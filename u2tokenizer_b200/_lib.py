"""ctypes binding of libu2b200.so (declared in include/u2b200.h).

There is deliberately NO fallback: if the shared library is missing or a call fails, a
RuntimeError is raised. PyTorch only supplies device memory and streams.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "libu2b200.so"
_lib = None


class GemmDesc(C.Structure):
    """Mirror of ``u2_gemm_desc`` (include/u2b200.h)."""
    _fields_ = [
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("zi", C.c_int32), ("zo", C.c_int32), ("b_zi_div", C.c_int32),
        ("lda", C.c_int64), ("a_stride_zi", C.c_int64), ("a_stride_zo", C.c_int64),
        ("ldb", C.c_int64), ("b_stride_zi", C.c_int64), ("b_stride_zo", C.c_int64),
        ("ldc", C.c_int64), ("c_stride_zi", C.c_int64), ("c_stride_zo", C.c_int64),
        ("c_dtype", C.c_int32), ("alpha", C.c_float),
        ("bias", C.c_void_p),
        ("act", C.c_int32),
        ("residual", C.c_void_p),
        ("ldr", C.c_int64),
        ("res_row_mod", C.c_int32),
        ("row_div", C.c_int32), ("row_stride", C.c_int32), ("row_off", C.c_int32),
        ("block_n", C.c_int32),
        ("a_mn", C.c_int32), ("b_mn", C.c_int32),
        ("epi_op", C.c_int32),
        ("rowvec", C.c_void_p),
        ("rv_stride_zi", C.c_int64), ("rv_stride_zo", C.c_int64),
        ("mul", C.c_void_p),
    ]


class SoftmaxDesc(C.Structure):
    """Mirror of ``u2_softmax_desc``."""
    _fields_ = [
        ("in_s0", C.c_int64), ("in_s1", C.c_int64), ("in_s2", C.c_int64),
        ("out_s0", C.c_int64), ("out_s1", C.c_int64), ("out_s2", C.c_int64),
        ("n0", C.c_int32), ("H", C.c_int32), ("S", C.c_int32), ("n", C.c_int32),
        ("scale", C.c_float),
        ("rel_bias", C.c_void_p),
        ("rel_max", C.c_int32),
        ("causal", C.c_int32), ("causal_off", C.c_int32),
        ("zero_pad_to", C.c_int32),
        ("window", C.c_int32),
    ]


class RopeDesc(C.Structure):
    """Mirror of ``u2_rope_desc``."""
    _fields_ = [
        ("rows", C.c_int64), ("ld", C.c_int64),
        ("dh", C.c_int32), ("n_q_heads", C.c_int32), ("n_k_heads", C.c_int32), ("n_v_heads", C.c_int32),
        ("q_norm_w", C.c_void_p), ("k_norm_w", C.c_void_p),
        ("eps", C.c_float),
        ("inv_freq", C.c_void_p),
        ("pos0", C.c_int32), ("pos_div", C.c_int32), ("pos_mod", C.c_int32),
        ("pos0_dev", C.c_void_p),
        ("k_cache", C.c_void_p), ("v_cache", C.c_void_p),
        ("Tmax", C.c_int32), ("rows_per_batch", C.c_int32),
        ("pos0_per_batch", C.c_int32),
    ]


class GemvDesc(C.Structure):
    """Mirror of ``u2_gemv_desc``."""
    _fields_ = [
        ("B", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("ldx", C.c_int64), ("ldw", C.c_int64), ("ldy", C.c_int64), ("ldr", C.c_int64),
        ("y_dtype", C.c_int32),
        ("residual", C.c_void_p),
        ("norm_gamma", C.c_void_p),
        ("norm_eps", C.c_float),
        ("silu_pair", C.c_int32),
    ]


class DlinearDesc(C.Structure):
    """Mirror of ``u2_dlinear_desc``."""
    _fields_ = [
        ("B", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("ldx", C.c_int64), ("ldw", C.c_int64), ("ldy", C.c_int64), ("ldr", C.c_int64), ("ldxg", C.c_int64),
        ("y_dtype", C.c_int32),
        ("ws", C.c_void_p), ("counters", C.c_void_p),
        ("ssq_in", C.c_void_p),
        ("eps", C.c_float),
        ("residual", C.c_void_p),
        ("silu_pair", C.c_int32),
        ("gamma_next", C.c_void_p),
        ("xg", C.c_void_p),
        ("ssq_out", C.c_void_p),
        ("ssq_zero", C.c_void_p),
        ("pdl", C.c_int32),
        ("dbg", C.c_void_p),
        ("ws_elems", C.c_int64),
        ("dep_flags", C.c_void_p), ("dep_shift", C.c_int32), ("out_flags", C.c_void_p),
        ("sched", C.c_int32),
        ("w_format", C.c_int32),
    ]


class FusedDecodeDesc(C.Structure):
    """Mirror of ``u2_fused_decode_desc``."""
    _fields_ = [
        ("B", C.c_int32), ("Hq", C.c_int32), ("Hkv", C.c_int32), ("dh", C.c_int32), ("Tmax", C.c_int32),
        ("pos", C.c_int32),
        ("pos_dev", C.c_void_p),
        ("ldq", C.c_int64), ("ldo", C.c_int64),
        ("q_norm_w", C.c_void_p), ("k_norm_w", C.c_void_p),
        ("eps", C.c_float),
        ("inv_freq", C.c_void_p),
        ("scale", C.c_float),
        ("kv_splits", C.c_int32), ("pdl", C.c_int32),
        ("pos_per_seq", C.c_int32),
        ("kv_src", C.c_void_p), ("ld_kv_src", C.c_int64),
        ("window", C.c_int32),
    ]


class DlinearNext(C.Structure):
    """Mirror of ``u2_dlinear_next``."""
    _fields_ = [
        ("pre_stages", C.c_int32), ("lookahead_units", C.c_int32), ("n", C.c_int32),
        ("w", C.c_void_p * 2),
        ("N", C.c_int32 * 2), ("K", C.c_int32 * 2),
        ("ldw", C.c_int64 * 2),
        ("units", C.c_int32 * 2),
        ("w_format", C.c_int32 * 2),
    ]


class FaDesc(C.Structure):
    """Mirror of ``u2_fa_desc``."""
    _fields_ = [
        ("B", C.c_int32), ("H", C.c_int32), ("Sq", C.c_int32), ("Sk", C.c_int32), ("dh", C.c_int32),
        ("scale", C.c_float),
        ("q_sb", C.c_int64), ("q_ss", C.c_int64), ("q_sh", C.c_int64),
        ("k_sb", C.c_int64), ("k_ss", C.c_int64), ("k_sh", C.c_int64),
        ("v_sb", C.c_int64), ("v_ss", C.c_int64), ("v_sh", C.c_int64),
        ("out_sb", C.c_int64), ("out_ss", C.c_int64),
        ("lse", C.c_void_p),
    ]


class LogprobDesc(C.Structure):
    """Mirror of ``u2_logprob_desc``."""
    _fields_ = [
        ("R", C.c_int32), ("V", C.c_int32), ("E", C.c_int32),
        ("ldh", C.c_int64), ("ldw", C.c_int64),
        ("labels", C.c_void_p), ("ws", C.c_void_p), ("ws_bytes", C.c_int64),
        ("lse", C.c_void_p), ("logit_sum", C.c_void_p), ("nll_acc", C.c_void_p),
    ]


class PreprocessInfo(C.Structure):
    """Mirror of ``u2_preprocess_info``."""
    _fields_ = [
        ("a_min", C.c_double), ("a_max", C.c_double),
        ("lo", C.c_int32 * 3), ("hi", C.c_int32 * 3), ("out", C.c_int32 * 3),
        ("sigma", C.c_float * 3), ("tail", C.c_int32 * 3), ("status", C.c_int32),
    ]


class PreprocessDesc(C.Structure):
    """Mirror of ``u2_preprocess_desc``."""
    _fields_ = [
        ("D", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("target", C.c_int32), ("pad_depth", C.c_int32),
        ("lower_pct", C.c_double), ("upper_pct", C.c_double),
        ("ws", C.c_void_p), ("ws_bytes", C.c_int64),
    ]


class SoftmaxBwdDesc(C.Structure):
    """Mirror of ``u2_softmax_bwd_desc`` (include/u2b200_train.h)."""
    _fields_ = [
        ("p_s0", C.c_int64), ("p_s1", C.c_int64), ("p_s2", C.c_int64),
        ("dp_s0", C.c_int64), ("dp_s1", C.c_int64), ("dp_s2", C.c_int64),
        ("ds_s0", C.c_int64), ("ds_s1", C.c_int64), ("ds_s2", C.c_int64),
        ("n0", C.c_int32), ("H", C.c_int32), ("S", C.c_int32), ("n", C.c_int32),
        ("zero_pad_to", C.c_int32),
    ]


class AdamWDesc(C.Structure):
    """Mirror of ``u2_adamw_desc``."""
    _fields_ = [
        ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("weight_decay", C.c_float),
        ("step", C.c_int32),
        ("grad_scale", C.c_void_p),
        ("seed", C.c_uint64), ("index_offset", C.c_int64),
    ]


class LoraDesc(C.Structure):
    """Mirror of ``u2_lora_desc`` (include/u2b200_train.h)."""
    _fields_ = [
        ("M", C.c_int32), ("K", C.c_int32), ("r", C.c_int32), ("n_adapters", C.c_int32),
        ("ldx", C.c_int64), ("ldu", C.c_int64),
        ("scale", C.c_float), ("p", C.c_float),
        ("seed", C.c_uint64),
        ("stream", C.c_int32 * 3),
        ("accumulate", C.c_int32),
    ]


LP_MAX_EOS, LP_MAX_BAD_WORDS, LP_MAX_BAD_TOKENS = 8, 256, 2048  # U2_LP_MAX_* of include/u2b200.h


class LogitsProcParams(C.Structure):
    """Mirror of ``u2_logits_proc_params`` (copied to device memory as raw bytes)."""
    _fields_ = [
        ("penalty", C.c_float), ("inv_penalty", C.c_float), ("ngram", C.c_int32), ("min_new", C.c_int32),
        ("n_eos", C.c_int32), ("n_bad", C.c_int32),
        ("eos", C.c_int32 * LP_MAX_EOS),
        ("bad_off", C.c_int32 * (LP_MAX_BAD_WORDS + 1)),
        ("bad_tok", C.c_int32 * LP_MAX_BAD_TOKENS),
    ]


class SlotState(C.Structure):
    """Mirror of ``u2_slot_state`` (one record per decode row, in device memory)."""
    _fields_ = [("seed", C.c_uint64), ("row", C.c_int32), ("count", C.c_int32), ("max_new", C.c_int32),
                ("done", C.c_int32)]


class SlotParams(C.Structure):
    """Mirror of ``u2_slot_params`` (copied to device memory as raw bytes)."""
    _fields_ = [("pad", C.c_int64), ("n_eos", C.c_int32), ("eos", C.c_int32 * LP_MAX_EOS), ("reserved", C.c_int32)]


class RowStoreParams(C.Structure):
    """Mirror of ``u2_row_store_params`` (copied to device memory as raw bytes)."""
    _fields_ = [("dst", C.c_void_p), ("ld_step", C.c_int64), ("ld_row", C.c_int64), ("steps", C.c_int32),
                ("reserved", C.c_int32)]


BEAM_MAX_BEAMS, BEAM_MAX_EOS, BEAM_MAX_KEEP = 16, 8, 144  # U2_BEAM_MAX_* of include/u2b200.h


class BeamParams(C.Structure):
    """Mirror of ``u2_beam_params`` (copied to device memory as raw bytes)."""
    _fields_ = [
        ("length_penalty", C.c_double),
        ("num_beams", C.c_int32), ("beams_to_keep", C.c_int32), ("early_stopping", C.c_int32),
        ("max_new_tokens", C.c_int32), ("n_eos", C.c_int32), ("reserved", C.c_int32),
        ("eos", C.c_int32 * BEAM_MAX_EOS),
    ]


class BeamStepDesc(C.Structure):
    """Mirror of ``u2_beam_step_desc``."""
    _fields_ = [
        ("params", C.c_void_p),
        ("prompts", C.c_int32), ("V", C.c_int32),
        ("cand_val", C.c_void_p), ("cand_tok", C.c_void_p),
        ("running", C.c_void_p), ("fin_score", C.c_void_p), ("fin_info", C.c_void_p), ("flags", C.c_void_p),
        ("ids", C.c_void_p),
        ("rec", C.c_void_p), ("ld_rec", C.c_int64), ("rec_rows", C.c_int32),
        ("kv_src", C.c_void_p), ("ld_kv_src", C.c_int64),
        ("pos_dev", C.c_void_p),
        ("hist", C.c_void_p), ("ld_hist", C.c_int64), ("hist_cap", C.c_int32),
        ("step_dev", C.c_void_p),
    ]


# name -> (restype, argtypes); every symbol include/u2b200.h / u2b200_train.h declares must be listed here
# (tests/test_abi.py cross-checks this table against the header and the built library).
_P, _I, _L, _F = C.c_void_p, C.c_int32, C.c_int64, C.c_float
SIGNATURES = {
    "u2_version": (C.c_int, []),
    "u2_last_error": (C.c_char_p, []),
    "u2_device_sm_count": (C.c_int, []),
    "u2_gemm_bf16": (C.c_int, [_P, _P, _P, C.POINTER(GemmDesc), _P]),
    "u2_layernorm_bf16": (C.c_int, [_P, _P, _P, _P, _P, _P, _L, _I, _L, _L, _L, _F, _P]),
    "u2_rmsnorm_bf16": (C.c_int, [_P, _P, _P, _P, _P, _L, _I, _L, _L, _L, _F, _P]),
    "u2_softmax_f32_bf16": (C.c_int, [_P, _P, C.POINTER(SoftmaxDesc), _P]),
    "u2_silu_mul_bf16": (C.c_int, [_P, _P, _L, _I, _L, _L, _I, _P]),
    "u2_patchify_f32_bf16": (C.c_int, [_P, _P, _L, _I, _I, _I, _I, _I, _I, _P]),
    "u2_patch_embed_f32_bf16": (C.c_int, [_P, _P, _P, _P, _P, _L, _I, _I, _I, _I, _I, _I, _I, _L, _P]),
    "u2_set_rows_bf16": (C.c_int, [_P, _P, _L, _L, _L, _I, _P]),
    "u2_vit_frame_rows_bf16": (C.c_int, [_P, _P, _L, _I, _I, _I, _P]),
    "u2_transpose_heads_bf16": (C.c_int, [_P, _P, _I, _I, _I, _I, _L, _L, _L, _L, _L, _L, _P]),
    "u2_spp_pool_bf16": (C.c_int, [_P, _P, _L, _I, _I, _I, _I, _I, _L, _L, _L, _I, _P]),
    "u2_multiscale_pool_bf16": (C.c_int, [_P, _P, _P, _F, _P, _I, _I, _I, _I, _P]),
    "u2_multiscale_pool_ws_elems": (C.c_int64, [_I, _I]),
    "u2_embed_splice_bf16": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _L, _P]),
    "u2_temporal_attention_bf16": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _L, _L, _F, _P, _I, _P]),
    "u2_rope_bf16": (C.c_int, [_P, C.POINTER(RopeDesc), _P]),
    "u2_decode_attention_bf16": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _L, _L, _F, _I, _P, _L, _P]),
    "u2_decode_attention_window_bf16": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _L, _L, _F, _I, _P, _L,
                                                  _I, _P]),
    "u2_gemv_bf16": (C.c_int, [_P, _P, _P, C.POINTER(GemvDesc), _P]),
    "u2_argmax_f32": (C.c_int, [_P, _P, _P, _I, _I, _L, _P]),
    "u2_dlinear_bf16": (C.c_int, [_P, _P, _P, C.POINTER(DlinearDesc), _P]),
    "u2_decode_attention_fused_bf16": (C.c_int, [_P, _P, _P, _P, C.POINTER(FusedDecodeDesc), _P]),
    "u2_decode_embed_bf16": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _L, _P]),
    "u2_flash_attention_d64_bf16": (C.c_int, [_P, _P, _P, _P, C.POINTER(FaDesc), _P]),
    "u2_sample_f32": (C.c_int, [_P, _P, _I, _I, _L, _F, _I, _F, C.c_uint64, _P, _I, _P]),
    "u2_sample_dev_f32": (C.c_int, [_P, _P, _I, _I, _L, _P, _P, _I, _P]),
    "u2_logits_process_f32": (C.c_int, [_P, _I, _I, _L, _P, _P, _L, _I, _P, _P, _I, _P]),
    "u2_sample_slots_f32": (C.c_int, [_P, _P, _I, _I, _L, _P, _P, _P]),
    "u2_logits_process_slots_f32": (C.c_int, [_P, _I, _I, _L, _P, _P, _L, _I, _P, _P, _P]),
    "u2_slot_update": (C.c_int, [_P, _I, _P, _P, _L, _P, _P, _P, _P]),
    "u2_store_rows_f32": (C.c_int, [_P, _I, _I, _L, _P, _P, _I, _P]),
    "u2_sample_out_f32": (C.c_int, [_P, _P, _I, _I, _L, _P, _P, _I, _P, _P, _P, _P]),
    "u2_pick_logprob_f32": (C.c_int, [_P, _I, _I, _L, _P, _P, _P]),
    "u2_slot_update_lp": (C.c_int, [_P, _I, _P, _P, _L, _P, _P, _P, _P, _P, _P]),
    "u2_topk_rows_f32": (C.c_int, [_P, _P, _I, _I, _I, _L, _L, _P]),
    "u2_log_softmax_f32": (C.c_int, [_P, _P, _I, _I, _L, _L, _P]),
    "u2_beam_topk_f32": (C.c_int, [_P, _L, _I, _I, _P, _P, _P, _P, _P, _P]),
    "u2_beam_step": (C.c_int, [C.POINTER(BeamStepDesc), _I, _P]),
    "u2_dlinear_ws_elems": (C.c_int64, [_I, _I]),
    "u2_dlinear_multi_bf16": (C.c_int, [_P, _P, _P, _P, _I, _P, _P, _I, _P, _P]),
    "u2_dlinear_pack_bf16": (C.c_int, [_P, _I, _I, _L, _P, _P, _P]),
    "u2_preprocess_ws_bytes": (C.c_int64, [_I, _I, _I]),
    "u2_preprocess_volume_f32": (C.c_int, [_P, _P, _P, C.POINTER(PreprocessDesc), _P]),
    "u2_logprob_ws_bytes": (C.c_int64, [_I, _I]),
    "u2_lmhead_logprob_bf16": (C.c_int, [_P, _P, _P, C.POINTER(LogprobDesc), _P]),
    # ---- training side (include/u2b200_train.h)
    "u2_transpose_bf16": (C.c_int, [_P, _P, _I, _I, _L, _L, _I, _L, _L, _P]),
    "u2_colsum_bf16": (C.c_int, [_P, _P, _L, _L, _L, _P]),
    "u2_gelu_bf16": (C.c_int, [_P, _P, _L, _P]),
    "u2_gelu_bwd_bf16": (C.c_int, [_P, _P, _P, _L, _P]),
    "u2_silu_mul_bwd_bf16": (C.c_int, [_P, _P, _P, _L, _I, _L, _L, _P]),
    "u2_layernorm_bwd_bf16": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _L, _I, _L, _L, _L, _L, _F, _P]),
    "u2_rmsnorm_bwd_bf16": (C.c_int, [_P, _P, _P, _P, _P, _P, _L, _I, _L, _L, _L, _L, _F, _P]),
    "u2_softmax_bwd_bf16": (C.c_int, [_P, _P, _P, C.POINTER(SoftmaxBwdDesc), _P]),
    "u2_relbias_grad_bf16": (C.c_int, [_P, _P, _I, _I, _I, _I, _L, _L, _L, _I, _P]),
    "u2_rowdot_bf16": (C.c_int, [_P, _P, _P, _I, _I, _I, _I, _L, _L, _L, _L, _L, _L, _P]),
    "u2_temporal_attention_bwd_bf16": (C.c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _L, _L, _L, _F, _P, _P, _I, _P]),
    "u2_rope_bwd_bf16": (C.c_int, [_P, _P, C.POINTER(RopeDesc), _P, _P, _P]),
    "u2_spp_pool_bwd_bf16": (C.c_int, [_P, _P, _L, _I, _I, _I, _I, _I, _L, _L, _L, _L, _I, _P]),
    "u2_multiscale_pool_bwd_bf16": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "u2_embed_scatter_add_bf16": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _L, _P]),
    "u2_group_sum_bf16": (C.c_int, [_P, _P, _L, _I, _I, _I, _L, _L, _P]),
    "u2_ce_bwd_f32_bf16": (C.c_int, [_P, _P, _P, _P, _P, _L, _I, _L, _L, _P]),
    "u2_dpo_loss_f32": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _F, _P]),
    "u2_adamw_bf16": (C.c_int, [_P, _P, _P, _P, _P, _L, C.POINTER(AdamWDesc), _P]),
    "u2_adamw_bf16_mom16": (C.c_int, [_P, _P, _P, _P, _P, _L, C.POINTER(AdamWDesc), _P]),
    "u2_adamw_f32grad": (C.c_int, [_P, _P, _P, _P, _P, _P, _L, C.POINTER(AdamWDesc), _P]),
    "u2_sumsq_bf16": (C.c_int, [_P, _P, _L, _P]),
    "u2_sumsq_f32": (C.c_int, [_P, _P, _L, _P]),
    "u2_add_bf16": (C.c_int, [_P, _P, _L, _P]),
    "u2_cast_f32_bf16": (C.c_int, [_P, _P, _L, _P]),
    "u2_cast_bf16_f32": (C.c_int, [_P, _P, _L, _P]),
    "u2_lora_down_bf16": (C.c_int, [_P, _P, _P, C.POINTER(LoraDesc), _P]),
    "u2_lora_wgrad_bf16": (C.c_int, [_P, _P, _P, C.POINTER(LoraDesc), _P]),
    "u2_lora_dgrad_bf16": (C.c_int, [_P, _P, _P, C.POINTER(LoraDesc), _P]),
}


def lib_path() -> Path:
    return _LIB_PATH


def load():
    """Load the library (once). Raises RuntimeError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise RuntimeError(
            f"{_LIB_PATH} is missing: build it with `python -m u2tokenizer_b200.build` "
            "(there is no CPU / PyTorch fallback for the hot path)")
    lib = C.CDLL(str(_LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


# kernels launched per entry point (u2_multiscale_pool_bf16: gate + gate sum + write, counted at its maximum)
KERNELS_PER_CALL = {"u2_multiscale_pool_bf16": 3, "u2_argmax_f32": 2, "u2_lmhead_logprob_bf16": 2,
                    "u2_preprocess_volume_f32": 14, "u2_multiscale_pool_bwd_bf16": 2}
_launches = 0


def launches() -> int:
    """Number of CUDA kernels this process has launched through the C ABI so far."""
    return _launches


def add_launches(n: int) -> None:
    """CUDA-graph replays re-launch the captured kernels without going through check()."""
    global _launches
    _launches += n


def check(rc: int, what: str) -> None:
    global _launches
    _launches += KERNELS_PER_CALL.get(what, 1)
    if rc != 0:
        msg = load().u2_last_error()
        raise RuntimeError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")
