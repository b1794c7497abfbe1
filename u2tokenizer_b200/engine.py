"""Host-side orchestration of the hot path over the C-ABI kernels (libu2b200.so).

`U2Engine` owns the device copies of the weights in the layouts the kernels want (fused QKV /
gate-up matrices, fp32 vectors) and sequences the kernel launches for

  * the vision front   : patch embed -> ViT3D -> final LN -> spatial pooling -> projector MLP
                         (reference src/model/u2_arch.py:96-99, multimodal_encoder/vit.py,
                          multimodal_projector/spatial_pooling_projector.py)
  * the mu2-tokenizer  : SVR (spatial + temporal attention, token selection, multi-scale pooling) and
                         TTA (self / visual-cross / text-cross attention, linear aggregation)
                         (reference src/model/u2tokenizer/{u2Tokenizer,svr,tta,rma,rope}.py)
  * the splice         : embed_tokens gather + visual tokens at positions 1..n_vis (u2_arch.py:118-121)
  * the decoder        : Qwen3 / Llama / Phi-3 prefill (tensor-core GEMMs) and KV-cached greedy decode
                         (weight-streaming GEMVs), i.e. what HF runs under super().forward()/generate()

All arithmetic happens in hand-written CUDA; torch provides memory, streams and CUDA graphs only.
"""
from __future__ import annotations

import math
from dataclasses import asdict, dataclass, replace
from typing import Dict, Iterable, List, Optional, Tuple

import torch

from . import _lib, ops
from .geometry import Geometry

BF16, F32 = torch.bfloat16, torch.float32
REL_MAX = 512  # RelativeMultiheadAttention(max_seq_len=512), reference rma.py:6,19


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


@dataclass(frozen=True)
class LogitsProcessors:
    """HF generate()'s repetition_penalty, no_repeat_ngram_size, bad_words_ids and min_new_tokens, applied by one
    kernel to every step's logits before the pick (ops.logits_process). The history is the generated tokens only.
    eos_token_ids: the ids min_new_tokens keeps out. Validated values: see modeling's _generate_logits_processors."""
    repetition_penalty: float = 1.0
    no_repeat_ngram_size: int = 0
    min_new_tokens: int = 0
    eos_token_ids: Tuple[int, ...] = ()
    bad_words_ids: Tuple[Tuple[int, ...], ...] = ()

    def neutral(self) -> bool:
        return (self.repetition_penalty == 1.0 and self.no_repeat_ngram_size == 0 and not self.bad_words_ids
                and (self.min_new_tokens == 0 or not self.eos_token_ids))


@dataclass(frozen=True)
class BeamSearch:
    """HF generate(num_beams, length_penalty, early_stopping, num_return_sequences) on the CUDA path (GenerationMixin.
    _beam_search): the beams of prompt b are rows b*K .. b*K+K-1 of one decode batch, they continue each other's KV cache
    through an indirection table, and the per-step selection and bookkeeping run inside the captured decode step
    (ops.beam_topk / ops.beam_step). early_stopping: True, False or "never". pad_token_id: fills the rows shorter than the
    longest returned hypothesis (HF's `pad_token_id or eos_token_id[0]`). Validated values: see modeling's
    _generate_beam_search."""
    num_beams: int
    length_penalty: float = 1.0
    early_stopping: object = False
    num_return_sequences: int = 1
    pad_token_id: Optional[int] = None


def eos_ids(eos_token_id) -> Tuple[int, ...]:
    """EOS ids given as None, an int, a list / tuple or a tensor, as a tuple of ints (empty for None)."""
    if eos_token_id is None:
        return ()
    if isinstance(eos_token_id, torch.Tensor):
        eos_token_id = eos_token_id.reshape(-1).tolist()
    elif not isinstance(eos_token_id, (list, tuple)):
        eos_token_id = [eos_token_id]
    return tuple(int(e) for e in eos_token_id)


@dataclass(frozen=True)
class GenerateRequest:
    """What the token-picking head of one generate() call does, handed to every decode step of the call.
    sampling: (temperature, top_k, top_p, seed), or None for greedy argmax. processors: a neutral configuration is kept
    as None, so it runs exactly as no configuration: no extra launch, the same captured graph. beam: num_beams > 1, or
    None; with it the sampling is ignored. eos_token_id: anything eos_ids() takes, kept as its tuple.
    output_scores / output_logits: every step also stores the scores the token was picked from / the raw logits into
    the row stores set by _set_row_store() (HF generate(output_scores, output_logits)). return_logprobs (continuous
    batching): every slot also records the log-prob of each pick. All three off: exactly the launches without them."""
    max_new_tokens: int
    eos_token_id: Tuple[int, ...] = ()
    sampling: Optional[Tuple[float, int, float, int]] = None
    processors: Optional[LogitsProcessors] = None
    beam: Optional[BeamSearch] = None
    output_scores: bool = False
    output_logits: bool = False
    return_logprobs: bool = False

    def __post_init__(self):
        object.__setattr__(self, "eos_token_id", eos_ids(self.eos_token_id))
        if self.processors is not None and self.processors.neutral():
            object.__setattr__(self, "processors", None)


SEED_STRIDE = 0x9E3779B97F4A7C15


def chunk_plan(B: int, n: int, cap: int, beam: bool) -> List[Tuple[torch.Tensor, int]]:
    """The decode chunks of a generate() call over B prompts with n rows each (row b * n + s is row s of prompt b) when
    one decode step carries at most cap rows: per chunk, the prompt of each of its rows (CPU int64) and the offset its
    sampled rows add to the request seed. Beam search takes windows of (cap // n) * n rows, so the beams of a prompt
    never straddle two chunks; the other modes take windows of cap rows. The sampler keys its random stream by
    (seed, step, row in the chunk), so multi-sample chunks (n > 1) move the seed by SEED_STRIDE per chunk; the chunks of
    a batch of one row per prompt all keep the request seed."""
    width = (cap // n) * n if beam else cap
    return [(torch.arange(r0, min(B * n, r0 + width)) // n, SEED_STRIDE * ci if n > 1 else 0)
            for ci, r0 in enumerate(range(0, B * n, width))]


class _Take:
    """Pops tensors out of the source state dict (so fused copies do not double peak memory)."""

    def __init__(self, sd: Dict[str, torch.Tensor], device):
        self.sd, self.dev = sd, device

    def has(self, k):
        return k in self.sd

    def bf(self, k) -> torch.Tensor:
        return self.sd.pop(k).to(device=self.dev, dtype=BF16).contiguous()

    def f32(self, k) -> torch.Tensor:
        # parameters are bf16-valued on the reference side at inference; keep those values, fp32 storage
        return self.sd.pop(k).to(device=self.dev, dtype=BF16).to(F32).contiguous()

    def cat_bf(self, keys) -> torch.Tensor:
        return torch.cat([self.bf(k) for k in keys], dim=0).contiguous()

    def cat_f32(self, keys) -> torch.Tensor:
        return torch.cat([self.f32(k) for k in keys], dim=0).contiguous()


@dataclass
class _SelfAttnW:  # RelativeMultiheadAttention / RotaryMultiheadAttention / the nn.MultiheadAttention fallback
    wqkv: torch.Tensor
    bqkv: torch.Tensor
    wd: torch.Tensor
    bd: torch.Tensor
    rel: Optional[torch.Tensor]
    seq_first: bool = False  # nn.MultiheadAttention with batch_first=False: dim 0 of the input is the sequence


@dataclass
class _CrossAttnW:  # MultiHeadCrossAttention
    wq: torch.Tensor
    bq: torch.Tensor
    wkv: torch.Tensor   # [2E, E] (k then v); linagg: [E, E] (k only)
    bkv: torch.Tensor
    wd: Optional[torch.Tensor]
    bd: Optional[torch.Tensor]


class U2Engine:
    def __init__(self, geom: Geometry, state_dict: Dict[str, torch.Tensor], device="cuda",
                 attn_workspace_bytes: int = 6 << 30, decode_impl: str = "tcgen05"):
        if not torch.cuda.is_available():
            raise RuntimeError("U2Engine needs a CUDA device: the hot path has no CPU implementation")
        from . import _lib
        _lib.load()  # fail loudly when the extension is missing
        self.g = geom
        self.dev = torch.device(device)
        self.attn_ws = attn_workspace_bytes
        self.decode_impl = decode_impl  # "tcgen05" (stream-K tensor-core linears) or "gemv" (CUDA-core GEMV)
        import os
        from . import _lib
        self.num_sms = int(_lib.load().u2_device_sm_count())
        self.fwd_graph = os.environ.get("U2_FWD_GRAPH", "1") != "0"  # replay repeated same-shape forwards as one CUDA graph
        self.attn_pdl = os.environ.get("U2_ATTN_PDL", "0") != "0"  # PDL launch of the split-KV decode attention
        self.pdl = os.environ.get("U2_PDL", "1") != "0"  # programmatic dependent launch between decode linears
        self.multi_op = os.environ.get("U2_MULTI_OP", "1") != "0"  # o_proj/gate-up/down/qkv chained in one launch
        self.fused_patch_embed = os.environ.get("U2_FUSED_PATCH_EMBED", "0") != "0"  # one-kernel gather + Linear (canonical patches); see DESIGN.md
        self.use_flash = os.environ.get("U2_FLASH", "1") != "0"  # fused wgmma attention where it applies (dh 64)
        self.fine_deps = os.environ.get("U2_FINE_DEPS", "0") != "0"  # per-tile flags instead of grid-wide waits
        self.dl_sched = int(os.environ.get("U2_DL_SCHED", "0"))  # 1: whole 64-row tiles per CTA; 0: stream-K / 128
        self.pre_stages = int(os.environ.get("U2_PRE_STAGES", "0"))  # 0 = fill the whole ring before the dependency
        self.l2_lookahead_units = int(os.environ.get("U2_L2_LOOKAHEAD", "0"))  # x16 KB per CTA at op boundaries
        self.l2_next_units = int(os.environ.get("U2_L2_NEXT", "-1"))            # x16 KB per CTA of the next gate|up
        if geom.vision_select_feature != "patch":
            raise NotImplementedError("only vision_select_feature='patch' is supported (the spp projector needs it)")
        t = _Take(dict(state_dict), self.dev)
        self._prep_vit(t)
        self._prep_projector(t)
        if geom.enable_u2tokenizer:
            self._prep_tokenizer(t)
        self._prep_decoder(t)
        self._gen_state = None
        self._fwd_state = None
        self._param_blocks = {}  # what -> [host arguments, device block]: see _param_block
        self.last_beam_scores = None  # fp32 [rows] scores of the hypotheses the last beam search returned

    # =========================================================================================
    # weight preparation
    # =========================================================================================
    def _prep_vit(self, t: _Take):
        g = self.g
        v = "model.vision_tower.vision_tower."
        self.pe_w = t.bf(v + "patch_embedding.patch_embeddings.1.weight")
        self.pe_b = t.f32(v + "patch_embedding.patch_embeddings.1.bias")
        self.pos = t.bf(v + "patch_embedding.position_embeddings").view(g.n_patches, g.vit_hidden)
        self.cls = t.bf(v + "cls_token").view(g.vit_hidden)
        self.vit = []
        for i in range(g.vit_layers):
            b = f"{v}blocks.{i}."
            self.vit.append(dict(
                ln1g=t.f32(b + "norm1.weight"), ln1b=t.f32(b + "norm1.bias"),
                wqkv=t.bf(b + "attn.qkv.weight"),
                bqkv=t.f32(b + "attn.qkv.bias") if t.has(b + "attn.qkv.bias") else None,
                wo=t.bf(b + "attn.out_proj.weight"), bo=t.f32(b + "attn.out_proj.bias"),
                ln2g=t.f32(b + "norm2.weight"), ln2b=t.f32(b + "norm2.bias"),
                w1=t.bf(b + "mlp.linear1.weight"), b1=t.f32(b + "mlp.linear1.bias"),
                w2=t.bf(b + "mlp.linear2.weight"), b2=t.f32(b + "mlp.linear2.bias")))
        self.vit_ng = t.f32(v + "norm.weight")
        self.vit_nb = t.f32(v + "norm.bias")

    def _prep_projector(self, t: _Take):
        g = self.g
        p = "model.mm_projector.projector."
        self.proj = [(t.bf(p + "0.weight"), t.f32(p + "0.bias"))]
        for i in range(1, int(g.proj_layer_num)):
            idx = 2 * i if g.proj_layer_type == "mlp" else i
            self.proj.append((t.bf(p + f"{idx}.weight"), t.f32(p + f"{idx}.bias")))

    def _self_attn_w(self, t: _Take, pre: str) -> _SelfAttnW:
        if self.g.attn_type not in ("rma", "rope"):
            # any other attn_type is torch.nn.MultiheadAttention in the reference (svr.py:17-18, tta.py:83-84):
            # packed q | k | v projection, called sequence-first
            return _SelfAttnW(wqkv=t.bf(pre + "in_proj_weight"), bqkv=t.f32(pre + "in_proj_bias"),
                              wd=t.bf(pre + "out_proj.weight"), bd=t.f32(pre + "out_proj.bias"), rel=None,
                              seq_first=True)
        rel = t.f32(pre + "relative_bias") if self.g.attn_type == "rma" else None
        return _SelfAttnW(
            wqkv=t.cat_bf([pre + "wq.weight", pre + "wk.weight", pre + "wv.weight"]),
            bqkv=t.cat_f32([pre + "wq.bias", pre + "wk.bias", pre + "wv.bias"]),
            wd=t.bf(pre + "dense.weight"), bd=t.f32(pre + "dense.bias"), rel=rel)

    def _cross_attn_w(self, t: _Take, pre: str, compress: bool = False) -> _CrossAttnW:
        if compress:
            # LinearAggregation never runs wv / dense (reference tta.py:47-48,62-65): drop them
            for k in ("wv.weight", "wv.bias", "dense.weight", "dense.bias"):
                t.sd.pop(pre + k, None)
            return _CrossAttnW(wq=t.bf(pre + "wq.weight"), bq=t.f32(pre + "wq.bias"),
                               wkv=t.bf(pre + "wk.weight"), bkv=t.f32(pre + "wk.bias"), wd=None, bd=None)
        return _CrossAttnW(wq=t.bf(pre + "wq.weight"), bq=t.f32(pre + "wq.bias"),
                           wkv=t.cat_bf([pre + "wk.weight", pre + "wv.weight"]),
                           bkv=t.cat_f32([pre + "wk.bias", pre + "wv.bias"]),
                           wd=t.bf(pre + "dense.weight"), bd=t.f32(pre + "dense.bias"))

    def _prep_tokenizer(self, t: _Take):
        g = self.g
        u = "model.u2tokenizer."
        self.queries = t.bf(u + "query_tokens").view(g.num_3d_query_token, g.hidden_size)
        self.svr = []
        for i in range(g.u2t_num_layers):
            l = f"{u}svt_module.attention_network.layers.{i}."
            self.svr.append((self._self_attn_w(t, l + "spatial_attention."),
                             self._self_attn_w(t, l + "temporal_attention.")))
        self.score_w = t.bf(u + "svt_module.token_selection.score_net.weight")
        self.score_b = t.f32(u + "svt_module.token_selection.score_net.bias")
        self.gate_w, self.gate_b = None, 0.0
        if g.enable_dmtp:
            self.gate_w = t.f32(u + "svt_module.dynamic_pool.gate_fc.weight").view(-1)
            self.gate_b = float(t.f32(u + "svt_module.dynamic_pool.gate_fc.bias").item())
        self.tta = []
        for i in range(g.u2t_num_layers):
            l = f"{u}tta_module.layers_vt.{i}."
            self.tta.append(dict(
                self_attn=self._self_attn_w(t, l + "self_attention."),
                vis=self._cross_attn_w(t, l + "visual_cross_attention."),
                txt=self._cross_attn_w(t, l + "text_cross_attention."),
                ns=(t.f32(l + "norm_self.weight"), t.f32(l + "norm_self.bias")),
                nv=(t.f32(l + "norm_cross_v.weight"), t.f32(l + "norm_cross_v.bias")),
                nt=(t.f32(l + "norm_cross_t.weight"), t.f32(l + "norm_cross_t.bias"))))
        self.linagg = self._cross_attn_w(t, u + "tta_module.layer_linagg.linear_aggregator.", compress=True)
        dh = g.hidden_size // g.u2t_num_heads
        self.u2t_inv_freq = (1.0 / (10000 ** (torch.arange(0, dh, 2, dtype=F32) / dh))).to(self.dev)

    def _prep_decoder(self, t: _Take):
        g = self.g
        self.embed = t.bf("model.embed_tokens.weight")
        self.layers = []
        phi3 = g.decoder_family == "phi3"
        for i in range(g.num_hidden_layers):
            l = f"model.layers.{i}."
            if phi3:
                # HF Phi3: qkv_proj is already the fused [q; k; v] layout, gate_up_proj is [gate; up] in halves
                # (modeling_phi3.py:58-62)
                wqkv = t.bf(l + "self_attn.qkv_proj.weight")
                gate, up = t.bf(l + "mlp.gate_up_proj.weight").chunk(2, dim=0)
            else:
                wqkv = t.cat_bf([l + "self_attn.q_proj.weight", l + "self_attn.k_proj.weight",
                                 l + "self_attn.v_proj.weight"])
                gate, up = t.bf(l + "mlp.gate_proj.weight"), t.bf(l + "mlp.up_proj.weight")
            self.layers.append(dict(
                ln1=t.f32(l + "input_layernorm.weight"),
                wqkv=wqkv,
                qn=t.f32(l + "self_attn.q_norm.weight") if g.qk_norm else None,
                kn=t.f32(l + "self_attn.k_norm.weight") if g.qk_norm else None,
                wo=t.bf(l + "self_attn.o_proj.weight"),
                ln2=t.f32(l + "post_attention_layernorm.weight"),
                # gate/up rows interleaved (gate_j, up_j) = rows (2j, 2j+1): one copy serves the prefill GEMM
                # (+ interleaved SiLU*mul) and the decode linear's in-epilogue pairing
                wgu=torch.stack([gate, up], dim=1).view(2 * g.intermediate_size, g.hidden_size).contiguous(),
                wdown=t.bf(l + "mlp.down_proj.weight")))
            del gate, up
        self.final_norm = t.f32("model.norm.weight")
        self.lm_head = self.embed if (g.tie_word_embeddings or not t.has("lm_head.weight")) else t.bf("lm_head.weight")
        self.inv_freq = self._decoder_inv_freq().to(self.dev)
        # The decode step streams every weight once per token, so it reads the lossless 13-bit packing of each matrix
        # that fits it (ops.dlinear_pack: 0.81 of the bf16 bytes); prefill and training keep the bf16 copies. A tied
        # head's packed copy serves the decode head only. Keys: (layer, name) and ("head",).
        self._packed = {}
        if self.decode_impl == "tcgen05" and all(
                k % 64 == 0 for k in (g.hidden_size, g.intermediate_size, g.num_attention_heads * g.head_dim)):
            mats = [((i, k), l[k]) for i, l in enumerate(self.layers) for k in ("wqkv", "wo", "wgu", "wdown")]
            for key, w in mats + [(("head",), self.lm_head)]:
                pk = ops.dlinear_pack(w)
                if pk is not None:
                    self._packed[key] = pk
        self._decode_bf16 = False  # True: the decode step streams the bf16 weights (reference runs and A/B measurements)

    def _decoder_inv_freq(self) -> torch.Tensor:
        """Default RoPE or the llama3 rescaling (HF modeling_rope_utils; reference config.json:49-56)."""
        g = self.g
        dh = g.head_dim
        inv = 1.0 / (g.rope_theta ** (torch.arange(0, dh, 2, dtype=F32) / dh))
        rs = g.rope_scaling
        if rs and rs.get("rope_type", rs.get("type")) == "llama3":
            factor, lo, hi = rs["factor"], rs["low_freq_factor"], rs["high_freq_factor"]
            old = rs["original_max_position_embeddings"]
            wavelen = 2 * math.pi / inv
            inv_l = torch.where(wavelen > old / lo, inv / factor, inv)
            smooth = (old / wavelen - lo) / (hi - lo)
            smoothed = (1 - smooth) * inv_l / factor + smooth * inv_l
            is_med = ~(wavelen < old / hi) & ~(wavelen > old / lo)
            inv = torch.where(is_med, smoothed, inv_l)
        elif rs:
            raise NotImplementedError(f"rope_scaling {rs} not supported")
        return inv

    # =========================================================================================
    # attention through the GEMM kernel (scores materialised in fp32, probabilities in bf16)
    # =========================================================================================
    def _attention(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, scale: float,
                   rel_bias: Optional[torch.Tensor] = None, causal: bool = False, window: int = 0):
        """q [b, Sq, h, dh], k/v [b, Sk, hk, dh] (strided views, dh contiguous), out [b, Sq, h*dh] view.
        softmax(q k^T * scale (+ rel bias) (+ causal mask, + sliding window when window > 0)) v, batched over (b, h) on
        the tensor cores."""
        b, Sq, h, dh = q.shape
        Sk, hk = k.shape[1], k.shape[2]
        Skp = _pad8(Sk)
        if dh == 64 and h == hk and rel_bias is None and not causal and self.use_flash:
            # fused wgmma attention: scores never leave the SM (the ViT tower, S = 2049); V is consumed as stored
            return ops.flash_attention_d64(q, k, v, out, scale)
        per_b = h * Sq * Skp * 6
        chunk = max(1, min(b, self.attn_ws // max(per_b, 1)))
        dev = q.device
        sc = torch.empty(chunk, h, Sq, Skp, device=dev, dtype=F32)
        pr = torch.empty(chunk, h, Sq, Skp, device=dev, dtype=BF16)
        for b0 in range(0, b, chunk):
            nb = min(chunk, b - b0)
            qq, kk, vv, oo = q[b0:b0 + nb], k[b0:b0 + nb], v[b0:b0 + nb], out[b0:b0 + nb]
            ops.gemm(qq, kk, sc, M=Sq, N=Sk, K=dh, lda=qq.stride(1), ldb=kk.stride(1), ldc=Skp, zi=h, zo=nb,
                     b_zi_div=h // hk, a_strides=(qq.stride(2), qq.stride(0)), b_strides=(kk.stride(2), kk.stride(0)),
                     c_strides=(Sq * Skp, h * Sq * Skp), alpha=scale)
            ops.softmax(sc, pr, n0=nb, H=h, S=Sq, n=Sk, in_strides=(h * Sq * Skp, Sq * Skp, Skp),
                        out_strides=(h * Sq * Skp, Sq * Skp, Skp), rel_bias=rel_bias, rel_max=REL_MAX, causal=causal,
                        causal_off=Sk - Sq, window=window if causal else 0)
            # P @ V with V [Sk, dh] as stored (MN-major B operand): no transposed copy of V
            ops.gemm(pr, vv, oo, M=Sq, N=dh, K=Sk, lda=Skp, ldb=vv.stride(1), ldc=oo.stride(1), zi=h, zo=nb,
                     b_zi_div=h // hk, a_strides=(Sq * Skp, h * Sq * Skp), b_strides=(vv.stride(2), vv.stride(0)),
                     c_strides=(dh, oo.stride(0)), b_mn=True)
        return out

    # =========================================================================================
    # vision front
    # =========================================================================================
    def encode_images(self, frames: torch.Tensor) -> torch.Tensor:
        """frames fp32 [F, 1, D, H, W] -> projected tokens bf16 [F, tokens_per_frame, E]
        (u2MetaForCausalLM.encode_images, reference u2_arch.py:96-99)."""
        g = self.g
        if frames.dim() != 5 or frames.shape[1] != 1 or g.image_channel != 1:
            raise NotImplementedError("single-channel volumes [F, 1, D, H, W] only")
        if list(frames.shape[2:]) != list(g.image_size):
            raise ValueError(f"frame size {list(frames.shape[2:])} != config.image_size {g.image_size}")
        Fr = frames.shape[0]
        Hd, P = g.vit_hidden, g.n_patches
        S = P + 1
        Sp = _pad8(S)
        vol = frames.to(device=self.dev, dtype=F32).contiguous().view(Fr, *g.image_size)
        x = torch.empty(Fr, Sp, Hd, device=self.dev, dtype=BF16)
        if self.fused_patch_embed and ops.patch_embed_supported(g.image_size, g.patch_size, Hd):
            # --- fused patch embedding: 5-D TMA slabs of the fp32 volume -> bf16 A operand in smem -> wgmma (+bias +pos)
            ops.patch_embed(vol, g.patch_size, self.pe_w, self.pe_b, self.pos, x)
        else:
            # --- brick gather -> GEMM (+bias +position table, rows scattered behind the cls row)
            rows = ops.patchify(vol, g.patch_size)
            ops.gemm(rows, self.pe_w, x, M=Fr * P, N=Hd, K=g.patch_dim, lda=g.patch_dim, ldb=g.patch_dim, ldc=Hd,
                     bias=self.pe_b, residual=self.pos, ldr=Hd, res_row_mod=P, row_remap=(P, Sp, 1))
            del rows
        ops.vit_frame_rows(x, self.cls, Fr, Sp, S)  # cls row + the 7 zero padding rows per frame (no full-buffer memset)
        # --- transformer blocks
        nh = g.vit_heads
        dh = Hd // nh
        x2 = x.view(Fr * Sp, Hd)
        y = torch.empty_like(x2)
        qkv = torch.empty(Fr * Sp, 3 * Hd, device=self.dev, dtype=BF16)
        ctx = torch.zeros(Fr, Sp, Hd, device=self.dev, dtype=BF16)
        hmid = torch.empty(Fr * Sp, g.vit_mlp, device=self.dev, dtype=BF16)
        qkv5 = qkv.view(Fr, Sp, 3, nh, dh)
        for w in self.vit:
            ops.layernorm(x2, w["ln1g"], w["ln1b"], 1e-5, out=y)
            ops.linear(y, w["wqkv"], w["bqkv"], out=qkv)
            self._attention(qkv5[:, :S, 0], qkv5[:, :S, 1], qkv5[:, :S, 2], ctx[:, :S], dh ** -0.5)
            ops.linear(ctx.view(Fr * Sp, Hd), w["wo"], w["bo"], residual=x2, out=x2)
            ops.layernorm(x2, w["ln2g"], w["ln2b"], 1e-5, out=y)
            ops.linear(y, w["w1"], w["b1"], act=ops.ACT_GELU, out=hmid)
            ops.linear(hmid, w["w2"], w["b2"], residual=x2, out=x2)
        ops.layernorm(x2, self.vit_ng, self.vit_nb, 1e-5, out=y)
        # --- drop cls + pooling + projector MLP
        npf = g.tokens_per_frame
        pooled = torch.empty(Fr, npf, Hd, device=self.dev, dtype=BF16)
        ops.spp_pool(y, pooled, frames=Fr, grid=g.grid, ps=g.proj_pooling_size, E=Hd, in_frame_stride=Sp, in_off=1,
                     ldx=Hd, sequence=(g.proj_pooling_type == "sequence"))
        z = pooled.view(Fr * npf, Hd)
        n = len(self.proj)
        for i, (w, b) in enumerate(self.proj):
            act = ops.ACT_GELU if (g.proj_layer_type == "mlp" and i < n - 1) else ops.ACT_NONE
            z = ops.linear(z, w, b, act=act)
        return z.view(Fr, npf, g.hidden_size)

    # =========================================================================================
    # mu2-tokenizer
    # =========================================================================================
    def _u2t_self_attention(self, x2: torch.Tensor, nb: int, S: int, w: _SelfAttnW,
                            residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        """RMA / RoPE self-attention over sequences of length S (reference rma.py:46-82, rope.py:62-91)."""
        g = self.g
        E, H = g.hidden_size, g.u2t_num_heads
        dh = E // H
        qkv = ops.linear(x2, w.wqkv, w.bqkv)
        if g.attn_type == "rope":
            ops.rope(qkv, rows=nb * S, ld=3 * E, dh=dh, n_q=H, n_k=H, inv_freq=self.u2t_inv_freq, pos_div=1, pos_mod=S)
        q5 = qkv.view(nb, S, 3, H, dh)
        ctx = torch.empty(nb, S, E, device=self.dev, dtype=BF16)
        if w.seq_first:
            # nn.MultiheadAttention fallback: the reference hands it [nb, S, E] with batch_first=False, so the attention
            # runs ALONG dim 0 (length nb) for each of the S positions: the same kernels on transposed views, no copies
            q5, ctx_v = q5.transpose(0, 1), ctx.transpose(0, 1)
            self._attention(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], ctx_v, 1.0 / math.sqrt(dh))
        else:
            self._attention(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], ctx, 1.0 / math.sqrt(dh), rel_bias=w.rel)
        return ops.linear(ctx.view(nb * S, E), w.wd, w.bd, residual=residual)

    def _u2t_temporal_attention(self, x2: torch.Tensor, B: int, C: int, N: int, w: _SelfAttnW) -> torch.Tensor:
        """Attention across the C frames of every (batch, token); rows stay in (b, c, n) order so the two
        permute+contiguous copies of the reference (svr.py:33,36) disappear."""
        g = self.g
        E, H = g.hidden_size, g.u2t_num_heads
        dh = E // H
        qkv = ops.linear(x2, w.wqkv, w.bqkv)
        if w.seq_first:
            # nn.MultiheadAttention fallback: the reference's [B*N, C, E] input is read sequence-first, i.e. attention
            # over the B*N (batch, token) pairs of every frame c. Rows are (b, c, n): for B = 1 that is plain attention
            # with the frames as the batch; B > 1 regroups the rows frame-major (the one copy this rare path pays).
            if B > 1:
                qkv = qkv.view(B, C, N, 3 * E).transpose(0, 1).contiguous()
            q5 = qkv.view(C, B * N, 3, H, dh)
            ctx = torch.empty(C, B * N, E, device=self.dev, dtype=BF16)
            self._attention(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], ctx, 1.0 / math.sqrt(dh))
            if B > 1:
                ctx = ctx.view(C, B, N, E).transpose(0, 1).contiguous()
            return ops.linear(ctx.view(B * C * N, E), w.wd, w.bd)
        if g.attn_type == "rope":
            ops.rope(qkv, rows=B * C * N, ld=3 * E, dh=dh, n_q=H, n_k=H, inv_freq=self.u2t_inv_freq, pos_div=N, pos_mod=C)
        ctx = torch.empty(B * C * N, E, device=self.dev, dtype=BF16)
        ops.temporal_attention(qkv, ctx, B=B, C_=C, N=N, H=H, dh=dh, scale=1.0 / math.sqrt(dh), rel_bias=w.rel,
                               rel_max=REL_MAX)
        return ops.linear(ctx, w.wd, w.bd)

    def _cross_attention(self, q_in: torch.Tensor, kv_in: torch.Tensor, B: int, Sq: int, Sk: int, w: _CrossAttnW,
                         residual: Optional[torch.Tensor]) -> torch.Tensor:
        """MultiHeadCrossAttention (reference tta.py:42-69), no mask; linagg when w.wd is None."""
        g = self.g
        E, H = g.hidden_size, g.u2t_num_heads
        dh = E // H
        q = ops.linear(q_in, w.wq, w.bq).view(B, Sq, H, dh)
        ctx = torch.empty(B, Sq, E, device=self.dev, dtype=BF16)
        if w.wd is None:
            k = ops.linear(kv_in, w.wkv, w.bkv).view(B, Sk, H, dh)
            v = kv_in.view(B, Sk, H, dh)
            self._attention(q, k, v, ctx, 1.0 / math.sqrt(dh))
            return ctx.view(B * Sq, E)
        kv = ops.linear(kv_in, w.wkv, w.bkv).view(B, Sk, 2, H, dh)
        self._attention(q, kv[:, :, 0], kv[:, :, 1], ctx, 1.0 / math.sqrt(dh))
        return ops.linear(ctx.view(B * Sq, E), w.wd, w.bd, residual=residual)

    def _token_selection_diff(self, x2: torch.Tensor, B: int, T: int) -> torch.Tensor:
        """DifferentiableTokenSelection (reference svr.py:101-117) without the 1024-iteration Python loop:
        scores^T = W_s X^T, softmax over the TOKEN axis, selected = softmax^T-weights @ X.
        (score_net.bias is constant along the softmax axis and cancels exactly.)"""
        g = self.g
        E, K = g.hidden_size, self.score_w.shape[0]
        Tp = _pad8(T)
        scT = torch.empty(K, B * T, device=self.dev, dtype=F32)
        ops.gemm(self.score_w, x2, scT, M=K, N=B * T, K=E, lda=E, ldb=E, ldc=B * T)
        pT = torch.empty(B, K, Tp, device=self.dev, dtype=BF16)
        ops.softmax(scT, pT, n0=B, H=1, S=K, n=T, in_strides=(T, 0, B * T), out_strides=(K * Tp, 0, Tp))
        sel = torch.empty(B, K, E, device=self.dev, dtype=BF16)
        # weights [K, T] @ X [T, E] with X as stored (MN-major B operand): no transposed copy of the tokens
        ops.gemm(pT, x2, sel, M=K, N=E, K=T, lda=Tp, ldb=E, ldc=E, zo=B, a_strides=(0, K * Tp), b_strides=(0, T * E),
                 c_strides=(0, K * E), b_mn=True)
        return sel

    def _token_selection_hard(self, x2: torch.Tensor, B: int, T: int) -> torch.Tensor:
        """TokenSelection (reference svr.py:75-91): Linear(E->1) scores, top-k over frames*tokens (sorted
        descending like torch.topk), gather. The scalar bias shifts every score alike and cannot change the
        selection."""
        g = self.g
        E, K = g.hidden_size, g.u2t_top_k
        if K > T:
            raise RuntimeError(f"selected index k out of range: top_k={K} > {T} tokens (torch.topk raises too)")
        sc = torch.empty(B * T, 1, device=self.dev, dtype=F32)
        ops.gemm(x2, self.score_w, sc, M=B * T, N=1, K=E, lda=E, ldb=E, ldc=1)
        idx = ops.topk_rows(sc.view(B, T), K, idx_offset_per_row=T)  # row-global indices into x2
        self.last_selection = idx
        return ops.embed_splice(idx, x2, None)

    def u2tokenizer(self, v_tokens: torch.Tensor, t_tokens: torch.Tensor) -> torch.Tensor:
        """u2Tokenizer.forward (reference u2Tokenizer.py:40-47): v_tokens [B, C, N, E], t_tokens [B, Lt, E]
        -> [B, num_3d_query_token, E]."""
        g = self.g
        B, C, N, E = v_tokens.shape
        Lt = t_tokens.shape[1]
        x = v_tokens.reshape(B * C * N, E)
        for sp, tp in self.svr:
            x = self._u2t_self_attention(x, B * C, N, sp)
            x = self._u2t_temporal_attention(x, B, C, N, tp)
        if g.enable_diffts:
            sel = self._token_selection_diff(x, B, C * N)
        else:
            sel = self._token_selection_hard(x, B, C * N)
        vis = ops.multiscale_pool(sel, self.gate_w, self.gate_b, g.enable_dmtp) if g.use_multi_scale else sel
        Mv = vis.shape[1]
        vis2 = vis.view(B * Mv, E)
        txt2 = t_tokens.reshape(B * Lt, E)
        Q = g.num_3d_query_token
        q = self.queries.unsqueeze(0).expand(B, Q, E).contiguous().view(B * Q, E)
        for w in self.tta:
            s = self._u2t_self_attention(q, B, Q, w["self_attn"], residual=q)
            s = ops.layernorm(s, w["ns"][0], w["ns"][1], 1e-5)
            v = self._cross_attention(s, vis2, B, Q, Mv, w["vis"], residual=s)
            v = ops.layernorm(v, w["nv"][0], w["nv"][1], 1e-5)
            t = self._cross_attention(v, txt2, B, Q, Lt, w["txt"], residual=v)
            q = ops.layernorm(t, w["nt"][0], w["nt"][1], 1e-5)
        out = self._cross_attention(q, vis2, B, Q, Mv, self.linagg, residual=None)
        return out.view(B, Q, E)

    # =========================================================================================
    # multimodal front (prepare_inputs_for_multimodal, reference u2_arch.py:101-122)
    # =========================================================================================
    def visual_tokens(self, images: torch.Tensor, question_ids: Optional[torch.Tensor]) -> torch.Tensor:
        g = self.g
        if g.enable_u2tokenizer:
            B, C = images.shape[0], images.shape[1]
            feats = self.encode_images(images.reshape(B * C, 1, *images.shape[2:]))
            v_tokens = feats.view(B, C, feats.shape[-2], feats.shape[-1])
            if question_ids is None:
                raise ValueError("question_ids is required when the mu2-tokenizer is enabled")
            t_tokens = ops.embed_splice(question_ids.to(self.dev), self.embed, None)
            return self.u2tokenizer(v_tokens, t_tokens)
        return self.encode_images(images)

    def multimodal_embeds(self, input_ids: torch.Tensor, images: torch.Tensor,
                          question_ids: Optional[torch.Tensor]) -> torch.Tensor:
        vis = self.visual_tokens(images, question_ids)
        return ops.embed_splice(input_ids.to(self.dev), self.embed, vis)

    def embed_tokens(self, input_ids: torch.Tensor) -> torch.Tensor:
        return ops.embed_splice(input_ids.to(self.dev), self.embed, None)

    def forward_logits(self, input_ids: torch.Tensor, images: torch.Tensor, question_ids: Optional[torch.Tensor],
                       use_graph: Optional[bool] = None) -> torch.Tensor:
        """Teacher-forced forward with images: vision tower -> mu2-tokenizer -> splice -> decoder prefill -> lm_head,
        [B, L, V] fp32 logits. The ~600 launches of one forward are short (a 256x256x128 study is ~6 ms of kernels), so
        from the second call with the same shapes on the whole sequence replays as ONE CUDA graph over static buffers
        (U2_FWD_GRAPH=0 keeps it eager)."""
        from . import _lib
        if use_graph is None:
            use_graph = self.fwd_graph
        key = (tuple(images.shape), images.dtype, tuple(input_ids.shape),
               None if question_ids is None else tuple(question_ids.shape))
        st = self._fwd_state if (self._fwd_state is not None and self._fwd_state["key"] == key) else None
        if st is None:
            self._fwd_state = None  # drop the previous graph (and its memory pool) first
            st = dict(key=key, calls=0, graph=None)
            self._fwd_state = st
        st["calls"] += 1

        def run(ids, im, q):
            emb = self.multimodal_embeds(ids, im, q)
            return self.lm_logits(self.prefill(emb))

        def capture():
            st["logits"] = run(st["ids"], st["images"], st["q"])

        if not use_graph or st["calls"] < 2:  # the first call runs eagerly (it also configures the kernels' attributes)
            return run(input_ids, images, question_ids)
        if st["graph"] is None:
            st["ids"] = input_ids.to(self.dev).clone()
            st["images"] = images.to(self.dev).clone()
            st["q"] = None if question_ids is None else question_ids.to(self.dev).clone()
            torch.cuda.synchronize()
        st["ids"].copy_(input_ids, non_blocking=True)
        st["images"].copy_(images, non_blocking=True)
        if st["q"] is not None:
            st["q"].copy_(question_ids, non_blocking=True)
        self._replay(st, capture)
        return st["logits"].clone()

    @staticmethod
    def _replay(st: dict, capture) -> None:
        """Replays the CUDA graph st["graph"], recording capture() into it first when it is None. _lib counts kernels as
        they are launched: a capture records them without running them, so its count (st["n"]) is taken back once and
        added on every replay."""
        if st["graph"] is None:
            graph = torch.cuda.CUDAGraph()
            n0 = _lib.launches()
            with torch.cuda.graph(graph):
                capture()
            st["n"] = _lib.launches() - n0
            _lib.add_launches(-st["n"])
            st["graph"] = graph
        st["graph"].replay()
        _lib.add_launches(st["n"])

    # =========================================================================================
    # decoder: prefill
    # =========================================================================================
    def new_cache(self, batch: int, max_len: int) -> "KVCache":
        return KVCache(self.g, batch, max_len, self.dev)

    def prefill(self, embeds: torch.Tensor, cache: Optional["KVCache"] = None) -> torch.Tensor:
        """Decoder stack over a full prompt [B, L, E] (causal, positions 0..L-1); fills `cache` when given.
        Returns the final-norm hidden states [B, L, E]."""
        g = self.g
        B, L, E = embeds.shape
        hq, hkv, dh, I = g.num_attention_heads, g.num_key_value_heads, g.head_dim, g.intermediate_size
        if cache is not None and (cache.batch != B or cache.max_len < L or cache.length != 0):
            raise ValueError("prefill needs an empty cache with matching batch and max_len >= prompt length")
        x = embeds.reshape(B * L, E).clone()
        y = torch.empty_like(x)
        nqkv = (hq + 2 * hkv) * dh
        qkv = torch.empty(B * L, nqkv, device=self.dev, dtype=BF16)
        ctx = torch.empty(B, L, hq * dh, device=self.dev, dtype=BF16)
        gu = torch.empty(B * L, 2 * I, device=self.dev, dtype=BF16)
        act = torch.empty(B * L, I, device=self.dev, dtype=BF16)
        q4 = qkv.view(B, L, hq + 2 * hkv, dh)
        for li, w in enumerate(self.layers):
            ops.rmsnorm(x, w["ln1"], g.rms_norm_eps, out=y)
            ops.linear(y, w["wqkv"], out=qkv)
            kc, vc = (cache.k[li], cache.v[li]) if cache is not None else (None, None)
            ops.rope(qkv, rows=B * L, ld=nqkv, dh=dh, n_q=hq, n_k=hkv, n_v=hkv if cache is not None else 0,
                     inv_freq=self.inv_freq, q_norm_w=w["qn"], k_norm_w=w["kn"], eps=g.rms_norm_eps, pos0=0, pos_div=1,
                     pos_mod=L, k_cache=kc, v_cache=vc, Tmax=cache.max_len if cache is not None else 0, rows_per_batch=L)
            self._attention(q4[:, :, :hq], q4[:, :, hq:hq + hkv], q4[:, :, hq + hkv:], ctx, 1.0 / math.sqrt(dh), causal=True,
                            window=g.window)
            ops.linear(ctx.view(B * L, hq * dh), w["wo"], residual=x, out=x)
            ops.rmsnorm(x, w["ln2"], g.rms_norm_eps, out=y)
            ops.linear(y, w["wgu"], out=gu)
            ops.silu_mul(gu, act, interleaved=True)
            ops.linear(act, w["wdown"], residual=x, out=x)
        if cache is not None:
            cache.set_length(L)
        ops.rmsnorm(x, self.final_norm, g.rms_norm_eps, out=y)
        return y.view(B, L, E)

    def lm_logits(self, hidden: torch.Tensor, out_dtype=F32) -> torch.Tensor:
        """lm_head over [.., E] hidden states -> [.., V] logits."""
        return ops.linear(hidden, self.lm_head, out_dtype=out_dtype)

    def token_logps(self, hidden: torch.Tensor, labels: torch.Tensor, *, want_lse=False, want_logit_sum=False,
                    nll_acc: Optional[torch.Tensor] = None):
        """log_softmax(lm_head(hidden))[labels] per position without materialising the [.., V] logits
        (reference: lm_head + trl selective_log_softmax, src/train/dpo_u2trainer.py:267-300). hidden [.., E] bf16,
        labels [..] int64 (< 0: ignored, log-probability 0). Returns (logp, lse or None, logit_sum or None), fp32 [..]."""
        shp = labels.shape
        h2 = hidden.reshape(-1, hidden.shape[-1])
        if not h2.is_contiguous():
            h2 = h2.contiguous()
        logp, lse, lsum = ops.lmhead_logprob(h2, self.lm_head, labels.reshape(-1).contiguous(), want_lse=want_lse,
                                             want_logit_sum=want_logit_sum, nll_acc=nll_acc)
        rs = lambda t: None if t is None else t.view(shp)
        return rs(logp), rs(lse), rs(lsum)

    # =========================================================================================
    # decoder: one KV-cached decode step (weight streaming)
    # =========================================================================================
    def _decode_buffers(self, B: int):
        g = self.g
        key = ("dec", B)
        if getattr(self, "_dec_key", None) != key:
            if getattr(self, "_gen_state", None) is not None:
                self._gen_state["graph"] = None  # a captured step points at the buffers that are about to be replaced
            hq, hkv, dh, I, E = g.num_attention_heads, g.num_key_value_heads, g.head_dim, g.intermediate_size, g.hidden_size
            d = self.dev
            self._dec = dict(
                x=torch.empty(B, E, device=d, dtype=BF16), qkv=torch.empty(B, (hq + 2 * hkv) * dh, device=d, dtype=BF16),
                ctx=torch.empty(B, hq * dh, device=d, dtype=BF16), act=torch.empty(B, I, device=d, dtype=BF16),
                logits=torch.empty(B, g.vocab_size, device=d, dtype=F32), ids=torch.zeros(B, 1, device=d, dtype=torch.int64),
                xg=torch.empty(B, E, device=d, dtype=BF16), xg2=torch.empty(B, E, device=d, dtype=BF16),
                ssq_a=torch.zeros(16, device=d, dtype=F32),
                ssq_b=torch.zeros(16, device=d, dtype=F32))
            max_n = max(g.vocab_size, 2 * I, (hq + 2 * hkv) * dh, E)
            shapes = [((hq + 2 * hkv) * dh, E), (E, hq * dh), (2 * I, E), (E, I), (g.vocab_size, E)]
            # two of each: consecutive ops of a chained launch overlap in time (fine-grained dataflow)
            wse = max(ops.dlinear_ws_elems(n, k) for n, k in shapes)
            self._dec["ws"] = ops.dlinear_new_ws(wse, device=d, lead=(2,))
            self._dec["counters"] = torch.zeros(2, (max_n + 63) // 64 + 8, device=d, dtype=torch.int32)
            self._dec["flags"] = torch.zeros(g.num_hidden_layers, 4, 256, device=d, dtype=torch.int32)
            self._dec["gridbar"] = torch.zeros(4 * g.num_hidden_layers, device=d, dtype=torch.int32)
            self._dec["step"] = torch.zeros(1, device=d, dtype=torch.int32)
            self._dec_key = key
        return self._dec

    def reset_decode_state(self, B: int):
        """Grid-barrier epochs / self-cleaning workspaces back to zero (start of a generation, or after an
        interrupted step)."""
        bufs = self._decode_buffers(B)
        for k in ("gridbar", "step", "counters", "ssq_a", "ssq_b", "flags"):
            bufs[k].zero_()
        bufs["ws"].view(torch.int32).fill_(-1)  # "empty slot" sentinel

    def _kv_splits(self, B: int) -> int:
        """CTAs per (sequence, KV head) in the decode attention: fill the SMs when B * Hkv is small
        (cfg 3: 4 * 8 = 32 pairs -> clusters of 4 = 128 CTAs). U2_ATTN_SPLIT=0/1 disables, 2/4/8 forces."""
        import os
        env = os.environ.get("U2_ATTN_SPLIT", "auto")
        if env != "auto":
            return max(1, int(env))
        pairs = B * self.g.num_key_value_heads
        s = 8
        while s > 1 and pairs * s > max(self.num_sms, pairs):
            s //= 2
        return s

    def _use_tc_decode(self, B: int) -> bool:
        g = self.g
        dims = (g.hidden_size, g.intermediate_size, g.num_attention_heads * g.head_dim)
        return self.decode_impl == "tcgen05" and B <= 16 and all(k % 64 == 0 for k in dims)

    def _decode_rows(self) -> int:
        """Sequences one decode step carries: 16 (the dlinear N) on the wgmma path, 8 (the GEMV batch) otherwise."""
        tc_rows = 16
        return tc_rows if self._use_tc_decode(tc_rows) else 8

    def decode_step_tc(self, cache: "KVCache", req: Optional[GenerateRequest] = None,
                       slots: Optional[dict] = None) -> torch.Tensor:
        """Decode step with every linear on the wgmma stream-K kernel and the RMSNorms folded into its
        epilogues. Launches per step: embed, qkv(0), then per layer [fused attention, one multi-op launch
        o_proj -> gate|up -> down -> next qkv (or lm_head)], argmax  =  2 launches per layer."""
        g = self.g
        B = cache.batch
        hq, hkv, dh = g.num_attention_heads, g.num_key_value_heads, g.head_dim
        bufs = self._decode_buffers(B)
        x, qkv, ctx, act, logits, ids, xg_a, xg_b = (bufs[k] for k in ("x", "qkv", "ctx", "act", "logits", "ids", "xg", "xg2"))
        ssq_a, ssq_b, ws, cnt, flags = bufs["ssq_a"], bufs["ssq_b"], bufs["ws"], bufs["counters"], bufs["flags"]
        gridbar, step = bufs["gridbar"], bufs["step"]
        eps = g.rms_norm_eps
        nl = len(self.layers)
        c0 = dict(ws=ws[0], counters=cnt[0], sched=self.dl_sched)
        c1 = dict(ws=ws[1], counters=cnt[1], sched=self.dl_sched)
        packed = {} if (self._decode_bf16 or self.dl_sched != 0) else self._packed  # the kM = 64 schedule reads bf16

        def launch_w(keys):
            """One launch's weights: all packed when every one of them is, else all bf16 (a launch has one format)."""
            pk = [packed.get(k) for k in keys]
            if all(p is not None for p in pk):
                return pk
            return [self.lm_head if k == ("head",) else self.layers[k[0]][k[1]] for k in keys]

        ops.decode_embed(ids, self.embed, self.layers[0]["ln1"], x, xg_b, ssq_b, ssq_a, step)
        ops.dlinear(xg_b, launch_w([(0, "wqkv")])[0], qkv, ssq_in=ssq_b, eps=eps, pdl=self.pdl, **c1)
        for li, w in enumerate(self.layers):
            ops.decode_attention_fused(qkv, cache.k[li], cache.v[li], ctx, B=B, Hq=hq, Hkv=hkv, dh=dh, Tmax=cache.max_len,
                                       inv_freq=self.inv_freq, scale=1.0 / math.sqrt(dh), pos_dev=cache.length_dev,
                                       q_norm_w=w["qn"], k_norm_w=w["kn"], eps=eps, kv_splits=self._kv_splits(B),
                                       pdl=self.pdl and self.attn_pdl, pos_per_seq=True, kv_src=cache.kv_src,
                                       window=g.window)
            last = li + 1 == nl
            g_next = self.final_norm if last else self.layers[li + 1]["ln1"]
            fl = flags[li] if (self.multi_op and self.fine_deps) else [None] * 4
            dep = lambda i, shift: dict(dep_flags=fl[i], dep_shift=shift) if fl[i] is not None else {}
            wo, wgu, wdown, wnext = launch_w([(li, "wo"), (li, "wgu"), (li, "wdown"), ("head",) if last else (li + 1, "wqkv")])
            chain = [
                (ctx, wo, x, dict(residual=x, gamma_next=w["ln2"], xg=xg_a, ssq_out=ssq_a, ssq_zero=ssq_b,
                                  out_flags=fl[0], **c0)),
                (xg_a, wgu, act, dict(ssq_in=ssq_a, eps=eps, silu_pair=True, out_flags=fl[1], **dep(0, 1), **c1)),
                (act, wdown, x, dict(residual=x, gamma_next=g_next, xg=xg_b, ssq_out=ssq_b, ssq_zero=ssq_a,
                                     out_flags=fl[2], **dep(1, 0), **c0)),
                (xg_b, wnext, logits if last else qkv, dict(ssq_in=ssq_b, eps=eps, **dep(2, 1), **c1)),
            ]
            if self.multi_op:
                # L2 look-ahead: next layer's o_proj (all of it) and the head of its gate|up stream
                nxt = () if (last or self.l2_next_units < 0) else tuple(
                    zip(launch_w([(li + 1, "wo"), (li + 1, "wgu")]), (1 << 20, self.l2_next_units)))
                ops.dlinear_multi(chain, gridbar=gridbar[li * 4:(li + 1) * 4], step_dev=step, pdl=self.pdl,
                                  lookahead_units=self.l2_lookahead_units, next_weights=nxt,
                                  pre_stages=self.pre_stages)
            else:
                for (xi, wi, yi, kw) in chain:
                    ops.dlinear(xi, wi, yi, pdl=self.pdl, **kw)
        self._pick_or_slot_pick(logits, ids.view(B), bufs["step"], req, cache, slots)
        return logits

    def _pick_or_slot_pick(self, logits, ids_out, step_dev, req, cache: "KVCache", slots: Optional[dict]):
        """The end of a decode step: the pick and cache.advance_device(), or with `slots` (a continuous-batching state)
        the per-slot pick and slot bookkeeping of _slot_pick."""
        if slots is None:
            self._pick_next(logits, ids_out, step_dev, req)
            cache.advance_device()
        else:
            self._slot_pick(logits, ids_out, slots, req, cache)

    def _slot_pick(self, logits: torch.Tensor, ids_out: torch.Tensor, st: dict, req: GenerateRequest,
                   cache: Optional["KVCache"] = None):
        """The token-picking head of continuous batching: _pick_next with the seed, RNG row and step (history length) of
        every row read from its slot record st['slots'], so each slot picks what its request would pick decoded alone;
        then ops.slot_update appends the picks to st['out'], finishes slots on EOS / max_new_tokens, feeds st['pad'] to
        finished slots and advances the cache lengths of the others. cache None: an admission's first pick, from the
        prefill logits (the host sets its lengths)."""
        if req.processors is not None:
            blk = self._param_block("logits processors", ops.logits_proc_params, self.g.vocab_size,
                                    **asdict(req.processors))
            ops.logits_process_slots(logits, blk, ids_out, st["hist"], st["slots"])
        lp = (st["lp_step"], st["lp"]) if req.return_logprobs else None
        if req.sampling is None:
            ops.argmax(logits, ids_out)
            if lp is not None:
                ops.pick_logprob(logits, ids_out, lp[0])
        else:
            params = self._param_block("sampling parameters", ops.sample_params, *req.sampling)
            if lp is not None:
                ops.sample_out(logits, params, ids_out, logprob=lp[0], slots=st["slots"])
            else:
                ops.sample_slots(logits, params, st["slots"], ids_out)
        ops.slot_update(ids_out, st["slots"], st["out"],
                        self._param_block("slot parameters", ops.slot_params, st["pad"], req.eos_token_id),
                        None if cache is None else cache.length_dev, None if cache is None else cache.length_plus1_dev,
                        lp=lp)

    def _pick_next(self, logits: torch.Tensor, ids_out: torch.Tensor, step_dev: Optional[torch.Tensor],
                   req: Optional[GenerateRequest], step: int = 0):
        """Greedy argmax (req None: plain argmax), or the sampled head (temperature -> top-k -> top-p -> multinomial)
        when the request samples (HF generate(do_sample=True, ...), reference eval/mrg.py:74-75). The request's logits
        processors rewrite the logits in place first, from the generation state's history of generated tokens.
        Beam search replaces all of it with the beam step (_beam_pick). The requested outputs are stored at the step:
        the raw logits before the processors, the scores (processed logits, or the sampler's warped row) after them."""
        if req is not None and req.output_logits:
            ops.store_rows(logits, self._row_store("logits"), step=step, step_dev=step_dev)
        if req is not None and req.beam is not None:
            return self._beam_pick(logits, ids_out, step_dev, req, step)
        if req is not None and req.processors is not None:
            blk = self._param_block("logits processors", ops.logits_proc_params, self.g.vocab_size,
                                    **asdict(req.processors))
            ops.logits_process(logits, blk, ids_out, self._gen_state["hist"], step=step, step_dev=step_dev)
        if req is None or req.sampling is None:
            if req is not None and req.output_scores:
                ops.store_rows(logits, self._row_store("scores"), step=step, step_dev=step_dev)
            ops.argmax(logits, ids_out)
        else:
            # parameters (seed included) are read from a device block: the captured decode graph survives a new
            # request's seed / temperature / top-k / top-p
            params = self._param_block("sampling parameters", ops.sample_params, *req.sampling)
            if req.output_scores:
                ops.sample_out(logits, params, ids_out, scores=self._row_store("scores"), step=step, step_dev=step_dev)
            else:
                ops.sample_dev(logits, params, ids_out, step=step, step_dev=step_dev)

    def _set_row_store(self, what: str, dst: torch.Tensor) -> None:
        """Points the `what` row store ("logits" or "scores") at dst, an fp32 [steps, rows, V] view: the decode steps of
        the chunk that follows store step t's rows into dst[t]. Call it before the chunk's first (eager) pick."""
        self._param_block(what + " store", ops.row_store_params, **ops.row_store_dst(dst))

    def _row_store(self, what: str) -> torch.Tensor:
        return self._param_blocks[what + " store"][1]

    def _param_block(self, what: str, make, *args, **kw) -> torch.Tensor:
        """The device block make(self.dev, *args, **kw) builds (ops.sample_params, logits_proc_params or beam_params),
        which the decode step reads. A captured decode graph keeps the block's address, so there is one block per
        `what`, allocated on first use and rewritten in place (make(..., out=block)) only when the arguments change:
        that is how a new request's values reach the graph without a new capture. A change during a capture would not
        be recorded, so it is refused."""
        host = (args, kw)
        blk = self._param_blocks.get(what)
        if blk is None:
            self._param_blocks[what] = blk = [host, make(self.dev, *args, **kw)]
        elif blk[0] != host:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError(f"{what} changed inside a CUDA-graph capture")
            make(self.dev, *args, out=blk[1], **kw)
            blk[0] = host
        return blk[1]

    def _beam_pick(self, logits: torch.Tensor, ids_out: torch.Tensor, step_dev: Optional[torch.Tensor],
                   req: GenerateRequest, step: int):
        """HF's beam step: log_softmax -> logits processors (on the log-probs) -> per-row top beams_to_keep of
        log-prob + running score -> per-prompt merge and bookkeeping, which also writes the next ids and reorders the
        cache indirection table and the processor history. logits keeps the raw logits."""
        st = self._gen_state
        bs, bm = st["beam"], req.beam
        blk = self._param_block("beam search parameters", ops.beam_params, num_beams=bm.num_beams,
                                length_penalty=bm.length_penalty, early_stopping=bm.early_stopping,
                                max_new_tokens=req.max_new_tokens, eos_token_ids=req.eos_token_id)
        lp = ops.log_softmax(logits, bs["lp"])
        if req.processors is not None:
            pblk = self._param_block("logits processors", ops.logits_proc_params, self.g.vocab_size,
                                     **asdict(req.processors))
            ops.logits_process(lp, pblk, ids_out, st["hist"], step=step, step_dev=step_dev)
        if req.output_scores:
            ops.store_rows(lp, self._row_store("scores"), step=step, step_dev=step_dev)
        ops.beam_topk(lp, bs["running"], bs["flags"], blk, bs["cand_val"], bs["cand_tok"])
        ops.beam_step(blk, bs, ids_out, st["cache"].kv_src, st["cache"].length_dev, V=logits.shape[1],
                      hist=st.get("hist"), step=step, step_dev=step_dev)

    def decode_step(self, cache: "KVCache", req: Optional[GenerateRequest] = None,
                    slots: Optional[dict] = None) -> torch.Tensor:
        """Consumes buffers['ids'] [B,1] (the last token of every sequence), appends sequence b to the cache at
        position cache.length_dev[b] (read on the device), leaves fp32 logits in buffers['logits'] and the next ids
        back in buffers['ids'], picked as `req` asks (None: greedy argmax). Launch sequence is CUDA-graph capturable.
        slots: the state of a continuous-batching call (_SlotDecoder), whose rows pick per slot (_slot_pick)."""
        g = self.g
        B = cache.batch
        if self._use_tc_decode(B):
            return self.decode_step_tc(cache, req, slots)
        hq, hkv, dh = g.num_attention_heads, g.num_key_value_heads, g.head_dim
        bufs = self._decode_buffers(B)
        x, qkv, ctx, act, logits, ids = (bufs[k] for k in ("x", "qkv", "ctx", "act", "logits", "ids"))
        ops.embed_splice(ids, self.embed, None, out=x)  # [B, 1, E] gathered straight into x
        nqkv = (hq + 2 * hkv) * dh
        for li, w in enumerate(self.layers):
            ops.gemv(x, w["wqkv"], qkv, norm_gamma=w["ln1"], norm_eps=g.rms_norm_eps)
            ops.rope(qkv, rows=B, ld=nqkv, dh=dh, n_q=hq, n_k=hkv, n_v=hkv, inv_freq=self.inv_freq, q_norm_w=w["qn"],
                     k_norm_w=w["kn"], eps=g.rms_norm_eps, pos0=0, pos_div=1, pos_mod=1, pos0_dev=cache.length_dev,
                     k_cache=cache.k[li], v_cache=cache.v[li], Tmax=cache.max_len, rows_per_batch=1, pos0_per_batch=True)
            ops.decode_attention(qkv, cache.k[li], cache.v[li], ctx, B=B, Hq=hq, Hkv=hkv, dh=dh, Tmax=cache.max_len,
                                 T_dev=cache.length_plus1_dev, ldq=nqkv, ldo=hq * dh, scale=1.0 / math.sqrt(dh),
                                 T_per_seq=True, kv_src=cache.kv_src, window=g.window)
            ops.gemv(ctx, w["wo"], x, residual=x)
            ops.gemv(x, w["wgu"], act, norm_gamma=w["ln2"], norm_eps=g.rms_norm_eps, silu_pair=True)
            ops.gemv(act, w["wdown"], x, residual=x)
        ops.gemv(x, self.lm_head, logits, norm_gamma=self.final_norm, norm_eps=g.rms_norm_eps)
        bufs["step"] += 1  # the gemv path has no decode_embed kernel to bump the step counter
        self._pick_or_slot_pick(logits, ids.view(B), bufs["step"], req, cache, slots)
        return logits

    # =========================================================================================
    # generation (reference u2llama.py:90-127): greedy, sampled, multi-sample and beam search through one driver
    # =========================================================================================
    @torch.no_grad()
    def generate(self, embeds: torch.Tensor, max_new_tokens: int, eos_token_id=None, do_sample: bool = False,
                 temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0, seed: int = 0, use_graph: bool = True,
                 num_return_sequences: int = 1, lengths=None, processors: Optional[LogitsProcessors] = None,
                 beam: Optional[BeamSearch] = None, output_scores: bool = False, output_logits: bool = False):
        """Greedy (do_sample=False) or sampled decoding; same loop, only the token-picking head differs.
        processors (optional): HF's repetition penalty / no-repeat n-gram / bad words / min new tokens, applied to every
        step's logits before the pick; every row of a chunk of rows keeps its own history of generated tokens.
        num_return_sequences > 1 (HF semantics: row b * n + s is sample s of prompt b) shares ONE vision + prefill pass:
        the prompt's KV rows are replicated into the decode cache (the reference's DPO-data workflow draws 8 samples per
        study by re-running the whole model per sample, green_refactored/pred_then_green.py:77-83).
        lengths [B] (optional): prompt b is embeds[b, :lengths[b]] (right padding after it); it decodes from position
        lengths[b] on, as if it ran alone. None = every prompt fills the whole width.
        beam (num_beams > 1): HF beam search instead of the greedy / sampled pick (do_sample and num_return_sequences are
        then ignored; the beam config carries its own num_return_sequences).
        output_scores / output_logits (HF generate's): the call returns (ids, scores, logits), each of the last two an fp32
        [max_new_tokens, rows, V] tensor (or None when not asked) whose step t holds every row's scores (greedy: the
        processed logits; sampled: the warped row, -inf where top-k / top-p dropped the token; beam: the processed
        log-probs of all num_beams rows of every prompt) / raw logits. They cost max_new_tokens * rows * V * 4 bytes each,
        allocated before decoding starts so that an out-of-memory error comes first; steps after a chunk of rows stopped
        early (every row hit EOS) hold 0."""
        lens = self._row_lengths(lengths, embeds.shape[0], embeds.shape[1])
        outputs = dict(output_scores=bool(output_scores), output_logits=bool(output_logits))
        if beam is not None and beam.num_beams > 1:
            return self._generate(embeds, GenerateRequest(max_new_tokens, eos_token_id, processors=processors,
                                                          beam=beam, **outputs), lens, use_graph)
        sampling = (float(temperature), int(top_k or 0), float(top_p), int(seed)) if do_sample else None
        req = GenerateRequest(max_new_tokens, eos_token_id, sampling, processors, **outputs)
        return self._generate(embeds, req, lens, use_graph, max(1, int(num_return_sequences)))

    def generate_greedy(self, embeds: torch.Tensor, max_new_tokens: int, eos_token_id=None,
                        use_graph: bool = True, return_margins: bool = False, force_ids: Optional[torch.Tensor] = None,
                        logits_out: Optional[list] = None, lengths=None,
                        processors: Optional[LogitsProcessors] = None):
        """Prefill on `embeds` [B, L, E], then max_new_tokens greedy decode steps. Returns new ids [B, n] (and the
        per-step top-1/top-2 logit margins when asked, for margin-aware parity checks). processors: as for generate();
        the margins and logits_out then hold the processed logits.
        force_ids [B, n] (parity tests): teacher forcing - the returned ids are still this engine's own picks, but the
        token fed to the next step is force_ids[:, step], so one near-tie cannot derail the rest of the comparison.
        logits_out: a list that receives a copy of every step's fp32 logits [B, V].
        return_margins, force_ids and logits_out need a batch that fits one decode step (_decode_rows()).
        lengths [B] (optional): prompt b is embeds[b, :lengths[b]]. The prefill runs over the padded width; causal
        attention keeps the real positions exact, and the cache rows from lengths[b] on are overwritten by the decode
        steps before any step reads them."""
        margins = [] if return_margins else None
        ids = self._generate(embeds, GenerateRequest(max_new_tokens, eos_token_id, processors=processors),
                             self._row_lengths(lengths, embeds.shape[0], embeds.shape[1]), use_graph,
                             margins=margins, force_ids=force_ids, logits_out=logits_out)
        return (ids, torch.stack(margins, dim=1)) if return_margins else ids

    def _generate(self, embeds: torch.Tensor, req: GenerateRequest, lens: torch.Tensor, use_graph: bool = True,
                  num_return_sequences: int = 1, margins: Optional[list] = None,
                  force_ids: Optional[torch.Tensor] = None, logits_out: Optional[list] = None) -> torch.Tensor:
        """The decode driver of every generate() mode. Every prompt gets n rows, num_beams for beam search and
        num_return_sequences otherwise, decoded in the chunks chunk_plan() lays out over the rows one decode step
        carries. With n > 1 the prompts are prefilled once and each chunk copies its rows' prompt KV from that cache;
        with n == 1 each chunk prefills its own prompts straight into its decode cache.
        lens: the CPU prompt lengths of _row_lengths(). margins / force_ids / logits_out: the hooks of generate_greedy()
        (logits_out also receives the raw logits of a beam search), for a request that fits one chunk.
        Greedy and sampled chunks that stop early are padded to the common width with the first EOS id; beam search
        returns n_ret hypotheses per prompt, best first, filled with HF's fill value (last_beam_scores: their scores,
        last_beam_indices: HF's beam_indices). With req.output_scores / output_logits: (ids, scores, logits), see
        generate()."""
        B, L, _ = embeds.shape
        cap, bm, eos = self._decode_rows(), req.beam, req.eos_token_id
        if bm is not None:
            K, n_ret = bm.num_beams, bm.num_return_sequences
            if K > cap:
                raise ValueError(f"num_beams={K} exceeds the {cap} rows one decode step carries on this path")
            if not 1 <= n_ret <= K:
                raise ValueError(f"num_return_sequences={n_ret} must be in 1..num_beams={K}")
            if len(eos) > _lib.BEAM_MAX_EOS:
                raise ValueError(f"beam search supports at most {_lib.BEAM_MAX_EOS} EOS ids, got {len(eos)}")
            fill = (bm.pad_token_id or eos[0]) if eos else -1
        n = bm.num_beams if bm is not None else num_return_sequences
        plan = chunk_plan(B, n, cap, bm is not None)
        if len(plan) > 1 and (margins is not None or force_ids is not None or logits_out is not None):
            raise ValueError(f"return_margins / force_ids / logits_out need at most {cap} rows, got {B * n}")
        stores = {}
        for what, on in (("scores", req.output_scores), ("logits", req.output_logits)):
            if on:  # steps x rows x V x 4 bytes, allocated before any decoding
                stores[what] = torch.zeros(req.max_new_tokens, B * n, self.g.vocab_size, device=self.dev, dtype=F32)
        if n > 1:
            pc = self.new_cache(B, L)
            logits0 = self.lm_logits(self._last_hidden(self.prefill(embeds, pc), lens))
        outs, seqs, scores, beam_idx = [], [], [], []
        r0 = 0
        for src, seed_off in plan:
            r = req if req.sampling is None else replace(req, sampling=(*req.sampling[:3], req.sampling[3] + seed_off))
            st = self._gen_state_for(len(src), L + req.max_new_tokens, r)
            cache = st["cache"]
            if n > 1:
                dev_src = src.to(self.dev)
                cache.k[:, :, :, :L].copy_(pc.k.index_select(1, dev_src))
                cache.v[:, :, :, :L].copy_(pc.v.index_select(1, dev_src))
                cache.set_length(lens[src])  # every row continues from its prompt's length
                chunk_logits0 = logits0.index_select(0, dev_src)
            else:
                cache.set_length(0)
                hidden = self.prefill(embeds[int(src[0]):int(src[-1]) + 1], cache)
                cache.set_length(lens[src])
                chunk_logits0 = self.lm_logits(self._last_hidden(hidden, lens[src]))
            for what, buf in stores.items():  # this chunk's rows of the caller's [steps, B * n, V]
                self._set_row_store(what, buf[:, r0:r0 + len(src)])
            if bm is not None:
                self._beam_loop(st, chunk_logits0, r, use_graph, logits_out)
                s, sc, bi = self._beam_backtrack(st["beam"], len(src) // K, K, n_ret, fill, row0=r0)
                seqs += s
                scores.append(sc)
                beam_idx += bi
            else:
                outs.append(self._decode_loop(st, chunk_logits0, r, use_graph, margins, force_ids, logits_out))
            r0 += len(src)
        extra = (stores.get("scores"), stores.get("logits")) if stores else ()
        if bm is not None:
            out = torch.full((len(seqs), max(len(x) for x in seqs)), fill, dtype=torch.int64)
            idx = torch.full(out.shape, -1, dtype=torch.int32)
            for i, (x, b) in enumerate(zip(seqs, beam_idx)):
                out[i, :len(x)] = torch.as_tensor(x, dtype=torch.int64)
                idx[i, :len(b)] = torch.as_tensor(b, dtype=torch.int32)
            self.last_beam_scores = torch.cat(scores)
            self.last_beam_indices = idx.to(self.dev)
            return (out.to(self.dev), *extra) if extra else out.to(self.dev)
        width = max(o.shape[1] for o in outs)
        if any(o.shape[1] != width for o in outs):  # chunks that hit EOS early: pad with EOS (masked by the caller)
            outs = [torch.nn.functional.pad(o, (0, width - o.shape[1]), value=eos[0]) for o in outs]
        out = torch.cat(outs, dim=0)
        return (out, *extra) if extra else out

    def _gen_state_for(self, B: int, cap: int, req: GenerateRequest, slot_width: int = 0):
        """The static KV cache and the captured decode-step graph are kept across calls with the same (batch, capacity,
        head configuration): capture + instantiation cost ~0.1 s, which would otherwise be paid per request. With logits
        processors the state also holds the history of generated tokens, int32 [B, cap]; with beam search (K > 1) the
        cache's indirection table and the beam buffers of ops.beam_step. slot_width > 0 (continuous batching): the slot
        records (ops.slot_state) and the generated tokens of every slot, int64 [B, slot_width]."""
        K = req.beam.num_beams if req.beam is not None else 1
        key = (B, cap, self.decode_impl, self.multi_op, self.fine_deps, req.sampling is not None,
               req.processors is not None, K, slot_width, req.output_scores, req.output_logits, req.return_logprobs)
        st = self._gen_state if (self._gen_state is not None and self._gen_state["key"] == key) else None
        if st is None:
            self._gen_state = None  # drop the old cache before allocating the new one
            st = dict(key=key, cache=self.new_cache(B, cap), graph=None)
            if req.processors is not None:
                st["hist"] = torch.zeros(B, cap, device=self.dev, dtype=torch.int32)
            if slot_width:
                st["slots"] = torch.zeros(B, ops.SLOT_STATE_BYTES, device=self.dev, dtype=torch.uint8)
                st["out"] = torch.zeros(B, slot_width, device=self.dev, dtype=torch.int64)
                if req.return_logprobs:
                    st["lp"] = torch.zeros(B, slot_width, device=self.dev, dtype=F32)
                    st["lp_step"] = torch.zeros(B, device=self.dev, dtype=F32)
            if K > 1:
                st["cache"].kv_src = torch.zeros(B, cap, device=self.dev, dtype=torch.int32)
                i32 = dict(device=self.dev, dtype=torch.int32)
                st["beam"] = dict(
                    lp=torch.empty(B, self.g.vocab_size, device=self.dev, dtype=F32),
                    cand_val=torch.empty(B, _lib.BEAM_MAX_KEEP, device=self.dev, dtype=F32),
                    cand_tok=torch.empty(B, _lib.BEAM_MAX_KEEP, **i32),
                    running=torch.empty(B, device=self.dev, dtype=F32),
                    fin_score=torch.empty(B, device=self.dev, dtype=F32),
                    fin_info=torch.empty(B, 4, **i32), flags=torch.empty(B // K, 2, **i32),
                    rec=torch.empty(cap, B, 2, **i32))
            self._gen_state = st
        return st

    @staticmethod
    def _row_lengths(lengths, B: int, L: int) -> torch.Tensor:
        """Per-row prompt lengths as a CPU int64 tensor [B] (None: every row is L long)."""
        if lengths is None:
            return torch.full((B,), L, dtype=torch.int64)
        lens = torch.as_tensor(lengths).to(device="cpu", dtype=torch.int64).reshape(-1)
        if lens.numel() != B:
            raise ValueError(f"lengths has {lens.numel()} entries for a batch of {B} prompts")
        if bool((lens < 1).any()) or bool((lens > L).any()):
            raise ValueError(f"prompt lengths {lens.tolist()} outside 1..{L} (the padded width)")
        return lens

    def _last_hidden(self, hidden: torch.Tensor, lens: torch.Tensor) -> torch.Tensor:
        """hidden[b, lens[b] - 1] for every row: the state the first new token of prompt b is picked from."""
        B = hidden.shape[0]
        return hidden[torch.arange(B, device=hidden.device), (lens - 1).to(hidden.device)]

    def _beam_loop(self, st, logits0: torch.Tensor, req: GenerateRequest, use_graph: bool, logits_out: Optional[list]):
        """The first beam step on the prefill logits, then up to max_new_tokens - 1 decode steps (the steps after the
        first replay one captured graph); every 16 steps the host checks whether every prompt is done."""
        cache, bs = st["cache"], st["beam"]
        R, K = cache.batch, req.beam.num_beams
        bufs = self._decode_buffers(R)
        self.reset_decode_state(R)
        bs["running"].view(-1, K).fill_(-1e9)[:, 0] = 0.0
        bs["fin_score"].fill_(-1e9)
        bs["fin_info"].copy_(torch.tensor([0, -1, 0, 0], dtype=torch.int32).expand(R, 4))
        bs["flags"].copy_(torch.tensor([1, 0], dtype=torch.int32).expand(R // K, 2))
        cache.kv_src.copy_(torch.arange(R, device=self.dev, dtype=torch.int32)[:, None].expand(R, cache.max_len))
        self._pick_next(logits0, bufs["ids"].view(R), None, req, step=0)
        if logits_out is not None:
            logits_out.append(logits0.float().clone())
        for step in range(1, req.max_new_tokens):
            if step % 16 == 1 and bool(bs["flags"][:, 1].all()):
                break
            if use_graph and (st["graph"] is not None or step >= 2):
                self._replay(st, lambda: self.decode_step(cache, req))
            else:
                self.decode_step(cache, req)
            if logits_out is not None:
                logits_out.append(bufs["logits"].clone())

    @staticmethod
    def _beam_backtrack(bs: dict, P: int, K: int, n_ret: int, fill: int, row0: int = 0):
        """The best n_ret finished hypotheses of every prompt, rebuilt from the per-step (token, parent beam) records,
        with their scores and HF's beam_indices: per step, the row (row0 + p * K + beam) the token was appended to."""
        info = bs["fin_info"].cpu().numpy()
        score = bs["fin_score"].cpu()
        rec = bs["rec"].cpu().numpy()
        seqs, keep, rows = [], [], []
        for p in range(P):
            for i in range(n_ret):
                r = p * K + i
                _, te, beam, tok = (int(x) for x in info[r])
                seq = [fill] * (te + 1)
                row = [-1] * (te + 1)
                if te >= 0:
                    seq[te] = tok
                    row[te] = row0 + p * K + beam
                    for s in range(te - 1, -1, -1):
                        seq[s] = int(rec[s, p * K + beam, 0])
                        beam = int(rec[s, p * K + beam, 1])
                        row[s] = row0 + p * K + beam
                seqs.append(seq)
                keep.append(r)
                rows.append(row)
        return seqs, score[keep], rows

    def _decode_loop(self, st, logits0: torch.Tensor, req: GenerateRequest, use_graph: bool,
                     margins: Optional[list] = None, force_ids: Optional[torch.Tensor] = None,
                     logits_out: Optional[list] = None):
        """Pick the first token from `logits0`, then run max_new_tokens - 1 decode steps on st['cache'] (whose length
        is the prompt length); the steps after the first replay one captured CUDA graph. margins: a list that receives
        every step's top-1/top-2 logit margins [B] (the steps then run eagerly)."""
        cache = st["cache"]
        B = cache.batch
        bufs = self._decode_buffers(B)
        self.reset_decode_state(B)
        out = torch.empty(B, req.max_new_tokens, device=self.dev, dtype=torch.int64)
        self._pick_next(logits0, bufs["ids"].view(B), None, req, step=0)
        out[:, 0] = bufs["ids"].view(B)
        if logits_out is not None:
            logits_out.append(logits0.float().clone())
        if force_ids is not None:
            force_ids = force_ids.to(self.dev, torch.int64)
            bufs["ids"].view(B).copy_(force_ids[:, 0])
        if margins is not None:
            t2 = logits0.topk(2, dim=-1).values
            margins.append(t2[:, 0] - t2[:, 1])
        eos = torch.as_tensor(req.eos_token_id, device=self.dev) if req.eos_token_id else None
        n_done = 1
        for step in range(1, req.max_new_tokens):
            if eos is not None and (step % 16 == 1) and bool(torch.isin(out[:, :n_done], eos).any(dim=1).all()):
                break
            if use_graph and margins is None and (st["graph"] is not None or step >= 2):
                # step 1 ran eagerly (warm-up + validation of the launch sequence); capture the same
                # sequence once - positions are read from the device, so every replay is a new step
                self._replay(st, lambda: self.decode_step(cache, req))
            else:
                lg = self.decode_step(cache, req)
                if margins is not None:
                    t2 = lg.topk(2, dim=-1).values
                    margins.append(t2[:, 0] - t2[:, 1])
            out[:, step] = bufs["ids"].view(B)
            if logits_out is not None:
                logits_out.append(bufs["logits"].clone())
            if force_ids is not None:
                bufs["ids"].view(B).copy_(force_ids[:, step])
            n_done += 1
        return out[:, :n_done]

    # =========================================================================================
    # continuous batching: finished decode rows are refilled with queued requests between graph replays
    # =========================================================================================
    @torch.no_grad()
    def generate_continuous(self, requests: Iterable["SlotRequest"], num_slots: int, eos_token_id=None,
                            pad_token_id: int = 0, do_sample: bool = False, temperature: float = 1.0, top_k: int = 50,
                            top_p: float = 1.0, num_return_sequences: int = 1,
                            processors: Optional[LogitsProcessors] = None, use_graph: bool = True,
                            return_logprobs: bool = False) -> Dict[str, list]:
        """Decodes every request of `requests` (read lazily) through num_slots decode rows; each request's n =
        num_return_sequences samples take n rows, admitted together as soon as n rows are free. Every row generates
        what generate() gives for its request alone: the same prefill, and a pick keyed by the request's seed, the
        sample's index and the request's own step. Returns {request_id: n token lists}, each up to and including the
        first EOS; with return_logprobs, n (tokens, log-probs) pairs instead, the log-prob of each token under the
        distribution it was picked from (log_softmax of its scores). Statistics of the call: last_continuous (steps,
        captures, admissions)."""
        cap = self._decode_rows()
        if not 1 <= num_slots <= cap:
            raise ValueError(f"num_slots={num_slots} outside 1..{cap} (the rows one decode step carries on this path)")
        if not 1 <= num_return_sequences <= num_slots:
            raise ValueError(f"num_return_sequences={num_return_sequences} outside 1..num_slots={num_slots}")
        sampling = (float(temperature), int(top_k or 0), float(top_p), 0) if do_sample else None
        # max_new_tokens and the seed live in the slots
        req = GenerateRequest(0, eos_token_id, sampling, processors, return_logprobs=bool(return_logprobs))
        dec = _SlotDecoder(self, req, num_slots, int(pad_token_id), use_graph)
        sched = SlotScheduler(dec, num_slots, num_return_sequences)
        out = sched.run(requests)
        self.last_continuous = dict(steps=sched.steps, captures=dec.captures, admissions=sched.admissions,
                                    capacity=sched.capacity)
        return out


SLOT_POLL_STEPS = 8  # decode steps between two polls of the slots' done flags (DESIGN.md, continuous batching)
SLOT_CAP_ROUND = 128


def slot_capacity(max_prompt: int, max_new_tokens: int) -> int:
    """KV capacity of a continuous-batching cache: the longest prompt admitted so far, rounded up to a multiple of 128,
    plus the largest max_new_tokens (a row's last decode step writes position prompt + max_new_tokens - 2)."""
    return -(-max_prompt // SLOT_CAP_ROUND) * SLOT_CAP_ROUND + max_new_tokens


@dataclass
class SlotRequest:
    """One request of a continuous-batching call as the engine takes it: the prompt's embeddings [1, L, E] (bf16, on the
    device; what generate() prefills for it alone), its own max_new_tokens and sampling seed."""
    request_id: str
    embeds: Optional[torch.Tensor]
    max_new_tokens: int
    seed: int = 0

    @property
    def prompt_len(self) -> int:
        return int(self.embeds.shape[1])


class SlotScheduler:
    """The host policy of continuous batching, over a backend that owns the device state (_SlotDecoder on the GPU):
      reserve(capacity, width)  make the cache hold `capacity` positions and `width` tokens per slot, keeping the live
                                slots (called before the first admission and whenever a request needs more);
      admit(request, slots)     prefill the request and start its n samples in the given slots;
      step()                    one decode step over every slot;
      snapshot() / read(h)      enqueue a copy of the slots' state without waiting; read it back (waits for the copy):
                                per slot its result (its generated tokens) when it is finished, else None.
    Free slots are taken lowest first. A request is pulled from the iterable only when a slot is free, and waits for n
    free slots. Every SLOT_POLL_STEPS steps the snapshot taken SLOT_POLL_STEPS steps earlier is read and a new one is
    enqueued: the host never waits on the step it just queued, so the device keeps the queued steps to run while the
    host retires and admits."""

    def __init__(self, backend, num_slots: int, samples: int = 1):
        self.b, self.S, self.n = backend, num_slots, samples
        self.steps = self.admissions = self.capacity = 0

    def run(self, requests) -> Dict[str, List[List[int]]]:
        it = iter(requests)
        free, owner = list(range(self.S)), [None] * self.S
        parts, results = {}, {}
        pending, exhausted, snap = None, False, None
        max_len = max_new = 0
        while True:
            while True:
                if pending is None:
                    if exhausted or not free:
                        break
                    pending = next(it, None)
                    if pending is None:
                        exhausted = True
                        break
                    if pending.request_id in parts or pending.request_id in results:
                        raise ValueError(f"duplicate request_id {pending.request_id!r}")
                    if pending.max_new_tokens < 1:
                        raise ValueError(f"request {pending.request_id!r}: max_new_tokens must be >= 1")
                if len(free) < self.n:
                    break
                slots, free = free[:self.n], free[self.n:]
                max_len, max_new = max(max_len, pending.prompt_len), max(max_new, pending.max_new_tokens)
                need = slot_capacity(max_len, max_new)
                if need > self.capacity:
                    self.b.reserve(need, max_new)
                    self.capacity = need
                self.b.admit(pending, slots)
                self.admissions += 1
                parts[pending.request_id] = [None] * self.n
                for j, s in enumerate(slots):
                    owner[s] = (pending.request_id, j)
                pending = None
            if all(o is None for o in owner):
                return results
            self.b.step()
            self.steps += 1
            if self.steps % SLOT_POLL_STEPS == 0:
                if snap is not None:
                    handle, owners_then = snap
                    for s, toks in enumerate(self.b.read(handle)):
                        # a slot refilled after the snapshot was taken shows its previous request's state: skip it
                        if toks is None or owner[s] is None or owner[s] != owners_then[s]:
                            continue
                        rid, j = owner[s]
                        parts[rid][j] = toks
                        owner[s] = None
                        free.append(s)
                        if all(p is not None for p in parts[rid]):
                            results[rid] = parts.pop(rid)
                    free.sort()
                snap = (self.b.snapshot(), list(owner))


class _SlotDecoder:
    """The device side of SlotScheduler on a U2Engine: a static cache of num_slots rows with their slot records, and
    one captured decode step (decode_step with slots) per (slots, capacity). Admissions, polls and cache growth run on
    the decode stream, between replays."""

    def __init__(self, eng: U2Engine, req: GenerateRequest, num_slots: int, pad: int, use_graph: bool):
        self.eng, self.req, self.S, self.pad, self.use_graph = eng, req, num_slots, pad, use_graph
        self.st, self.captures = None, 0
        eng.reset_decode_state(num_slots)
        self.ids = eng._decode_buffers(num_slots)["ids"].view(num_slots)

    def reserve(self, capacity: int, width: int):
        old, eng = self.st, self.eng
        st = eng._gen_state_for(self.S, capacity, self.req, slot_width=width)
        st["pad"] = self.pad
        if old is None:
            # no slot holds a request yet: every record is done (pad fed, lengths frozen at 0)
            st["slots"].copy_(ops.slot_state([0] * self.S, [0] * self.S, [1] * self.S, done=[1] * self.S))
            st["cache"].set_length(0)
        else:
            # a longer prompt or max_new_tokens arrived: the live slots move to the larger cache
            T0, w0 = old["cache"].max_len, old["out"].shape[1]
            for a, b in ((st["cache"].k, old["cache"].k), (st["cache"].v, old["cache"].v)):
                a[:, :, :, :T0].copy_(b)
            for name in ("length_dev", "length_plus1_dev"):
                getattr(st["cache"], name).copy_(getattr(old["cache"], name))
            st["slots"].copy_(old["slots"])
            st["out"][:, :w0].copy_(old["out"])
            if "lp" in st:
                st["lp"][:, :w0].copy_(old["lp"])
            if "hist" in st:
                st["hist"][:, :T0].copy_(old["hist"])
        self.st = st

    def admit(self, r: SlotRequest, slots: List[int]):
        """generate()'s batch-1 prefill of the request, its KV rows copied into each of its slots (as the n > 1 path
        of _generate copies them), and the first pick from the prefill logits with the request's own (seed, row) head."""
        eng, st, n = self.eng, self.st, len(slots)
        L = r.prompt_len
        pc = eng.new_cache(1, L)
        hidden = eng.prefill(r.embeds, pc)
        logits0 = eng.lm_logits(eng._last_hidden(hidden, torch.tensor([L])))
        logits0 = logits0.index_select(0, torch.zeros(n, dtype=torch.int64, device=eng.dev))
        first = dict(slots=ops.slot_state([r.seed] * n, range(n), [r.max_new_tokens] * n).to(eng.dev),
                     out=torch.empty(n, 1, device=eng.dev, dtype=torch.int64), pad=self.pad)
        if "hist" in st:
            first["hist"] = torch.zeros(n, 1, device=eng.dev, dtype=torch.int32)  # count 0: no history is read
        if "lp" in st:
            first["lp"] = torch.empty(n, 1, device=eng.dev, dtype=F32)
            first["lp_step"] = torch.empty(n, device=eng.dev, dtype=F32)
        ids = torch.empty(n, device=eng.dev, dtype=torch.int64)
        eng._slot_pick(logits0, ids, first, self.req)
        cache = st["cache"]
        for s in slots:
            cache.k[:, s, :, :L].copy_(pc.k[:, 0])
            cache.v[:, s, :, :L].copy_(pc.v[:, 0])
        idx = torch.tensor(slots, device=eng.dev)
        cache.length_dev.index_fill_(0, idx, L)
        cache.length_plus1_dev.index_fill_(0, idx, L + 1)
        st["slots"].index_copy_(0, idx, first["slots"])
        st["out"][:, 0].index_copy_(0, idx, first["out"][:, 0])
        if "lp" in st:
            st["lp"][:, 0].index_copy_(0, idx, first["lp"][:, 0])
        self.ids.index_copy_(0, idx, ids)
        if "hist" in st:
            st["hist"].index_fill_(0, idx, 0)

    def step(self):
        st = self.st
        run = lambda: self.eng.decode_step(st["cache"], self.req, slots=st)
        if not self.use_graph or not st.get("warm"):
            run()  # the first step on a new state runs eagerly (it also configures the kernels' attributes)
            st["warm"] = True
            return
        if st["graph"] is None:
            self.captures += 1
        self.eng._replay(st, run)

    def snapshot(self):
        st = self.st
        recs = torch.empty(st["slots"].shape, dtype=torch.uint8, pin_memory=True)
        out = torch.empty(st["out"].shape, dtype=torch.int64, pin_memory=True)
        recs.copy_(st["slots"], non_blocking=True)
        out.copy_(st["out"], non_blocking=True)
        lp = None
        if "lp" in st:
            lp = torch.empty(st["lp"].shape, dtype=F32, pin_memory=True)
            lp.copy_(st["lp"], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        return ev, recs, out, lp

    @staticmethod
    def read(handle) -> list:
        """Per slot its tokens, or (tokens, log-probs) with return_logprobs, when it is finished; else None."""
        ev, recs, out, lp = handle
        ev.synchronize()
        f = ops.slot_state_fields(recs)
        done = [(s, c) for s, (c, d) in enumerate(zip(f["count"].tolist(), f["done"].tolist())) if d]
        res = [None] * out.shape[0]
        for s, c in done:
            res[s] = out[s, :c].tolist() if lp is None else (out[s, :c].tolist(), lp[s, :c].tolist())
        return res


class KVCache:
    """Static KV cache [layers][B, Hkv, Tmax, dh] bf16 + the current length of every sequence on the device
    (int32 [B], so the decode step's launch parameters never change and the step can live in a CUDA graph; prompts of
    different lengths decode side by side, each at its own position). `length` is the longest row's length."""

    def __init__(self, g: Geometry, batch: int, max_len: int, device):
        self.batch, self.max_len = batch, max_len
        shape = (g.num_hidden_layers, batch, g.num_key_value_heads, max_len, g.head_dim)
        self.k = torch.zeros(shape, device=device, dtype=BF16)
        self.v = torch.zeros(shape, device=device, dtype=BF16)
        self.length = 0
        self.length_dev = torch.zeros(batch, device=device, dtype=torch.int32)
        self.length_plus1_dev = torch.ones(batch, device=device, dtype=torch.int32)
        self.kv_src = None  # beam search: int32 [B, max_len], the cache row holding position t of sequence b

    def set_length(self, n):
        """n: one length for every sequence, or the per-sequence lengths [B]."""
        lens = torch.as_tensor(n)
        if lens.dim() == 0:
            n = int(lens)
            self.length = n
            self.length_dev.fill_(n)
            self.length_plus1_dev.fill_(n + 1)
            return
        lens = lens.to(device="cpu", dtype=torch.int32).reshape(-1)
        if lens.numel() != self.batch:
            raise ValueError(f"{lens.numel()} lengths for a cache of {self.batch} sequences")
        if bool((lens < 0).any()) or bool((lens > self.max_len).any()):
            raise ValueError(f"lengths {lens.tolist()} outside 0..{self.max_len}")
        self.length = int(lens.max())
        self.length_dev.copy_(lens)
        self.length_plus1_dev.copy_(lens + 1)

    def advance_device(self):
        self.length_dev.add_(1)
        self.length_plus1_dev.add_(1)
        self.length += 1
