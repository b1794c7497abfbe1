#!/usr/bin/env python
"""Benchmark of the mu2-LLM hot path (driver contract: one JSON line on stdout from rank 0).

A "step" is one pass of the hot path over one batch of synthetic CT volumes: vision front ->
mu2-tokenizer -> splice -> decoder prefill -> greedy decode of `new_tokens` report tokens, called
through the reference-facing HuggingFace-style API (`model.generate(images, input_ids,
question_ids=..., max_new_tokens=..., do_sample=False)`).

  value : volumes/s with the inputs already resident in HBM when the timed region starts
  e2e   : the same call with HOST (pinned) inputs, H2D copies and the D2H read of the ids timed
  roofline : the dominant kernel (decode-step weight-streaming GEMV, HBM-bound) timed live with
             CUDA events in isolation, algorithmic bytes / time vs MEASURED_PEAKS.json
  cpu_baseline / --impl reference : the fp32 oracle port (oracle/u2_oracle.py, a restatement of the
             reference's PyTorch forward) timed on this box's host cores on a bounded sample

Workloads (BASELINE.json configs): cfg3 (default) = mu2-Qwen3-8B greedy generate 256 tokens, batch 4,
256^3 volumes (8 frames); cfg2 = mu2-Qwen3-1.7B forward, one 256x256x128 volume.
Multi-GPU: pure data parallel replicas (independent volumes, no data-path collective), weak scaling.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def log(*a):
    print(*a, file=sys.stderr, flush=True)


# ------------------------------------------------------------------------------------------------
# workloads
# ------------------------------------------------------------------------------------------------
def make_geometry(workload: str):
    from u2tokenizer_b200.configuration import QWEN3_1P7B, QWEN3_8B, U2Qwen3Config
    from u2tokenizer_b200.geometry import Geometry
    if workload == "cfg3":
        cfg = U2Qwen3Config(**QWEN3_8B)
        spec = dict(model="mu2-Qwen3-8B", batch=4, frames=8, new_tokens=256, n_question=32, lt=512, mode="generate")
    elif workload == "cfg2":
        cfg = U2Qwen3Config(**QWEN3_1P7B)
        spec = dict(model="mu2-Qwen3-1.7B", batch=1, frames=4, new_tokens=0, n_question=32, lt=512, mode="forward")
    elif workload == "cfg4":
        # BASELINE configs[3]: mu2-Qwen3-8B, global batch 16 on 8 GPUs = 2 volumes / GPU, three raw scales (64 / 128 / 256)^3
        # brought to [8, 32, 256, 256] by the reference's resize-and-pad rule (u2Transform.py:74-94,120: zero frames behind the
        # real depth), teacher-forced sequences of 512 tokens (train_stage1.py:104), forward + backward + ZeRO-1 AdamW step
        cfg = U2Qwen3Config(**QWEN3_8B)
        spec = dict(model="mu2-Qwen3-8B", batch=2, frames=8, new_tokens=0, n_question=32, lt=512, seq=512, mode="train")
    elif workload == "cfg5":
        # BASELINE configs[4]: stage-2 DPO step, one preference pair / GPU (chosen + rejected = 2 sequences of 1024 tokens
        # over the same study), policy forward + backward and frozen-reference forward (dpo_u2trainer.py:185-359)
        cfg = U2Qwen3Config(**QWEN3_8B)
        spec = dict(model="mu2-Qwen3-8B", batch=2, frames=8, new_tokens=0, n_question=32, lt=1024, seq=1024, mode="dpo")
    elif workload == "tiny_train":
        cfg = U2Qwen3Config(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                            num_key_value_heads=2, head_dim=64, vocab_size=1024, image_size=[16, 64, 64],
                            vit_hidden_size=128, vit_mlp_dim=256, vit_num_layers=2, vit_num_heads=2, u2t_num_layers=2,
                            u2t_top_k=16, num_3d_query_token=16, tie_word_embeddings=False)
        spec = dict(model="tiny", batch=2, frames=2, new_tokens=0, n_question=8, lt=16, seq=48, mode="train")
    elif workload == "tiny_dpo":
        cfg = U2Qwen3Config(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                            num_key_value_heads=2, head_dim=64, vocab_size=1024, image_size=[16, 64, 64],
                            vit_hidden_size=128, vit_mlp_dim=256, vit_num_layers=2, vit_num_heads=2, u2t_num_layers=2,
                            u2t_top_k=16, num_3d_query_token=16, tie_word_embeddings=False)
        spec = dict(model="tiny", batch=2, frames=2, new_tokens=0, n_question=8, lt=16, seq=48, mode="dpo")
    elif workload == "tiny":  # plumbing check only
        cfg = U2Qwen3Config(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                            num_key_value_heads=2, head_dim=64, vocab_size=1024, image_size=[16, 64, 64],
                            vit_hidden_size=128, vit_mlp_dim=256, vit_num_layers=2, vit_num_heads=4, u2t_num_layers=2,
                            u2t_top_k=16, num_3d_query_token=16, tie_word_embeddings=False)
        spec = dict(model="tiny", batch=2, frames=2, new_tokens=8, n_question=8, lt=16, mode="generate")
    else:
        raise SystemExit(f"unknown workload {workload}")
    return cfg, Geometry.from_hf(cfg), spec


def build_model(cfg, geom, seed=0):
    """Random-init weights of the real architecture, generated on the device (no network for checkpoints)."""
    from u2tokenizer_b200.modeling import U2Qwen3ForCausalLM
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device("cuda"):
            model = U2Qwen3ForCausalLM(cfg)
    finally:
        torch.set_default_dtype(prev)
    sd = synthetic_state_dict(geom, seed=seed, device="cuda", dtype=torch.bfloat16)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    del sd
    model.eval()
    torch.cuda.empty_cache()
    return model


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index, self.proc, self.lines = index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for ln in self.proc.stdout:
            self.lines.append(ln.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            pass
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1]))
            except ValueError:
                continue
            for n, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "samples": len(sm), "reasons": sorted(reasons)}


def measured_peaks():
    # fallback: NVIDIA's H100 SXM data sheet (3.35 TB/s HBM3, 989 dense BF16 TFLOP/s at up to 700 W), never reached
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d.get("hbm_gbs", 3350.0), d.get("bf16_tflops_sustained", 989.0), "measured"
    return 3350.0, 989.0, "data sheet"


# ------------------------------------------------------------------------------------------------
# roofline probe: the dominant kernel timed live (CUDA events, kernel launched alone in a loop over
# all decoder layers' weights so the working set (>= 4 GB) is far larger than the 50 MB L2)
# ------------------------------------------------------------------------------------------------
def roofline_probe(model, spec, geom):
    from u2tokenizer_b200 import ops
    eng = model.engine()
    hbm, tf, src = measured_peaks()
    if spec["mode"] == "generate":
        # dominant kernel of the generate workload: the decode-step linear chain launch
        # (dlinear_wgmma_kernel: o_proj -> gate|up -> down -> next qkv in ONE launch, 386 MB of weights for 8B)
        B = spec["batch"]
        hq, hkv, dh, I, E = (geom.num_attention_heads, geom.num_key_value_heads, geom.head_dim, geom.intermediate_size,
                             geom.hidden_size)
        bufs = eng._decode_buffers(B)
        eng.reset_decode_state(B)
        x, qkv, ctx, act, xg_a, xg_b = (bufs[k] for k in ("x", "qkv", "ctx", "act", "xg", "xg2"))
        ctx.normal_()
        x.normal_()
        c0 = dict(ws=bufs["ws"][0], counters=bufs["counters"][0], sched=eng.dl_sched)
        c1 = dict(ws=bufs["ws"][1], counters=bufs["counters"][1], sched=eng.dl_sched)
        nl = len(eng.layers)

        def chain(li):
            w, wn = eng.layers[li], eng.layers[(li + 1) % nl]
            fl = bufs["flags"][li] if eng.fine_deps else [None] * 4
            dep = lambda i, shift: dict(dep_flags=fl[i], dep_shift=shift) if fl[i] is not None else {}
            return [(ctx, w["wo"], x, dict(residual=x, gamma_next=w["ln2"], xg=xg_a, ssq_out=bufs["ssq_a"], ssq_zero=bufs["ssq_b"], out_flags=fl[0], **c0)),
                    (xg_a, w["wgu"], act, dict(ssq_in=bufs["ssq_a"], eps=geom.rms_norm_eps, silu_pair=True, out_flags=fl[1], **dep(0, 1), **c1)),
                    (act, w["wdown"], x, dict(residual=x, gamma_next=wn["ln1"], xg=xg_b, ssq_out=bufs["ssq_b"], ssq_zero=bufs["ssq_a"], out_flags=fl[2], **dep(1, 0), **c0)),
                    (xg_b, wn["wqkv"], qkv, dict(ssq_in=bufs["ssq_b"], eps=geom.rms_norm_eps, **dep(2, 1), **c1))]

        def sweep():
            bufs["step"] += 1
            for li in range(nl):
                ops.dlinear_multi(chain(li), gridbar=bufs["gridbar"][li * 4:(li + 1) * 4], step_dev=bufs["step"], pdl=eng.pdl)
        st = torch.cuda.current_stream()
        sweep()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        reps = 3
        e0.record(st)
        for _ in range(reps):
            sweep()
        e1.record(st)
        torch.cuda.synchronize()
        eng.reset_decode_state(B)
        sec = e0.elapsed_time(e1) / 1e3 / (reps * nl)
        nq = (hq + 2 * hkv) * dh
        w_bytes = 2 * (E * hq * dh + 2 * I * E + E * I + nq * E)
        act_bytes = 2 * B * (hq * dh + 3 * E + 2 * E + 2 * I + 2 * E + nq)  # activations in/out of the four linears
        alg_bytes = w_bytes + act_bytes
        ach = alg_bytes / sec / 1e9
        return {"bound": "hbm", "kernel": "dlinear_wgmma_kernel<128> (decode chain: o_proj+gate|up+down+qkv in one launch)",
                "achieved": round(ach, 1), "peak": hbm, "unit": "GB/s", "frac": round(ach / hbm, 4),
                "peak_source": src, "bytes_per_launch": alg_bytes,
                "us_per_launch": round(sec * 1e6, 2),
                "note": "timed live with CUDA events over all layers' weights (13.9 GB working set >> 50 MB L2)"}
    # forward workloads: the ViT MLP GEMM (largest share of tensor work)
    Fr = spec["batch"] * spec["frames"]
    M = Fr * 2056
    a = torch.randn(M, geom.vit_hidden, device="cuda").bfloat16()
    w = eng.vit[0]["w1"]
    out = torch.empty(M, geom.vit_mlp, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):
        ops.linear(a, w, eng.vit[0]["b1"], act=ops.ACT_GELU, out=out)
    # the kernel is short (< 100 us): replay 10 launches from a CUDA graph so that the host's launch path is not what
    # gets timed (operands stay L2-resident between launches, as they are inside the model's own launch sequence)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(10):
            ops.linear(a, w, eng.vit[0]["b1"], act=ops.ACT_GELU, out=out)
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(3):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    sec = e0.elapsed_time(e1) / 1e3 / 30
    fl = 2.0 * M * geom.vit_mlp * geom.vit_hidden
    ach = fl / sec / 1e12
    return {"bound": "tensor", "kernel": "gemm_bf16_wgmma_kernel (ViT MLP fc1 + GELU)", "achieved": round(ach, 1), "peak": tf,
            "unit": "TFLOP/s", "frac": round(ach / tf, 4), "traffic": None, "peak_source": src,
            "flops_per_launch": fl, "us_per_launch": round(sec * 1e6, 2)}


def extra_rooflines(model, spec, geom):
    """Secondary kernels named by BASELINE.json's north star, timed live (CUDA events, inputs larger than L2):
    the 3-D patch-embed brick gather (HBM) and the decoder prefill gate|up GEMM (tensor pipe)."""
    from u2tokenizer_b200 import ops
    eng = model.engine()
    hbm, tf, src = measured_peaks()
    out = []
    ev = lambda: torch.cuda.Event(enable_timing=True)
    # --- the WHOLE 3-D patch-embedding op (SURVEY.md section 8d: 97.0 MB of algorithmic traffic per 256^3 volume = fp32 volume in,
    # bf16 tokens out, weights once; 25.8 GFLOP): brick gather + GEMM (+bias +position table, rows placed behind the cls
    # row) + cls / padding rows, 32 frames = 4 volumes per pass, two buffer sets alternated (537 MB >> 50 MB L2)
    Fr = 32
    D0, D1, D2 = geom.image_size
    P, Hd, pd = geom.n_patches, geom.vit_hidden, geom.patch_dim
    S, Sp = P + 1, (P + 1 + 7) // 8 * 8
    vols = [torch.rand(Fr, D0, D1, D2, device="cuda") for _ in range(2)]
    rows = [torch.empty(Fr * P, pd, device="cuda", dtype=torch.bfloat16) for _ in range(2)]
    xs = [torch.empty(Fr, Sp, Hd, device="cuda", dtype=torch.bfloat16) for _ in range(2)]

    def gather(i):
        ops.patchify(vols[i], geom.patch_size, out=rows[i])

    def embed_unfused(i):
        gather(i)
        ops.gemm(rows[i], eng.pe_w, xs[i], M=Fr * P, N=Hd, K=pd, lda=pd, ldb=pd, ldc=Hd, bias=eng.pe_b, residual=eng.pos, ldr=Hd,
                 res_row_mod=P, row_remap=(P, Sp, 1))
        ops.vit_frame_rows(xs[i], eng.cls, Fr, Sp, S)

    fused = eng.fused_patch_embed and ops.patch_embed_supported(geom.image_size, geom.patch_size, Hd)

    def embed(i):
        if not fused:
            return embed_unfused(i)
        ops.patch_embed(vols[i], geom.patch_size, eng.pe_w, eng.pe_b, eng.pos, xs[i])
        ops.vit_frame_rows(xs[i], eng.cls, Fr, Sp, S)

    def timed_us(fn, reps=8):
        for i in range(2):
            fn(i)
        e0, e1 = ev(), ev()
        torch.cuda.synchronize()
        e0.record()
        for r in range(reps):
            fn(r % 2)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / reps
    us_op, us_gather = timed_us(embed), timed_us(gather)
    us_unfused = timed_us(embed_unfused) if fused else us_op
    by_op = Fr * (D0 * D1 * D2 * 4 + P * Hd * 2) + (pd * Hd + P * Hd + Hd) * 2
    fl_op = 2.0 * Fr * P * pd * Hd
    out.append({"kernel": ("3-D patch embedding, whole op (patch_embed_wgmma_kernel: 5-D TMA slabs -> in-smem fp32->bf16 A operand -> "
                           "wgmma, bias + position epilogue; + vit_frame_rows_kernel)") if fused else
                          "3-D patch embedding, whole op (patchify_tma_kernel + gemm_bf16_wgmma_kernel<128> + vit_frame_rows_kernel)",
                "bound": "hbm / tensor (arithmetic intensity 266 FLOP/B vs ridge 218)", "achieved": round(by_op / us_op / 1e3, 1),
                "peak": hbm, "unit": "GB/s", "frac": round(by_op / us_op / 1e3 / hbm, 4), "bytes_per_launch": by_op,
                "us_per_launch": round(us_op, 2), "tensor_achieved_tflops": round(fl_op / us_op / 1e6, 1),
                "tensor_frac": round(fl_op / us_op / 1e6 / tf, 4), "peak_source": src,
                "unfused_us_per_launch": round(us_unfused, 2),
                "note": "algorithmic bytes = 97.0 MB per volume (SURVEY 8d); the unfused variant (gather + GEMM, "
                        f"{round(us_unfused, 1)} us) writes and re-reads bf16 im2col rows that are NOT counted; its gather alone moves "
                        f"its own 100.7 MB per volume at {round(Fr * D0 * D1 * D2 * 6 / us_gather / 1e3 / hbm, 3)} of the HBM peak "
                        f"({round(us_gather, 1)} us)"})
    del vols, rows, xs
    # --- decoder prefill GEMM (gate|up): M = batch * prompt rows
    M = max(spec["batch"], 1) * (geom.num_3d_query_token + spec["n_question"])
    E, I = geom.hidden_size, geom.intermediate_size
    a = (torch.randn(M, E, device="cuda") * 0.05).bfloat16()
    c = torch.empty(M, 2 * I, device="cuda", dtype=torch.bfloat16)
    nl = len(eng.layers)
    for li in range(min(nl, 4)):
        ops.linear(a, eng.layers[li]["wgu"], out=c)
    e0, e1 = ev(), ev()
    torch.cuda.synchronize()
    e0.record()
    for li in range(nl):
        ops.linear(a, eng.layers[li]["wgu"], out=c)
    e1.record()
    torch.cuda.synchronize()
    sec = e0.elapsed_time(e1) / 1e3 / nl
    fl = 2.0 * M * 2 * I * E
    out.append({"kernel": f"gemm_bf16_wgmma_kernel<128> (decoder prefill gate|up, M={M} N={2 * I} K={E})", "bound": "tensor",
                "achieved": round(fl / sec / 1e12, 1), "peak": tf, "unit": "TFLOP/s", "frac": round(fl / sec / 1e12 / tf, 4),
                "flops_per_launch": fl, "us_per_launch": round(sec * 1e6, 2), "peak_source": src})
    return out


# ------------------------------------------------------------------------------------------------
# CPU baseline: the oracle port on host cores, bounded sample, extrapolated by layer counts
# ------------------------------------------------------------------------------------------------
def cpu_baseline(geom, spec, budget_note=True):
    """Times the fp32 oracle (a restatement of the reference's PyTorch forward) on the host cores.
    Bounded sample (about 10-30 s of CPU work): ONE volume through the WHOLE vision path at full depth (patch embedding,
    all ViT blocks, projector, all SVR / TTA layers, DiffTS, DMTP, linear aggregation - measured, not extrapolated), then
    two decoder layers at the prompt length and for 8 cached decode tokens plus a 32k-row slice of the lm_head, scaled
    by the decoder's layer count / vocabulary (the extrapolated share is reported)."""
    import copy
    from oracle import u2_oracle as O
    from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict
    try:
        avail = len(os.sched_getaffinity(0))
    except AttributeError:
        avail = os.cpu_count() or 1

    def best_threads(fn):
        """The box may report far more logical CPUs than it can run well: pick the fastest thread count (median of 3)."""
        best, best_t = avail, float("inf")
        for n in sorted({min(avail, c) for c in (8, 16, 32, 64, 128, avail)}):
            torch.set_num_threads(n)
            fn()
            ts = []
            for _ in range(3):
                t0 = time.perf_counter()
                fn()
                ts.append(time.perf_counter() - t0)
            dt = statistics.median(ts)
            if dt < best_t:
                best, best_t = n, dt
        return best

    E, I = geom.hidden_size, geom.intermediate_size
    a_big, b_big = torch.randn(2056 * 2, 768), torch.randn(768, 3072)          # one ViT MLP GEMM over two frames
    a_vec, b_vec = torch.randn(1, E), torch.randn(E, 2 * I)                     # one decode-step gate|up GEMV
    n_big = best_threads(lambda: a_big @ b_big)
    n_vec = best_threads(lambda: a_vec @ b_vec)
    cores = max(n_big, n_vec)
    torch.set_num_threads(n_big)
    g1 = copy.deepcopy(geom)
    n_dec = 2
    g1.num_hidden_layers = n_dec
    g1.vocab_size = min(geom.vocab_size, 8192)  # lm_head timed separately below on a 32k-row slice of the real width
    sd = {k: v.float() for k, v in synthetic_state_dict(g1, seed=0, device="cpu", dtype=torch.bfloat16).items()}
    images, ids, qids = synthetic_inputs(g1, batch=1, frames=spec["frames"], n_question=spec["n_question"], lt=spec["lt"])
    t = {}

    def timed(name, fn):
        t0 = time.perf_counter()
        r = fn()
        t[name] = time.perf_counter() - t0
        return r

    with torch.no_grad():
        O.vit_block(sd, "model.vision_tower.vision_tower.blocks.0.", torch.randn(1, 2049, geom.vit_hidden), g1.vit_heads)  # warm
        timed("vision_tokenizer_full_depth", lambda: O.visual_tokens(sd, images, qids, g1))
        L = ids.shape[1]
        emb = torch.randn(1, L, E) * 0.02
        (_, past) = timed("dec_prefill_%d_layers" % n_dec, lambda: O.decoder_forward(sd, emb, g1, return_hidden=True))
        n_tok = 8
        torch.set_num_threads(n_vec)

        def dec():
            p = past
            for _ in range(n_tok):
                _, p = O.decoder_forward(sd, torch.randn(1, 1, E) * 0.02, g1, p, return_hidden=True)
        dec()
        timed("dec_decode_%d_tokens_%d_layers" % (n_tok, n_dec), dec)
        head = torch.randn(min(geom.vocab_size, 32768), E)
        hx = torch.randn(1, E)
        hx @ head.t()
        timed("lm_head_32k_rows", lambda: hx @ head.t())
    log("[cpu_baseline] parts (s):", {k: round(v, 4) for k, v in t.items()}, "threads gemm/gemv", n_big, n_vec, "of", avail)
    nl_d = geom.num_hidden_layers
    vision = t["vision_tokenizer_full_depth"]
    prefill = nl_d / n_dec * t["dec_prefill_%d_layers" % n_dec]
    head_tok = t["lm_head_32k_rows"] * geom.vocab_size / head.shape[0]
    per_tok = nl_d / n_dec * t["dec_decode_%d_tokens_%d_layers" % (n_tok, n_dec)] / n_tok + head_tok
    per_volume = vision + prefill + spec["new_tokens"] * per_tok + (head_tok if spec["new_tokens"] else head_tok * L)
    vols = 1.0 / per_volume
    measured = sum(t.values())
    sample = (f"oracle port (fp32 torch eager, {n_big} threads for the GEMM phases / {n_vec} for decode, best of a sweep over "
              f"{avail} logical CPUs): ONE volume x {spec['frames']} frames through the whole vision + mu2-tokenizer path at full "
              f"depth (measured: {vision:.1f} s), {n_dec} of {nl_d} decoder layers at prefill L={L} and for {n_tok} cached tokens, "
              f"a 32k-row lm_head slice; decoder scaled by {nl_d}/{n_dec} layers, {spec['new_tokens']} new tokens per volume; "
              f"{measured:.1f} s of CPU work measured, vision share of the estimated step {vision / per_volume:.1%} measured "
              f"directly, the remaining {1 - vision / per_volume:.1%} extrapolated from the decoder sample")
    return {"value": vols, "unit": "volumes/s", "cores": cores, "kind": "port", "sample": sample,
            "per_volume_s": per_volume, "tokens_per_s": (1.0 / per_tok) if spec["new_tokens"] else None,
            "parts_s": {k: round(v, 4) for k, v in t.items()}}


def gpu_eager_baseline(model, geom, spec, inputs, steps=2):
    """Same-box GPU comparator (SURVEY.md section 2d: "the kernel to beat on the same box"): the reference modules'
    arithmetic (the oracle functions) in bf16 under STOCK PyTorch eager - cuBLAS GEMMs, torch SDPA / flash attention,
    ATen elementwise kernels - on the same GPU, same weights, same inputs, same timed region as `value`."""
    from oracle import u2_oracle as O
    images, ids, qids = inputs
    sd = {k: v for k, v in model.state_dict().items()}
    if "lm_head.weight" not in sd:
        sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    O.USE_SDPA = True
    try:
        def run():
            with torch.no_grad():
                if spec["mode"] == "generate":
                    return O.greedy_generate(sd, ids, images.to(torch.bfloat16), qids, geom, spec["new_tokens"])[0]
                return O.forward_logits(sd, ids, images.to(torch.bfloat16), qids, geom)[:, -1].float().argmax(-1)
        run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            r = run()
        e1.record()
        torch.cuda.synchronize()
    finally:
        O.USE_SDPA = False
    ms = e0.elapsed_time(e1) / steps
    B = spec["batch"]
    return {"value": round(B / (ms / 1e3), 4), "unit": "volumes/s", "ms_per_step": round(ms, 2),
            "tokens_per_s": round(B * spec["new_tokens"] / (ms / 1e3), 1) if spec["new_tokens"] else None,
            "kind": "oracle functions (the reference modules' arithmetic) in bf16 under stock PyTorch eager: cuBLAS + torch SDPA, "
                    "same GPU / weights / inputs / timed region; HF-style Python decode loop with a concatenated KV cache",
            "steps": steps}


# ------------------------------------------------------------------------------------------------
# training workloads (cfg 4: SFT step, cfg 5: DPO step): forward + backward + ZeRO-1 gradient exchange + fused AdamW
# ------------------------------------------------------------------------------------------------
def train_flops(g, B, C, L, Lt):
    """Forward FLOPs of one training sample batch (2 * M * N * K over every contraction on the path) and the step total:
    backward = dgrad + wgrad of every Linear (2x forward) + the attention backward (2.5x its forward, incl. the recomputed
    ViT scores); patch embedding has no dgrad."""
    Hd, P, E, H = g.vit_hidden, g.n_patches, g.hidden_size, g.u2t_num_heads
    S = P + 1
    F_ = B * C
    N, Q, K = g.tokens_per_frame, g.num_3d_query_token, g.u2t_top_k
    lin = att = 0.0
    pe = 2.0 * F_ * P * g.patch_dim * Hd
    lin += g.vit_layers * 2.0 * F_ * S * (3 * Hd * Hd + Hd * Hd + 2 * Hd * g.vit_mlp)
    att += g.vit_layers * 4.0 * F_ * S * S * Hd
    lin += 2.0 * F_ * N * (Hd * E + E * E)                                         # projector
    rows = F_ * N
    lin += g.u2t_num_layers * 2 * 2.0 * rows * 4 * E * E                            # SVR: spatial + temporal, qkv + dense
    att += g.u2t_num_layers * (4.0 * F_ * N * N * E + 4.0 * B * N * C * C * E)
    T_ = C * N
    if g.enable_diffts:
        lin += 2.0 * B * T_ * K * E * 2
    Mv = K + K // 2 + K // 4 if g.use_multi_scale else K
    lin += g.u2t_num_layers * 2.0 * B * (Q * 4 * E * E + Q * 2 * E * E + Mv * 2 * E * E + Q * 2 * E * E + Lt * 2 * E * E)
    att += g.u2t_num_layers * 4.0 * B * Q * (Q + Mv + Lt) * E
    lin += 2.0 * B * (Q + Mv) * E * E
    att += 4.0 * B * Q * Mv * E
    hq, hkv, dh, I = g.num_attention_heads, g.num_key_value_heads, g.head_dim, g.intermediate_size
    lin += g.num_hidden_layers * 2.0 * B * L * (E * (hq + 2 * hkv) * dh + hq * dh * E + 3 * E * I)
    att += g.num_hidden_layers * 2.0 * B * L * L * hq * dh                          # causal: half of 4 * L^2
    head = 2.0 * B * L * E * g.vocab_size
    fwd = pe + lin + att + head
    step = 2.0 * pe + 3.0 * lin + 3.5 * att + 4.0 * head                            # head: fused fwd + recomputed logits + 2 grads
    return fwd, step


def train_batch(geom, spec, rank, world):
    """Synthetic training batch of the shapes the reference's collator yields (train_stage1.py:244-250): images
    [B, 8, 32, 256, 256] with the three raw scales' zero-padded depth, input_ids = <im_patch> x 256 + question + answer,
    labels = -100 on the visual / question part, question_ids right-padded to Lt."""
    from u2tokenizer_b200.synthetic import synthetic_inputs
    B, C, L = spec["batch"], spec["frames"], spec["seq"]
    images, ids, qids = synthetic_inputs(geom, batch=B, frames=C, n_question=spec["n_question"], lt=spec["lt"], seed=4321 + rank)
    for b in range(B):   # cfg 4: raw depth 64 / 128 / 256 -> 2 / 4 / 8 real frames, the rest is F.pad zeros
        depth = (64, 128, 256)[(rank * B + b) % 3]
        images[b, depth // 32:] = 0
    gen = torch.Generator().manual_seed(99 + rank)
    n_prompt = ids.shape[1]
    if spec["mode"] == "dpo":
        # one preference pair: chosen and rejected share the study and the prompt (dpo_u2trainer.py:151-183)
        images = images[:1].expand(2, *images.shape[1:]).contiguous()
        ids, qids = ids[:1].expand(2, -1).contiguous(), qids[:1].expand(2, -1).contiguous()
    ans = torch.randint(1, max(16, geom.vocab_size - 16), (ids.shape[0], L - n_prompt), generator=gen)
    ids = torch.cat([ids, ans], dim=1)
    labels = ids.clone()
    labels[:, :n_prompt] = -100
    mask = torch.zeros_like(ids)
    mask[:, n_prompt:] = 1
    return images, ids, qids, labels, mask


def run_train_steps(te, spec, geom, batch, steps, warmup, dist=None, ref_model=None, e2e=False):
    """W warm-up + K timed optimizer steps; per-phase device times (CUDA events on the compute stream):
    forward | backward (with the overlapped reduce-scatters in flight) | exposed gradient exchange (what is left of the
    reduce-scatter when the backward's last kernel has finished) | clip + fused AdamW + all-gather.
    e2e: a second timed loop of K steps in which every step copies its batch from PINNED HOST memory (what a DataLoader
    with pin_memory hands over) and reads the loss back to the host; returned as the 5th element (ms, bytes in, bytes out)."""
    from u2tokenizer_b200 import _lib, parallel
    images, ids, qids, labels, mask = [t.cuda() for t in batch]
    beta = 0.1
    host = [t.contiguous().pin_memory() for t in batch] if e2e else None

    def step(ev=None, from_host=False):
        nonlocal images, ids, qids, labels, mask
        if from_host:
            images, ids, qids, labels, mask = [t.cuda(non_blocking=True) for t in host]
        te.zero_grad()
        if ev: ev[0].record()
        if spec["mode"] == "dpo":
            with torch.no_grad():
                ref = ref_model.sequence_logps(images, ids, qids, mask)
            if ev: ev[1].record()
            out = te.dpo_forward_backward(images, ids, qids, mask, ref, beta)
        else:
            out = te.forward_loss(images, ids, qids, labels)
            if ev: ev[1].record()
            te.backward()
        if ev: ev[2].record()
        if te.comm_stream is not None:
            torch.cuda.current_stream().wait_stream(te.comm_stream)
        if ev: ev[3].record()
        te.optimizer_step()
        if ev: ev[4].record()
        return out

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
            torch.cuda.synchronize()
    for _ in range(max(warmup, 1)):
        out = step()
    te.sync_params()
    barrier()
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(5)] for _ in range(steps)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n0 = _lib.launches()
    e0.record()
    for i in range(steps):
        out = step(evs[i])
    te.sync_params()   # the last step's parameter all-gather belongs to the timed region
    e1.record()
    barrier()
    ms = parallel.max_over_ranks(e0.elapsed_time(e1), device="cuda")
    ph = [0.0] * 4
    for ev in evs:
        for j in range(4):
            ph[j] += ev[j].elapsed_time(ev[j + 1]) / steps
    names = ("ref_forward" if spec["mode"] == "dpo" else "forward", "policy_fwd_bwd" if spec["mode"] == "dpo" else "backward",
             "exposed_reduce_scatter", "clip_adamw")   # the parameter all-gather overlaps the next step's forward
    phases = {n: round(parallel.max_over_ranks(v, device="cuda"), 3) for n, v in zip(names, ph)}
    n_launch = _lib.launches() - n0
    if not e2e:
        return ms, n_launch, phases, out
    barrier()
    e0.record()
    d2h = 0
    for i in range(steps):
        o = step(from_host=True)
        o = o.float().cpu()             # the loss (DPO: loss / reward accuracy / margin) back on the host, every step
        d2h = o.numel() * 4
    te.sync_params()
    e1.record()
    barrier()
    ms_e2e = parallel.max_over_ranks(e0.elapsed_time(e1), device="cuda")
    h2d = sum(t.numel() * t.element_size() for t in host)
    return ms, n_launch, phases, out, (ms_e2e, h2d, d2h)


def train_main(args, cfg, geom, spec, base, rank, local_rank, world, dist):
    """`--workload cfg4|cfg5`: one JSON line for the training step."""
    from u2tokenizer_b200 import _lib, parallel
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    from u2tokenizer_b200.train import TrainEngine
    log(f"[rank {rank}] building {spec['model']} training state ...")
    sd = synthetic_state_dict(geom, seed=0, device="cuda", dtype=torch.bfloat16)
    te = TrainEngine(geom, sd, device="cuda", world_size=world, rank=rank)
    ref_model = None
    if spec["mode"] == "dpo":
        ref_model = TrainEngine(geom, sd, device="cuda", world_size=1, rank=0, trainable={k: False for k in ("vit", "proj", "u2t", "dec", "embed", "head")})
        ref_model.Gm = ref_model.Gv = None   # frozen reference: no gradient buffers
    del sd
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    n_mat = te.lay.mat_total
    need_f32 = n_mat / world * 12
    mom = torch.float32 if need_f32 + 40e9 < free else torch.bfloat16
    te.init_optimizer(lr=4e-6, weight_decay=0.0, max_grad_norm=1.0, moment_dtype=mom)   # script/ct_rate_stage1.sh:36-38
    batch = train_batch(geom, spec, rank, world)
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    ms, launches, phases, out, (ms_e2e, h2d, d2h) = run_train_steps(te, spec, geom, batch, args.steps, max(args.warmup, 3), dist,
                                                                    ref_model, e2e=True)
    clocks = sampler.stop() if rank == 0 else None
    if rank != 0:
        return
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, {"loss": out})
    B = spec["batch"] if spec["mode"] != "dpo" else 1   # DPO: one study per pair
    n_tok = batch[1].shape[0] * batch[1].shape[1]
    fwd_fl, step_fl = train_flops(geom, batch[1].shape[0], spec["frames"], spec["seq"], spec["lt"])
    if spec["mode"] == "dpo":
        step_fl += fwd_fl
    hbm, tf, src = measured_peaks()
    per_step = ms / args.steps
    compute_ms = per_step - phases["exposed_reduce_scatter"] - phases["clip_adamw"]
    out_d = dict(base)
    out_d.update({"value": round(world * B * args.steps / (ms / 1e3), 4), "ms_per_step": round(per_step, 3), "dtype": "bf16",
                  "tokens_per_sec": round(world * n_tok * args.steps / (ms / 1e3), 1), "gpu_launches": int(launches), "clocks": clocks,
                  "phases_ms": phases, "loss": [float(x) for x in out.flatten()[:3]] if out.numel() > 1 else float(out),
                  "optimizer": f"AdamW, ZeRO-1 over {world} rank(s): fp32 master, {str(mom).split('.')[-1]} moments, "
                               f"{te.lay.n_buckets} gradient buckets of {te.lay.bucket} bf16 elements, max_grad_norm 1.0",
                  "roofline": {"bound": "tensor", "kernel": "training step (all wgmma GEMMs: forward, dgrad, wgrad, attention)",
                               "achieved": round(step_fl / (compute_ms / 1e3) / 1e12, 1), "peak": tf, "unit": "TFLOP/s",
                               "frac": round(step_fl / (compute_ms / 1e3) / 1e12 / tf, 4), "traffic": None, "peak_source": src,
                               "flops_per_step": step_fl, "note": "algorithmic FLOPs of forward + backward per rank / (forward + backward ms)"},
                  "e2e": {"value": round(world * B * args.steps / (ms_e2e / 1e3), 4), "unit": "volumes/s",
                          "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h), "ms_per_step": round(ms_e2e / args.steps, 3),
                          "note": "every step copies its batch (fp32 volumes, ids, labels / masks) from pinned host memory and "
                                  "reads the loss back; h2d / d2h bytes are per rank"}})
    out_d["scaling"] = "weak"
    out_d["config"]["parallelism"] = f"dp{world}: ZeRO-1 (bucketed NCCL reduce-scatter overlapped with the backward, sharded fused AdamW, all-gather)"
    print(json.dumps(out_d), flush=True)


def train_substep(model, rank, local_rank, world, dist, steps=3, warmup=3):
    """cfg 4 training step (2 volumes / GPU, 512-token sequences) on the model the generate benchmark just used: its
    parameters move into the training engine's flat buffer (no second copy), every rank joins the ZeRO-1 exchange.
    The training state costs 4 bytes per parameter on every rank (bf16 weights and gradients) plus 8 / world (fp32
    master and bf16 moments, sharded): for the 8B model on fewer ranks than that needs (one 80 GB H100 holds 4 + 8
    bytes x 8.2e9 = 98 GB only with offloading) the step trains mu2-Qwen3-1.7B at the same batch geometry instead."""
    import gc
    from u2tokenizer_b200 import parallel
    cfg4, geom4, spec4 = make_geometry("cfg4")
    n_par = sum(p.numel() for p in model.parameters())
    own = n_par * (4 + 8 / world) > 0.6 * torch.cuda.mem_get_info()[1]
    if own:
        model.invalidate_engine()
        cfg_s, geom4, _ = make_geometry("cfg2")
        spec4 = dict(spec4, model="mu2-Qwen3-1.7B")
        model = build_model(cfg_s, geom4)
    model.invalidate_engine()
    gc.collect()
    torch.cuda.empty_cache()
    model.train()
    te = model.train_engine(world_size=world, rank=rank)
    try:
        gc.collect()
        torch.cuda.empty_cache()
        free, total = torch.cuda.mem_get_info()
        mom = torch.float32 if te.lay.mat_total / world * 12 + 40e9 < free else torch.bfloat16
        te.init_optimizer(lr=4e-6, weight_decay=0.0, max_grad_norm=1.0, moment_dtype=mom)
        batch = train_batch(geom4, spec4, rank, world)
        ms, launches, phases, out, (ms_e2e, h2d, d2h) = run_train_steps(te, spec4, geom4, batch, steps, warmup, dist, e2e=True)
        n_tok = batch[1].shape[0] * batch[1].shape[1]
        fwd_fl, step_fl = train_flops(geom4, batch[1].shape[0], spec4["frames"], spec4["seq"], spec4["lt"])
        hbm, tf, src = measured_peaks()
        per = ms / steps
        comp = per - phases["exposed_reduce_scatter"] - phases["clip_adamw"]
        return {"workload": f"cfg4: {spec4['model']} training step, 2 volumes / GPU (raw depth 64 / 128 / 256 zero-padded to 8 frames), "
                            "512-token sequences, forward + backward + ZeRO-1 (bucketed NCCL reduce-scatter overlapped with the "
                            "backward, sharded fused AdamW, all-gather overlapped with the next forward)",
                "value": round(world * spec4["batch"] * steps / (ms / 1e3), 4), "unit": "volumes/s", "ms_per_step": round(per, 3),
                "tokens_per_sec": round(world * n_tok * steps / (ms / 1e3), 1), "phases_ms": phases, "steps": steps, "warmup": warmup,
                "gpu_launches": int(launches), "loss": float(out),
                "e2e": {"value": round(world * spec4["batch"] * steps / (ms_e2e / 1e3), 4), "unit": "volumes/s",
                        "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h)},
                "optimizer": f"AdamW, ZeRO-1 over {world} rank(s), fp32 master, {str(mom).split('.')[-1]} moments, "
                             f"{te.lay.n_buckets} buckets of {te.lay.bucket} bf16 gradients",
                "tensor_frac_fwd_bwd": round(step_fl / (comp / 1e3) / 1e12 / tf, 4), "flops_per_step": step_fl}
    finally:
        te.sync_params()
        torch.cuda.synchronize()
        model.__dict__.pop("_u2_train_engine", None)
        te.Gm = te.Gv = te.opt = None
        te.tape = []
        del te
        model.eval()
        if own:
            del model
        gc.collect()
        torch.cuda.empty_cache()


def cfg2_forward_substep(steps=10, warmup=3):
    """BASELINE configs[1] (cfg 2) next to the headline: mu2-Qwen3-1.7B, ONE 256 x 256 x 128 study (4 frames), 288-token
    teacher-forced forward through model(images=, input_ids=, question_ids=) on one GPU. Device-resident and end-to-end
    (pinned host inputs copied every step, the last position's argmax read back) timings, CUDA events."""
    from u2tokenizer_b200 import _lib
    from u2tokenizer_b200.synthetic import synthetic_inputs
    cfg2, geom2, spec2 = make_geometry("cfg2")
    m = build_model(cfg2, geom2)
    try:
        images, ids, qids = synthetic_inputs(geom2, batch=spec2["batch"], frames=spec2["frames"], n_question=spec2["n_question"],
                                             lt=spec2["lt"], seed=1234)
        h = [t.pin_memory() for t in (images, ids, qids)]
        d = [t.cuda() for t in h]

        def run(im, i, q):
            return m(images=im, input_ids=i, question_ids=q).logits[:, -1].float().argmax(-1)

        def timed(fn):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n0 = _lib.launches()
            e0.record()
            for _ in range(steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / steps, (_lib.launches() - n0) // steps
        for _ in range(warmup):
            run(*d)
        ms, launches = timed(lambda: run(*d))
        ms_e2e, _ = timed(lambda: run(*[t.cuda(non_blocking=True) for t in h]).cpu())
        fwd_fl, _ = train_flops(geom2, spec2["batch"], spec2["frames"], ids.shape[1], spec2["lt"])
        hbm, tf, src = measured_peaks()
        return {"workload": "cfg2: mu2-Qwen3-1.7B forward, one 256x256x128 study (4 frames), 288-token sequence, 1 GPU",
                "value": round(spec2["batch"] / (ms / 1e3), 3), "unit": "volumes/s", "ms_per_step": round(ms, 3), "steps": steps,
                "warmup": warmup, "gpu_launches_per_step": int(launches),
                "e2e": {"value": round(spec2["batch"] / (ms_e2e / 1e3), 3), "unit": "volumes/s",
                        "h2d_bytes_per_step": int(sum(t.numel() * t.element_size() for t in h)), "d2h_bytes_per_step": 8},
                "tensor_frac": round(fwd_fl / (ms / 1e3) / 1e12 / tf, 4), "flops_per_step": fwd_fl,
                "note": "repeated same-shape forwards replay one CUDA graph over static buffers (engine.forward_logits)"}
    finally:
        del m
        torch.cuda.empty_cache()


def dump_outputs(d, arrays):
    """Outputs of the timed path as float64 .npy files, so that two builds can be compared output for output (the inputs
    and weights are generated from fixed seeds). Token ids are exact in float64."""
    import numpy as np
    os.makedirs(d, exist_ok=True)
    for name, t in arrays.items():
        np.save(os.path.join(d, f"{name}.npy"), t.detach().double().cpu().numpy())


# ------------------------------------------------------------------------------------------------
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default=os.environ.get("U2_BENCH_WORKLOAD", "cfg3"))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the timed path returned in its last timed step as DIR/<name>.npy (float64)")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    cfg, geom, spec = make_geometry(args.workload)
    metric = "ct_volumes_per_sec"
    base = {"metric": metric, "unit": "volumes/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "data": "synthetic",
            "config": {"workload": f"{args.workload}: {spec['model']} {spec['mode']}, batch {spec['batch']}/GPU, "
                                   f"{spec['frames']} frames of {'x'.join(map(str, geom.image_size))} per volume, "
                                   f"{spec['new_tokens']} new tokens, prompt {geom.num_3d_query_token + spec['n_question']} "
                                   f"tokens, question pad {spec['lt']}",
                       "batch_per_gpu": spec["batch"], "frames": spec["frames"], "new_tokens": spec["new_tokens"],
                       "parallelism": f"dp{args.gpus} (independent replicas, no data-path collective)",
                       "l2": "weights (>= 3.4 GB) and volumes (67 MB each) exceed the 50 MB L2; no explicit flush"}}

    if args.impl == "reference":
        if rank != 0:
            return
        t0 = time.time()
        vals = []
        cb = None
        for _ in range(1):  # one bounded sample (about 10-30 s of CPU work + the weight generation)
            cb = cpu_baseline(geom, spec)
            vals.append(cb["value"])
        v = statistics.median(vals)
        out = dict(base)
        out.update({"impl": "reference", "value": v, "ms_per_step": 1e3 * spec["batch"] / v, "dtype": "f32",
                    "n_gpus": args.gpus, "cpu_baseline": {k: cb[k] for k in ("value", "unit", "cores", "kind", "sample")},
                    "e2e": {"value": v, "unit": "volumes/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
                    "tokens_per_sec": cb["tokens_per_s"], "wall_s": round(time.time() - t0, 1)})
        out["cpu_baseline"]["value"] = v
        print(json.dumps(out), flush=True)
        return

    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (H100); there is no CPU path for the product")
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    from u2tokenizer_b200 import _lib, parallel
    from u2tokenizer_b200.synthetic import synthetic_inputs
    if spec["mode"] in ("train", "dpo"):
        train_main(args, cfg, geom, spec, base, rank, local_rank, world, dist)
        if dist is not None:
            dist.destroy_process_group()
        return
    log(f"[rank {rank}] building {spec['model']} ...")
    model = build_model(cfg, geom)
    images, ids, qids = synthetic_inputs(geom, batch=spec["batch"], frames=spec["frames"], n_question=spec["n_question"],
                                         lt=spec["lt"], seed=1234 + rank)
    h_images, h_ids, h_q = images.pin_memory(), ids.pin_memory(), qids.pin_memory()
    d_images, d_ids, d_q = h_images.cuda(), h_ids.cuda(), h_q.cuda()
    B = spec["batch"]

    def run(im, i, q):
        if spec["mode"] == "generate":
            return model.generate(im, i, question_ids=q, max_new_tokens=spec["new_tokens"], do_sample=False)
        return model(images=im, input_ids=i, question_ids=q).logits[:, -1].float().argmax(-1)

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
            torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = _lib.launches()
        e0.record()
        for _ in range(steps):
            r = fn()
        e1.record()
        barrier()
        ms = parallel.max_over_ranks(e0.elapsed_time(e1), device="cuda")  # device time, slowest rank
        return ms, _lib.launches() - n0, r

    for _ in range(max(args.warmup, 3)):
        run(d_images, d_ids, d_q)
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    prof = os.environ.get("U2_PROFILE_TIMED", "0") != "0"  # cudaProfilerStart/Stop around the timed region only
    if prof:
        torch.cuda.profiler.start()
    ms_dev, launches, res = timed(lambda: run(d_images, d_ids, d_q), args.steps)
    if prof:
        torch.cuda.profiler.stop()
    if rank == 0 and args.dump_outputs:
        dump_outputs(args.dump_outputs, {"generated_ids" if spec["mode"] == "generate" else "next_token_ids": res})

    def e2e_step():
        out = run(h_images.cuda(non_blocking=True), h_ids.cuda(non_blocking=True), h_q.cuda(non_blocking=True))
        return out.cpu()
    e2e_step()
    ms_e2e, _, res_h = timed(e2e_step, args.steps)
    clocks = sampler.stop() if rank == 0 else None
    n_new = int(res.shape[1]) if spec["mode"] == "generate" else 0
    out = None
    if rank == 0:
        vols = world * B * args.steps
        value = vols / (ms_dev / 1e3)
        e2e_v = vols / (ms_e2e / 1e3)
        out = dict(base)
        out.update({"value": round(value, 4), "ms_per_step": round(ms_dev / args.steps, 3), "dtype": "bf16",
                    "tokens_per_sec": round(world * B * n_new * args.steps / (ms_dev / 1e3), 2) if n_new else None,
                    "e2e": {"value": round(e2e_v, 4), "unit": "volumes/s",
                            "h2d_bytes_per_step": int(h_images.numel() * 4 + h_ids.numel() * 8 + h_q.numel() * 8),
                            "d2h_bytes_per_step": int(res_h.numel() * res_h.element_size()),
                            "tokens_per_sec": round(world * B * n_new * args.steps / (ms_e2e / 1e3), 2) if n_new else None},
                    "gpu_launches": int(launches), "clocks": clocks})
        try:
            out["roofline"] = roofline_probe(model, spec, geom)
        except Exception as e:  # the probe must never cost the bench line
            out["roofline"] = {"error": repr(e)}
        try:
            out["roofline_other_kernels"] = extra_rooflines(model, spec, geom)
        except Exception as e:
            out["roofline_other_kernels"] = [{"error": repr(e)}]
        if world == 1 and os.environ.get("U2_BENCH_GPU_EAGER", "1") != "0":
            try:
                out["gpu_eager_baseline"] = gpu_eager_baseline(model, geom, spec, (d_images, d_ids, d_q))
                out["gpu_eager_baseline"]["speedup_of_value"] = round(out["value"] / out["gpu_eager_baseline"]["value"], 2)
            except Exception as e:
                out["gpu_eager_baseline"] = {"error": repr(e)}
            torch.cuda.empty_cache()
    # ---- the training step of the same model on the same ranks (cfg 4: forward + backward + ZeRO-1 gradient exchange + fused
    # AdamW) - the one place where the data-parallel job has a real collective. Every rank takes part; a watchdog makes sure
    # that a failure in here can never cost the generate line above.
    if args.workload == "cfg3" and os.environ.get("U2_BENCH_TRAIN", "1") != "0":
        def bail():
            if rank == 0 and out is not None:
                out["train_step"] = {"error": "training sub-measurement exceeded its time limit"}
                print(json.dumps(out), flush=True)
            os._exit(0)
        wd = threading.Timer(float(os.environ.get("U2_BENCH_TRAIN_TIMEOUT", "420")), bail)
        wd.daemon = True
        wd.start()
        try:
            ts = train_substep(model, rank, local_rank, world, dist, steps=args.steps, warmup=args.warmup)
        except Exception as e:
            ts = {"error": repr(e)}
        wd.cancel()
        if out is not None:
            out["train_step"] = ts
    if rank != 0:
        if dist is not None:
            dist.destroy_process_group()
        return
    if world == 1 and args.workload == "cfg3" and os.environ.get("U2_BENCH_CFG2", "1") != "0":
        try:
            out["cfg2_forward"] = cfg2_forward_substep(steps=args.steps, warmup=args.warmup)
        except Exception as e:
            out["cfg2_forward"] = {"error": repr(e)}
    if world == 1 and not args.no_cpu_baseline:
        try:
            del model
            torch.cuda.empty_cache()
            cb = cpu_baseline(geom, spec)
            out["cpu_baseline"] = {k: cb[k] for k in ("value", "unit", "cores", "kind", "sample")}
            out["cpu_baseline"]["tokens_per_s"] = cb["tokens_per_s"]
        except Exception as e:
            out["cpu_baseline"] = {"error": repr(e)}
    if dist is not None:
        dist.destroy_process_group()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
