"""mu2-Phi-3-mini at the cfg 3 geometry (batch 4, 8 frames of 32x256x256 per volume, prompt 288 tokens, 256 greedy
tokens) on random-init weights: volumes/s of generate(), the decode step, its effective weight-stream bandwidth, and
the head_dim-96 decode attention alone at T ~ 1024 (batch 4) and at a window-bound T = 4000 > 2047 (one request).

    python tools/phi3_probe.py [--out FILE]

Prints one JSON line. Nothing is written to the tree unless --out names a file there."""
import argparse
import json
import math
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from u2tokenizer_b200 import ops  # noqa: E402
from u2tokenizer_b200.configuration import PHI3_MINI_4K, U2Phi3Config  # noqa: E402
from u2tokenizer_b200.engine import U2Engine  # noqa: E402
from u2tokenizer_b200.geometry import Geometry  # noqa: E402
from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict  # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def attention_tbps(g, B, T, window, splits):
    Hq, Hkv, dh = g.num_attention_heads, g.num_key_value_heads, g.head_dim
    Tmax = T + 8
    kc = torch.randn(B, Hkv, Tmax, dh, device="cuda").bfloat16()
    vc = torch.randn_like(kc)
    qkv = torch.randn(B, (Hq + 2 * Hkv) * dh, device="cuda").bfloat16()
    out = torch.empty(B, Hq * dh, device="cuda", dtype=torch.bfloat16)
    pos = torch.full((B,), T - 1, device="cuda", dtype=torch.int32)
    inv = 1.0 / (g.rope_theta ** (torch.arange(0, dh, 2, device="cuda").float() / dh))
    ms = timed(lambda: ops.decode_attention_fused(qkv, kc, vc, out, B=B, Hq=Hq, Hkv=Hkv, dh=dh, Tmax=Tmax, inv_freq=inv,
                                                  scale=1 / math.sqrt(dh), pos_dev=pos, kv_splits=splits,
                                                  pos_per_seq=True, window=window), 200)
    keys = min(T, window) if window else T
    return ms, B * Hkv * keys * dh * 2 * 2 / (ms * 1e-3) / 1e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    g = Geometry.from_hf(U2Phi3Config(**PHI3_MINI_4K))
    sd = synthetic_state_dict(g, seed=0, device="cuda", dtype=torch.bfloat16, bigram=1.0)
    eng = U2Engine(g, sd, device="cuda")
    del sd
    torch.cuda.empty_cache()
    B, frames, new = 4, 8, 256
    images, ids, qids = synthetic_inputs(g, batch=B, frames=frames, n_question=32, lt=512, device="cuda")
    run = lambda n: eng.generate(eng.multimodal_embeds(ids, images, qids), max_new_tokens=n)
    run(new)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    reps = 3
    for _ in range(reps):
        run(new)
    torch.cuda.synchronize()
    total_s = (time.perf_counter() - t0) / reps
    t_short = timed(lambda: run(32), 3)
    t_long = timed(lambda: run(new), 3)
    step_ms = (t_long - t_short) / (new - 32)
    E, I, V = g.hidden_size, g.intermediate_size, g.vocab_size
    nqkv = (g.num_attention_heads + 2 * g.num_key_value_heads) * g.head_dim
    w_bytes = 2 * (g.num_hidden_layers * (nqkv * E + E * g.num_attention_heads * g.head_dim + 2 * I * E + E * I) + V * E)
    kv_bytes_per_step = 2 * 2 * g.num_hidden_layers * B * g.num_key_value_heads * g.head_dim * (ids.shape[1] + new // 2)
    splits = eng._kv_splits(B)
    a1024 = attention_tbps(g, B, 1024, g.window, splits)
    along = attention_tbps(g, 1, 4000, g.window, eng._kv_splits(1))
    along_nowin = attention_tbps(g, 1, 4000, 0, eng._kv_splits(1))
    res = dict(
        workload="mu2-Phi-3-mini greedy generate, batch 4, 8 frames of 32x256x256, prompt 288, 256 new tokens",
        gpu=torch.cuda.get_device_name(), volumes_per_s=round(B / total_s, 4), generate_s=round(total_s, 4),
        decode_step_ms=round(step_ms, 4), decode_weight_gb=round(w_bytes / 1e9, 3),
        decode_kv_gb_mean_per_step=round(kv_bytes_per_step / 1e9, 3),
        decode_step_effective_tbps=round((w_bytes + kv_bytes_per_step) / (step_ms * 1e-3) / 1e12, 3),
        attn_T1024_B4=dict(ms_per_layer=round(a1024[0], 4), tbps=round(a1024[1], 3), kv_splits=splits),
        attn_T4000_B1_window2047=dict(ms_per_layer=round(along[0], 4), tbps=round(along[1], 3)),
        attn_T4000_B1_no_window=dict(ms_per_layer=round(along_nowin[0], 4), tbps=round(along_nowin[1], 3)),
    )
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
