"""Packed (13-bit, lossless) vs bf16 decode-linear weights at the Qwen3-8B widths, alternated in one process.

  ops    : every decode linear alone (ops.dlinear, 4 sequences) over LAYERS distinct layers' weights (working set far
           above the 50 MB L2): time per launch, bytes moved and the bf16-equivalent bytes, outputs compared bit for bit.
  chain  : the 4-op chained launch (o_proj -> gate|up -> down -> next qkv) over the same layers.
  decode : generate_greedy at cfg 3 (mu2-Qwen3-8B, 4 sequences, 256 new tokens) with the engine's packed weights and
           with its bf16 weights (the private U2Engine._decode_bf16 switch): ms per generate and per step, ids compared,
           peak memory of the generate phase.
The GPU name, power limit and clocks are printed with the numbers; --out PATH also writes them as one JSON file.
usage: python tools/packed_ab.py [ops] [chain] [decode] [--layers 36] [--rounds 3] [--reps 5] [--out PATH]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from u2tokenizer_b200 import ops  # noqa: E402

E, I, NQ, V = 4096, 12288, 6144, 151936
B = 4


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"unknown ({e})"
    return f"{torch.cuda.get_device_name(0)} | name, power limit, SM clock, max SM clock, mem clock: {q}"


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def packed_bytes(N, K):
    return -(-N // 128) * (K // 64) * ops.DLIN_PACKED_UNIT_BYTES


def make_layers(n):
    rnd = lambda N, K: (torch.randn(N, K, device="cuda") * K ** -0.5).bfloat16()
    layers = []
    for _ in range(n):
        w = dict(wo=rnd(E, E), wgu=rnd(2 * I, E), wdn=rnd(E, I), wqkv=rnd(NQ, E))
        pk = {k: ops.dlinear_pack(v) for k, v in w.items()}
        assert all(p is not None for p in pk.values()), "synthetic weights must pack"
        layers.append((w, pk))
    return layers


def run_ops(layers, rounds, reps):
    shapes = dict(wqkv=(NQ, E), wo=(E, E), wgu=(2 * I, E), wdn=(E, I))
    ws = ops.dlinear_new_ws(max(ops.dlinear_ws_elems(n, k) for n, k in shapes.values()))
    cnt = torch.zeros((2 * I + 63) // 64 + 8, device="cuda", dtype=torch.int32)
    res = {}
    for name, (N, K) in shapes.items():
        x = (torch.randn(B, K, device="cuda") * 0.5).bfloat16()
        ys = {f: torch.empty(len(layers), B, N, device="cuda", dtype=torch.float32) for f in ("bf16", "packed")}

        def sweep(fmt):
            for li, (w, pk) in enumerate(layers):
                ops.dlinear(x, w[name] if fmt == "bf16" else pk[name], ys[fmt][li], ws=ws, counters=cnt)
        for fmt in ("bf16", "packed"):
            sweep(fmt)
        torch.cuda.synchronize()
        equal = bool(torch.equal(ys["bf16"], ys["packed"]))
        t = {"bf16": [], "packed": []}
        for _ in range(rounds):
            for fmt in ("bf16", "packed"):
                t[fmt].append(timed(lambda: sweep(fmt), reps) * 1e3 / len(layers))
        bf_bytes, pk_bytes = 2 * N * K, packed_bytes(N, K)
        r = dict(N=N, K=K, equal=equal, bf16_bytes=bf_bytes, packed_bytes=pk_bytes)
        for fmt in t:
            us = sorted(t[fmt])
            moved = bf_bytes if fmt == "bf16" else pk_bytes
            r[fmt] = dict(us_per_launch=[round(v, 2) for v in t[fmt]], median_us=round(us[len(us) // 2], 2),
                          moved_TBps=round(moved / us[len(us) // 2] / 1e6, 3),
                          bf16_equiv_TBps=round(bf_bytes / us[len(us) // 2] / 1e6, 3))
        r["speedup"] = round(r["bf16"]["median_us"] / r["packed"]["median_us"], 3)
        print(json.dumps({name: r}), flush=True)
        res[name] = r
    return res


def run_chain(layers, rounds, reps):
    n = len(layers)
    ws = ops.dlinear_new_ws(max(ops.dlinear_ws_elems(a, b) for a, b in ((E, E), (2 * I, E), (E, I), (NQ, E))), lead=(2,))
    cnt = torch.zeros(2, (2 * I + 63) // 64 + 8, device="cuda", dtype=torch.int32)
    gridbar = torch.zeros(4 * n, device="cuda", dtype=torch.int32)
    step = torch.zeros(1, device="cuda", dtype=torch.int32)
    ln = (1 + 0.1 * torch.randn(E, device="cuda"))
    ssq_a, ssq_b = torch.zeros(16, device="cuda"), torch.zeros(16, device="cuda")
    x0 = (torch.randn(B, E, device="cuda")).bfloat16()
    ctx = (torch.randn(B, E, device="cuda")).bfloat16()
    x, xg, xg2 = x0.clone(), torch.empty_like(x0), torch.empty_like(x0)
    act = torch.empty(B, I, device="cuda", dtype=torch.bfloat16)
    qkv = torch.empty(B, NQ, device="cuda", dtype=torch.bfloat16)

    def one_pass(fmt):
        step.add_(1)
        for l, (w, pk) in enumerate(layers):
            ww = w if fmt == "bf16" else pk
            c0, c1 = dict(ws=ws[0], counters=cnt[0]), dict(ws=ws[1], counters=cnt[1])
            chain = [(ctx, ww["wo"], x, dict(residual=x, gamma_next=ln, xg=xg, ssq_out=ssq_a, ssq_zero=ssq_b, **c0)),
                     (xg, ww["wgu"], act, dict(ssq_in=ssq_a, silu_pair=True, **c1)),
                     (act, ww["wdn"], x, dict(residual=x, gamma_next=ln, xg=xg2, ssq_out=ssq_b, ssq_zero=ssq_a, **c0)),
                     (xg2, ww["wqkv"], qkv, dict(ssq_in=ssq_b, **c1))]
            ops.dlinear_multi(chain, gridbar=gridbar[4 * l:4 * l + 4], step_dev=step)

    outs = {}
    for fmt in ("bf16", "packed"):
        x.copy_(x0)
        ssq_a.zero_(); ssq_b.zero_()
        one_pass(fmt)
        torch.cuda.synchronize()
        outs[fmt] = (x.clone(), act.clone(), qkv.clone())
    equal = all(torch.equal(a, b) for a, b in zip(outs["bf16"], outs["packed"]))
    t = {"bf16": [], "packed": []}
    for _ in range(rounds):
        for fmt in ("bf16", "packed"):
            one_pass(fmt)
            t[fmt].append(timed(lambda: one_pass(fmt), reps) * 1e3 / n)
    bf_bytes = 2 * (E * E + 2 * I * E + E * I + NQ * E)
    pk_bytes = sum(packed_bytes(a, b) for a, b in ((E, E), (2 * I, E), (E, I), (NQ, E)))
    r = dict(equal_one_pass=equal, bf16_bytes=bf_bytes, packed_bytes=pk_bytes)
    for fmt in t:
        us = sorted(t[fmt])
        r[fmt] = dict(us_per_launch=[round(v, 1) for v in t[fmt]], median_us=round(us[len(us) // 2], 1),
                      bf16_equiv_TBps=round(bf_bytes / us[len(us) // 2] / 1e6, 3))
    r["speedup"] = round(r["bf16"]["median_us"] / r["packed"]["median_us"], 3)
    print(json.dumps({"chain": r}), flush=True)
    return r


def run_decode(rounds):
    import bench
    cfg, geom, spec = bench.make_geometry("cfg3")
    model = bench.build_model(cfg, geom)
    eng = model.engine()
    n_new = 256
    L = geom.num_3d_query_token + spec["n_question"]
    gen = torch.Generator(device="cuda").manual_seed(7)
    emb = (torch.randn(spec["batch"], L, geom.hidden_size, device="cuda", generator=gen) * 0.02).bfloat16()
    packed_mb = sum(p.buf.numel() for p in eng._packed.values()) / 2 ** 20
    res = dict(packed_matrices=len(eng._packed), packed_MiB=round(packed_mb, 1), ms_per_generate={}, ids_equal=None)
    ids = {}
    for fmt in ("bf16", "packed"):
        eng._decode_bf16 = fmt == "bf16"
        eng._gen_state = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ids[fmt] = eng.generate_greedy(emb, n_new)
        torch.cuda.synchronize()
        res[f"peak_GiB_{fmt}"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    res["ids_equal"] = bool(torch.equal(ids["bf16"], ids["packed"]))
    for fmt in ("bf16", "packed"):
        res["ms_per_generate"][fmt] = []
    for _ in range(rounds):
        for fmt in ("bf16", "packed"):
            eng._decode_bf16 = fmt == "bf16"
            eng._gen_state = None
            eng.generate_greedy(emb, n_new)  # capture
            torch.cuda.synchronize()
            ms = timed(lambda: eng.generate_greedy(emb, n_new), 1)
            res["ms_per_generate"][fmt].append(round(ms, 2))
    for fmt in ("bf16", "packed"):
        v = sorted(res["ms_per_generate"][fmt])
        res[f"ms_per_step_{fmt}"] = round(v[len(v) // 2] / n_new, 4)
    eng._decode_bf16 = False
    print(json.dumps({"decode": res}), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("modes", nargs="*", default=["ops", "chain"])
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5, help="passes over all layers per timed round")
    ap.add_argument("--out", default=None, help="JSON file for the results (default: printed only)")
    args = ap.parse_args()
    out = dict(gpu=gpu_info())
    print(out["gpu"], flush=True)
    torch.manual_seed(0)
    if "ops" in args.modes or "chain" in args.modes:
        layers = make_layers(args.layers)
        if "ops" in args.modes:
            out["ops"] = run_ops(layers, args.rounds, args.reps)
        if "chain" in args.modes:
            out["chain"] = run_chain(layers, args.rounds, args.reps)
        del layers
        torch.cuda.empty_cache()
    if "decode" in args.modes:
        out["decode"] = run_decode(args.rounds)
    out["gpu_after"] = gpu_info()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
