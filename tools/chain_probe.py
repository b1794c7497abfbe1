"""In-kernel timeline (globaltimer stamps) of the 4-op decode chain launch at Qwen3-8B shapes."""
import os, sys, torch
sys.path.insert(0, ".")
from u2tokenizer_b200 import ops
B, E, I, NQ = 4, 4096, 12288, 6144
dev = "cuda"
rnd = lambda *s, sc=1.0: (torch.randn(*s, device=dev) * sc)
nlay = 6
W = [dict(wo=rnd(E, E, sc=E ** -0.5).bfloat16(), wgu=rnd(2 * I, E, sc=E ** -0.5).bfloat16(), wdn=rnd(E, I, sc=I ** -0.5).bfloat16(),
          wqkv=rnd(NQ, E, sc=E ** -0.5).bfloat16()) for _ in range(nlay)]
ln = 1 + 0.1 * rnd(E)
tiles = (2 * I + 127) // 128
ws = ops.dlinear_new_ws(max(ops.dlinear_ws_elems(n, k) for n, k in ((E, E), (2 * I, E), (E, I), (NQ, E))), device=dev, lead=(2,)); cnt = torch.zeros(2, tiles * 2 + 8, device=dev, dtype=torch.int32)
FINE = os.environ.get("U2_FINE_DEPS", "0") != "0"
flags = torch.zeros(nlay, 4, 256, device=dev, dtype=torch.int32)
gridbar = torch.zeros(4 * nlay, device=dev, dtype=torch.int32); step = torch.zeros(1, device=dev, dtype=torch.int32)
ssq_a, ssq_b = torch.zeros(16, device=dev), torch.zeros(16, device=dev)
x = rnd(B, E).bfloat16(); xg = torch.empty_like(x); xg2 = torch.empty_like(x); ctx = rnd(B, E).bfloat16()
act = torch.empty(B, I, device=dev, dtype=torch.bfloat16); qkv = torch.empty(B, NQ, device=dev, dtype=torch.bfloat16)
dbg = torch.zeros(132 * 4 * 8, device=dev, dtype=torch.int64)
def chain(l, d=None):
    w = W[l]
    sc = int(os.environ.get("U2_DL_SCHED", "0"))
    c0 = dict(ws=ws[0], counters=cnt[0], sched=sc); c1 = dict(ws=ws[1], counters=cnt[1], sched=sc)
    fl = flags[l] if FINE else [None] * 4
    dep = lambda i, sh: dict(dep_flags=fl[i], dep_shift=sh) if FINE else {}
    return [(ctx, w["wo"], x, dict(residual=x, gamma_next=ln, xg=xg, ssq_out=ssq_a, ssq_zero=ssq_b, dbg=d, out_flags=fl[0], **c0)),
            (xg, w["wgu"], act, dict(ssq_in=ssq_a, silu_pair=True, out_flags=fl[1], **dep(0, 1), **c1)),
            (act, w["wdn"], x, dict(residual=x, gamma_next=ln, xg=xg2, ssq_out=ssq_b, ssq_zero=ssq_a, out_flags=fl[2], **dep(1, 0), **c0)),
            (xg2, w["wqkv"], qkv, dict(ssq_in=ssq_b, **dep(2, 1), **c1))]
for it in range(3):
    step += 1
    for l in range(nlay):
        ops.dlinear_multi(chain(l), gridbar=gridbar[4 * l:4 * l + 4], step_dev=step)
torch.cuda.synchronize()
import os
LA = int(os.environ.get("U2_L2_LOOKAHEAD", "24")); NX = int(os.environ.get("U2_L2_NEXT", "20"))
nxw = lambda l: ((W[(l + 1) % nlay]["wo"], 1 << 20), (W[(l + 1) % nlay]["wgu"], NX)) if NX >= 0 else ()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
step += 1
e0.record()
for l in range(nlay):
    ops.dlinear_multi(chain(l), gridbar=gridbar[4 * l:4 * l + 4], step_dev=step, lookahead_units=LA, next_weights=nxw(l), pre_stages=int(os.environ.get("U2_PRE_STAGES", "0")))
e1.record(); torch.cuda.synchronize()
print(f"chain launch: {e0.elapsed_time(e1) * 1e3 / nlay:.1f} us each (stream-only bound {2 * (E * E + 2 * I * E + E * I + NQ * E) / 6.4e6:.1f} us)")
step += 1
ops.dlinear_multi(chain(2, dbg), gridbar=gridbar[8:12], step_dev=step, lookahead_units=LA, next_weights=nxw(2), pre_stages=int(os.environ.get("U2_PRE_STAGES", "0"))); torch.cuda.synchronize()
d = dbg.view(132, 4, 8).cpu()
t0 = d[:, 0, 0].min().item()
rel = (d - t0).float() / 1e3
names = ["Wpre", "dep ok", "1st full", "last commit", "last acc", "epi done", "fin wait", "fin got"]
for oi, on in enumerate(["o_proj", "gate_up", "down", "qkv"]):
    print(f"{on:8s} " + " | ".join(f"{n} {rel[:, oi, i].min():.1f}/{rel[:, oi, i].median():.1f}/{rel[:, oi, i].max():.1f}" for i, n in enumerate(names[:6])))
    fin = d[:, oi, 6] > 0
    if fin.any():
        fw, fg, ed = rel[fin, oi, 6], rel[fin, oi, 7], rel[fin, oi, 5]
        print(f"         finalisers ({int(fin.sum())}): wait-start {fw.min():.1f}/{fw.median():.1f}/{fw.max():.1f} | sums in {fg.min():.1f}/{fg.median():.1f}/{fg.max():.1f} | done {ed.min():.1f}/{ed.median():.1f}/{ed.max():.1f}")
