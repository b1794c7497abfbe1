"""The 4-op decode chain launch (o_proj -> gate|up -> down -> next qkv) at Qwen3-8B shapes: launch time without and
with the L2 look-ahead prefetches, and the in-kernel timeline (globaltimer stamps) of every op boundary.
The name and power limit of the GPU are printed with the numbers.

The chain runs over NLAY distinct layers' weights (2.3 GB for 6 layers, far above the 50 MB L2), so each launch
streams its weights from HBM as in a decode step. The two configurations alternate, ROUNDS rounds each.
Per boundary i -> i+1 the gap is, per CTA, from the last MMA of op i (its last weight stage landed and was
consumed) to the first stage of op i+1 landing at the MMA warpgroup: the time this SM's tensor pipe waits on
the dependency. Usage: python tools/chain_probe.py [--layers 6] [--rounds 5] [--reps 20]."""
import argparse, os, subprocess, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from u2tokenizer_b200 import ops

ap = argparse.ArgumentParser()
ap.add_argument("--layers", type=int, default=6)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--reps", type=int, default=20, help="passes over all layers per timed round")
args = ap.parse_args()

B, E, I, NQ = 4, 4096, 12288, 6144
dev = "cuda"
torch.manual_seed(0)
rnd = lambda *s, sc=1.0: (torch.randn(*s, device=dev) * sc)
nlay = args.layers
W = [dict(wo=rnd(E, E, sc=E ** -0.5).bfloat16(), wgu=rnd(2 * I, E, sc=E ** -0.5).bfloat16(), wdn=rnd(E, I, sc=I ** -0.5).bfloat16(),
          wqkv=rnd(NQ, E, sc=E ** -0.5).bfloat16()) for _ in range(nlay)]
ln = 1 + 0.1 * rnd(E)
tiles = (2 * I + 127) // 128
ws = ops.dlinear_new_ws(max(ops.dlinear_ws_elems(n, k) for n, k in ((E, E), (2 * I, E), (E, I), (NQ, E))), device=dev, lead=(2,)); cnt = torch.zeros(2, tiles * 2 + 8, device=dev, dtype=torch.int32)
gridbar = torch.zeros(4 * nlay, device=dev, dtype=torch.int32); step = torch.zeros(1, device=dev, dtype=torch.int32)
ssq_a, ssq_b = torch.zeros(16, device=dev), torch.zeros(16, device=dev)
x = rnd(B, E).bfloat16(); xg = torch.empty_like(x); xg2 = torch.empty_like(x); ctx = rnd(B, E).bfloat16()
act = torch.empty(B, I, device=dev, dtype=torch.bfloat16); qkv = torch.empty(B, NQ, device=dev, dtype=torch.bfloat16)
nsm = torch.cuda.get_device_properties(0).multi_processor_count
dbg = torch.zeros(nlay, nsm * 4 * 8, device=dev, dtype=torch.int64)
NAMES = ["o_proj", "gate_up", "down", "qkv"]


def chain(l, d=None):
    w = W[l]
    c0 = dict(ws=ws[0], counters=cnt[0]); c1 = dict(ws=ws[1], counters=cnt[1])
    return [(ctx, w["wo"], x, dict(residual=x, gamma_next=ln, xg=xg, ssq_out=ssq_a, ssq_zero=ssq_b, dbg=d, **c0)),
            (xg, w["wgu"], act, dict(ssq_in=ssq_a, silu_pair=True, **c1)),
            (act, w["wdn"], x, dict(residual=x, gamma_next=ln, xg=xg2, ssq_out=ssq_b, ssq_zero=ssq_a, **c0)),
            (xg2, w["wqkv"], qkv, dict(ssq_in=ssq_b, **c1))]


def staging(l, on):
    """dlinear_multi arguments of layer l's launch. "la": the L2 look-ahead (U2_L2_LOOKAHEAD tiles per CTA beyond
    the ring at in-launch boundaries; the next layer's o_proj and U2_L2_NEXT tiles per CTA of its gate|up)."""
    if not on:
        return {}
    nw = W[(l + 1) % nlay]
    return dict(lookahead_units=LA, next_weights=((nw["wo"], 1 << 20), (nw["wgu"], NX)))


LA, NX = int(os.environ.get("U2_L2_LOOKAHEAD", "12")), int(os.environ.get("U2_L2_NEXT", "12"))
CONFIGS = {"off": False, "la": True}


def one_pass(on, with_dbg=False):
    step.add_(1)
    for l in range(nlay):
        ops.dlinear_multi(chain(l, dbg[l] if with_dbg else None), gridbar=gridbar[4 * l:4 * l + 4], step_dev=step,
                          **staging(l, on))


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        pl = f"unknown ({e})"
    return f"{name}, power limit / max SM clock: {pl}"


print(gpu_info())
for on in CONFIGS.values():
    for _ in range(3):
        one_pass(on)
torch.cuda.synchronize()

per_launch = {k: [] for k in CONFIGS}
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for r in range(args.rounds):
    for k, on in CONFIGS.items():
        one_pass(on)
        e0.record()
        for _ in range(args.reps):
            one_pass(on)
        e1.record(); torch.cuda.synchronize()
        per_launch[k].append(e0.elapsed_time(e1) * 1e3 / (args.reps * nlay))
wbytes = 2 * (E * E + 2 * I * E + E * I + NQ * E)
for k, v in per_launch.items():
    v = sorted(v)
    med = v[len(v) // 2]
    print(f"chain launch, staging {k:3s}: median {med:.1f} us (min {v[0]:.1f}, max {v[-1]:.1f}, {len(v)} rounds x "
          f"{args.reps * nlay} launches)  {wbytes / med / 1e6:.2f} TB/s of weights")

for k, on in CONFIGS.items():
    one_pass(on, with_dbg=True); torch.cuda.synchronize()
    d = dbg.view(nlay, nsm, 4, 8).cpu()
    for i in range(3):
        gap = (d[:, :, i + 1, 2] - d[:, :, i, 3]).float().flatten() / 1e3
        q = torch.quantile(gap, torch.tensor([0.1, 0.5, 0.9]))
        print(f"staging {k:3s} boundary {NAMES[i]:>7s} -> {NAMES[i + 1]:7s}: gap p10/median/p90 "
              f"{q[0]:.1f}/{q[1]:.1f}/{q[2]:.1f} us")
    span = (d[:, :, 3, 5].max(dim=1).values - d[:, :, 0, 0].min(dim=1).values).float() / 1e3
    print(f"staging {k:3s} first stamp -> last epilogue, median over layers: {span.median():.1f} us")
