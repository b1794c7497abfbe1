"""Timeline of the decode linear kernel from in-kernel globaltimer stamps + back-to-back launch timing."""
import sys, torch
sys.path.insert(0, ".")
from u2tokenizer_b200 import ops
B = 4
def probe(N, K, reps=40, nw=24, pdl=True):
    ws = ops.dlinear_new_ws(ops.dlinear_ws_elems(N, K)); cnt = torch.zeros((N + 63) // 64, device="cuda", dtype=torch.int32)
    x = torch.randn(B, K, device="cuda").bfloat16()
    W = [(torch.randn(N, K, device="cuda") * 0.02).bfloat16() for _ in range(nw)]
    out = torch.empty(B, N, device="cuda", dtype=torch.bfloat16)
    dbg = torch.zeros(132 * 8, device="cuda", dtype=torch.int64)
    for w in W: ops.dlinear(x, w, out, ws=ws, counters=cnt, pdl=pdl)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for r in range(reps):
        ops.dlinear(x, W[r % nw], out, ws=ws, counters=cnt, pdl=pdl)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    torch.cuda.synchronize()
    d = dbg.view(132, 8).cpu()
    t0 = d[:, 0].min().item()
    rel = (d - t0).float() / 1e3
    names = ["entry", "setup", "x-wait", "1st full", "last commit", "epi got", "epi done", "exit"]
    mb = N * K * 2 / 1e6
    print(f"N={N} K={K} pdl={pdl}: {us:.2f} us/launch back-to-back ({mb / us / 1e3:.2f} TB/s)")
    print("   stamp (us, min/median/max over CTAs): " + " | ".join(f"{n} {rel[:, i].min():.1f}/{rel[:, i].median():.1f}/{rel[:, i].max():.1f}" for i, n in enumerate(names)))
for pdl in (True, False):
    probe(4096, 4096, pdl=pdl); probe(6144, 4096, pdl=pdl); probe(24576, 4096, pdl=pdl); probe(4096, 12288, pdl=pdl)
