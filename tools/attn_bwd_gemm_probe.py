"""The two short-K GEMMs of the ViT attention backward (K = head_dim = 64, S = 2049, bf16 S x S output per (frame, head)):
P = exp(scale * q.k - lse) and dS = P * (dO.V^T - D), both formed in the GEMM epilogue - next to the same product with a
plain bf16 / fp32 epilogue. usage: python tools/attn_bwd_gemm_probe.py [frames] [reps]"""
import sys
import os
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from u2tokenizer_b200 import ops

b = int(sys.argv[1]) if len(sys.argv) > 1 else 16
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
h, S, dh = 12, 2049, 64
Sp = (S + 7) // 8 * 8
g = torch.Generator(device="cuda").manual_seed(3)
qkv = torch.randn(b, Sp, 3, h, dh, device="cuda", generator=g).bfloat16()
q, k, v = qkv[:, :S, 0], qkv[:, :S, 1], qkv[:, :S, 2]
do = torch.randn(b, S, h, dh, device="cuda", generator=g).bfloat16()
scale = dh ** -0.5
lse = torch.logsumexp(torch.einsum("bqhd,bkhd->bhqk", q[:1].float(), k[:1].float()) * scale, -1).repeat(b, 1, 1).contiguous()
D = torch.randn(b, h, S, device="cuda", generator=g) * 0.1
pr = torch.empty(b, h, S, Sp, device="cuda", dtype=torch.bfloat16)
f32 = torch.empty(b, h, S, Sp, device="cuda", dtype=torch.float32) if b <= 16 else None
common = dict(M=S, N=S, K=dh, ldc=Sp, zi=h, zo=b, c_strides=(S * Sp, h * S * Sp))
qa = dict(lda=q.stride(1), ldb=k.stride(1), a_strides=(q.stride(2), q.stride(0)), b_strides=(k.stride(2), k.stride(0)))
da = dict(lda=do.stride(1), ldb=v.stride(1), a_strides=(do.stride(2), do.stride(0)), b_strides=(v.stride(2), v.stride(0)))
runs = {
    "plain bf16": lambda: ops.gemm(q, k, pr, alpha=scale, **qa, **common),
    "P = exp(s - lse)": lambda: ops.gemm(q, k, pr, alpha=scale, epi_op=1, rowvec=lse, rv_strides=(S, h * S), **qa, **common),
    "dS = P * (dP - D)": lambda: ops.gemm(do, v, pr, epi_op=2, rowvec=D, rv_strides=(S, h * S), mul=pr, **da, **common),
}
if f32 is not None:
    runs["plain fp32"] = lambda: ops.gemm(q, k, f32, alpha=scale, **qa, **common)
fl = 2.0 * b * h * S * S * dh
for name, fn in runs.items():
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    tiles = b * h * ((S + 127) // 128) * ((S + 255) // 256)
    print(f"{name:20s} {ms * 1e3:8.1f} us  {fl / ms / 1e9:6.0f} TFLOP/s  {b * h * S * Sp * 2 / ms / 1e6:6.0f} GB/s written  "
          f"{ms * 1e3 / (tiles / 132):.2f} us per tile and SM", flush=True)
