"""Parity of the wgmma GEMM (u2_gemm_bf16) against fp32 torch.matmul on the same bf16 inputs."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, b, alpha=1.0, bias=None, act=0, residual=None):
    y = alpha * (a.float() @ b.float().t())
    if bias is not None:
        y = y + bias
    if act == 1:
        y = torch.nn.functional.gelu(y)
    elif act == 2:
        y = torch.nn.functional.silu(y)
    if residual is not None:
        y = y + residual.float()
    return y


def _check(out, ref, tol=1e-2):
    err = (out.float() - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-6
    assert err / scale < tol, f"max abs err {err} (scale {scale})"


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 256, 128), (256, 128, 512), (1000, 776, 328),
                                   (4096, 4096, 4096), (130, 64, 72), (2049, 2304, 768), (5, 16, 8)])
@pytest.mark.parametrize("block_n", [0, 64, 128, 256])
def test_gemm_plain(M, N, K, block_n):
    from u2tokenizer_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    b = torch.randn(N, K, device="cuda", generator=g).bfloat16()
    out = ops.linear(a, b, block_n=block_n)
    torch.cuda.synchronize()
    _check(out, _ref(a, b))


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_gemm_epilogue(act, out_dtype):
    from u2tokenizer_b200 import ops
    M, N, K = 777, 1032, 520
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    b = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g).bfloat16()
    out = ops.linear(a, b, bias, act=act, residual=res, out_dtype=out_dtype, alpha=0.5)
    torch.cuda.synchronize()
    assert out.dtype == out_dtype
    _check(out, _ref(a, b, 0.5, bias, act, res))


def test_gemm_batched_gqa_and_remap():
    """QK^T-style batched call: A [b, S, hq, d], B [b, Sk, hkv, d] (GQA sharing), fp32 scores."""
    from u2tokenizer_b200 import ops
    b_, S, Sk, hq, hkv, d = 2, 200, 333, 8, 2, 64
    g = torch.Generator(device="cuda").manual_seed(11)
    q = torch.randn(b_, S, hq, d, device="cuda", generator=g).bfloat16()
    k = torch.randn(b_, Sk, hkv, d, device="cuda", generator=g).bfloat16()
    ldc = (Sk + 7) // 8 * 8
    sc = torch.zeros(b_, hq, S, ldc, device="cuda", dtype=torch.float32)
    ops.gemm(q, k, sc, M=S, N=Sk, K=d, lda=hq * d, ldb=hkv * d, ldc=ldc, zi=hq, zo=b_,
             b_zi_div=hq // hkv, a_strides=(d, S * hq * d), b_strides=(d, Sk * hkv * d),
             c_strides=(S * ldc, hq * S * ldc), alpha=0.125)
    torch.cuda.synchronize()
    kk = k.repeat_interleave(hq // hkv, dim=2)
    ref = 0.125 * torch.einsum("bshd,bthd->bhst", q.float(), kk.float())
    _check(sc[..., :Sk], ref)
    assert sc[..., Sk:].abs().max().item() == 0.0


def test_gemm_row_remap_and_table_residual():
    """Patch-embed style epilogue: rows scattered into a padded [frames, 2056, N] layout + pos table."""
    from u2tokenizer_b200 import ops
    frames, P, N, K, S_pad = 3, 256, 768, 1024, 264
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn(frames * P, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.03).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    pos = torch.randn(P, N, device="cuda", generator=g).bfloat16()
    out = torch.zeros(frames, S_pad, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, w, out, M=frames * P, N=N, K=K, lda=K, ldb=K, ldc=N, bias=bias, residual=pos, ldr=N,
             res_row_mod=P, row_remap=(P, S_pad, 1))
    torch.cuda.synchronize()
    ref = (a.float() @ w.float().t() + bias).view(frames, P, N) + pos.float()
    _check(out[:, 1:1 + P], ref)
    assert out[:, 0].abs().max().item() == 0.0 and out[:, 1 + P:].abs().max().item() == 0.0
