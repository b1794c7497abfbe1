"""Training path on the GPU: every backward kernel against torch autograd on the same inputs, the transposed-operand
GEMM against torch.matmul, and the whole forward + backward (TrainEngine) against the autograd gradients of the fp32
oracle (oracle/u2_oracle.py on CUDA; its gradients are pinned against the reference modules' and HF's in
tests/test_oracle_grad_pin.py).

Tolerances (bf16 activations / gradients, fp32 accumulation): per tensor max|d - ref| / max|ref| <= 4e-2 and cosine >=
0.995 for gradients of the full model (they pass through ~20 bf16-rounded layers), 2e-2 for single kernels."""
import math

import pytest
import torch
import torch.nn.functional as F

from common import cosine, rel_err, tiny_geometry
from oracle import u2_oracle as O
from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _ops():
    from u2tokenizer_b200 import ops, train_ops
    return ops, train_ops


def close(a, b, tol=2e-2, what=""):
    e, c = rel_err(a.float().cpu(), b.float().cpu()), cosine(a.float().cpu(), b.float().cpu())
    assert e < tol and c > 0.999, f"{what}: rel_err {e:.4g} cos {c:.6f}"


# ------------------------------------------------------------------------------------------------
# GEMM with transposed (MN-major) operands
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (200, 72, 136), (65, 24, 65), (1024, 768, 2056), (96, 1024, 520)])
@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, False), (True, True)])
def test_gemm_transposed_operands(M, N, K, a_mn, b_mn):
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g).to(BF)
    B = torch.randn(N, K, device="cuda", generator=g).to(BF)
    ref = A.float() @ B.float().t()
    Kp, Mp, Np = (K + 7) // 8 * 8, (M + 7) // 8 * 8, (N + 7) // 8 * 8
    if a_mn:
        a_mem = torch.zeros(K, Mp, device="cuda", dtype=BF)
        a_mem[:, :M] = A.t()
        lda = Mp
    else:
        a_mem = torch.zeros(M, Kp, device="cuda", dtype=BF)
        a_mem[:, :K] = A
        lda = Kp
    if b_mn:
        b_mem = torch.zeros(K, Np, device="cuda", dtype=BF)
        b_mem[:, :N] = B.t()
        ldb = Np
    else:
        b_mem = torch.zeros(N, Kp, device="cuda", dtype=BF)
        b_mem[:, :K] = B
        ldb = Kp
    for bn in (0, 64, 128, 256):
        out = torch.empty(M, N, device="cuda", dtype=torch.float32)
        ops.gemm(a_mem, b_mem, out, M=M, N=N, K=K, lda=lda, ldb=ldb, ldc=N, a_mn=a_mn, b_mn=b_mn, block_n=bn)
        close(out, ref, 1e-2, f"gemm a_mn={a_mn} b_mn={b_mn} block_n={bn}")


def test_gemm_transposed_batched_accumulate():
    """Batched P^T @ dO with strided views (the attention backward's dV) and accumulation into a bf16 C."""
    ops, T = _ops()
    b, h, Sq, Sk, dh = 2, 3, 40, 33, 24
    Skp = 40
    g = torch.Generator(device="cuda").manual_seed(1)
    P = torch.randn(b, h, Sq, Skp, device="cuda", generator=g).to(BF)
    do = torch.randn(b, Sq, h, dh, device="cuda", generator=g).to(BF)
    base = torch.randn(b, Sk, h, dh, device="cuda", generator=g).to(BF)
    out = base.clone()
    ops.gemm(P, do, out, M=Sk, N=dh, K=Sq, lda=Skp, ldb=do.stride(1), ldc=out.stride(1), zi=h, zo=b,
             a_strides=(Sq * Skp, h * Sq * Skp), b_strides=(do.stride(2), do.stride(0)), c_strides=(out.stride(2), out.stride(0)),
             a_mn=True, b_mn=True, alpha=0.5, residual=out, ldr=out.stride(1))
    ref = base.float() + 0.5 * torch.einsum("bhqk,bqhd->bkhd", P[..., :Sk].float(), do.float())
    close(out, ref, 2e-2, "batched P^T dO accumulate")


def test_flash_lse_and_fused_attention_backward_epilogues():
    """The ViT attention backward without fp32 score / dP round trips: LSE out of the fused forward, P rebuilt in the score
    GEMM's epilogue, dS formed in the dP GEMM's epilogue (in place) - against explicit fp32 attention."""
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(11)
    b, S, h, dh = 2, 300, 3, 64
    Skp = (S + 7) // 8 * 8
    qkv = torch.randn(b, S, 3, h, dh, device="cuda", generator=g).to(BF)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    do = torch.randn(b, S, h, dh, device="cuda", generator=g).to(BF)
    scale = dh ** -0.5
    sc = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * scale
    P = torch.softmax(sc, -1)
    O = torch.einsum("bhqk,bkhd->bqhd", P, v.float())
    out = torch.empty(b, S, h * dh, device="cuda", dtype=BF)
    lse = torch.empty(b, h, S, device="cuda")
    ops.flash_attention_d64(q, k, v, out, scale, lse=lse)
    close(out.view(b, S, h, dh), O, 2e-2, "flash out")
    assert float((lse - torch.logsumexp(sc, -1)).abs().max()) < 2e-2
    pr = torch.empty(b, h, S, Skp, device="cuda", dtype=BF)
    ops.gemm(q, k, pr, M=S, N=S, K=dh, lda=q.stride(1), ldb=k.stride(1), ldc=Skp, zi=h, zo=b, a_strides=(q.stride(2), q.stride(0)),
             b_strides=(k.stride(2), k.stride(0)), c_strides=(S * Skp, h * S * Skp), alpha=scale, epi_op=1, rowvec=lse,
             rv_strides=(S, h * S))
    close(pr[..., :S], P, 2e-2, "P from the score GEMM epilogue")
    D = T.rowdot(do, out.view(b, S, h, dh))
    close(D, (do.float() * O).sum(-1).permute(0, 2, 1), 2e-2, "rowdot")
    dP = torch.einsum("bqhd,bkhd->bhqk", do.float(), v.float())
    dS = P * (dP - (dP * P).sum(-1, keepdim=True))
    ops.gemm(do, v, pr, M=S, N=S, K=dh, lda=do.stride(1), ldb=v.stride(1), ldc=Skp, zi=h, zo=b, a_strides=(do.stride(2), do.stride(0)),
             b_strides=(v.stride(2), v.stride(0)), c_strides=(S * Skp, h * S * Skp), epi_op=2, rowvec=D, rv_strides=(S, h * S), mul=pr)
    close(pr[..., :S], dS, 3e-2, "dS from the dP GEMM epilogue (in place)")


def test_linear_dgrad_wgrad():
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(300, 136, device="cuda", generator=g).to(BF)
    w = (torch.randn(72, 136, device="cuda", generator=g) * 0.1).to(BF)
    dy = torch.randn(300, 72, device="cuda", generator=g).to(BF)
    close(T.linear_dgrad(dy, w), dy.float() @ w.float(), 1e-2, "dgrad")
    gw = torch.zeros(72, 136, device="cuda", dtype=BF)
    T.linear_wgrad(dy, x, gw, accumulate=True)
    T.linear_wgrad(dy, x, gw, accumulate=True)
    close(gw, 2 * dy.float().t() @ x.float(), 1e-2, "wgrad x2")


# ------------------------------------------------------------------------------------------------
# row-wise / elementwise backward kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E", [96, 768, 4096])
def test_norm_backward(E):
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(E)
    rows = 77
    x = torch.randn(rows, E, device="cuda", generator=g).to(BF)
    dy = torch.randn(rows, E, device="cuda", generator=g).to(BF)
    dres = torch.randn(rows, E, device="cuda", generator=g).to(BF)
    gamma = (1 + 0.1 * torch.randn(E, device="cuda", generator=g))
    beta = 0.1 * torch.randn(E, device="cuda", generator=g)
    for rms in (False, True):
        xr = x.float().requires_grad_(True)
        gr = gamma.clone().requires_grad_(True)
        br = beta.clone().requires_grad_(True)
        y = F.layer_norm(xr, (E,), gr, br, 1e-5) if not rms else gr * (xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-6))
        y.backward(dy.float())
        dg = torch.zeros(E, device="cuda")
        db = torch.zeros(E, device="cuda")
        if rms:
            dx = T.rmsnorm_bwd(x, gamma, dy, dres=dres, dgamma=dg, eps=1e-6)
        else:
            dx = T.layernorm_bwd(x, gamma, dy, dres=dres, dgamma=dg, dbeta=db, eps=1e-5)
        close(dx, xr.grad + dres.float(), 2e-2, f"norm dx rms={rms}")
        close(dg, gr.grad, 2e-2, f"norm dgamma rms={rms}")
        if not rms:
            close(db, br.grad, 2e-2, "norm dbeta")
        # in place on the pending gradient, frozen gamma
        pend = dres.clone()
        (T.rmsnorm_bwd if rms else T.layernorm_bwd)(x, gamma, dy, dres=pend, out=pend, eps=1e-6 if rms else 1e-5)
        close(pend, xr.grad + dres.float(), 2e-2, "norm dx in place")


def test_gelu_silu_backward():
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    x = (2 * torch.randn(64, 256, device="cuda", generator=g)).to(BF)
    dy = torch.randn(64, 256, device="cuda", generator=g).to(BF)
    xr = x.float().requires_grad_(True)
    F.gelu(xr).backward(dy.float())
    close(T.gelu(x), F.gelu(x.float()), 1e-2, "gelu")
    close(T.gelu_bwd(x, dy), xr.grad, 1e-2, "gelu bwd")
    gu = torch.randn(50, 512, device="cuda", generator=g).to(BF)
    da = torch.randn(50, 256, device="cuda", generator=g).to(BF)
    gur = gu.float().requires_grad_(True)
    (F.silu(gur[:, :256]) * gur[:, 256:]).backward(da.float())
    close(T.silu_mul_bwd(gu, da), gur.grad, 1e-2, "silu_mul bwd")
    close(ops.silu_mul(gu, interleaved=False), F.silu(gu.float()[:, :256]) * gu.float()[:, 256:], 1e-2, "silu_mul fwd")


@pytest.mark.parametrize("n", [5, 33, 256, 1792, 2049, 9000])
def test_softmax_backward_and_relbias(n):
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(n)
    n0, H, S = 2, 3, 7
    npad = (n + 7) // 8 * 8
    sc = torch.randn(n0, H, S, npad, device="cuda", generator=g)
    P = torch.empty(n0, H, S, npad, device="cuda", dtype=BF)
    st = (H * S * npad, S * npad, npad)
    ops.softmax(sc, P, n0=n0, H=H, S=S, n=n, in_strides=st, out_strides=st, zero_pad_to=npad)
    dP = torch.randn(n0, H, S, npad, device="cuda", generator=g)
    Pf = P.float()[..., :n]
    ref = Pf * (dP[..., :n] - (dP[..., :n] * Pf).sum(-1, keepdim=True))
    dS = torch.empty_like(P)
    T.softmax_bwd(P, dP, dS, n0=n0, H=H, S=S, n=n, p_strides=st, dp_strides=st, ds_strides=st, zero_pad_to=npad)
    close(dS[..., :n], ref, 2e-2, "softmax bwd")
    assert float(dS[..., n:].abs().max()) == 0.0 if npad > n else True
    if n <= 512 and S <= 512:
        rel_max = 512
        drel = torch.zeros(2 * rel_max - 1, H, device="cuda")
        T.relbias_grad(dS, drel, n0=n0, H=H, S=S, n=n, strides=st, rel_max=rel_max)
        want = torch.zeros_like(drel)
        d = dS.float()
        for i in range(S):
            for j in range(n):
                want[j - i + rel_max - 1] += d[:, :, i, j].sum(0)
        close(drel, want, 2e-2, "relbias grad")


@pytest.mark.parametrize("C,dh,rel", [(3, 16, True), (8, 64, True), (8, 512, True), (64, 64, False)])
def test_temporal_attention_backward(C, dh, rel):
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(C + dh)
    B, N, H = 2, 5, 2
    E = H * dh
    qkv = torch.randn(B * C * N, 3 * E, device="cuda", generator=g).to(BF)
    dout = torch.randn(B * C * N, E, device="cuda", generator=g).to(BF)
    table = (0.3 * torch.randn(1023, H, device="cuda", generator=g)) if rel else None
    scale = 1 / math.sqrt(dh)
    q = qkv.float().requires_grad_(True)
    tb = table.clone().requires_grad_(True) if rel else None
    x = q.view(B, C, N, 3, H, dh).permute(3, 0, 2, 4, 1, 5)  # [3, B, N, H, C, dh]
    s = (x[0] @ x[1].transpose(-1, -2)) * scale
    if rel:
        pos = torch.arange(C, device="cuda")
        s = s + tb[pos[None, :] - pos[:, None] + 511].permute(2, 0, 1)
    o = torch.softmax(s, -1) @ x[2]                          # [B, N, H, C, dh]
    o = o.permute(0, 3, 1, 2, 4).reshape(B * C * N, E)
    out = torch.empty(B * C * N, E, device="cuda", dtype=BF)
    ops.temporal_attention(qkv, out, B=B, C_=C, N=N, H=H, dh=dh, scale=scale, rel_bias=table.view(-1) if rel else None)
    close(out, o, 2e-2, "temporal fwd")
    o.backward(dout.float())
    dqkv = torch.empty_like(qkv)
    drel = torch.zeros(1023 * H, device="cuda") if rel else None
    T.temporal_attention_bwd(qkv, dout, dqkv, B=B, C_=C, N=N, H=H, dh=dh, scale=scale, rel_bias=table.view(-1) if rel else None,
                             drel=drel)
    close(dqkv, q.grad, 2e-2, "temporal dqkv")
    if rel:
        close(drel.view(1023, H), tb.grad, 2e-2, "temporal drel")


@pytest.mark.parametrize("dh,norm", [(32, True), (64, False), (128, True)])
def test_rope_backward(dh, norm):
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(dh)
    rows, nq, nk, nv, Lx = 24, 4, 2, 2, 12
    ld = (nq + nk + nv) * dh
    x = torch.randn(rows, ld, device="cuda", generator=g).to(BF)
    dy = torch.randn(rows, ld, device="cuda", generator=g).to(BF)
    inv = 1.0 / (10000 ** (torch.arange(0, dh, 2, device="cuda").float() / dh))
    wq = (1 + 0.1 * torch.randn(dh, device="cuda", generator=g)) if norm else None
    wk = (1 + 0.1 * torch.randn(dh, device="cuda", generator=g)) if norm else None
    xr = x.float().requires_grad_(True)
    wqr = wq.clone().requires_grad_(True) if norm else None
    wkr = wk.clone().requires_grad_(True) if norm else None
    h = xr.view(rows, nq + nk + nv, dh)
    pos = (torch.arange(rows, device="cuda") % Lx).float()
    fr = torch.outer(pos, inv)
    cos, sin = torch.cat((fr, fr), -1).cos()[:, None], torch.cat((fr, fr), -1).sin()[:, None]

    def rot(t, w):
        if w is not None:
            t = w * (t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6))
        return t * cos + O._rotate_half(t) * sin
    y = torch.cat((rot(h[:, :nq], wqr), rot(h[:, nq:nq + nk], wkr), h[:, nq + nk:]), 1).reshape(rows, ld)
    y.backward(dy.float())
    fwd = x.clone()
    ops.rope(fwd, rows=rows, ld=ld, dh=dh, n_q=nq, n_k=nk, n_v=0, inv_freq=inv, q_norm_w=wq, k_norm_w=wk, eps=1e-6, pos_div=1,
             pos_mod=Lx)
    close(fwd, y, 2e-2, "rope fwd")
    dx = dy.clone()
    dwq = torch.zeros(dh, device="cuda") if norm else None
    dwk = torch.zeros(dh, device="cuda") if norm else None
    T.rope_bwd(dx, x, rows=rows, ld=ld, dh=dh, n_q=nq, n_k=nk, inv_freq=inv, q_norm_w=wq, k_norm_w=wk, eps=1e-6, pos_div=1,
               pos_mod=Lx, dq_norm_w=dwq, dk_norm_w=dwk)
    close(dx, xr.grad, 2e-2, "rope dx")
    if norm:
        close(dwq, wqr.grad, 2e-2, "rope dq_norm")
        close(dwk, wkr.grad, 2e-2, "rope dk_norm")


def test_pool_backward():
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(5)
    Fr, grid, ps, E = 3, (4, 4, 4), 2, 96
    S = 64 + 1
    Sp = 72
    dy = torch.randn(Fr, 8, E, device="cuda", generator=g).to(BF)
    x = torch.randn(Fr, Sp, E, device="cuda", generator=g).to(BF)
    xr = x.float().requires_grad_(True)
    t = xr[:, 1:65].view(Fr, 4, 4, 4, E).permute(0, 4, 1, 2, 3)
    F.avg_pool3d(t, 2, 2).permute(0, 2, 3, 4, 1).reshape(Fr, 8, E).backward(dy.float())
    dx = torch.full((Fr * Sp, E), 7.0, device="cuda", dtype=BF)
    T.spp_pool_bwd(dy, dx, frames=Fr, grid=grid, ps=ps, E=E, in_frame_stride=Sp, in_off=1, ldx=E, rows_per_frame=Sp)
    close(dx.view(Fr, Sp, E), xr.grad, 1e-2, "spp_pool bwd")
    # multi-scale pooling, dynamic gate
    for dyn in (True, False):
        for K in (8, 10):
            B = 2
            xs = torch.randn(B, K, E, device="cuda", generator=g).to(BF)
            gw = 0.2 * torch.randn(E, device="cuda", generator=g)
            n_out = K + K // 2 + K // 4
            dyy = torch.randn(B, n_out, E, device="cuda", generator=g).to(BF)
            sd = {"g.gate_fc.weight": gw.view(1, E).clone().requires_grad_(True), "g.gate_fc.bias": torch.zeros(1, device="cuda")}
            xr = xs.float().requires_grad_(True)
            ref = O.multi_scale_pool(sd, "g.", xr, dyn)
            y, logits = T.multiscale_pool_fwd(xs, gw if dyn else None, dyn)
            close(y, ref, 2e-2, "msp fwd")
            ref.backward(dyy.float())
            dgw = torch.zeros(E, device="cuda")
            dx = T.multiscale_pool_bwd(xs, dyy, gw if dyn else None, logits, dgw if dyn else None, dyn)
            close(dx, xr.grad, 2e-2, f"msp dx dyn={dyn} K={K}")
            if dyn and K == 10:  # with K % 4 == 0 the three gates see the same mean and the gate gradient is exactly 0
                close(dgw, sd["g.gate_fc.weight"].grad.view(-1), 5e-2, "msp dgate_w")


def test_scatter_groupsum_colsum_transpose():
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(6)
    B, L, E, V, nv = 2, 9, 64, 50, 4
    ids = torch.randint(0, V, (B, L), device="cuda", generator=g)
    ids[0, 3] = ids[1, 5] = ids[0, 7]  # repeated rows: the adds must accumulate
    dr = torch.randn(B, L, E, device="cuda", generator=g).to(BF)
    dt = torch.zeros(V, E, device="cuda", dtype=BF)
    dvis = torch.empty(B * nv, E, device="cuda", dtype=BF)
    T.embed_scatter_add(ids, dr, dt, dvis, nv)
    want = torch.zeros(V, E, device="cuda")
    for b in range(B):
        for l in range(L):
            if not (1 <= l <= nv):
                want[ids[b, l]] += dr[b, l].float()
    close(dt, want, 2e-2, "embed scatter")
    close(dvis.view(B, nv, E), dr[:, 1:1 + nv], 1e-6, "splice grad")
    x = torch.randn(12, 6, 16, device="cuda", generator=g).to(BF)  # rows, hq = 6 (hkv 2 x G 3), dh 16
    out = torch.zeros(12, 2 * 16, device="cuda", dtype=BF)
    T.group_sum(x, out, rows=12, heads=2, G=3, dh=16, ld_in=96, ld_out=32)
    close(out.view(12, 2, 16), x.float().view(12, 2, 3, 16).sum(2), 1e-2, "group_sum")
    m = torch.randn(1000, 136, device="cuda", generator=g).to(BF)
    acc = torch.ones(136, device="cuda")
    T.colsum(m, acc)
    close(acc, 1 + m.float().sum(0), 1e-2, "colsum")
    close(T.transpose(m), m.t(), 1e-6, "transpose")


def test_ce_and_dpo_heads():
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(7)
    R, V = 12, 1000
    logits = 3 * torch.randn(R, V, device="cuda", generator=g)
    labels = torch.randint(0, V, (R,), device="cuda", generator=g)
    coef = torch.rand(R, device="cuda", generator=g)
    coef[3] = 0
    lr = logits.clone().requires_grad_(True)
    lp = torch.log_softmax(lr, -1).gather(1, labels[:, None]).squeeze(1)
    (-(coef * lp).sum()).backward()
    dl = T.ce_bwd(logits, torch.logsumexp(logits, -1), labels, coef)
    close(dl, lr.grad, 2e-2, "ce bwd")
    P, L = 3, 10
    pt = -torch.rand(2 * P, L, device="cuda", generator=g)
    ref = -3 * torch.rand(2 * P, device="cuda", generator=g)
    mask = (torch.rand(2 * P, L, device="cuda", generator=g) > 0.3)
    ptr = pt.clone().requires_grad_(True)
    s = (ptr * mask).sum(-1)
    x = 0.1 * ((s[:P] - s[P:]) - (ref[:P] - ref[P:]))
    loss = -F.logsigmoid(x).mean()
    loss.backward()
    st, cf = T.dpo_loss(pt, ref, mask.to(torch.uint8), 0.1)
    assert abs(float(st[0]) - float(loss)) < 1e-5
    close(-cf, ptr.grad, 1e-4, "dpo coef")


def test_adamw_matches_torch():
    ops, T = _ops()
    g = torch.Generator(device="cuda").manual_seed(8)
    n = 4096
    p0 = torch.randn(n, device="cuda", generator=g)
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    master, m, v = p0.clone(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pout = torch.empty(n, device="cuda", dtype=BF)
    scale = torch.full((1,), 0.5, device="cuda")
    for step in range(1, 4):
        gr = torch.randn(n, device="cuda", generator=g).to(BF)
        ref.grad = gr.float() * 0.5
        opt.step()
        T.adamw(master, m, v, gr, pout, lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1, step=step, grad_scale=scale)
        assert float((master - ref.data).abs().max()) < 1e-5
        close(pout, ref.data, 1e-2, "adamw bf16 out")
    acc = torch.zeros(1, device="cuda")
    T.sumsq(gr, acc)
    assert abs(float(acc) - float(gr.float().pow(2).sum())) / float(acc) < 1e-4


# ------------------------------------------------------------------------------------------------
# whole model: forward + backward against the oracle's autograd
# ------------------------------------------------------------------------------------------------
def _oracle_loss_and_grads(sd16, g, images, ids, qids, labels):
    sd = {k: v.float().cuda().requires_grad_(True) for k, v in sd16.items()}
    logits = O.forward_logits(sd, ids.cuda(), images.cuda(), qids.cuda(), g)
    loss = O.causal_lm_loss(logits, labels.cuda())
    loss.backward()
    return float(loss), {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in sd.items()}


def _labels(ids, n_vis):
    lab = ids.clone()
    lab[:, :n_vis + 1] = -100
    return lab


CASES = {
    "qwen3_rma_diffts_dmtp": dict(),
    "rope": dict(attn_type="rope"),
    "hard_selection_plain_pool": dict(enable_diffts=False, enable_dmtp=False, u2t_top_k=8),
    "llama_tied": dict(qk_norm=False, tie_word_embeddings=True, head_dim=32, rope_theta=500000.0),
    "sequence_pool_no_multiscale": dict(proj_pooling_type="sequence", use_multi_scale=False),
    # ViT head_dim 64: fused wgmma attention forward + probabilities recomputed in the backward (the production ViT-B path)
    "vit_head_dim_64_flash_recompute": dict(vit_hidden=128, vit_heads=2, vit_mlp=256),
}


@pytest.mark.parametrize("case", list(CASES))
def test_forward_backward_matches_oracle_autograd(case):
    from u2tokenizer_b200.train import TrainEngine
    g = tiny_geometry(**CASES[case])
    sd16 = synthetic_state_dict(g, seed=21, device="cpu", dtype=BF)
    # N(0, 0.02) query tokens make every TTA attention uniform (scores ~ 0) and its gradients pure cancellation noise:
    # give them O(1) entries so that the TTA / linear-aggregation backward is actually exercised
    sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
    images, ids, qids = synthetic_inputs(g, batch=2, frames=3, n_question=7, lt=12)
    labels = _labels(ids, g.num_3d_query_token)
    ref_loss, ref_g = _oracle_loss_and_grads(sd16, g, images, ids, qids, labels)
    te = TrainEngine(g, sd16, device="cuda")
    te.zero_grad()
    loss = te.forward_backward(images.cuda(), ids.cuda(), qids.cuda(), labels.cuda())
    torch.cuda.synchronize()
    assert abs(float(loss) - ref_loss) < 2e-2 * max(1.0, abs(ref_loss)), (float(loss), ref_loss)
    L = te.lay
    bad, worst = [], (0.0, "")
    skip_zero = n_noise = 0
    # gradients that are mathematically (near) zero - k-projection biases under the softmax shift invariance, gates that
    # see identical inputs, score nets behind a nearly uniform softmax - are cancellation noise in ANY bf16 pipeline: a
    # tensor also passes when its absolute error is below 2e-3 of the largest gradient entry of the whole model
    gmax = max(v.abs().max().item() for v in ref_g.values())
    for n in L.mat_names + L.vec_names:
        got = te.grad(n).float().cpu()
        if n == "lm_head.weight" and te.tied:
            continue
        want = ref_g[n].cpu()
        if n == "model.embed_tokens.weight" and te.tied and "lm_head.weight" in ref_g:
            pass  # the oracle ties through the same tensor: its gradient already holds both uses
        scale = want.abs().max().item()
        if scale < 1e-9:
            skip_zero += 1
            assert got.abs().max().item() < 1e-4, f"{n}: oracle gradient is zero, got {got.abs().max().item()}"
            continue
        e, c = rel_err(got, want), cosine(got, want)
        if e < 4e-2 and c > 0.995:
            if e > worst[0]:
                worst = (e, n)
            continue
        if (got - want).abs().max().item() < 2e-3 * gmax:
            n_noise += 1
            continue
        bad.append((n, round(e, 4), round(c, 5), got.abs().max().item(), scale))
    print(f"[{case}] loss {float(loss):.5f} (oracle {ref_loss:.5f}); {len(L.mat_names + L.vec_names)} parameters: worst rel_err "
          f"among the directly compared {worst[0]:.4g} at {worst[1]}; {n_noise} below the noise floor (|err| < 2e-3 * {gmax:.3g}), "
          f"{skip_zero} identically zero")
    for b_ in bad:
        print("   BAD", b_)
    assert not bad, bad[:6]


def test_frozen_vision_tower_and_module_backward():
    """model(**batch).loss.backward() through the HF-style surface (reference train_stage1.py:244-250) with
    freeze_vision_tower: p.grad of the trainable parameters equals the oracle's, the tower gets none."""
    from u2tokenizer_b200.configuration import U2Qwen3Config
    from u2tokenizer_b200.geometry import Geometry
    from u2tokenizer_b200.modeling import U2Qwen3ForCausalLM
    cfg = U2Qwen3Config(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                        head_dim=32, vocab_size=512, image_size=[16, 64, 64], vit_hidden_size=96, vit_mlp_dim=192,
                        vit_num_layers=2, vit_num_heads=4, u2t_num_layers=2, u2t_top_k=8, num_3d_query_token=8,
                        tie_word_embeddings=False, rope_theta=1e6)
    g = Geometry.from_hf(cfg)
    sd16 = synthetic_state_dict(g, seed=5, device="cpu", dtype=BF)
    sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(BF)
    try:
        with torch.device("cuda"):
            model = U2Qwen3ForCausalLM(cfg)
    finally:
        torch.set_default_dtype(prev)
    model.load_state_dict(sd16, strict=False)
    model.get_model().vision_tower.requires_grad_(False)
    model.train()
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=6, lt=10)
    labels = _labels(ids, g.num_3d_query_token)
    ref_loss, ref_g = _oracle_loss_and_grads(sd16, g, images, ids, qids, labels)
    out = model(images=images.cuda(), input_ids=ids.cuda(), labels=labels.cuda(), question_ids=qids.cuda(),
                attention_mask=torch.ones_like(ids).cuda())
    out.loss.backward()
    assert abs(float(out.loss) - ref_loss) < 2e-2 * max(1.0, abs(ref_loss))
    bad = []
    gmax = max(v.abs().max().item() for v in ref_g.values())
    for n, p in model.named_parameters():
        if n.startswith("model.vision_tower."):
            assert p.grad is None
            continue
        want = ref_g[n].cpu()
        if want.abs().max().item() < 1e-9:
            continue
        assert p.grad is not None, n
        got = p.grad.float().cpu()
        e, c = rel_err(got, want), cosine(got, want)
        if not (e < 5e-2 and c > 0.99) and (got - want).abs().max().item() >= 2e-3 * gmax:
            bad.append((n, round(e, 4), round(c, 5)))
    for b_ in bad:
        print("   BAD", b_)
    assert not bad, bad[:6]
    # an optimizer step through torch (in place on the flat buffer) is seen by the next forward
    before = float(out.loss)
    torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=0.05).step()
    after = float(model(images=images.cuda(), input_ids=ids.cuda(), labels=labels.cuda(), question_ids=qids.cuda()).loss)
    assert after < before, (before, after)


def test_gradient_slots_overwrite_accumulate_and_stale_clear():
    """The matrix-gradient buffer is never memset: the first wgrad after zero_grad() overwrites its slot, a second
    backward() before the next zero_grad() adds (micro-batch accumulation), and a slot that holds an earlier step's
    gradient but is not written in the current step (its group was frozen in between) reads as zero."""
    from u2tokenizer_b200.train import TrainEngine
    g = tiny_geometry()
    sd16 = synthetic_state_dict(g, seed=8, device="cpu", dtype=BF)
    sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
    ia, ida, qa = synthetic_inputs(g, batch=2, frames=2, n_question=6, lt=10, seed=1)
    ib, idb, qb = synthetic_inputs(g, batch=2, frames=2, n_question=6, lt=10, seed=2)
    la, lb = _labels(ida, g.num_3d_query_token), _labels(idb, g.num_3d_query_token)

    def run(te, im, ids, q, lab):
        return te.forward_backward(im.cuda(), ids.cuda(), q.cuda(), lab.cuda())

    fresh = TrainEngine(g, sd16, device="cuda")
    fresh.zero_grad()
    run(fresh, ib, idb, qb, lb)
    te = TrainEngine(g, sd16, device="cuda")
    te.zero_grad()
    run(te, ia, ida, qa, la)
    ga = te.Gm.clone()
    te.zero_grad()
    run(te, ib, idb, qb, lb)          # step 2 on another batch: no trace of step 1 (atomics reorder the last bits only)
    gmax = fresh.Gm.float().abs().max().item()
    assert (te.Gm.float() - fresh.Gm.float()).abs().max().item() <= 4e-3 * gmax
    close(te.Gv, fresh.Gv, 1e-3, "vector gradients of step 2")
    assert (ga.float() - fresh.Gm.float()).abs().max().item() > 0.05 * gmax   # the two batches do differ
    # accumulation: A then B without zero_grad in between
    te.zero_grad()
    run(te, ia, ida, qa, la)
    gva = te.Gv.clone()
    run(te, ib, idb, qb, lb)
    want = ga.float() + fresh.Gm.float()
    err = (te.Gm.float() - want).abs().max().item()
    assert err <= 2e-2 * want.abs().max().item() + 1e-6, err
    close(te.Gv, gva + fresh.Gv, 1e-3, "accumulated vector gradients")
    # a group that stops training: its slots are cleared when the step does not write them
    vit_w = "model.vision_tower.vision_tower.blocks.0.mlp.linear1.weight"
    assert te.grad(vit_w).abs().max().item() > 0
    te.trainable["vit"] = False
    te.zero_grad()
    run(te, ib, idb, qb, lb)
    assert te.grad(vit_w).abs().max().item() == 0
    dec_w = "model.layers.0.mlp.down_proj.weight"
    assert (te.grad(dec_w).float() - fresh.grad(dec_w).float()).abs().max().item() <= 4e-3 * gmax


def test_module_backward_accumulates_over_micro_batches():
    """HF Trainer with gradient_accumulation_steps = 2: loss.backward() twice before optimizer.step(). autograd keeps the
    returned gradient views as p.grad, so the second backward adds into the same slots in place."""
    from u2tokenizer_b200.configuration import U2Qwen3Config
    from u2tokenizer_b200.geometry import Geometry
    from u2tokenizer_b200.modeling import U2Qwen3ForCausalLM
    cfg = U2Qwen3Config(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                        head_dim=32, vocab_size=512, image_size=[16, 64, 64], vit_hidden_size=96, vit_mlp_dim=192,
                        vit_num_layers=2, vit_num_heads=4, u2t_num_layers=2, u2t_top_k=8, num_3d_query_token=8,
                        tie_word_embeddings=False, rope_theta=1e6)
    g = Geometry.from_hf(cfg)
    sd16 = synthetic_state_dict(g, seed=5, device="cpu", dtype=BF)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(BF)
    try:
        with torch.device("cuda"):
            model = U2Qwen3ForCausalLM(cfg)
    finally:
        torch.set_default_dtype(prev)
    model.load_state_dict(sd16, strict=False)
    model.train()
    batches = []
    for seed in (1, 2):
        im, ids, q = synthetic_inputs(g, batch=2, frames=2, n_question=6, lt=10, seed=seed)
        batches.append(dict(images=im.cuda(), input_ids=ids.cuda(), labels=_labels(ids, g.num_3d_query_token).cuda(),
                            question_ids=q.cuda()))
    single = []
    for b in batches:
        model.zero_grad(set_to_none=True)
        model(**b).loss.backward()
        single.append({n: p.grad.float().clone() for n, p in model.named_parameters() if p.grad is not None})
    model.zero_grad(set_to_none=True)
    for b in batches:
        model(**b).loss.backward()
    n_checked = 0
    gmax = max((single[0][n] + single[1][n]).abs().max().item() for n in single[0])
    for n, p in model.named_parameters():
        if n not in single[0]:
            continue
        want = single[0][n] + single[1][n]
        scale = want.abs().max().item()
        if scale < 1e-9:
            continue
        err = (p.grad.float() - want).abs().max().item()
        # cancellation-noise gradients (score net behind a nearly uniform softmax, ~1e-6 here) are not reproducible to
        # their own scale from run to run (fp32 atomics upstream): same criterion as the oracle comparison above
        assert err <= 2e-2 * scale + 1e-6 or err < 2e-3 * gmax, (n, err, scale, gmax)
        n_checked += 1
    assert n_checked > 50


def test_train_step_zero1_single_gpu_matches_torch_adamw():
    """TrainEngine.optimizer_step (world size 1: buckets, clipping, fused AdamW) against torch.optim.AdamW driven with the
    engine's own gradients; three steps, loss decreases."""
    from u2tokenizer_b200.train import TrainEngine
    g = tiny_geometry()
    sd16 = synthetic_state_dict(g, seed=9, device="cpu", dtype=BF)
    te = TrainEngine(g, sd16, device="cuda", bucket_elems=50_000)   # several buckets
    assert te.lay.n_buckets > 2
    te.init_optimizer(lr=1e-3, weight_decay=0.01, max_grad_norm=1.0)
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=6, lt=10)
    labels = _labels(ids, g.num_3d_query_token)
    L = te.lay
    ref_m = torch.nn.Parameter(te.W[:L.mat_total].float().clone())
    ref_v = torch.nn.Parameter(te.W[L.mat_total:].float().clone())
    opt = torch.optim.AdamW([ref_m, ref_v], lr=1e-3, weight_decay=0.01)
    losses = []
    for it in range(3):
        te.zero_grad()
        losses.append(float(te.forward_backward(images.cuda(), ids.cuda(), qids.cuda(), labels.cuda())))
        ref_m.grad, ref_v.grad = te.Gm.float().clone(), te.Gv.clone()
        torch.nn.utils.clip_grad_norm_([ref_m, ref_v], 1.0)
        opt.step()
        te.optimizer_step()
        assert float((te.opt["m_master"] - ref_m.data).abs().max()) < 2e-5, it
        assert float((te.opt["v_master"] - ref_v.data).abs().max()) < 2e-5, it
        close(te.W[:L.mat_total], ref_m.data, 1e-2, "bf16 params after the step")
    assert losses[2] < losses[0], losses


def test_dpo_step_matches_oracle_autograd():
    """Policy side of the stage-2 DPO step (reference dpo_u2trainer.py:185-359 + trl's sigmoid loss, beta 0.1): loss,
    reward statistics and every parameter gradient against autograd through the oracle's forward, selective log-softmax
    and -logsigmoid(beta * ((pc - pr) - (rc - rr)))."""
    from u2tokenizer_b200.train import TrainEngine
    g = tiny_geometry()
    sd16 = synthetic_state_dict(g, seed=31, device="cpu", dtype=BF)
    sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
    images, ids, qids = synthetic_inputs(g, batch=1, frames=2, n_question=6, lt=10)
    gen = torch.Generator().manual_seed(3)
    n_prompt = ids.shape[1]
    ans = torch.randint(1, g.vocab_size - 16, (2, 9), generator=gen)          # chosen / rejected completions
    ids2 = torch.cat([ids.expand(2, -1), ans], 1)
    images2, qids2 = images.expand(2, *images.shape[1:]).contiguous(), qids.expand(2, -1).contiguous()
    mask = torch.zeros_like(ids2)
    mask[:, n_prompt:] = 1
    mask[1, -2:] = 0                                                           # a shorter rejected completion
    ref_logps = torch.tensor([-30.0, -28.5])
    beta = 0.1
    sd = {k: v.float().cuda().requires_grad_(True) for k, v in sd16.items()}
    logits = O.forward_logits(sd, ids2.cuda(), images2.cuda(), qids2.cuda(), g)
    ptl, allp, _ = O.dpo_per_token_logps(logits, ids2.cuda(), mask.cuda())
    x = beta * ((allp[0] - allp[1]) - (ref_logps[0] - ref_logps[1]).cuda())
    loss = -F.logsigmoid(x)
    loss.backward()
    te = TrainEngine(g, sd16, device="cuda")
    te.zero_grad()
    st = te.dpo_forward_backward(images2.cuda(), ids2.cuda(), qids2.cuda(), mask.cuda(), ref_logps.cuda(), beta)
    torch.cuda.synchronize()
    assert abs(float(st[0]) - float(loss)) < 2e-2 * max(1.0, float(loss)), (st, float(loss))
    seq = te.sequence_logps(images2.cuda(), ids2.cuda(), qids2.cuda(), mask.cuda())
    close(seq, allp.detach(), 2e-2, "summed sequence log-probabilities")
    L = te.lay
    gmax = max(v.grad.abs().max().item() for v in sd.values() if v.grad is not None)
    bad = []
    for n in L.mat_names + L.vec_names:
        want = sd[n].grad
        if want is None or want.abs().max().item() < 1e-9:
            continue
        got = te.grad(n).float().cpu()
        want = want.cpu()
        e, c = rel_err(got, want), cosine(got, want)
        if not (e < 4e-2 and c > 0.995) and (got - want).abs().max().item() >= 2e-3 * gmax:
            bad.append((n, round(e, 4), round(c, 5)))
    assert not bad, bad[:6]
