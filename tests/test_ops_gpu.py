"""Each CUDA op (C ABI) against the same arithmetic in fp32 torch on identical bf16 inputs."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def close(out, ref, tol=1e-2):
    err = (out.float() - ref.float()).abs().max().item()
    scale = ref.float().abs().max().item() + 1e-6
    assert err / scale < tol, f"max abs err {err:.4g} vs scale {scale:.4g}"


@pytest.mark.parametrize("E", [96, 768, 2048, 4096])
@pytest.mark.parametrize("with_res", [False, True])
def test_layernorm_rmsnorm(E, with_res):
    from u2tokenizer_b200 import ops
    g = gen(E)
    x = torch.randn(37, E, device=DEV, generator=g).bfloat16()
    r = torch.randn(37, E, device=DEV, generator=g).bfloat16() if with_res else None
    gamma = 1 + 0.1 * torch.randn(E, device=DEV, generator=g)
    beta = 0.1 * torch.randn(E, device=DEV, generator=g)
    xs = x.float() + (r.float() if with_res else 0)
    y = ops.layernorm(x, gamma, beta, 1e-5, residual=r)
    close(y, F.layer_norm(xs, (E,), gamma, beta, 1e-5))
    so = torch.empty_like(x) if with_res else None
    y = ops.rmsnorm(x, gamma, 1e-6, residual=r, sum_out=so)
    if with_res:
        close(so, xs, 5e-3)
        xs = so.float()
    close(y, gamma * xs * torch.rsqrt(xs.pow(2).mean(-1, keepdim=True) + 1e-6))


@pytest.mark.parametrize("S,n", [(7, 7), (256, 256), (40, 1792), (33, 2049), (64, 300), (5, 8200), (3, 16384)])
@pytest.mark.parametrize("mode", ["plain", "rel", "causal"])
def test_softmax(S, n, mode):
    from u2tokenizer_b200 import ops
    if mode == "rel" and (S != n or n > 512):
        pytest.skip("relative bias needs square S<=512")
    if mode == "causal" and S > n:
        pytest.skip()
    B, H = 2, 3
    g = gen(S * 31 + n)
    ld = (n + 7) // 8 * 8
    sc = torch.randn(B, H, S, ld, device=DEV, generator=g) * 3
    out = torch.full((B, H, S, ld), 7.0, device=DEV, dtype=torch.bfloat16)
    rel = torch.randn(1023, H, device=DEV, generator=g) if mode == "rel" else None
    off = n - S
    ops.softmax(sc, out, n0=B, H=H, S=S, n=n, in_strides=(H * S * ld, S * ld, ld), out_strides=(H * S * ld, S * ld, ld),
                scale=0.5, rel_bias=rel, rel_max=512, causal=(mode == "causal"), causal_off=off, zero_pad_to=ld)
    ref = sc[..., :n] * 0.5
    if rel is not None:
        pos = torch.arange(n, device=DEV)
        ref = ref + rel[pos[None, :] - pos[:, None] + 511].permute(2, 0, 1)[None]
    if mode == "causal":
        i = torch.arange(S, device=DEV)[:, None]
        j = torch.arange(n, device=DEV)[None, :]
        ref = ref.masked_fill(j > i + off, float("-inf"))
    close(out[..., :n], torch.softmax(ref, -1), 1e-2)
    assert out[..., n:].abs().max().item() == 0 if ld > n else True


def test_silu_mul():
    from u2tokenizer_b200 import ops
    gu = torch.randn(50, 2 * 768, device=DEV, generator=gen(1)).bfloat16()
    close(ops.silu_mul(gu), F.silu(gu[:, :768].float()) * gu[:, 768:].float())
    close(ops.silu_mul(gu, interleaved=True), F.silu(gu[:, 0::2].float()) * gu[:, 1::2].float())


def test_patchify():
    from u2tokenizer_b200 import ops
    vol = torch.rand(3, 8, 32, 48, device=DEV, generator=gen(2))
    p = (4, 16, 16)
    out = ops.patchify(vol, p)
    x = vol.view(3, 1, 2, 4, 2, 16, 3, 16).permute(0, 2, 4, 6, 3, 5, 7, 1).reshape(3 * 12, 1024)
    assert torch.equal(out, x.bfloat16())


def test_set_rows_transpose():
    from u2tokenizer_b200 import ops
    g = gen(3)
    x = torch.zeros(4, 10, 64, device=DEV, dtype=torch.bfloat16)
    v = torch.randn(64, device=DEV, generator=g).bfloat16()
    ops.set_rows(x, v, 4, 10, 0)
    assert torch.equal(x[:, 0], v.expand(4, 64)) and x[:, 1:].abs().max().item() == 0
    B, S, H, Dh = 2, 45, 3, 40
    t = torch.randn(B, S, 3 * H * Dh, device=DEV, generator=g).bfloat16()  # fused qkv; take the V part
    ld = 48
    out = torch.full((B, H, Dh, ld), 5.0, device=DEV, dtype=torch.bfloat16)
    ops.transpose_heads(t[:, :, 2 * H * Dh:], out, B=B, S=S, H=H, Dh=Dh, in_strides=(S * 3 * H * Dh, 3 * H * Dh, Dh),
                        out_strides=(H * Dh * ld, Dh * ld), ld_out=ld)
    ref = t[:, :, 2 * H * Dh:].view(B, S, H, Dh).permute(0, 2, 3, 1)
    assert torch.equal(out[..., :S], ref) and out[..., S:].abs().max().item() == 0


@pytest.mark.parametrize("sequence", [False, True])
def test_spp_pool(sequence):
    from u2tokenizer_b200 import ops
    Fr, g0, g1, g2, E, S_pad = 3, 4, 6, 8, 96, 200
    x = torch.randn(Fr, S_pad, E, device=DEV, generator=gen(4)).bfloat16()
    n_out = (g0 // 2) * (g1 // 2) * (g2 // 2)
    out = torch.empty(Fr, n_out, E, device=DEV, dtype=torch.bfloat16)
    ops.spp_pool(x, out, frames=Fr, grid=(g0, g1, g2), ps=2, E=E, in_frame_stride=S_pad, in_off=1, ldx=E, sequence=sequence)
    tok = x[:, 1:1 + g0 * g1 * g2].float()
    if sequence:
        ref = F.avg_pool1d(tok.permute(0, 2, 1), 8, 8).permute(0, 2, 1)
    else:
        ref = F.avg_pool3d(tok.view(Fr, g0, g1, g2, E).permute(0, 4, 1, 2, 3), 2, 2).permute(0, 2, 3, 4, 1).reshape(Fr, -1, E)
    close(out, ref, 5e-3)


@pytest.mark.parametrize("K", [1024, 8, 7, 3, 1])
@pytest.mark.parametrize("dynamic", [True, False])
def test_multiscale_pool(K, dynamic):
    from u2tokenizer_b200 import ops
    B, E = 2, 256
    g = gen(K)
    x = torch.randn(B, K, E, device=DEV, generator=g).bfloat16()
    w = torch.randn(E, device=DEV, generator=g) * 0.3
    bias = 0.1
    out = ops.multiscale_pool(x, w, bias, dynamic)
    xf = x.float()
    pooled, gates = [], []
    for s in (1, 2, 4):
        if K >= s:
            p = F.avg_pool1d(xf.permute(0, 2, 1), s, s).permute(0, 2, 1)
            pooled.append(p)
            gates.append(p.mean(1) @ w[:, None] + bias)
    if dynamic:
        wts = torch.softmax(torch.cat(gates, 1), 1)
        ref = torch.cat([p * wts[:, i].view(-1, 1, 1) for i, p in enumerate(pooled)], 1)
    else:
        ref = torch.cat(pooled, 1)
    assert out.shape == ref.shape
    close(out, ref, 1e-2)


def test_embed_splice():
    from u2tokenizer_b200 import ops
    g = gen(6)
    table = torch.randn(100, 64, device=DEV, generator=g).bfloat16()
    ids = torch.randint(0, 100, (2, 12), device=DEV, generator=g)
    vis = torch.randn(2, 5, 64, device=DEV, generator=g).bfloat16()
    out = ops.embed_splice(ids, table, vis)
    emb = table[ids]
    ref = torch.cat((emb[:, :1], vis, emb[:, 6:]), 1)
    assert torch.equal(out, ref)
    assert torch.equal(ops.embed_splice(ids, table, None), emb)


@pytest.mark.parametrize("C_,dh", [(8, 512), (3, 32), (1, 64), (16, 256), (32, 64), (33, 64), (64, 64), (100, 32)])
@pytest.mark.parametrize("rel", [True, False])
def test_temporal_attention(C_, dh, rel):
    from u2tokenizer_b200 import ops
    B, N, H = 2, 5, 4
    E = H * dh
    g = gen(C_ * dh)
    qkv = torch.randn(B * C_ * N, 3 * E, device=DEV, generator=g).bfloat16()
    bias = torch.randn(1023, H, device=DEV, generator=g) if rel else None
    out = torch.empty(B * C_ * N, E, device=DEV, dtype=torch.bfloat16)
    ops.temporal_attention(qkv, out, B=B, C_=C_, N=N, H=H, dh=dh, scale=1 / math.sqrt(dh), rel_bias=bias)
    t = qkv.float().view(B, C_, N, 3, H, dh)
    q, k, v = (t[:, :, :, i].permute(0, 2, 3, 1, 4) for i in range(3))  # [B, N, H, C, dh]
    sc = q @ k.transpose(-1, -2) / math.sqrt(dh)
    if rel:
        pos = torch.arange(C_, device=DEV)
        sc = sc + bias[pos[None, :] - pos[:, None] + 511].permute(2, 0, 1)[None, None]
    ref = (torch.softmax(sc, -1) @ v).permute(0, 3, 1, 2, 4).reshape(B * C_ * N, E)
    close(out, ref, 1e-2)


@pytest.mark.parametrize("dh", [32, 64, 128])
@pytest.mark.parametrize("qk_norm", [True, False])
def test_rope_and_cache(dh, qk_norm):
    from u2tokenizer_b200 import ops
    B, S, Hq, Hkv, Tmax, pos0 = 2, 9, 4, 2, 32, 5
    g = gen(dh)
    ld = (Hq + 2 * Hkv) * dh
    x = torch.randn(B * S, ld, device=DEV, generator=g).bfloat16()
    x0 = x.clone()
    inv = 1.0 / (10000 ** (torch.arange(0, dh, 2, device=DEV).float() / dh))
    qw = 1 + 0.1 * torch.randn(dh, device=DEV, generator=g) if qk_norm else None
    kw = 1 + 0.1 * torch.randn(dh, device=DEV, generator=g) if qk_norm else None
    kc = torch.zeros(B, Hkv, Tmax, dh, device=DEV, dtype=torch.bfloat16)
    vc = torch.zeros_like(kc)
    ops.rope(x, rows=B * S, ld=ld, dh=dh, n_q=Hq, n_k=Hkv, n_v=Hkv, inv_freq=inv, q_norm_w=qw, k_norm_w=kw, eps=1e-6,
             pos0=pos0, pos_div=1, pos_mod=S, k_cache=kc, v_cache=vc, Tmax=Tmax, rows_per_batch=S)
    t = x0.float().view(B, S, Hq + 2 * Hkv, dh)
    q, k, v = t[:, :, :Hq], t[:, :, Hq:Hq + Hkv], t[:, :, Hq + Hkv:]
    if qk_norm:
        q = qw * q * torch.rsqrt(q.pow(2).mean(-1, keepdim=True) + 1e-6)
        k = kw * k * torch.rsqrt(k.pow(2).mean(-1, keepdim=True) + 1e-6)
    pos = torch.arange(pos0, pos0 + S, device=DEV).float()
    fr = torch.outer(pos, inv)
    emb = torch.cat((fr, fr), -1)
    cos, sin = emb.cos()[None, :, None], emb.sin()[None, :, None]
    rot = lambda u: torch.cat((-u[..., dh // 2:], u[..., :dh // 2]), -1)
    qr, kr = q * cos + rot(q) * sin, k * cos + rot(k) * sin
    got = x.float().view(B, S, Hq + 2 * Hkv, dh)
    close(got[:, :, :Hq], qr, 1e-2)
    close(got[:, :, Hq:Hq + Hkv], kr, 1e-2)
    assert torch.equal(got[:, :, Hq + Hkv:], v)
    close(kc[:, :, pos0:pos0 + S].permute(0, 2, 1, 3), kr, 1e-2)
    assert torch.equal(vc[:, :, pos0:pos0 + S].permute(0, 2, 1, 3).float(), v)
    assert kc[:, :, :pos0].abs().max().item() == 0 and kc[:, :, pos0 + S:].abs().max().item() == 0


@pytest.mark.parametrize("dh,T", [(128, 545), (64, 17), (32, 3), (128, 1)])
def test_decode_attention(dh, T):
    from u2tokenizer_b200 import ops
    B, Hq, Hkv, Tmax = 3, 8, 2, 600
    g = gen(T)
    q = torch.randn(B, Hq * dh, device=DEV, generator=g).bfloat16()
    kc = torch.randn(B, Hkv, Tmax, dh, device=DEV, generator=g).bfloat16()
    vc = torch.randn(B, Hkv, Tmax, dh, device=DEV, generator=g).bfloat16()
    out = torch.empty(B, Hq * dh, device=DEV, dtype=torch.bfloat16)
    Td = torch.tensor([T], device=DEV, dtype=torch.int32)
    for kw in (dict(T=T), dict(T_dev=Td)):
        out.zero_()
        ops.decode_attention(q, kc, vc, out, B=B, Hq=Hq, Hkv=Hkv, dh=dh, Tmax=Tmax, ldq=Hq * dh, ldo=Hq * dh,
                             scale=1 / math.sqrt(dh), **kw)
        qq = q.float().view(B, Hq, 1, dh)
        kk = kc[:, :, :T].float().repeat_interleave(Hq // Hkv, 1)
        vv = vc[:, :, :T].float().repeat_interleave(Hq // Hkv, 1)
        ref = (torch.softmax(qq @ kk.transpose(-1, -2) / math.sqrt(dh), -1) @ vv).reshape(B, Hq * dh)
        close(out, ref, 1e-2)


@pytest.mark.parametrize("B", [1, 4, 8])
@pytest.mark.parametrize("N,K", [(4096, 2048), (1000, 328), (24576, 4096), (151936, 1024)])
def test_gemv(B, N, K):
    from u2tokenizer_b200 import ops
    g = gen(B * N + K)
    x = torch.randn(B, K, device=DEV, generator=g).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) * K ** -0.5).bfloat16()
    res = torch.randn(B, N, device=DEV, generator=g).bfloat16()
    out = torch.empty(B, N, device=DEV, dtype=torch.bfloat16)
    ops.gemv(x, w, out, residual=res)
    close(out, x.float() @ w.float().t() + res.float())
    outf = torch.empty(B, N, device=DEV, dtype=torch.float32)
    gamma = 1 + 0.1 * torch.randn(K, device=DEV, generator=g)
    ops.gemv(x, w, outf, norm_gamma=gamma, norm_eps=1e-6)
    xn = (gamma * x.float() * torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + 1e-6))
    close(outf, xn @ w.float().t(), 1e-2)
    if N % 2 == 0:
        o2 = torch.empty(B, N // 2, device=DEV, dtype=torch.bfloat16)
        ops.gemv(x, w, o2, silu_pair=True)
        y = x.float() @ w.float().t()
        close(o2, F.silu(y[:, 0::2]) * y[:, 1::2], 2e-2)


def test_argmax():
    from u2tokenizer_b200 import ops
    lg = torch.randn(4, 151936, device=DEV, generator=gen(9))
    lg[1, 77] = 100.0
    lg[1, 5000] = 100.0  # tie -> first index
    assert torch.equal(ops.argmax(lg), lg.argmax(-1))
    assert ops.argmax(lg)[1].item() == 77


@pytest.mark.parametrize("sched", [0, 1])
@pytest.mark.parametrize("B", [1, 4, 16])
@pytest.mark.parametrize("N,K", [(4096, 4096), (1000, 320), (6144, 2048), (24576, 4096), (4096, 12288), (151936, 1024)])
def test_dlinear(B, N, K, sched):
    """wgmma decode linear (swap-AB + stream-K): plain, fused-norm scale, residual + next-norm prep, silu pair."""
    from u2tokenizer_b200 import ops
    g = gen(B * N + K + 1)
    x = torch.randn(B, K, device=DEV, generator=g).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) * K ** -0.5).bfloat16()
    ws = ops.dlinear_new_ws(ops.dlinear_ws_elems(N, K), device=DEV)
    cnt = torch.zeros((N + 63) // 64 + 1, device=DEV, dtype=torch.int32)  # + the ticket of the ssq_out sum
    ref = x.float() @ w.float().t()
    # (a) fp32 output, fused RMSNorm scale
    ssq = torch.zeros(16, device=DEV)
    ssq[:B] = torch.rand(B, device=DEV, generator=g) * K + 1.0
    out = torch.empty(B, N, device=DEV)
    for _ in range(2):  # twice: the workspace must come back clean
        ops.dlinear(x, w, out, ws=ws, counters=cnt, ssq_in=ssq, eps=1e-6, sched=sched)
        close(out, ref * torch.rsqrt(ssq[:B] / K + 1e-6)[:, None])
    assert cnt.abs().max().item() == 0
    # (b) residual (in place) + xg + ssq_out + ssq_zero
    res = torch.randn(B, N, device=DEV, generator=g).bfloat16()
    xres = res.clone()
    gam = 1 + 0.1 * torch.randn(N, device=DEV, generator=g)
    xg = torch.empty(B, N, device=DEV, dtype=torch.bfloat16)
    sso = torch.zeros(16, device=DEV)
    ssz = torch.ones(16, device=DEV)
    ops.dlinear(x, w, xres, ws=ws, counters=cnt, residual=xres, gamma_next=gam, xg=xg, ssq_out=sso, ssq_zero=ssz, sched=sched)
    want = (ref + res.float())
    close(xres, want)
    close(xg, xres.float() * gam, 1e-2)
    close(sso[:B], xres.float().pow(2).sum(-1), 1e-3)
    # the sums of squares are added up in a fixed order: the same launch again gives the same bits
    xres2, sso2 = res.clone(), torch.zeros(16, device=DEV)
    ops.dlinear(x, w, xres2, ws=ws, counters=cnt, residual=xres2, gamma_next=gam, xg=xg, ssq_out=sso2, ssq_zero=ssz, sched=sched)
    assert torch.equal(sso2, sso) and torch.equal(xres2, xres)
    assert cnt.abs().max().item() == 0 and bool((ws.view(torch.int32) == -1).all())
    assert ssz.abs().max().item() == 0
    # (c) silu pair on interleaved rows
    if N % 2 == 0:
        act = torch.empty(B, N // 2, device=DEV, dtype=torch.bfloat16)
        ops.dlinear(x, w, act, ws=ws, counters=cnt, silu_pair=True, sched=sched)
        close(act, F.silu(ref[:, 0::2]) * ref[:, 1::2], 2e-2)
    assert cnt.abs().max().item() == 0


def test_decode_embed():
    from u2tokenizer_b200 import ops
    g = gen(77)
    table = torch.randn(50, 256, device=DEV, generator=g).bfloat16()
    ids = torch.tensor([[3], [49], [0]], device=DEV)
    gam = 1 + 0.1 * torch.randn(256, device=DEV, generator=g)
    x = torch.empty(3, 256, device=DEV, dtype=torch.bfloat16)
    xg = torch.empty_like(x)
    ssq, ssz = torch.zeros(16, device=DEV), torch.ones(16, device=DEV)
    stepc = torch.zeros(1, device=DEV, dtype=torch.int32)
    ops.decode_embed(ids, table, gam, x, xg, ssq, ssz, stepc)
    assert stepc.item() == 1
    e = table[ids.view(-1)]
    assert torch.equal(x, e)
    close(xg, e.float() * gam, 1e-2)
    close(ssq[:3], e.float().pow(2).sum(-1), 1e-4)
    assert ssz[:3].abs().max().item() == 0


@pytest.mark.parametrize("dh,Hq,Hkv", [(128, 32, 8), (128, 16, 8), (64, 32, 8), (32, 4, 2), (64, 8, 8)])
@pytest.mark.parametrize("pos", [0, 5, 290, 543])
@pytest.mark.parametrize("qk_norm", [True, False])
@pytest.mark.parametrize("splits", [1, 4])
def test_decode_attention_fused(dh, Hq, Hkv, pos, qk_norm, splits):
    """Fused q/k-norm + RoPE + cache append + attention vs the unfused kernels' arithmetic in fp32 torch
    (splits > 1: the split-KV cluster variant, partial results merged over distributed shared memory)."""
    _check_decode_attention_fused(dh, Hq, Hkv, pos, qk_norm, splits, Tmax=600)


@pytest.mark.parametrize("splits,pos,Tmax", [(2, 1100, 1200), (8, 3, 64), (8, 2500, 2600), (2, 31, 600), (4, 1024, 1200)])
@pytest.mark.parametrize("dh,Hq,Hkv", [(128, 32, 8), (64, 8, 8), (32, 4, 2)])
def test_decode_attention_fused_split_rounds(dh, Hq, Hkv, splits, pos, Tmax):
    """More keys than one round of the cluster covers (S x 256), fewer keys than CTAs, group boundaries."""
    _check_decode_attention_fused(dh, Hq, Hkv, pos, True, splits, Tmax=Tmax)


def _check_decode_attention_fused(dh, Hq, Hkv, pos, qk_norm, splits, Tmax):
    from u2tokenizer_b200 import ops
    B = 3
    g = gen(dh * 7 + pos + Hq)
    ld = (Hq + 2 * Hkv) * dh
    qkv = torch.randn(B, ld, device=DEV, generator=g).bfloat16()
    kc = torch.randn(B, Hkv, Tmax, dh, device=DEV, generator=g).bfloat16()
    vc = torch.randn(B, Hkv, Tmax, dh, device=DEV, generator=g).bfloat16()
    kc0, vc0 = kc.clone(), vc.clone()
    inv = 1.0 / (1e6 ** (torch.arange(0, dh, 2, device=DEV).float() / dh))
    qw = 1 + 0.1 * torch.randn(dh, device=DEV, generator=g) if qk_norm else None
    kw = 1 + 0.1 * torch.randn(dh, device=DEV, generator=g) if qk_norm else None
    out = torch.empty(B, Hq * dh, device=DEV, dtype=torch.bfloat16)
    pd = torch.tensor([pos], device=DEV, dtype=torch.int32)
    ops.decode_attention_fused(qkv, kc, vc, out, B=B, Hq=Hq, Hkv=Hkv, dh=dh, Tmax=Tmax, inv_freq=inv,
                               scale=1 / math.sqrt(dh), pos_dev=pd, q_norm_w=qw, k_norm_w=kw, eps=1e-6, kv_splits=splits)
    t = qkv.float().view(B, Hq + 2 * Hkv, dh)
    q, k, v = t[:, :Hq], t[:, Hq:Hq + Hkv], t[:, Hq + Hkv:]
    if qk_norm:
        q = qw * q * torch.rsqrt(q.pow(2).mean(-1, keepdim=True) + 1e-6)
        k = kw * k * torch.rsqrt(k.pow(2).mean(-1, keepdim=True) + 1e-6)
    fr = pos * inv
    emb = torch.cat((fr, fr))
    rot = lambda u: torch.cat((-u[..., dh // 2:], u[..., :dh // 2]), -1)
    q = (q * emb.cos() + rot(q) * emb.sin()).bfloat16().float()
    k = (k * emb.cos() + rot(k) * emb.sin()).bfloat16().float()
    close(kc[:, :, pos], k, 1e-2)
    assert torch.equal(vc[:, :, pos].float(), v)
    keep = torch.ones(Tmax, dtype=torch.bool, device=DEV)
    keep[pos] = False
    assert torch.equal(kc[:, :, keep], kc0[:, :, keep]) and torch.equal(vc[:, :, keep], vc0[:, :, keep])
    K = kc[:, :, :pos + 1].float().repeat_interleave(Hq // Hkv, 1)
    V = vc[:, :, :pos + 1].float().repeat_interleave(Hq // Hkv, 1)
    ref = (torch.softmax(q[:, :, None] @ K.transpose(-1, -2) / math.sqrt(dh), -1) @ V).reshape(B, Hq * dh)
    close(out, ref, 1e-2)


@pytest.mark.parametrize("sched,fine", [(0, False), (0, True), (1, False)])
@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("E,I,NQ", [(4096, 12288, 6144), (256, 512, 384), (2048, 6144, 4096)])
def test_dlinear_multi_chain(B, E, I, NQ, sched, fine):
    """o_proj -> gate|up -> down -> qkv in ONE launch (grid barriers inside) == the same four ops launched
    one by one == fp32 torch. Run for several 'steps' so the barrier epochs and self-cleaning state cycle."""
    from u2tokenizer_b200 import ops
    g = gen(E + I + B)
    rnd = lambda *s, sc=1.0: (torch.randn(*s, device=DEV, generator=g) * sc)
    wo, wgu, wdn, wqkv = (rnd(E, E, sc=E ** -0.5).bfloat16(), rnd(2 * I, E, sc=E ** -0.5).bfloat16(),
                          rnd(E, I, sc=I ** -0.5).bfloat16(), rnd(NQ, E, sc=E ** -0.5).bfloat16())
    ln2, ln1n = 1 + 0.1 * rnd(E), 1 + 0.1 * rnd(E)
    tiles = (max(2 * I, NQ, E) + 127) // 128
    eps = 1e-6

    def run(multi, ctx0, x0):
        ws = ops.dlinear_new_ws(max(ops.dlinear_ws_elems(n, k) for n, k in ((E, E), (2 * I, E), (E, I), (NQ, E))), device=DEV, lead=(2,))
        cnt = torch.zeros(2, tiles * 2 + 8, device=DEV, dtype=torch.int32)
        flags = torch.zeros(4, 256, device=DEV, dtype=torch.int32)
        use_fine = fine and multi
        fl = flags if use_fine else [None] * 4
        dep = lambda i, shift: dict(dep_flags=fl[i], dep_shift=shift) if use_fine else {}
        xg2 = torch.empty(B, E, device=DEV, dtype=torch.bfloat16)
        gridbar = torch.zeros(4, device=DEV, dtype=torch.int32); step = torch.zeros(1, device=DEV, dtype=torch.int32)
        ssq_a, ssq_b = torch.zeros(16, device=DEV), torch.zeros(16, device=DEV)
        x, xg = x0.clone(), torch.empty(B, E, device=DEV, dtype=torch.bfloat16)
        act = torch.empty(B, I, device=DEV, dtype=torch.bfloat16)
        qkv = torch.empty(B, NQ, device=DEV, dtype=torch.bfloat16)
        outs = []
        for it in range(3):
            step += 1
            ssq_b.fill_(123.0)  # must be reset by op 0
            ctx = (ctx0 * (1 + 0.1 * it)).bfloat16()
            c0 = dict(ws=ws[0], counters=cnt[0], sched=sched)
            c1 = dict(ws=ws[1], counters=cnt[1], sched=sched)
            chain = [(ctx, wo, x, dict(residual=x, gamma_next=ln2, xg=xg, ssq_out=ssq_a, ssq_zero=ssq_b, out_flags=fl[0], **c0)),
                     (xg, wgu, act, dict(ssq_in=ssq_a, eps=eps, silu_pair=True, out_flags=fl[1], **dep(0, 1), **c1)),
                     (act, wdn, x, dict(residual=x, gamma_next=ln1n, xg=xg2, ssq_out=ssq_b, ssq_zero=ssq_a, out_flags=fl[2], **dep(1, 0), **c0)),
                     (xg2, wqkv, qkv, dict(ssq_in=ssq_b, eps=eps, **dep(2, 1), **c1))]
            if multi:
                ops.dlinear_multi(chain, gridbar=gridbar, step_dev=step)
            else:
                for (a, w, y, kw) in chain:
                    ops.dlinear(a, w, y, **kw)
            torch.cuda.synchronize()
            outs.append((x.clone(), qkv.clone(), act.clone()))
        assert cnt.abs().max().item() == 0
        return outs

    ctx0 = rnd(B, E)
    x0 = rnd(B, E).bfloat16()
    single = run(False, ctx0, x0)
    multi = run(True, ctx0, x0)
    # fp32 torch reference of the chain (bf16 rounding points as in the kernels)
    x = x0.float()
    for it in range(3):
        ctx = (ctx0 * (1 + 0.1 * it)).bfloat16().float()
        x = (ctx @ wo.float().t() + x).bfloat16().float()
        h = (x * ln2).bfloat16().float() @ wgu.float().t() * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)
        a = (F.silu(h[:, 0::2].bfloat16().float()) * h[:, 1::2].bfloat16().float()).bfloat16().float()
        x = (a @ wdn.float().t() + x).bfloat16().float()
        q = (x * ln1n).bfloat16().float() @ wqkv.float().t() * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)
        for outs in (single, multi):
            close(outs[it][0], x, 2e-2)
            close(outs[it][1], q, 3e-2)
            close(outs[it][2], a, 3e-2)


@pytest.mark.parametrize("T,K", [(2048, 1024), (24, 8), (8192, 1024), (100, 100), (5, 1), (16384, 1024), (9000, 3)])
def test_topk_rows(T, K):
    """Index work: bit-exact against torch.topk (sorted descending) on the same fp32 scores, ties included."""
    from u2tokenizer_b200 import ops
    g = gen(T + K)
    sc = torch.randn(3, T, device=DEV, generator=g)
    sc[1, T // 2] = sc[1, T // 3]          # an exact tie
    sc[2] = torch.round(sc[2] * 4) / 4     # many ties
    got = ops.topk_rows(sc, K)
    vals = torch.gather(sc, 1, got)
    ref_vals = torch.topk(sc, K, dim=1).values
    assert torch.equal(vals, ref_vals)                       # same multiset of values in the same order
    assert (got.sort(dim=1).values.diff(dim=1) != 0).all() if K > 1 else True   # no index twice
    # torch leaves the order among equal scores unspecified; ours is deterministic: lower index first
    if K > 1:
        tie = vals[:, 1:] == vals[:, :-1]
        assert (got[:, 1:][tie] > got[:, :-1][tie]).all()
    off = ops.topk_rows(sc, K, idx_offset_per_row=T)
    assert torch.equal(off, got + torch.arange(3, device=DEV)[:, None] * T)


@pytest.mark.parametrize("Sq,Sk", [(2049, 2049), (128, 128), (300, 77), (1, 1), (130, 257)])
def test_flash_attention_d64(Sq, Sk):
    """Fused wgmma attention (ViT head_dim 64) vs fp32 torch on the same bf16 q/k/v, incl. ragged tails."""
    from u2tokenizer_b200 import ops
    B, H, dh = 2, 3, 64
    g = gen(Sq * 3 + Sk)
    Sp = (max(Sq, Sk) + 7) // 8 * 8
    qkv = torch.randn(B, Sp, 3, H, dh, device=DEV, generator=g).bfloat16()   # fused layout like the ViT qkv Linear
    q, k, v = qkv[:, :Sq, 0], qkv[:, :Sk, 1], qkv[:, :Sk, 2]
    out = torch.zeros(B, Sp, H * dh, device=DEV, dtype=torch.bfloat16)
    scale = dh ** -0.5
    ops.flash_attention_d64(q, k, v, out[:, :Sq], scale)  # V consumed in place (MN-major operand of the PV product)
    ref = torch.softmax(torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * scale, -1)
    ref = torch.einsum("bhqk,bkhd->bqhd", ref, v.float()).reshape(B, Sq, H * dh)
    close(out[:, :Sq], ref, 1e-2)
    assert out[:, Sq:].abs().max().item() == 0 if Sp > Sq else True


@pytest.mark.parametrize("temperature,top_k,top_p", [(1.0, 0, 1.0), (0.7, 50, 0.9), (1.3, 5, 1.0), (1.0, 0, 0.5)])
def test_sampling_distribution(temperature, top_k, top_p):
    """Statistical parity with the HF warper chain (temperature -> top-k -> top-p) + multinomial: empirical token
    frequencies over many draws match the filtered distribution; filtered-out tokens are never drawn."""
    from u2tokenizer_b200 import ops
    V, n = 300, 40000
    g = gen(int(temperature * 10) + top_k)
    row = torch.randn(V, device=DEV, generator=g) * 2.0
    logits = row.expand(1024, V).contiguous()
    # reference distribution (HF semantics)
    x = row.double() / temperature
    if top_k > 0:
        kth = x.topk(top_k).values[-1]
        x = x.masked_fill(x < kth, float("-inf"))
    p = torch.softmax(x, -1)
    if top_p < 1.0:
        sp, si = p.sort(descending=True)
        cum = sp.cumsum(0)
        keep_sorted = (cum - sp) < top_p          # keep tokens until the mass reaches top_p (the crossing one included)
        keep = torch.zeros(V, dtype=torch.bool, device=DEV)
        keep[si[keep_sorted]] = True
        p = torch.where(keep, p, torch.zeros_like(p))
        p = p / p.sum()
    counts = torch.zeros(V, device=DEV, dtype=torch.float64)
    draws = 0
    step = 0
    while draws < n:
        ids = ops.sample(logits, temperature=temperature, top_k=top_k, top_p=top_p, seed=1234, step=step)
        counts += torch.bincount(ids, minlength=V).double()
        draws += ids.numel()
        step += 1
    freq = counts / draws
    assert (freq[p == 0] == 0).all(), "a filtered-out token was drawn"
    # total-variation distance; sampling noise ~ sqrt(support / draws)
    tv = 0.5 * (freq - p).abs().sum().item()
    assert tv < 0.03, tv
    # same (seed, step) -> same draw; different rows decorrelated
    a = ops.sample(logits, temperature=temperature, top_k=top_k, top_p=top_p, seed=7, step=3)
    b2 = ops.sample(logits, temperature=temperature, top_k=top_k, top_p=top_p, seed=7, step=3)
    assert torch.equal(a, b2) and a.unique().numel() > 1


@pytest.mark.parametrize("image,hidden,frames", [([8, 128, 256], 96, 3), ([32, 256, 256], 768, 5)])
def test_patch_embed_fused(image, hidden, frames):
    """One-kernel patch embedding (5-D TMA slabs -> converted A operand -> wgmma, + bias + position table) against the
    MONAI restatement in the oracle and against the unfused gather + GEMM path, canonical 4 x 16 x 16 patches."""
    from oracle import u2_oracle as O
    from u2tokenizer_b200 import ops
    patch = [4, 16, 16]
    assert ops.patch_embed_supported(image, patch, hidden)
    gen = torch.Generator(device="cuda").manual_seed(hidden)
    vol = torch.rand(frames, *image, device="cuda", generator=gen)
    K = 4 * 16 * 16
    P = (image[0] // 4) * (image[1] // 16) * (image[2] // 16)
    w = (torch.randn(hidden, K, device="cuda", generator=gen) * K ** -0.5).bfloat16()
    b = 0.1 * torch.randn(hidden, device="cuda", generator=gen)
    pos = (0.1 * torch.randn(P, hidden, device="cuda", generator=gen)).bfloat16()
    Sp = (P + 1 + 7) // 8 * 8
    out = torch.full((frames, Sp, hidden), 7.0, device="cuda", dtype=torch.bfloat16)
    ops.patch_embed(vol, patch, w, b, pos, out)
    sd = {"v.patch_embedding.patch_embeddings.1.weight": w.float(), "v.patch_embedding.patch_embeddings.1.bias": b,
          "v.patch_embedding.position_embeddings": pos.float()[None]}
    ref = O.patch_embed(sd, "v.", vol[:, None], patch)
    got = out[:, 1:1 + P].float()
    e = ((got - ref).abs().max() / ref.abs().max()).item()
    assert e < 1e-2, e
    assert float(out[:, 0].float().min()) == 7.0 and float(out[:, P + 1:].float().min()) == 7.0   # cls / padding rows untouched
    rows = ops.patchify(vol, patch)
    x2 = torch.empty_like(out)
    ops.gemm(rows, w, x2, M=frames * P, N=hidden, K=K, lda=K, ldb=K, ldc=hidden, bias=b, residual=pos, ldr=hidden, res_row_mod=P,
             row_remap=(P, Sp, 1))
    assert float((x2[:, 1:1 + P].float() - got).abs().max()) <= 2 ** -6 * float(ref.abs().max())
