"""The training step at the widths the 8B benchmark trains (μ²Qwen3-8B: E 4096, 32 query / 8 KV heads of 128, I 12288,
V 151936, 512- and 1024-token sequences; Phi-3-mini's head_dim 96 and 2047-key window), and the optimizer it runs.

Every kernel is compared with a plain high-precision reference of the same operation on the same bf16 inputs: fp32
autograd with TF32 off, fp64 where a sum is long, and for the fused AdamW an fp64 emulation of the kernel's own
arithmetic. The file runs in a few minutes on one H100 and every test stays below 40 GB of device memory."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from common import cosine, rel_err, tiny_geometry
from oracle import u2_oracle as O
from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
F64 = torch.float64
GRID_PASS = 132 * 16 * 256 * 4     # elements one grid-stride pass of the AdamW kernels covers (capped grid x 4 per thread)


def _ops():
    from u2tokenizer_b200 import ops, train_ops
    return ops, train_ops


@pytest.fixture(autouse=True)
def fp32_references():
    """Reference matmuls in true fp32 (TF32 off, restored afterwards); each test's peak device memory below 40 GB."""
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
    peak = torch.cuda.max_memory_allocated()
    torch.cuda.empty_cache()
    print(f"peak device memory {peak / 2 ** 30:.2f} GiB")
    assert peak < 40e9, f"peak device memory {peak / 1e9:.1f} GB"


def close(a, b, tol=2e-2, what=""):
    e, c = rel_err(a.double(), b.double()), cosine(a.double(), b.double())
    assert e < tol and c > 0.999, f"{what}: rel_err {e:.4g} cos {c:.6f}"


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------
# optimizer
# ------------------------------------------------------------------------------------------------
def _f32(x):
    """The value of a Python float after the C ABI stores it in a float."""
    return float(np.float32(x))


def _bf16_floor_ceil(x):
    """fp32 x -> (largest bf16 <= x, smallest bf16 >= x), as fp32."""
    t = x.view(torch.int32) & -65536                      # toward zero
    tv = t.view(torch.float32)
    away = torch.where(tv == x, t, t + 65536).view(torch.float32)
    pos = x >= 0
    return torch.where(pos, tv, away), torch.where(pos, away, tv)


def _adamw_fp64(w, m, v, g, *, lr, b1, b2, eps, wd, step, gs):
    """One fused-AdamW step in fp64 from the fp32 constants the kernel holds (beta^step rounded to fp32 like powf).
    Returns the new master, the fp32 m / v before they are stored, and per-element bounds of the fp32 rounding the
    kernel adds to each of the three."""
    lr, b1, b2, eps, wd, gs = (_f32(x) for x in (lr, b1, b2, eps, wd, gs))
    u = 2.0 ** -24                                        # unit roundoff of fp32
    gj = g * gs
    ma, mb = b1 * m, (1 - b1) * gj                        # 1 - beta is exact in fp32
    va, vb = b2 * v, (1 - b2) * gj * gj
    m1, v1 = ma + mb, va + vb
    p1, p2 = _f32(b1 ** step), _f32(b2 ** step)
    bc1, bc2 = 1 - p1, 1 - p2
    denom = v1.sqrt() / math.sqrt(bc2) + eps
    coef = lr / bc1 / denom
    upd = coef * m1
    w1 = w * (1 - lr * wd) - upd
    tol_m = 8 * u * (ma.abs() + mb.abs())                 # g * gs, two products, one sum
    tol_v = 8 * u * (va + vb)
    # powf is within 4 ulp (CUDA C Programming Guide); 1 - beta^step amplifies that by beta^step / (1 - beta^step)
    e_pow = 8 * u * (p1 / bc1 + 0.5 * p2 / bc2)
    tol_w = (8 * u * (w * (1 - lr * wd)).abs() + coef * tol_m
             + upd.abs() * (64 * u + e_pow + 0.5 * tol_v / v1.clamp_min(1e-300)))
    return w1, m1, v1, tol_w, tol_m, tol_v


def _adam_state(n, seed):
    """fp32 master, bf16 m / v / gradient of a run in progress (a few exact zeros: fresh state, zero gradients)."""
    g_ = _gen(seed)
    w = torch.randn(n, device="cuda", generator=g_)
    m = (0.05 * torch.randn(n, device="cuda", generator=g_)).to(BF)
    v = (0.05 * torch.randn(n, device="cuda", generator=g_)).square().to(BF)
    gr = torch.randn(n, device="cuda", generator=g_).to(BF)
    m[1::7], v[1::7], gr[2::11] = 0, 0, 0
    return w, m, v, gr


@pytest.mark.parametrize("n", [4, 7 * 2 ** 20 + 4])
@pytest.mark.parametrize("scaled", [False, True])
def test_adamw_bf16_moments_one_step_against_fp64_emulation(n, scaled):
    """u2_adamw_bf16_mom16, one step, against its own arithmetic in fp64: n = 4 and n over three grid-stride passes,
    grad_scale NULL and a device scalar, bias correction at steps 1 / 2 / 1000 / 100000, weight decay 0 and 0.1.
    The master (computed from the unrounded fp32 moments) matches to a few fp32 ulps; each stored moment is one of the
    two bf16 neighbours of the exact value (its fp32 rounding included); the bf16 parameter copy is the master rounded
    to nearest."""
    ops, T = _ops()
    assert n == 4 or n > 3 * GRID_PASS
    w0, m0, v0, gr = _adam_state(n, seed=n % 1000)
    gs = 0.37
    scale = torch.full((1,), gs, device="cuda") if scaled else None
    g64 = gr.to(F64)
    for step in (1, 2, 1000, 100000):
        for wd in (0.0, 0.1):
            kw = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=wd, step=step)
            w, m, v = w0.clone(), m0.clone(), v0.clone()
            pout = torch.empty(n, device="cuda", dtype=BF)
            T.adamw(w, m, v, gr, pout, grad_scale=scale, **kw)
            w1, m1, v1, tol_w, tol_m, tol_v = _adamw_fp64(w0.to(F64), m0.to(F64), v0.to(F64), g64, lr=1e-3, b1=0.9,
                                                          b2=0.999, eps=1e-8, wd=wd, step=step, gs=gs if scaled else 1.0)
            err = (w.to(F64) - w1).abs()
            bad = err > tol_w
            assert not bad.any(), (f"step {step} wd {wd}: {int(bad.sum())} masters off, worst {float(err.max()):.3g} "
                                   f"(tolerance there {float(tol_w[err.argmax()]):.3g})")
            for name, got, x, tol in (("m", m, m1, tol_m), ("v", v, v1, tol_v)):
                lo, _ = _bf16_floor_ceil((x - tol).float())
                _, hi = _bf16_floor_ceil((x + tol).float())
                s = got.float()
                out = (s < lo) | (s > hi)
                assert not out.any(), f"step {step} wd {wd}: {int(out.sum())} stored {name} outside their bf16 neighbours"
            assert torch.equal(pout, w.to(BF)), "bf16 parameter copy != master rounded to nearest"


def test_adamw_bf16_moments_track_fp32_adamw_over_3000_steps():
    """Drift of the bf16-moment state against fp32 AdamW (torch.optim.AdamW fed the same gradients): 1 M parameters
    from 0, lr 4e-6 (the benchmark's), pure-noise gradients whose scale decays 10x over 3000 steps. With
    round-to-nearest moments v can only grow once (1 - beta2)|g^2 - v| drops below half a bf16 ulp of v: the median
    v / v_fp32 reaches ~4.4 and the weights drift ~18 % away by step 3000. Unbiased (stochastic) rounding keeps both
    at the fp32 run's."""
    ops, T = _ops()
    n, steps, lr = 2 ** 20, 3000, 4e-6
    gen = _gen(0)
    ref = torch.nn.Parameter(torch.zeros(n, device="cuda"))
    opt = torch.optim.AdamW([ref], lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)
    master = torch.zeros(n, device="cuda")
    m = torch.zeros(n, device="cuda", dtype=BF)
    v = torch.zeros(n, device="cuda", dtype=BF)
    rows = []
    for t in range(1, steps + 1):
        gr = (1e-2 * 10 ** (-(t - 1) / steps) * torch.randn(n, device="cuda", generator=gen)).to(BF)
        ref.grad = gr.float()
        opt.step()
        T.adamw(master, m, v, gr, None, lr=lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, step=t)
        if t in (500, 1000, 3000):
            ratio = float((v.float() / opt.state[ref]["exp_avg_sq"]).median())
            div = float((master - ref.data).norm() / ref.data.norm())
            rows.append((t, ratio, div))
    print("\nstep | median v_bf16 / v_fp32 | |w_bf16 - w_fp32| / |w_fp32|")
    for t, ratio, div in rows:
        print(f"{t:5d} | {ratio:.4f} | {div:.3e}")
    for t, ratio, div in rows:
        assert 0.9 <= ratio <= 1.1 and div < 5e-2, f"step {t}: median v ratio {ratio:.3f}, weight divergence {div:.3g}"


def test_adamw_bf16_moment_rounding_is_reproducible_and_split_invariant():
    """The stochastic rounding draws from (seed, step, global element index) only: the same call twice gives the same
    bits, and one call on a whole buffer gives the same bits as two calls on its halves with index offsets (how ZeRO-1
    slices and buckets cut it). Another step, seed or offset gives different bits; the master never depends on them."""
    ops, T = _ops()
    n = 3 * 2 ** 20 + 8
    h = n // 2
    base = 3 * 2 ** 32 + 12                     # past 2^32: the high word of the index is hashed too
    w0, m0, v0, gr = _adam_state(n, seed=5)

    def run(step=7, seed=0x5EED, off=base, split=False):
        w, m, v = w0.clone(), m0.clone(), v0.clone()
        kw = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, step=step, seed=seed)
        if split:
            T.adamw(w[:h], m[:h], v[:h], gr[:h], None, index_offset=off, **kw)
            T.adamw(w[h:], m[h:], v[h:], gr[h:], None, index_offset=off + h, **kw)
        else:
            T.adamw(w, m, v, gr, None, index_offset=off, **kw)
        return w, m.view(torch.int16), v.view(torch.int16)

    w, m, v = run()
    for other in (run(), run(split=True)):
        assert torch.equal(other[0], w) and torch.equal(other[1], m) and torch.equal(other[2], v)
    for kw in (dict(step=8), dict(seed=0x5EEE), dict(off=base + 4)):
        w2, m2, v2 = run(**kw)
        if "step" not in kw:
            assert torch.equal(w2, w)
        # about half the elements sit between their two bf16 neighbours far enough to flip
        assert (m2 != m).float().mean() > 0.1 and (v2 != v).float().mean() > 0.1, kw


def test_adamw_bf16_moment_rounding_is_unbiased():
    """E[stored moment] = the fp32 moment: from m = v = 0 a step stores (1 - beta1) g and (1 - beta2) g^2 (fp32), each
    value drawn 2^16 times per step over 8 steps; every draw is one of its two bf16 neighbours and their mean is the
    fp32 value within 5 standard errors of a Bernoulli draw between them."""
    ops, T = _ops()
    K, R, steps = 16, 2 ** 16, 8
    vals = torch.randn(K, device="cuda", generator=_gen(3)).to(BF)
    gr = vals.repeat_interleave(R)
    n = K * R
    b1, b2 = torch.tensor(0.9, device="cuda"), torch.tensor(0.999, device="cuda")
    xm = (1 - b1) * vals.float()                 # fp32 arithmetic, as the kernel does it
    xv = ((1 - b2) * vals.float()) * vals.float()
    draws = {"m": [], "v": []}
    for step in range(1, steps + 1):
        w = torch.zeros(n, device="cuda")
        m = torch.zeros(n, device="cuda", dtype=BF)
        v = torch.zeros(n, device="cuda", dtype=BF)
        T.adamw(w, m, v, gr, None, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, step=step, seed=11)
        draws["m"].append(m.view(K, R))
        draws["v"].append(v.view(K, R))
    for name, x in (("m", xm), ("v", xv)):
        s = torch.cat(draws[name], 1).float()    # [K, steps * R]
        lo, hi = _bf16_floor_ceil(x)
        assert bool(((s == lo[:, None]) | (s == hi[:, None])).all()), f"{name}: a draw is not a bf16 neighbour"
        N = s.shape[1]
        p = ((x.double() - lo.double()) / (hi.double() - lo.double()).clamp_min(1e-300))
        se = (hi.double() - lo.double()) * (p * (1 - p) / N).sqrt()
        bias = s.double().mean(1) - x.double()
        assert bool((bias.abs() <= 5 * se).all()), f"{name}: mean - x = {bias.tolist()}, standard errors {se.tolist()}"


def test_adamw_f32grad_matches_torch():
    """u2_adamw_f32grad (every vector parameter, every step) against torch.optim.AdamW over 5 steps, n over three
    grid-stride passes, grad_scale and weight decay on. The fp32 parameter mirror holds bf16-representable values: the
    master rounded to nearest, the same as the bf16 copy."""
    ops, T = _ops()
    n, lr = 7 * 2 ** 20 + 4, 1e-3
    gen = _gen(8)
    p0 = torch.randn(n, device="cuda", generator=gen)
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref], lr=lr, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    master, m, v = p0.clone(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pout = torch.empty(n, device="cuda", dtype=BF)
    p32 = torch.full((n,), float("nan"), device="cuda")
    scale = torch.full((1,), 0.37, device="cuda")
    for step in range(1, 6):
        gr = torch.randn(n, device="cuda", generator=gen)
        ref.grad = gr * 0.37
        opt.step()
        T.adamw(master, m, v, gr, pout, lr=lr, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1, step=step,
                grad_scale=scale, param_out_f32=p32)
        st = opt.state[ref]
        d = (master - ref.data).abs()
        assert bool((d <= 2 ** -20 * ref.data.abs() + step * lr * 1e-5).all()), (step, float(d.max()))
        for name, got, want in (("m", m, st["exp_avg"]), ("v", v, st["exp_avg_sq"])):
            assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max()), (step, name)
        assert torch.equal(pout, master.to(BF))
        assert torch.equal(p32, master.to(BF).float())


@pytest.mark.parametrize("dtype", [BF, torch.float32])
def test_sumsq_large_n_accumulates(dtype):
    """sum of squares over 2.5e8 elements (more than the 8B model's largest gradient bucket) against an fp64 sum,
    relative error < 1e-5; the kernel adds into out (the clipping norm sums several buckets into one scalar)."""
    ops, T = _ops()
    n = 250_000_000
    x = torch.randn(n, device="cuda", generator=_gen(4)).add_(0.5).to(dtype)
    ref = sum(float(c.to(F64).square().sum()) for c in x.split(2 ** 25))
    s0 = 0.25 * ref
    out = torch.full((1,), s0, device="cuda")
    T.sumsq(x, out)
    got = float(out) - float(np.float32(s0))
    assert abs(got - ref) / ref < 1e-5, (got, ref)
    small = x[:8]
    out = torch.ones(1, device="cuda")
    T.sumsq(small, out)
    T.sumsq(small, out)
    want = 1 + 2 * float(small.to(F64).square().sum())
    assert abs(float(out) - want) <= 1e-6 * want, (float(out), want)


def _labels(ids, n_vis):
    lab = ids.clone()
    lab[:, :n_vis + 1] = -100
    return lab


@pytest.mark.parametrize("clip", ["active", "inactive"])
def test_optimizer_step_bf16_moments_against_fp32_adamw(clip):
    """TrainEngine.optimizer_step with moment_dtype=torch.bfloat16 (the single-GPU benchmark's optimizer): several
    buckets, 5 steps, gradient clipping active (threshold half the first gradient norm) or inactive (4x it), against
    torch.optim.AdamW with fp32 moments driven by the engine's own gradients. In the first steps an AdamW update is at
    most ~lr per element (|m^| / sqrt(v^) <= 1.011 for t <= 5 by Cauchy-Schwarz); bf16 moments change an update by a
    small fraction of that, so per element |master - fp32 master| <= steps * lr * 0.05. The vector region keeps fp32
    moments and matches to 2e-5; the bf16 parameters are the masters rounded to nearest."""
    from u2tokenizer_b200.train import TrainEngine
    g = tiny_geometry()
    sd16 = synthetic_state_dict(g, seed=9, device="cpu", dtype=BF)
    te = TrainEngine(g, sd16, device="cuda", bucket_elems=50_000)
    L = te.lay
    assert L.n_buckets > 2
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=6, lt=10)
    labels = _labels(ids, g.num_3d_query_token)
    batch = (images.cuda(), ids.cuda(), qids.cuda(), labels.cuda())
    te.zero_grad()
    te.forward_backward(*batch)
    norm0 = math.sqrt(float(te.Gm.float().square().sum()) + float(te.Gv.square().sum()))
    max_norm = 0.5 * norm0 if clip == "active" else 4.0 * norm0
    lr = 1e-3
    te.init_optimizer(lr=lr, weight_decay=0.01, max_grad_norm=max_norm, moment_dtype=BF)
    ref_m = torch.nn.Parameter(te.opt["m_master"].clone())
    ref_v = torch.nn.Parameter(te.opt["v_master"].clone())
    opt = torch.optim.AdamW([ref_m, ref_v], lr=lr, weight_decay=0.01)
    worst = 0.0
    for it in range(1, 6):
        te.zero_grad()
        te.forward_backward(*batch)
        ref_m.grad, ref_v.grad = te.Gm.float().clone(), te.Gv.clone()
        total = float(torch.nn.utils.clip_grad_norm_([ref_m, ref_v], max_norm))
        assert (total > max_norm) == (clip == "active"), (total, max_norm)
        opt.step()
        te.optimizer_step()
        d = float((te.opt["m_master"] - ref_m.data).abs().max())
        worst = max(worst, d / (it * lr))
        assert d <= it * lr * 0.05, (it, d)
        assert float((te.opt["v_master"] - ref_v.data).abs().max()) < 2e-5, it
        assert torch.equal(te.W[:L.mat_total], te.opt["m_master"].to(BF))
    print(f"max |master - fp32 master| / (steps * lr) = {worst:.3g}")


# ------------------------------------------------------------------------------------------------
# decoder backward kernels at production shapes
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E", [2048, 3072, 4096])
def test_rmsnorm_backward_production_widths(E):
    """RMSNorm backward at the decoder widths of Qwen3-1.7B / Phi-3-mini / Qwen3-8B over 2048 rows, with the residual
    branch's gradient (dres) and in place on it as the training path calls it; dgamma accumulates over all rows."""
    ops, T = _ops()
    gen = _gen(E)
    rows = 2048
    x = torch.randn(rows, E, device="cuda", generator=gen).to(BF)
    dy = torch.randn(rows, E, device="cuda", generator=gen).to(BF)
    dres = torch.randn(rows, E, device="cuda", generator=gen).to(BF)
    gamma = 1 + 0.1 * torch.randn(E, device="cuda", generator=gen)
    xr = x.to(F64).requires_grad_(True)
    gr = gamma.to(F64).requires_grad_(True)
    (gr * (xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-6))).backward(dy.to(F64))
    dg = torch.ones(E, device="cuda")
    dx = T.rmsnorm_bwd(x, gamma, dy, dres=dres, dgamma=dg, eps=1e-6)
    close(dx, xr.grad + dres.to(F64), 2e-2, "rmsnorm dx")
    close(dg - 1, gr.grad, 2e-2, "rmsnorm dgamma")
    pend = dres.clone()
    T.rmsnorm_bwd(x, gamma, dy, dres=pend, out=pend, dgamma=dg, eps=1e-6)
    assert torch.equal(pend, dx)
    close(dg - 1, 2 * gr.grad, 2e-2, "rmsnorm dgamma accumulated")


@pytest.mark.parametrize("dh,nq,nk,theta,norm", [(128, 32, 8, 1e6, True), (96, 32, 32, 1e4, False)])
def test_rope_backward_production_heads(dh, nq, nk, theta, norm):
    """RoPE (+ Qwen3 q/k RMSNorm) forward and backward on the decoder's fused qkv rows: Qwen3-8B (dh 128, 32 / 8
    heads, theta 1e6, q/k norm) and Phi-3-mini (dh 96, 32 / 32, theta 1e4), 2 x 1024 rows with positions up to 1023;
    dq_norm / dk_norm are summed over every row and head."""
    ops, T = _ops()
    gen = _gen(dh + nk)
    B, Lx = 2, 1024
    rows, nv = B * Lx, nk
    ld = (nq + nk + nv) * dh
    x = torch.randn(rows, ld, device="cuda", generator=gen).to(BF)
    dy = torch.randn(rows, ld, device="cuda", generator=gen).to(BF)
    inv = 1.0 / (theta ** (torch.arange(0, dh, 2, device="cuda").float() / dh))
    wq = (1 + 0.1 * torch.randn(dh, device="cuda", generator=gen)) if norm else None
    wk = (1 + 0.1 * torch.randn(dh, device="cuda", generator=gen)) if norm else None
    xr = x.to(F64).requires_grad_(True)
    wqr = wq.to(F64).requires_grad_(True) if norm else None
    wkr = wk.to(F64).requires_grad_(True) if norm else None
    h = xr.view(rows, nq + nk + nv, dh)
    fr = torch.outer((torch.arange(rows, device="cuda") % Lx).to(F64), inv.to(F64))
    cos, sin = torch.cat((fr, fr), -1).cos()[:, None], torch.cat((fr, fr), -1).sin()[:, None]

    def rot(t, w):
        if w is not None:
            t = w * (t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6))
        return t * cos + O._rotate_half(t) * sin
    y = torch.cat((rot(h[:, :nq], wqr), rot(h[:, nq:nq + nk], wkr), h[:, nq + nk:]), 1).reshape(rows, ld)
    y.backward(dy.to(F64))
    fwd = x.clone()
    ops.rope(fwd, rows=rows, ld=ld, dh=dh, n_q=nq, n_k=nk, n_v=0, inv_freq=inv, q_norm_w=wq, k_norm_w=wk, eps=1e-6,
             pos_div=1, pos_mod=Lx)
    close(fwd, y, 2e-2, "rope fwd")
    dx = dy.clone()
    dwq = torch.zeros(dh, device="cuda") if norm else None
    dwk = torch.zeros(dh, device="cuda") if norm else None
    T.rope_bwd(dx, x, rows=rows, ld=ld, dh=dh, n_q=nq, n_k=nk, inv_freq=inv, q_norm_w=wq, k_norm_w=wk, eps=1e-6, pos0=0,
               pos_div=1, pos_mod=Lx, dq_norm_w=dwq, dk_norm_w=dwk)
    close(dx, xr.grad, 2e-2, "rope dx")
    if norm:
        close(dwq, wqr.grad, 2e-2, "rope dq_norm")
        close(dwk, wkr.grad, 2e-2, "rope dk_norm")


@pytest.mark.parametrize("I", [6144, 8192, 12288])
def test_silu_mul_backward_halves_layout(I):
    """SiLU(gate) * up and its backward in the [gate | up] halves layout of the training path (interleaved=False) at
    the MLP widths of Qwen3-1.7B, Phi-3-mini and Qwen3-8B, 1024 rows."""
    ops, T = _ops()
    gen = _gen(I)
    rows = 1024
    gu = (2 * torch.randn(rows, 2 * I, device="cuda", generator=gen)).to(BF)
    da = torch.randn(rows, I, device="cuda", generator=gen).to(BF)
    gur = gu.float().requires_grad_(True)
    y = F.silu(gur[:, :I]) * gur[:, I:]
    y.backward(da.float())
    close(ops.silu_mul(gu, interleaved=False), y, 1e-2, "silu_mul fwd")
    close(T.silu_mul_bwd(gu, da), gur.grad, 1e-2, "silu_mul bwd")


@pytest.mark.parametrize("S,window", [(512, 0), (1024, 0), (2304, 0), (2304, 2047)])
def test_softmax_backward_causal_rows(S, window):
    """dS = P * (dP - rowsum(dP * P)) on causal rows (S = Sk, keys padded to Skp > Sk) and with Phi-3's 2047-key window
    on 2304 keys, out of place and in place as the attention backward runs it: masked keys and the padding get exact
    zeros."""
    ops, T = _ops()
    gen = _gen(S + window)
    n0, H = 2, 4
    Skp = S + 8
    st = (H * S * Skp, S * Skp, Skp)
    sc = 4 * torch.randn(n0, H, S, Skp, device="cuda", generator=gen)
    P = torch.empty(n0, H, S, Skp, device="cuda", dtype=BF)
    ops.softmax(sc, P, n0=n0, H=H, S=S, n=S, in_strides=st, out_strides=st, causal=True, causal_off=0, zero_pad_to=Skp,
                window=window)
    del sc
    i = torch.arange(S, device="cuda")[:, None]
    j = torch.arange(S, device="cuda")[None, :]
    visible = (j <= i) & ((j > i - window) if window else True)
    assert float(P[..., :S].float().masked_fill(visible, 0).abs().max()) == 0.0
    dP = torch.randn(n0, H, S, Skp, device="cuda", generator=gen)
    Pf = P[..., :S].to(F64)
    ref = Pf * (dP[..., :S].to(F64) - (dP[..., :S].to(F64) * Pf).sum(-1, keepdim=True))
    dS = torch.full_like(P, 1.0)
    T.softmax_bwd(P, dP, dS, n0=n0, H=H, S=S, n=S, p_strides=st, dp_strides=st, ds_strides=st, zero_pad_to=Skp)
    close(dS[..., :S], ref, 2e-2, "softmax bwd")
    assert float(dS[..., :S].float().masked_fill(visible, 0).abs().max()) == 0.0
    assert float(dS[..., S:].abs().max()) == 0.0
    T.softmax_bwd(P, dP, P, n0=n0, H=H, S=S, n=S, p_strides=st, dp_strides=st, ds_strides=st, zero_pad_to=Skp)
    assert torch.equal(P, dS)


@pytest.mark.parametrize("V", [151936, 32064])
def test_ce_backward_vocab_widths(V):
    """dlogits = coef * (softmax - onehot) at the Qwen3 and Phi-3 vocabularies, 1024 rows, lse from the fused lm_head
    log-prob kernel (as the training path takes it); rows with coef 0 (unlabelled) come out exactly zero."""
    ops, T = _ops()
    gen = _gen(V)
    R, E = 1024, 512
    h = torch.randn(R, E, device="cuda", generator=gen).to(BF)
    W = (torch.randn(V, E, device="cuda", generator=gen) * (3 / math.sqrt(E))).to(BF)
    labels = torch.randint(0, V, (R,), device="cuda", generator=gen)
    labels[:8], labels[8:16] = V - 1, 0
    coef = torch.rand(R, device="cuda", generator=gen)
    coef[::7] = 0
    lab = torch.where(coef > 0, labels, torch.full_like(labels, -1))
    _, lse, _ = ops.lmhead_logprob(h, W, lab, want_lse=True)
    logits = h.float() @ W.float().t()
    assert float((lse - torch.logsumexp(logits, -1)).abs().max()) < 1e-3
    lr_ = logits.clone().requires_grad_(True)
    lp = torch.log_softmax(lr_, -1).gather(1, labels[:, None]).squeeze(1)
    (-(coef * lp).sum()).backward()
    dl = T.ce_bwd(logits, lse, lab.clamp_min(0), coef)
    close(dl, lr_.grad, 2e-2, "ce bwd")
    assert float(dl[coef == 0].float().abs().max()) == 0.0


def test_embed_scatter_add_repeated_ids_is_exact():
    """Embedding gradient at V = 151936 with half of 2 x 1024 rows on 16 hot ids (~64 bf16 atomic adds per element).
    Row gradients and the table hold small integers, so every partial sum is an integer below 256 and exact in bf16 in
    any order: the result must equal the fp32 index_add exactly (a lost or misplaced add shows)."""
    ops, T = _ops()
    gen = _gen(12)
    V, E, B, L = 151936, 2048, 2, 1024
    ids = torch.randint(0, V, (B, L), device="cuda", generator=gen)
    hot = torch.randint(0, V, (16,), device="cuda", generator=gen)
    hot[0], hot[1] = 0, V - 1
    ids.view(-1)[::2] = hot[torch.randint(0, 16, (B * L // 2,), device="cuda", generator=gen)]
    assert int(torch.bincount(ids.view(-1), minlength=V).max()) <= 125
    drows = torch.randint(-2, 3, (B, L, E), device="cuda", generator=gen).to(BF)
    dt0 = torch.randint(-4, 5, (V, E), device="cuda", generator=gen).to(BF)
    dt = dt0.clone()
    T.embed_scatter_add(ids, drows, dt, None)
    want = dt0.float().index_add_(0, ids.view(-1), drows.view(-1, E).float())
    assert torch.equal(dt.float(), want)


# ------------------------------------------------------------------------------------------------
# the decoder's causal GQA attention composite
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def engine():
    from u2tokenizer_b200.train import TrainEngine
    g = tiny_geometry()
    return TrainEngine(g, synthetic_state_dict(g, seed=0, device="cpu", dtype=BF), device="cuda")


@pytest.mark.parametrize("dh,hq,hkv,L,window", [(128, 32, 8, 512, 0), (128, 16, 8, 1024, 0), (96, 32, 32, 1024, 0),
                                               (96, 32, 32, 2304, 2047)])
def test_causal_gqa_attention_backward(engine, dh, hq, hkv, L, window):
    """TrainEngine.attention(causal=True) as the decoder runs it (q / k / v views of one fused qkv buffer; scores GEMM,
    causal / windowed softmax, P @ V; backward: softmax_bwd, P^T @ dO and dS^T @ Q with group_sum over the G query
    heads of a KV head, dQ GEMM with the GQA batch divisor) against fp32 attention with the KV heads repeated, B = 2.
    Queries are scaled so that most rows put more than half their probability on one key: a near-uniform softmax
    would hide errors in dS."""
    from u2tokenizer_b200.train import Var
    te = engine
    B, G = 2, hq // hkv
    nh = hq + 2 * hkv
    scale = 1.0 / math.sqrt(dh)
    gen = _gen(dh * L + hq)
    qkv = torch.randn(B, L, nh, dh, device="cuda", generator=gen)
    qkv[:, :, :hq] *= 8
    qkv = qkv.to(BF)
    dout = torch.randn(B, L, hq * dh, device="cuda", generator=gen).to(BF)
    qv = lambda t: t.view(B, L, nh, dh)[:, :, :hq]
    kv_ = lambda t: t.view(B, L, nh, dh)[:, :, hq:hq + hkv]
    vv_ = lambda t: t.view(B, L, nh, dh)[:, :, hq + hkv:]
    var = Var(qkv.clone())
    te.tape = []
    out = te.attention(var, qv, var, kv_, var, vv_, (B, L, hq * dh), scale, causal=True, group="dec", window=window)
    out.g = dout.clone()
    te.run_backward()
    ctx = out.v.float()

    q = qv(qkv).float().transpose(1, 2).requires_grad_(True)      # [B, hq, L, dh]
    k = kv_(qkv).float().transpose(1, 2).requires_grad_(True)
    v = vv_(qkv).float().transpose(1, 2).requires_grad_(True)
    i = torch.arange(L, device="cuda")[:, None]
    j = torch.arange(L, device="cuda")[None, :]
    visible = (j <= i) & ((j > i - window) if window else True)
    s = (q @ k.repeat_interleave(G, 1).transpose(-1, -2)) * scale
    p = torch.softmax(s.masked_fill(~visible, float("-inf")), -1)
    del s
    peaked = float((p.amax(-1) > 0.5).float().mean())
    assert peaked > 0.5, f"only {peaked:.2f} of the rows are peaked"
    ref = p @ v.repeat_interleave(G, 1)
    ref.backward(dout.float().view(B, L, hq, dh).transpose(1, 2))
    del p
    close(ctx.view(B, L, hq, dh), ref.detach().transpose(1, 2), 2e-2, "ctx")
    close(qv(var.g).float(), q.grad.transpose(1, 2), 2e-2, "dQ")
    close(kv_(var.g).float(), k.grad.transpose(1, 2), 2e-2, "dK")
    close(vv_(var.g).float(), v.grad.transpose(1, 2), 2e-2, "dV")


# ------------------------------------------------------------------------------------------------
# one decoder layer at full width through the whole engine
# ------------------------------------------------------------------------------------------------
LAYER_CASES = {
    # E 4096: the vocabulary is cut to 32768 so that the fp32 oracle's embedding, head and their gradients fit the
    # memory budget next to the 8B-wide layer
    "qwen3_8b_L512": (dict(hidden_size=4096, intermediate_size=12288, num_attention_heads=32, num_key_value_heads=8,
                           head_dim=128, vocab_size=32768), 512),
    "qwen3_8b_L1024": (dict(hidden_size=4096, intermediate_size=12288, num_attention_heads=32, num_key_value_heads=8,
                            head_dim=128, vocab_size=32768), 1024),
    "qwen3_1.7b_L512": (dict(hidden_size=2048, intermediate_size=6144, num_attention_heads=16, num_key_value_heads=8,
                             head_dim=128, vocab_size=151936), 512),
    "phi3_mini_L512": (dict(hidden_size=3072, intermediate_size=8192, num_attention_heads=32, num_key_value_heads=32,
                            head_dim=96, vocab_size=32064, qk_norm=False, rms_norm_eps=1e-5, rope_theta=1e4,
                            decoder_family="phi3", sliding_window=2047), 512),
}


@pytest.mark.parametrize("case", list(LAYER_CASES))
def test_full_width_decoder_layer_matches_oracle_autograd(case):
    """TrainEngine.forward_backward with ONE decoder layer at the Qwen3-8B, Qwen3-1.7B and Phi-3-mini widths (a tiny
    vision side and one tokenizer layer at the decoder width), B = 2, 512 tokens (and 1024 for 8B): the loss and every
    parameter gradient against autograd through the fp32 oracle (tests/phi3_oracle.py for Phi-3), with the criterion
    of test_train_gpu.py: rel_err < 4e-2 and cosine > 0.995, or an absolute error below 2e-3 of the largest gradient
    entry of the model."""
    import phi3_oracle as P3
    from u2tokenizer_b200.train import TrainEngine
    over, L = LAYER_CASES[case]
    g = tiny_geometry(num_hidden_layers=1, u2t_num_layers=1, **over)
    sd16 = synthetic_state_dict(g, seed=41, device="cuda", dtype=BF)
    sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
    n_vis = g.num_3d_query_token
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=L - n_vis, lt=L)
    assert ids.shape[1] == L
    labels = _labels(ids, n_vis).cuda()
    images, ids, qids = images.cuda(), ids.cuda(), qids.cuda()
    sd = {k: v.float().requires_grad_(True) for k, v in sd16.items()}
    if g.decoder_family == "phi3":
        ref = O.causal_lm_loss(P3.decoder_forward(sd, O.multimodal_embeds(sd, ids, images, qids, g), g)[0], labels)
    else:
        ref = O.causal_lm_loss(O.forward_logits(sd, ids, images, qids, g), labels)
    ref.backward()
    ref_loss = float(ref.detach())
    ref_g = {k: v.grad for k, v in sd.items()}
    del sd, ref
    te = TrainEngine(g, sd16, device="cuda")
    del sd16
    te.zero_grad()
    loss = float(te.forward_backward(images, ids, qids, labels))
    assert abs(loss - ref_loss) < 2e-2 * max(1.0, abs(ref_loss)), (loss, ref_loss)
    lay = te.lay
    gmax = max(v.abs().max().item() for v in ref_g.values() if v is not None)
    bad, n_cmp = [], 0
    for n in lay.mat_names + lay.vec_names:
        if n == "lm_head.weight" and te.tied:
            continue
        got = te.grad(n).float()
        want = ref_g[n] if ref_g[n] is not None else torch.zeros_like(got)
        n_cmp += 1
        if want.abs().max().item() < 1e-9:
            assert got.abs().max().item() < 1e-4, n
            continue
        e, c = rel_err(got, want), cosine(got, want)
        if (e < 4e-2 and c > 0.995) or (got - want).abs().max().item() < 2e-3 * gmax:
            continue
        bad.append((n, round(e, 4), round(c, 5)))
    assert n_cmp > 20 and any(n.startswith("model.layers.0.") for n in lay.mat_names)
    assert not bad, bad[:6]
