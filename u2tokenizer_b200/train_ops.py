"""Python-side wrappers of the training kernels (include/u2b200_train.h): torch tensors in, C-ABI calls underneath.
Like ops.py: CUDA only, no PyTorch fallback; shapes / strides are validated here, arithmetic happens in csrc/."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib, ops
from .ops import BF16, F32, _need_cuda, _ptr, _stream


def _rows2d(t: torch.Tensor) -> torch.Tensor:
    t2 = t.reshape(-1, t.shape[-1]) if t.dim() != 2 else t
    if t2.stride(1) != 1:
        raise ValueError("last dim must be contiguous")
    return t2


def transpose(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [..., R, C] (last dim contiguous, leading dims collapsible) -> [..., C, R]."""
    _need_cuda(x)
    R, Cc = x.shape[-2], x.shape[-1]
    xb = x.reshape(-1, R, Cc)
    if xb.stride(2) != 1:
        xb = xb.contiguous()
    nb = xb.shape[0]
    if out is None:
        out = torch.empty(*x.shape[:-2], Cc, R, device=x.device, dtype=BF16)
    ob = out.view(-1, Cc, R)
    _lib.check(_lib.load().u2_transpose_bf16(xb.data_ptr(), ob.data_ptr(), R, Cc, xb.stride(1), ob.stride(1), nb,
                                             xb.stride(0) if nb > 1 else 0, ob.stride(0) if nb > 1 else 0, _stream()),
               "u2_transpose_bf16")
    return out


def colsum(x: torch.Tensor, out: torch.Tensor, rows: Optional[int] = None, cols: Optional[int] = None,
           ld: Optional[int] = None) -> torch.Tensor:
    """out[c] += sum_r x[r, c] (out fp32, accumulated)."""
    _need_cuda(x, out)
    if rows is None:
        x2 = _rows2d(x)
        rows, cols, ld = x2.shape[0], x2.shape[1], x2.stride(0)
    if out.dtype != F32:
        raise TypeError("colsum accumulates into fp32")
    _lib.check(_lib.load().u2_colsum_bf16(x.data_ptr(), out.data_ptr(), rows, cols, ld, _stream()), "u2_colsum_bf16")
    return out


def gelu(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need_cuda(x)
    if not x.is_contiguous():
        raise ValueError("gelu expects a contiguous tensor")
    if out is None:
        out = torch.empty_like(x)
    _lib.check(_lib.load().u2_gelu_bf16(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "u2_gelu_bf16")
    return out


def gelu_bwd(x_pre: torch.Tensor, dy: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need_cuda(x_pre, dy)
    if not (x_pre.is_contiguous() and dy.is_contiguous()):
        raise ValueError("gelu_bwd expects contiguous tensors")
    if out is None:
        out = torch.empty_like(dy)
    _lib.check(_lib.load().u2_gelu_bwd_bf16(x_pre.data_ptr(), dy.data_ptr(), out.data_ptr(), dy.numel(), _stream()),
               "u2_gelu_bwd_bf16")
    return out


def silu_mul_bwd(gate_up: torch.Tensor, dact: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need_cuda(gate_up, dact)
    g2, d2 = _rows2d(gate_up), _rows2d(dact)
    I = g2.shape[1] // 2
    if out is None:
        out = torch.empty_like(g2)
    if out.stride(0) != g2.stride(0):
        raise ValueError("silu_mul_bwd: dgu must share gate_up's row stride")
    _lib.check(_lib.load().u2_silu_mul_bwd_bf16(g2.data_ptr(), d2.data_ptr(), out.data_ptr(), g2.shape[0], I, g2.stride(0),
                                                d2.stride(0), _stream()), "u2_silu_mul_bwd_bf16")
    return out


def layernorm_bwd(x, gamma, dy, *, dres=None, out=None, dgamma=None, dbeta=None, eps=1e-5):
    _need_cuda(x, gamma, dy, dres, out, dgamma, dbeta)
    x2, g2 = _rows2d(x), _rows2d(dy)
    if out is None:
        out = torch.empty_like(x2)
    o2 = _rows2d(out)
    r2 = _rows2d(dres) if dres is not None else None
    _lib.check(_lib.load().u2_layernorm_bwd_bf16(x2.data_ptr(), gamma.data_ptr(), g2.data_ptr(), _ptr(r2), o2.data_ptr(),
                                                 _ptr(dgamma), _ptr(dbeta), x2.shape[0], x2.shape[1], x2.stride(0),
                                                 g2.stride(0), r2.stride(0) if r2 is not None else 0, o2.stride(0), eps,
                                                 _stream()), "u2_layernorm_bwd_bf16")
    return out


def rmsnorm_bwd(x, gamma, dy, *, dres=None, out=None, dgamma=None, eps=1e-6):
    _need_cuda(x, gamma, dy, dres, out, dgamma)
    x2, g2 = _rows2d(x), _rows2d(dy)
    if out is None:
        out = torch.empty_like(x2)
    o2 = _rows2d(out)
    r2 = _rows2d(dres) if dres is not None else None
    _lib.check(_lib.load().u2_rmsnorm_bwd_bf16(x2.data_ptr(), gamma.data_ptr(), g2.data_ptr(), _ptr(r2), o2.data_ptr(),
                                               _ptr(dgamma), x2.shape[0], x2.shape[1], x2.stride(0), g2.stride(0),
                                               r2.stride(0) if r2 is not None else 0, o2.stride(0), eps, _stream()),
               "u2_rmsnorm_bwd_bf16")
    return out


def softmax_bwd(P: torch.Tensor, dP: torch.Tensor, dS: torch.Tensor, *, n0: int, H: int, S: int, n: int, p_strides,
                dp_strides, ds_strides, zero_pad_to: int = 0):
    _need_cuda(P, dP, dS)
    if P.dtype != BF16 or dP.dtype != F32 or dS.dtype != BF16:
        raise TypeError("softmax_bwd: P / dS bf16, dP fp32")
    d = _lib.SoftmaxBwdDesc()
    d.p_s0, d.p_s1, d.p_s2 = p_strides
    d.dp_s0, d.dp_s1, d.dp_s2 = dp_strides
    d.ds_s0, d.ds_s1, d.ds_s2 = ds_strides
    d.n0, d.H, d.S, d.n, d.zero_pad_to = n0, H, S, n, zero_pad_to
    _lib.check(_lib.load().u2_softmax_bwd_bf16(P.data_ptr(), dP.data_ptr(), dS.data_ptr(), C.byref(d), _stream()),
               "u2_softmax_bwd_bf16")
    return dS


def relbias_grad(dS: torch.Tensor, drel: torch.Tensor, *, n0: int, H: int, S: int, n: int, strides, rel_max: int = 512):
    _need_cuda(dS, drel)
    _lib.check(_lib.load().u2_relbias_grad_bf16(dS.data_ptr(), drel.data_ptr(), n0, H, S, n, strides[0], strides[1],
                                                strides[2], rel_max, _stream()), "u2_relbias_grad_bf16")
    return drel


def rowdot(a: torch.Tensor, c: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """a, c bf16 views [B, S, H, dh] (dh contiguous) -> fp32 [B, H, S] of sum_d a * c."""
    _need_cuda(a, c, out)
    B, S, H, dh = a.shape
    if out is None:
        out = torch.empty(B, H, S, device=a.device, dtype=F32)
    _lib.check(_lib.load().u2_rowdot_bf16(a.data_ptr(), c.data_ptr(), out.data_ptr(), B, S, H, dh, a.stride(0), a.stride(1),
                                          a.stride(2), c.stride(0), c.stride(1), c.stride(2), _stream()), "u2_rowdot_bf16")
    return out


def temporal_attention_bwd(qkv, dout, dqkv, *, B, C_, N, H, dh, scale, rel_bias=None, drel=None, rel_max=512):
    _need_cuda(qkv, dout, dqkv, rel_bias, drel)
    _lib.check(_lib.load().u2_temporal_attention_bwd_bf16(qkv.data_ptr(), dout.data_ptr(), dqkv.data_ptr(), B, C_, N, H, dh,
                                                          qkv.stride(-2), dout.stride(-2), dqkv.stride(-2), scale,
                                                          _ptr(rel_bias), _ptr(drel), rel_max, _stream()),
               "u2_temporal_attention_bwd_bf16")
    return dqkv


def rope_bwd(dx: torch.Tensor, x_raw: Optional[torch.Tensor], *, rows: int, ld: int, dh: int, n_q: int, n_k: int, inv_freq,
             q_norm_w=None, k_norm_w=None, eps: float = 1e-6, pos0: int = 0, pos_div: int = 1, pos_mod: int = 1,
             dq_norm_w=None, dk_norm_w=None):
    _need_cuda(dx, x_raw, inv_freq, q_norm_w, k_norm_w, dq_norm_w, dk_norm_w)
    d = _lib.RopeDesc()
    d.rows, d.ld, d.dh = rows, ld, dh
    d.n_q_heads, d.n_k_heads, d.n_v_heads = n_q, n_k, 0
    d.q_norm_w, d.k_norm_w, d.eps = _ptr(q_norm_w), _ptr(k_norm_w), eps
    d.inv_freq = inv_freq.data_ptr()
    d.pos0, d.pos_div, d.pos_mod = pos0, pos_div, pos_mod
    _lib.check(_lib.load().u2_rope_bwd_bf16(dx.data_ptr(), _ptr(x_raw), C.byref(d), _ptr(dq_norm_w), _ptr(dk_norm_w),
                                            _stream()), "u2_rope_bwd_bf16")
    return dx


def spp_pool_bwd(dy: torch.Tensor, dx: torch.Tensor, *, frames: int, grid, ps: int, E: int, in_frame_stride: int, in_off: int,
                 ldx: int, rows_per_frame: int, sequence: bool = False):
    _need_cuda(dy, dx)
    _lib.check(_lib.load().u2_spp_pool_bwd_bf16(dy.data_ptr(), dx.data_ptr(), frames, grid[0], grid[1], grid[2], ps, E,
                                                in_frame_stride, in_off, ldx, rows_per_frame, int(sequence), _stream()),
               "u2_spp_pool_bwd_bf16")
    return dx


def multiscale_pool_fwd(x: torch.Tensor, gate_w: Optional[torch.Tensor], dynamic: bool):
    """Forward that also returns the [B, 3] gate logits the backward needs (u2_multiscale_pool_bf16)."""
    _need_cuda(x, gate_w)
    B, K, E = x.shape
    x = x.contiguous()
    n_out = K + (K // 2 if K >= 2 else 0) + (K // 4 if K >= 4 else 0)
    out = torch.empty(B, n_out, E, device=x.device, dtype=BF16)
    ws = torch.zeros(int(_lib.load().u2_multiscale_pool_ws_elems(B, K)), device=x.device, dtype=F32)
    # gate_fc.bias shifts the three logits alike and cancels in the softmax over the scales: 0 is exact
    _lib.check(_lib.load().u2_multiscale_pool_bf16(x.data_ptr(), out.data_ptr(), _ptr(gate_w), 0.0, ws.data_ptr(), B, K, E,
                                                   int(dynamic), _stream()), "u2_multiscale_pool_bf16")
    return out, ws[:3 * B].view(B, 3)


def multiscale_pool_bwd(x, dy, gate_w, logits, dgate_w, dynamic: bool):
    _need_cuda(x, dy, gate_w, logits, dgate_w)
    B, K, E = x.shape
    dx = torch.empty_like(x)
    ws = torch.empty(B, 8, device=x.device, dtype=F32)
    _lib.check(_lib.load().u2_multiscale_pool_bwd_bf16(x.data_ptr(), dy.data_ptr(), dx.data_ptr(), _ptr(gate_w), _ptr(logits),
                                                       _ptr(dgate_w), ws.data_ptr(), B, K, E, int(dynamic), _stream()),
               "u2_multiscale_pool_bwd_bf16")
    return dx


def embed_scatter_add(ids: torch.Tensor, drows: torch.Tensor, dtable: Optional[torch.Tensor], dvis: Optional[torch.Tensor],
                      n_vis: int = 0):
    _need_cuda(ids, drows, dtable, dvis)
    ids = ids.long().contiguous()
    B, L = ids.shape
    E = drows.shape[-1]
    if not drows.is_contiguous():
        raise ValueError("embed_scatter_add expects contiguous row gradients")
    vocab = dtable.shape[0] if dtable is not None else 0
    _lib.check(_lib.load().u2_embed_scatter_add_bf16(ids.data_ptr(), drows.data_ptr(), _ptr(dtable), _ptr(dvis), B, L, E,
                                                     n_vis if dvis is not None else 0, vocab, _stream()),
               "u2_embed_scatter_add_bf16")


def group_sum(x: torch.Tensor, out: torch.Tensor, *, rows: int, heads: int, G: int, dh: int, ld_in: int, ld_out: int):
    _need_cuda(x, out)
    _lib.check(_lib.load().u2_group_sum_bf16(x.data_ptr(), out.data_ptr(), rows, heads, G, dh, ld_in, ld_out, _stream()),
               "u2_group_sum_bf16")
    return out


def ce_bwd(logits: torch.Tensor, lse: torch.Tensor, labels: torch.Tensor, coef: torch.Tensor,
           out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 logits [R, V] -> bf16 dlogits = coef[r] * (softmax - onehot(labels))."""
    _need_cuda(logits, lse, labels, coef, out)
    R, V = logits.shape
    if logits.dtype != F32 or logits.stride(1) != 1:
        raise TypeError("ce_bwd expects fp32 logits rows")
    if out is None:
        out = torch.empty(R, V, device=logits.device, dtype=BF16)
    _lib.check(_lib.load().u2_ce_bwd_f32_bf16(logits.data_ptr(), out.data_ptr(), lse.data_ptr(), labels.data_ptr(),
                                              coef.data_ptr(), R, V, logits.stride(0), out.stride(0), _stream()),
               "u2_ce_bwd_f32_bf16")
    return out


def dpo_loss(per_tok: torch.Tensor, ref_sum: torch.Tensor, mask: torch.Tensor, beta: float):
    """per_tok fp32 [2P, L], ref_sum fp32 [2P], mask uint8 [2P, L] -> (stats fp32 [3] = loss, accuracy, margin;
    coef fp32 [2P, L] = -dloss/dlogp)."""
    _need_cuda(per_tok, ref_sum, mask)
    P2, L = per_tok.shape
    out = torch.empty(3, device=per_tok.device, dtype=F32)
    coef = torch.empty(P2, L, device=per_tok.device, dtype=F32)
    _lib.check(_lib.load().u2_dpo_loss_f32(per_tok.data_ptr(), ref_sum.data_ptr(), mask.data_ptr(), out.data_ptr(),
                                           coef.data_ptr(), P2 // 2, L, beta, _stream()), "u2_dpo_loss_f32")
    return out, coef


def _adam_desc(lr, beta1, beta2, eps, weight_decay, step, grad_scale, seed, index_offset):
    d = _lib.AdamWDesc()
    d.lr, d.beta1, d.beta2, d.eps, d.weight_decay = lr, beta1, beta2, eps, weight_decay
    d.step = int(step)
    d.grad_scale = _ptr(grad_scale)
    d.seed = int(seed) & (2 ** 64 - 1)
    d.index_offset = int(index_offset)
    return d


def adamw(master, m, v, grad, param_out, *, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, step=1, grad_scale=None,
          param_out_f32=None, seed=0, index_offset=0):
    """Fused AdamW over a flat shard (torch.optim.AdamW semantics). grad bf16 -> u2_adamw_bf16, fp32 -> u2_adamw_f32grad;
    bf16 m / v -> u2_adamw_bf16_mom16, whose stochastic rounding of the moments draws from (seed, step, index_offset +
    element index)."""
    _need_cuda(master, m, v, grad, param_out, grad_scale, param_out_f32)
    n = master.numel()
    d = _adam_desc(lr, beta1, beta2, eps, weight_decay, step, grad_scale, seed, index_offset)
    lib = _lib.load()
    if grad.dtype == BF16 and m.dtype == BF16:
        _lib.check(lib.u2_adamw_bf16_mom16(master.data_ptr(), m.data_ptr(), v.data_ptr(), grad.data_ptr(), _ptr(param_out), n,
                                           C.byref(d), _stream()), "u2_adamw_bf16_mom16")
    elif grad.dtype == BF16:
        _lib.check(lib.u2_adamw_bf16(master.data_ptr(), m.data_ptr(), v.data_ptr(), grad.data_ptr(), _ptr(param_out), n,
                                     C.byref(d), _stream()), "u2_adamw_bf16")
    else:
        _lib.check(lib.u2_adamw_f32grad(master.data_ptr(), m.data_ptr(), v.data_ptr(), grad.data_ptr(), _ptr(param_out),
                                        _ptr(param_out_f32), n, C.byref(d), _stream()), "u2_adamw_f32grad")


def sumsq(x: torch.Tensor, out: torch.Tensor):
    _need_cuda(x, out)
    lib = _lib.load()
    if x.dtype == BF16:
        _lib.check(lib.u2_sumsq_bf16(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "u2_sumsq_bf16")
    else:
        _lib.check(lib.u2_sumsq_f32(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "u2_sumsq_f32")
    return out


def add_(dst: torch.Tensor, src: torch.Tensor) -> torch.Tensor:
    """dst += src (bf16, contiguous, same shape)."""
    _need_cuda(dst, src)
    if dst.shape != src.shape or not dst.is_contiguous() or not src.is_contiguous():
        raise ValueError("add_: contiguous tensors of the same shape")
    _lib.check(_lib.load().u2_add_bf16(dst.data_ptr(), src.data_ptr(), dst.numel(), _stream()), "u2_add_bf16")
    return dst


def cast(src: torch.Tensor, dst: torch.Tensor):
    """dtype plumbing between the flat buffers (bf16 <-> fp32)."""
    _need_cuda(src, dst)
    lib = _lib.load()
    if src.dtype == F32 and dst.dtype == BF16:
        _lib.check(lib.u2_cast_f32_bf16(src.data_ptr(), dst.data_ptr(), src.numel(), _stream()), "u2_cast_f32_bf16")
    elif src.dtype == BF16 and dst.dtype == F32:
        _lib.check(lib.u2_cast_bf16_f32(src.data_ptr(), dst.data_ptr(), src.numel(), _stream()), "u2_cast_bf16_f32")
    else:
        raise TypeError("cast: bf16 <-> fp32 only")
    return dst


# ------------------------------------------------------------------------------------------------
# linear-layer gradients on the wgmma GEMM (transposed operands, no transposed copies)
# ------------------------------------------------------------------------------------------------
def linear_dgrad(dy: torch.Tensor, w: torch.Tensor, out: Optional[torch.Tensor] = None, *, accumulate: bool = False,
                 alpha: float = 1.0) -> torch.Tensor:
    """dx [M, K] = dy [M, N] @ w [N, K]  (w stored [N, K]: the contraction index N is its row index -> MN-major B)."""
    dy2 = _rows2d(dy)
    M, N = dy2.shape
    K = w.shape[1]
    if out is None:
        out = torch.empty(M, K, device=dy.device, dtype=BF16)
    o2 = _rows2d(out)
    ops.gemm(dy2, w, o2, M=M, N=K, K=N, lda=dy2.stride(0), ldb=w.stride(0), ldc=o2.stride(0), b_mn=True, alpha=alpha,
             residual=o2 if accumulate else None, ldr=o2.stride(0) if accumulate else 0)
    return out


def linear_wgrad(dy: torch.Tensor, x: torch.Tensor, out: torch.Tensor, *, accumulate: bool = False) -> torch.Tensor:
    """dw [N, K] (+)= dy [M, N]^T @ x [M, K]  (both operands MN-major: the contraction index M is their row index)."""
    dy2, x2 = _rows2d(dy), _rows2d(x)
    M, N = dy2.shape
    K = x2.shape[1]
    ops.gemm(dy2, x2, out, M=N, N=K, K=M, lda=dy2.stride(0), ldb=x2.stride(0), ldc=out.stride(0), a_mn=True, b_mn=True,
             residual=out if accumulate else None, ldr=out.stride(0) if accumulate else 0)
    return out


# ------------------------------------------------------------------------------------------------
# LoRA adapters (csrc/lora.cu): the masked down-projection and its two masked gradients
# ------------------------------------------------------------------------------------------------
def _lora_desc(x2: torch.Tensor, u2: torch.Tensor, A: torch.Tensor, r: int, scale: float, p: float, seed: int, streams,
               accumulate: bool = False):
    M, K = x2.shape
    nA = A.shape[0] // r
    if A.shape != (nA * r, K) or not A.is_contiguous() or not 1 <= nA <= 3:
        raise ValueError(f"lora: A must be the contiguous stack [n_adapters * r, K] of 1-3 adapters, got {tuple(A.shape)}")
    if u2.shape != (M, nA * r) or u2.stride(1) != 1:
        raise ValueError(f"lora: U / dU must be [M, n_adapters * r] = [{M}, {nA * r}] with contiguous rows")
    if len(streams) != nA:
        raise ValueError("lora: one mask stream per adapter")
    d = _lib.LoraDesc()
    d.M, d.K, d.r, d.n_adapters = M, K, r, nA
    d.ldx, d.ldu = x2.stride(0), u2.stride(0)
    d.scale, d.p = float(scale), float(p)
    d.seed = int(seed) & (2 ** 64 - 1)
    for j, s_ in enumerate(streams):
        d.stream[j] = int(s_)
    d.accumulate = int(bool(accumulate))
    return d


def lora_down(x: torch.Tensor, A: torch.Tensor, r: int, scale: float, *, p: float = 0.0, seed: int = 0, streams=(0,),
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """U [M, n * r] = scale * (D_j o x) A_j^T for the n = A.shape[0] // r stacked adapters sharing x [M, K]."""
    _need_cuda(x, A, out)
    x2 = _rows2d(x)
    if out is None:
        out = torch.empty(x2.shape[0], A.shape[0], device=x.device, dtype=BF16)
    d = _lora_desc(x2, out, A, r, scale, p, seed, streams)
    _lib.check(_lib.load().u2_lora_down_bf16(x2.data_ptr(), A.data_ptr(), out.data_ptr(), C.byref(d), _stream()),
               "u2_lora_down_bf16")
    return out


def lora_wgrad(du: torch.Tensor, x: torch.Tensor, dA: torch.Tensor, r: int, scale: float, *, p: float = 0.0, seed: int = 0,
               streams=(0,), accumulate: bool = False) -> torch.Tensor:
    """dA_j (+)= scale * dU_j^T (D_j o x) into the stacked gradient dA [n * r, K]."""
    _need_cuda(du, x, dA)
    x2 = _rows2d(x)
    if not dA.is_contiguous():
        raise ValueError("lora_wgrad: dA must be contiguous")
    d = _lora_desc(x2, _rows2d(du), dA, r, scale, p, seed, streams, accumulate)
    _lib.check(_lib.load().u2_lora_wgrad_bf16(du.data_ptr(), x2.data_ptr(), dA.data_ptr(), C.byref(d), _stream()),
               "u2_lora_wgrad_bf16")
    return dA


def lora_dgrad(du: torch.Tensor, A: torch.Tensor, dx: torch.Tensor, r: int, scale: float, *, p: float = 0.0, seed: int = 0,
               streams=(0,)) -> torch.Tensor:
    """dx += sum_j D_j o (scale * dU_j A_j), in place."""
    _need_cuda(du, A, dx)
    dx2 = _rows2d(dx)
    d = _lora_desc(dx2, _rows2d(du), A, r, scale, p, seed, streams)
    _lib.check(_lib.load().u2_lora_dgrad_bf16(du.data_ptr(), A.data_ptr(), dx2.data_ptr(), C.byref(d), _stream()),
               "u2_lora_dgrad_bf16")
    return dx
