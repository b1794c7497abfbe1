"""Python-side operator wrappers: torch tensors in, C-ABI calls (libu2b200.so) underneath.

Every function here launches hand-written sm_90a kernels on the current torch CUDA stream; none
of them has a PyTorch fallback. Shapes/strides are validated here, arithmetic happens in csrc/.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import GemmDesc

BF16 = torch.bfloat16
F32 = torch.float32

ACT_NONE, ACT_GELU, ACT_SILU = 0, 1, 2
DT_BF16, DT_F32 = 0, 1


def _stream() -> int:
    # the device index is passed explicitly: without it torch.cuda.current_stream() re-resolves the current device
    # through its availability checks on every call, host time that the launch-bound training forward pays per kernel
    return torch.cuda.current_stream(torch.cuda.current_device()).cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need_cuda(*ts: torch.Tensor) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("u2tokenizer_b200 ops run on CUDA tensors only (no CPU fallback)")


def gemm(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, *, M: int, N: int, K: int,
         lda: int, ldb: int, ldc: int,
         zi: int = 1, zo: int = 1, b_zi_div: int = 1,
         a_strides=(0, 0), b_strides=(0, 0), c_strides=(0, 0),
         alpha: float = 1.0, bias: Optional[torch.Tensor] = None, act: int = ACT_NONE,
         residual: Optional[torch.Tensor] = None, ldr: int = 0, res_row_mod: int = 0,
         row_remap=(0, 0, 0), block_n: int = 0, a_mn: bool = False, b_mn: bool = False,
         epi_op: int = 0, rowvec: Optional[torch.Tensor] = None, rv_strides=(0, 0),
         mul: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Raw (batched, strided) GEMM: C[z] = act(alpha * A[z] @ B[z']^T + bias) + residual.
    a_mn / b_mn: the operand is stored transposed ([K][M] / [K][N], lda / ldb = stride between contraction indices)."""
    _need_cuda(a, b, c, bias, residual)
    if a.dtype != BF16 or b.dtype != BF16:
        raise TypeError("gemm operands must be bf16")
    if c.dtype not in (BF16, F32):
        raise TypeError("gemm output must be bf16 or fp32")
    if bias is not None and bias.dtype != F32:
        raise TypeError("gemm bias must be fp32")
    if residual is not None and residual.dtype != BF16:
        raise TypeError("gemm residual must be bf16")
    d = GemmDesc()
    d.M, d.N, d.K = M, N, K
    d.zi, d.zo, d.b_zi_div = zi, zo, b_zi_div
    d.lda, d.a_stride_zi, d.a_stride_zo = lda, a_strides[0], a_strides[1]
    d.ldb, d.b_stride_zi, d.b_stride_zo = ldb, b_strides[0], b_strides[1]
    d.ldc, d.c_stride_zi, d.c_stride_zo = ldc, c_strides[0], c_strides[1]
    d.c_dtype = DT_BF16 if c.dtype == BF16 else DT_F32
    d.alpha = alpha
    d.bias = _ptr(bias)
    d.act = act
    d.residual = _ptr(residual)
    d.ldr = ldr
    d.res_row_mod = res_row_mod
    d.row_div, d.row_stride, d.row_off = row_remap
    d.block_n = block_n
    d.a_mn, d.b_mn = int(a_mn), int(b_mn)
    _need_cuda(rowvec, mul)
    d.epi_op = int(epi_op)  # 1: exp(v - rowvec[row]); 2: mul * (v - rowvec[row])   (attention backward, see u2b200.h)
    d.rowvec = _ptr(rowvec)
    d.rv_stride_zi, d.rv_stride_zo = rv_strides
    d.mul = _ptr(mul)
    lib = _lib.load()
    if GEMM_TRACE is not None:   # tuning aid (tools/gemm_trace.py): per-call CUDA events keyed by shape / operand layout
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _lib.check(lib.u2_gemm_bf16(a.data_ptr(), b.data_ptr(), c.data_ptr(), C.byref(d), _stream()),
               "u2_gemm_bf16")
    if GEMM_TRACE is not None:
        e1.record()
        GEMM_TRACE.append(((M, N, K, zi * zo, int(a_mn), int(b_mn), "f32" if c.dtype == F32 else "bf16", int(bias is not None),
                            int(act), int(residual is not None), int(epi_op)), e0, e1))
    return c


GEMM_TRACE = None   # set to a list to record (key, start event, end event) per gemm() call


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
           act: int = ACT_NONE, residual: Optional[torch.Tensor] = None,
           out: Optional[torch.Tensor] = None, out_dtype: torch.dtype = BF16,
           alpha: float = 1.0, block_n: int = 0) -> torch.Tensor:
    """y = act(x @ w^T + bias) + residual for x [..., K] (last dim contiguous), w [N, K]."""
    K = x.shape[-1]
    N = w.shape[0]
    if w.shape[1] != K:
        raise ValueError(f"linear: weight {tuple(w.shape)} does not match input K={K}")
    x2 = x.reshape(-1, K)
    if x2.stride(1) != 1:
        x2 = x2.contiguous()
    if w.stride(1) != 1:
        w = w.contiguous()
    M = x2.shape[0]
    if out is None:
        out = torch.empty(*x.shape[:-1], N, device=x.device, dtype=out_dtype)
    o2 = out.view(-1, N) if out.is_contiguous() else out
    r2 = None
    ldr = 0
    if residual is not None:
        r2 = residual.reshape(-1, N)
        if r2.stride(1) != 1:
            r2 = r2.contiguous()
        ldr = r2.stride(0)
    gemm(x2, w, o2, M=M, N=N, K=K, lda=x2.stride(0), ldb=w.stride(0), ldc=o2.stride(0),
         alpha=alpha, bias=bias, act=act, residual=r2, ldr=ldr, block_n=block_n)
    return out


# ------------------------------------------------------------------------------------------------
# row-wise ops
# ------------------------------------------------------------------------------------------------
def _rows2d(t: torch.Tensor) -> torch.Tensor:
    t2 = t.reshape(-1, t.shape[-1]) if t.dim() != 2 else t
    if t2.stride(1) != 1:
        raise ValueError("last dim must be contiguous")
    return t2


def layernorm(x, gamma, beta, eps=1e-5, residual=None, out=None, sum_out=None):
    _need_cuda(x, gamma, beta, residual)
    x2 = _rows2d(x)
    if out is None:
        out = torch.empty_like(x2)
    o2 = _rows2d(out)
    r2 = _rows2d(residual) if residual is not None else None
    s2 = _rows2d(sum_out) if sum_out is not None else None
    if s2 is not None and s2.stride(0) != o2.stride(0):
        raise ValueError("sum_out must share out's row stride")
    _lib.check(_lib.load().u2_layernorm_bf16(x2.data_ptr(), _ptr(r2), gamma.data_ptr(), _ptr(beta), o2.data_ptr(),
                                             _ptr(s2), x2.shape[0], x2.shape[1], x2.stride(0),
                                             r2.stride(0) if r2 is not None else 0, o2.stride(0), eps, _stream()),
               "u2_layernorm_bf16")
    return out.view(x.shape) if out.numel() == x.numel() and out.is_contiguous() else out


def rmsnorm(x, gamma, eps=1e-6, residual=None, out=None, sum_out=None):
    _need_cuda(x, gamma, residual)
    x2 = _rows2d(x)
    if out is None:
        out = torch.empty_like(x2)
    o2 = _rows2d(out)
    r2 = _rows2d(residual) if residual is not None else None
    s2 = _rows2d(sum_out) if sum_out is not None else None
    if s2 is not None and s2.stride(0) != o2.stride(0):
        raise ValueError("sum_out must share out's row stride")
    _lib.check(_lib.load().u2_rmsnorm_bf16(x2.data_ptr(), _ptr(r2), gamma.data_ptr(), o2.data_ptr(), _ptr(s2),
                                           x2.shape[0], x2.shape[1], x2.stride(0),
                                           r2.stride(0) if r2 is not None else 0, o2.stride(0), eps, _stream()),
               "u2_rmsnorm_bf16")
    return out.view(x.shape) if out.numel() == x.numel() and out.is_contiguous() else out


def softmax(scores: torch.Tensor, out: torch.Tensor, *, n0: int, H: int, S: int, n: int,
            in_strides, out_strides, scale: float = 1.0, rel_bias: Optional[torch.Tensor] = None,
            rel_max: int = 0, causal: bool = False, causal_off: int = 0, zero_pad_to: int = 0, window: int = 0):
    """fp32 score rows -> bf16 probabilities (see u2_softmax_desc). window > 0 (causal only): key j of query i is
    visible iff i + causal_off - window < j <= i + causal_off (a sliding window; 0 = none)."""
    _need_cuda(scores, out, rel_bias)
    d = _lib.SoftmaxDesc()
    d.in_s0, d.in_s1, d.in_s2 = in_strides
    d.out_s0, d.out_s1, d.out_s2 = out_strides
    d.n0, d.H, d.S, d.n = n0, H, S, n
    d.scale = scale
    d.rel_bias = _ptr(rel_bias)
    d.rel_max = rel_max
    d.causal, d.causal_off = int(causal), causal_off
    d.zero_pad_to = zero_pad_to
    d.window = int(window or 0)
    _lib.check(_lib.load().u2_softmax_f32_bf16(scores.data_ptr(), out.data_ptr(), C.byref(d), _stream()),
               "u2_softmax_f32_bf16")
    return out


def silu_mul(gate_up: torch.Tensor, out: Optional[torch.Tensor] = None, interleaved: bool = False) -> torch.Tensor:
    _need_cuda(gate_up)
    g2 = _rows2d(gate_up)
    I = g2.shape[1] // 2
    if out is None:
        out = torch.empty(g2.shape[0], I, device=g2.device, dtype=BF16)
    _lib.check(_lib.load().u2_silu_mul_bf16(g2.data_ptr(), out.data_ptr(), g2.shape[0], I, g2.stride(0),
                                            out.stride(0), int(interleaved), _stream()), "u2_silu_mul_bf16")
    return out


# ------------------------------------------------------------------------------------------------
# layout ops
# ------------------------------------------------------------------------------------------------
def patchify(vol: torch.Tensor, patch_size, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """vol fp32 [F, D0, D1, D2] (single channel, contiguous) -> bf16 [F * n_patches, p0*p1*p2]."""
    _need_cuda(vol)
    if vol.dtype != F32 or not vol.is_contiguous():
        raise TypeError("patchify expects a contiguous fp32 volume")
    F_, d0, d1, d2 = vol.shape
    p0, p1, p2 = patch_size
    npatch = (d0 // p0) * (d1 // p1) * (d2 // p2)
    if out is None:
        out = torch.empty(F_ * npatch, p0 * p1 * p2, device=vol.device, dtype=BF16)
    _lib.check(_lib.load().u2_patchify_f32_bf16(vol.data_ptr(), out.data_ptr(), F_, d0, d1, d2, p0, p1, p2,
                                                _stream()), "u2_patchify_f32_bf16")
    return out


def patch_embed_supported(image_size, patch_size, hidden: int) -> bool:
    """Geometries the fused patch-embedding kernel covers (see u2_patch_embed_f32_bf16)."""
    d0, d1, d2 = image_size
    p0, p1, p2 = patch_size
    if d0 % p0 or d1 % p1 or d2 % p2:
        return False
    return p2 == 16 and d2 // p2 == 16 and p1 % 4 == 0 and (d1 // p1) % 8 == 0 and d2 <= 256 and hidden % 32 == 0


def patch_embed(vol: torch.Tensor, patch_size, w: torch.Tensor, bias: torch.Tensor, pos: torch.Tensor,
                out: torch.Tensor) -> torch.Tensor:
    """Fused gather + Linear + bias + position embedding: vol fp32 [F, D0, D1, D2] -> out bf16 [F, Sp, N] rows 1..P."""
    _need_cuda(vol, w, bias, pos, out)
    if vol.dtype != F32 or not vol.is_contiguous() or w.dtype != BF16 or bias.dtype != F32 or pos.dtype != BF16:
        raise TypeError("patch_embed: fp32 contiguous volume, bf16 weight / position table, fp32 bias")
    F_, d0, d1, d2 = vol.shape
    p0, p1, p2 = patch_size
    N = w.shape[0]
    if out.shape[0] != F_ or out.shape[2] != N or not out.is_contiguous() or not w.is_contiguous() or not pos.is_contiguous():
        raise ValueError("patch_embed: out must be contiguous [frames, rows, N]")
    _lib.check(_lib.load().u2_patch_embed_f32_bf16(vol.data_ptr(), w.data_ptr(), bias.data_ptr(), pos.data_ptr(), out.data_ptr(),
                                                   F_, d0, d1, d2, p0, p1, p2, N, out.shape[1], _stream()),
               "u2_patch_embed_f32_bf16")
    return out


def set_rows(dst: torch.Tensor, vec: torch.Tensor, n_rows: int, row_stride: int, row_off: int):
    _need_cuda(dst, vec)
    E = vec.numel()
    _lib.check(_lib.load().u2_set_rows_bf16(dst.data_ptr(), vec.data_ptr(), n_rows, row_stride, row_off, E,
                                            _stream()), "u2_set_rows_bf16")
    return dst


def vit_frame_rows(dst: torch.Tensor, cls: torch.Tensor, frames: int, Sp: int, S: int):
    """dst [frames, Sp, E]: cls row + zeroed padding rows (everything the patch-embed GEMM does not write)."""
    _need_cuda(dst, cls)
    _lib.check(_lib.load().u2_vit_frame_rows_bf16(dst.data_ptr(), cls.data_ptr(), frames, Sp, S, cls.numel(), _stream()),
               "u2_vit_frame_rows_bf16")
    return dst


def transpose_heads(x: torch.Tensor, out: torch.Tensor, *, B: int, S: int, H: int, Dh: int,
                    in_strides, out_strides, ld_out: int):
    """in[b][s][h][d] -> out[b][h][d][s(pad ld_out)]; strides in elements: in (sb, ss, sh), out (sb, sh)."""
    _need_cuda(x, out)
    _lib.check(_lib.load().u2_transpose_heads_bf16(x.data_ptr(), out.data_ptr(), B, S, H, Dh, in_strides[0],
                                                   in_strides[1], in_strides[2], out_strides[0], out_strides[1],
                                                   ld_out, _stream()), "u2_transpose_heads_bf16")
    return out


def spp_pool(x: torch.Tensor, out: torch.Tensor, *, frames: int, grid, ps: int, E: int,
             in_frame_stride: int, in_off: int, ldx: int, sequence: bool = False):
    _need_cuda(x, out)
    _lib.check(_lib.load().u2_spp_pool_bf16(x.data_ptr(), out.data_ptr(), frames, grid[0], grid[1], grid[2], ps, E,
                                            in_frame_stride, in_off, ldx, int(sequence), _stream()),
               "u2_spp_pool_bf16")
    return out


def multiscale_pool(x: torch.Tensor, gate_w: Optional[torch.Tensor], gate_bias: float, dynamic: bool) -> torch.Tensor:
    """x bf16 [B, K, E] -> [B, K + K//2 + K//4, E] (scales that do not fit are skipped)."""
    _need_cuda(x, gate_w)
    B, K, E = x.shape
    x = x.contiguous()
    n_out = K + (K // 2 if K >= 2 else 0) + (K // 4 if K >= 4 else 0)
    out = torch.empty(B, n_out, E, device=x.device, dtype=BF16)
    ws = torch.empty(int(_lib.load().u2_multiscale_pool_ws_elems(B, K)), device=x.device, dtype=F32)
    _lib.check(_lib.load().u2_multiscale_pool_bf16(x.data_ptr(), out.data_ptr(), _ptr(gate_w), gate_bias,
                                                   ws.data_ptr(), B, K, E, int(dynamic), _stream()),
               "u2_multiscale_pool_bf16")
    return out


def embed_splice(ids: torch.Tensor, table: torch.Tensor, vis: Optional[torch.Tensor],
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need_cuda(ids, table, vis)
    if ids.dtype != torch.int64:
        ids = ids.long()
    ids = ids.contiguous()
    B, L = ids.shape
    E = table.shape[1]
    n_vis = 0 if vis is None else vis.shape[1]
    if vis is not None:
        vis = vis.contiguous()
    if out is None:
        out = torch.empty(B, L, E, device=table.device, dtype=BF16)
    _lib.check(_lib.load().u2_embed_splice_bf16(ids.data_ptr(), table.data_ptr(), _ptr(vis), out.data_ptr(), B, L, E,
                                                n_vis, table.shape[0], _stream()), "u2_embed_splice_bf16")
    return out


# ------------------------------------------------------------------------------------------------
# small attention pieces
# ------------------------------------------------------------------------------------------------
def temporal_attention(qkv: torch.Tensor, out: torch.Tensor, *, B: int, C_: int, N: int, H: int, dh: int,
                       scale: float, rel_bias: Optional[torch.Tensor], rel_max: int = 512):
    _need_cuda(qkv, out, rel_bias)
    _lib.check(_lib.load().u2_temporal_attention_bf16(qkv.data_ptr(), out.data_ptr(), B, C_, N, H, dh,
                                                      qkv.stride(-2), out.stride(-2), scale, _ptr(rel_bias),
                                                      rel_max, _stream()), "u2_temporal_attention_bf16")
    return out


def rope(x: torch.Tensor, *, rows: int, ld: int, dh: int, n_q: int, n_k: int, n_v: int = 0,
         inv_freq: torch.Tensor, q_norm_w=None, k_norm_w=None, eps: float = 1e-6,
         pos0: int = 0, pos_div: int = 1, pos_mod: int = 1, pos0_dev=None,
         k_cache=None, v_cache=None, Tmax: int = 0, rows_per_batch: int = 1, pos0_per_batch: bool = False):
    """pos0_per_batch: pos0 = pos0_dev[row // rows_per_batch] (int32 [batch], one position per sequence)."""
    _need_cuda(x, inv_freq, q_norm_w, k_norm_w, k_cache, v_cache, pos0_dev)
    d = _lib.RopeDesc()
    d.rows, d.ld, d.dh = rows, ld, dh
    d.n_q_heads, d.n_k_heads, d.n_v_heads = n_q, n_k, n_v
    d.q_norm_w, d.k_norm_w, d.eps = _ptr(q_norm_w), _ptr(k_norm_w), eps
    d.inv_freq = inv_freq.data_ptr()
    d.pos0, d.pos_div, d.pos_mod = pos0, pos_div, pos_mod
    d.pos0_dev = _ptr(pos0_dev)
    d.k_cache, d.v_cache = _ptr(k_cache), _ptr(v_cache)
    d.Tmax, d.rows_per_batch = Tmax, rows_per_batch
    d.pos0_per_batch = 1 if pos0_per_batch else 0
    _lib.check(_lib.load().u2_rope_bf16(x.data_ptr(), C.byref(d), _stream()), "u2_rope_bf16")
    return x


def decode_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, out: torch.Tensor, *,
                     B: int, Hq: int, Hkv: int, dh: int, Tmax: int, T: int = 0, T_dev=None, ldq: int, ldo: int,
                     scale: float, T_per_seq: bool = False, kv_src: Optional[torch.Tensor] = None, window: int = 0):
    """T_per_seq: sequence b attends over T_dev[b] keys (int32 [B]).
    kv_src (beam search): int32 [B, >= Tmax]; key t of sequence b is read from cache row kv_src[b, t].
    window > 0: sliding window, sequence b attends over its last `window` keys only (u2_decode_attention_window_bf16)."""
    _need_cuda(q, k_cache, v_cache, out, T_dev, kv_src)
    _check_kv_src(kv_src, B, Tmax)
    if window:
        _lib.check(_lib.load().u2_decode_attention_window_bf16(
            q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), out.data_ptr(), B, Hq, Hkv, dh, Tmax, T, _ptr(T_dev),
            ldq, ldo, scale, 1 if T_per_seq else 0, _ptr(kv_src), kv_src.stride(0) if kv_src is not None else 0,
            int(window), _stream()), "u2_decode_attention_window_bf16")
        return out
    _lib.check(_lib.load().u2_decode_attention_bf16(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                                    out.data_ptr(), B, Hq, Hkv, dh, Tmax, T, _ptr(T_dev), ldq, ldo,
                                                    scale, 1 if T_per_seq else 0, _ptr(kv_src),
                                                    kv_src.stride(0) if kv_src is not None else 0, _stream()),
               "u2_decode_attention_bf16")
    return out


def _check_kv_src(kv_src: Optional[torch.Tensor], B: int, Tmax: int) -> None:
    if kv_src is not None and (kv_src.dtype != torch.int32 or kv_src.dim() != 2 or kv_src.shape[0] != B
                               or kv_src.shape[1] < Tmax or kv_src.stride(1) != 1):
        raise ValueError(f"kv_src must be int32 [{B}, >= {Tmax}] with unit column stride")


def gemv(x: torch.Tensor, w: torch.Tensor, out: torch.Tensor, *, residual=None, norm_gamma=None,
         norm_eps: float = 1e-6, silu_pair: bool = False):
    """Decode-step linear: x [B<=8, K] bf16, w [N, K] bf16 -> out [B, N or N/2] (bf16 or fp32)."""
    _need_cuda(x, w, out, residual, norm_gamma)
    d = _lib.GemvDesc()
    d.B, d.N, d.K = x.shape[0], w.shape[0], w.shape[1]
    d.ldx, d.ldw, d.ldy = x.stride(0), w.stride(0), out.stride(0)
    d.ldr = residual.stride(0) if residual is not None else 0
    d.y_dtype = DT_BF16 if out.dtype == BF16 else DT_F32
    d.residual = _ptr(residual)
    d.norm_gamma = _ptr(norm_gamma)
    d.norm_eps = norm_eps
    d.silu_pair = int(silu_pair)
    _lib.check(_lib.load().u2_gemv_bf16(x.data_ptr(), w.data_ptr(), out.data_ptr(), C.byref(d), _stream()),
               "u2_gemv_bf16")
    return out


_argmax_scratch = {}


def argmax(logits: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need_cuda(logits)
    B, V = logits.shape
    if out is None:
        out = torch.empty(B, device=logits.device, dtype=torch.int64)
    sc = _argmax_scratch.get(logits.device)
    if sc is None:
        sc = _argmax_scratch[logits.device] = torch.zeros(1024, device=logits.device, dtype=torch.int64)
    _lib.check(_lib.load().u2_argmax_f32(logits.data_ptr(), out.data_ptr(), sc.data_ptr(), B, V, logits.stride(0),
                                         _stream()), "u2_argmax_f32")
    return out


DLIN_W_BF16, DLIN_W_PACKED13 = 0, 1  # U2_DLIN_W_* of include/u2b200.h
DLIN_PACKED_UNIT_BYTES = 13328       # one packed 128 x 64 unit


class PackedWeight:
    """A decode-linear weight in the lossless 13-bit packing of u2_dlinear_pack_bf16: ``buf`` holds the units of the
    [N, K] bf16 matrix it was made from (uint8, ceil(N / 128) * K / 64 * 13 328 bytes)."""

    def __init__(self, buf: torch.Tensor, N: int, K: int):
        self.buf, self.N, self.K = buf, N, K

    @property
    def shape(self):
        return (self.N, self.K)


def dlinear_pack(w: torch.Tensor) -> Optional[PackedWeight]:
    """Pack a bf16 [N, K] weight (K % 64 == 0) for ops.dlinear / ops.dlinear_multi. Returns None when a 128 x 64 unit
    spans more than 31 nonzero exponents above its base (the matrix must then stay in bf16)."""
    _need_cuda(w)
    if w.dtype != BF16 or w.dim() != 2 or w.stride(1) != 1:
        raise ValueError("dlinear_pack: w must be a bf16 [N, K] matrix with unit column stride")
    N, K = w.shape
    buf = torch.empty(-(-N // 128) * (K // 64) * DLIN_PACKED_UNIT_BYTES, device=w.device, dtype=torch.uint8)
    bad = torch.zeros(1, device=w.device, dtype=torch.int32)
    _lib.check(_lib.load().u2_dlinear_pack_bf16(w.data_ptr(), N, K, w.stride(0), buf.data_ptr(), bad.data_ptr(),
                                                _stream()), "u2_dlinear_pack_bf16")
    return PackedWeight(buf, N, K) if int(bad.item()) == 0 else None


def _dlinear_w(w):
    """(data pointer, N, K, ldw, U2_DLIN_W_*) of a bf16 tensor or a PackedWeight."""
    if isinstance(w, PackedWeight):
        _need_cuda(w.buf)
        return w.buf.data_ptr(), w.N, w.K, w.K, DLIN_W_PACKED13
    _need_cuda(w)
    return w.data_ptr(), w.shape[0], w.shape[1], w.stride(0), DLIN_W_BF16


def _dlinear_desc(x, w, out, *, ws, counters, ssq_in=None, eps=1e-6, residual=None, silu_pair=False, gamma_next=None,
                  xg=None, ssq_out=None, ssq_zero=None, pdl=True, dbg=None, sched=0, dep_flags=None, dep_shift=1,
                  out_flags=None):
    _need_cuda(x, out, ws, counters, ssq_in, residual, gamma_next, xg, ssq_out, ssq_zero)
    d = _lib.DlinearDesc()
    _, d.N, d.K, d.ldw, d.w_format = _dlinear_w(w)
    d.B = x.shape[0]
    if counters.numel() < (d.N + 63) // 64 + (ssq_out is not None):
        raise ValueError("dlinear counters too small: ceil(N / 64) int32, + 1 with ssq_out")
    d.ws_elems = ws.numel()
    d.ldx, d.ldy = x.stride(0), out.stride(0)
    d.ldr = residual.stride(0) if residual is not None else 0
    d.ldxg = xg.stride(0) if xg is not None else 0
    d.y_dtype = DT_BF16 if out.dtype == BF16 else DT_F32
    d.ws, d.counters = ws.data_ptr(), counters.data_ptr()
    d.ssq_in = _ptr(ssq_in)
    d.eps = eps
    d.residual = _ptr(residual)
    d.silu_pair = int(silu_pair)
    d.gamma_next = _ptr(gamma_next)
    d.xg = _ptr(xg)
    d.ssq_out = _ptr(ssq_out)
    d.ssq_zero = _ptr(ssq_zero)
    d.pdl = int(pdl)
    d.dbg = _ptr(dbg)
    _need_cuda(dep_flags, out_flags)
    d.dep_flags, d.dep_shift, d.out_flags = _ptr(dep_flags), dep_shift, _ptr(out_flags)
    d.sched = int(sched)  # 0 = stream-K over 128-row tiles, 1 = whole 64-row tiles (no reduction)
    return d


def dlinear_ws_elems(N: int, K: int) -> int:
    """fp32 workspace elements the stream-K schedule needs for an N x K decode linear (needs a CUDA device)."""
    return int(_lib.load().u2_dlinear_ws_elems(N, K))


def dlinear_new_ws(n_elems: int, device="cuda", lead=()) -> torch.Tensor:
    """Workspace for the stream-K split-tile slots: fp32 view of all-ones words (the 'empty slot' sentinel)."""
    return torch.full((*lead, max(int(n_elems), 4)), -1, device=device, dtype=torch.int32).view(F32)


def dlinear(x: torch.Tensor, w, out: torch.Tensor, **kw):
    """Decode-step linear on wgmma (see u2_dlinear_desc): x [B<=16, K] bf16, w [N, K] bf16 or its PackedWeight."""
    d = _dlinear_desc(x, w, out, **kw)
    _lib.check(_lib.load().u2_dlinear_bf16(x.data_ptr(), _dlinear_w(w)[0], out.data_ptr(), C.byref(d), _stream()),
               "u2_dlinear_bf16")
    return out


def dlinear_multi(ops_list, *, gridbar: torch.Tensor, step_dev: torch.Tensor, pdl: bool = True,
                  lookahead_units: int = 0, next_weights=(), pre_stages: int = 0):
    """Several dependent decode linears in ONE launch. ops_list: [(x, w, out, kwargs), ...] (max 4); the weights are
    either all bf16 or all PackedWeight. next_weights: [(w, units_per_cta), ...] (max 2) to warm L2 for the next launch."""
    n = len(ops_list)
    descs = (_lib.DlinearDesc * n)()
    xs, ws_, ys = (C.c_void_p * n)(), (C.c_void_p * n)(), (C.c_void_p * n)()
    for i, (x, w, out, kw) in enumerate(ops_list):
        descs[i] = _dlinear_desc(x, w, out, **kw)
        xs[i], ws_[i], ys[i] = x.data_ptr(), _dlinear_w(w)[0], out.data_ptr()
    _need_cuda(gridbar, step_dev)
    nx = _lib.DlinearNext()
    nx.lookahead_units = lookahead_units
    nx.pre_stages = pre_stages
    nx.n = len(next_weights)
    for j, (wn, units) in enumerate(next_weights):
        nx.w[j], nx.N[j], nx.K[j], nx.ldw[j], nx.w_format[j] = _dlinear_w(wn)
        nx.units[j] = units
    _lib.check(_lib.load().u2_dlinear_multi_bf16(xs, ws_, ys, descs, n, gridbar.data_ptr(), step_dev.data_ptr(),
                                                 int(pdl), C.byref(nx), _stream()), "u2_dlinear_multi_bf16")


def decode_embed(ids: torch.Tensor, table: torch.Tensor, gamma: torch.Tensor, x: torch.Tensor, xg: torch.Tensor,
                 ssq: torch.Tensor, ssq_zero: Optional[torch.Tensor], step_counter: Optional[torch.Tensor] = None):
    _need_cuda(ids, table, gamma, x, xg, ssq, ssq_zero, step_counter)
    _lib.check(_lib.load().u2_decode_embed_bf16(ids.data_ptr(), table.data_ptr(), gamma.data_ptr(), x.data_ptr(),
                                                xg.data_ptr(), ssq.data_ptr(), _ptr(ssq_zero), _ptr(step_counter),
                                                ids.numel(),
                                                table.shape[1], table.shape[0], _stream()), "u2_decode_embed_bf16")
    return x


def decode_attention_fused(qkv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, out: torch.Tensor, *,
                           B: int, Hq: int, Hkv: int, dh: int, Tmax: int, inv_freq: torch.Tensor, scale: float,
                           pos: int = 0, pos_dev=None, q_norm_w=None, k_norm_w=None, eps: float = 1e-6, kv_splits: int = 1,
                           pdl: bool = False, pos_per_seq: bool = False, kv_src: Optional[torch.Tensor] = None,
                           window: int = 0):
    """q/k norm + RoPE + KV-cache append + GQA attention for one new token per sequence (one launch).
    window > 0: sliding window, the new token at position pos attends keys [max(0, pos - window + 1), pos] only.
    kv_splits in {2, 4, 8}: a cluster of that many CTAs per (sequence, KV head) splits the cached keys.
    pos_per_seq: sequence b's new token sits at position pos_dev[b] (int32 [B]) instead of pos_dev[0].
    kv_src (beam search): int32 [B, >= Tmax]; the cached key / value t < pos of sequence b is read from cache row
    kv_src[b, t] (the new token is appended to and read from row b). None: every sequence reads its own row."""
    _need_cuda(qkv, k_cache, v_cache, out, inv_freq, pos_dev, q_norm_w, k_norm_w, kv_src)
    _check_kv_src(kv_src, B, Tmax)
    d = _lib.FusedDecodeDesc()
    d.B, d.Hq, d.Hkv, d.dh, d.Tmax, d.pos = B, Hq, Hkv, dh, Tmax, pos
    d.pos_dev = _ptr(pos_dev)
    d.ldq, d.ldo = qkv.stride(0), out.stride(0)
    d.q_norm_w, d.k_norm_w, d.eps = _ptr(q_norm_w), _ptr(k_norm_w), eps
    d.inv_freq = inv_freq.data_ptr()
    d.scale = scale
    d.kv_splits = int(kv_splits)
    d.pdl = 1 if pdl else 0
    d.pos_per_seq = 1 if pos_per_seq else 0
    d.kv_src = _ptr(kv_src)
    d.ld_kv_src = kv_src.stride(0) if kv_src is not None else 0
    d.window = int(window or 0)
    _lib.check(_lib.load().u2_decode_attention_fused_bf16(qkv.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                                          out.data_ptr(), C.byref(d), _stream()),
               "u2_decode_attention_fused_bf16")
    return out


def topk_rows(scores: torch.Tensor, k: int, idx_offset_per_row: int = 0) -> torch.Tensor:
    """Indices of the k largest entries of every row of fp32 `scores` [rows, T], sorted descending."""
    _need_cuda(scores)
    if scores.dtype != F32 or scores.stride(1) != 1:
        raise TypeError("topk_rows expects fp32 rows")
    rows, T = scores.shape
    out = torch.empty(rows, k, device=scores.device, dtype=torch.int64)
    _lib.check(_lib.load().u2_topk_rows_f32(scores.data_ptr(), out.data_ptr(), rows, T, k, scores.stride(0),
                                            idx_offset_per_row, _stream()), "u2_topk_rows_f32")
    return out


def flash_attention_d64(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, scale: float,
                        lse: Optional[torch.Tensor] = None):
    """Fused non-causal attention for head_dim 64: q [B,Sq,H,64], k / v [B,Sk,H,64] (strided views, d contiguous: the
    slices of a fused QKV activation are consumed in place), out [B,Sq,H*64] view."""
    _need_cuda(q, k, v, out)
    B, Sq, H, dh = q.shape
    Sk = k.shape[1]
    if dh != 64 or q.stride(3) != 1 or k.stride(3) != 1 or v.stride(3) != 1 or out.stride(2) != 1 or v.shape != k.shape:
        raise ValueError("flash_attention_d64: head_dim must be 64 with a contiguous last dim, v shaped like k")
    d = _lib.FaDesc()
    d.B, d.H, d.Sq, d.Sk, d.dh, d.scale = B, H, Sq, Sk, dh, scale
    d.q_sb, d.q_ss, d.q_sh = q.stride(0), q.stride(1), q.stride(2)
    d.k_sb, d.k_ss, d.k_sh = k.stride(0), k.stride(1), k.stride(2)
    d.v_sb, d.v_ss, d.v_sh = v.stride(0), v.stride(1), v.stride(2)
    d.out_sb, d.out_ss = out.stride(0), out.stride(1)
    _need_cuda(lse)
    if lse is not None and (lse.dtype != F32 or not lse.is_contiguous() or lse.numel() != B * H * Sq):
        raise ValueError("flash_attention_d64: lse must be contiguous fp32 [B, H, Sq]")
    d.lse = _ptr(lse)
    _lib.check(_lib.load().u2_flash_attention_d64_bf16(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(),
                                                       C.byref(d), _stream()), "u2_flash_attention_d64_bf16")
    return out


def sample(logits: torch.Tensor, out: Optional[torch.Tensor] = None, *, temperature: float = 1.0, top_k: int = 50,
           top_p: float = 1.0, seed: int = 0, step: int = 0, step_dev=None) -> torch.Tensor:
    """ids ~ multinomial(top_p(top_k(softmax(logits / temperature)))) per row (HF sampling warper chain)."""
    _need_cuda(logits, step_dev)
    B, V = logits.shape
    if out is None:
        out = torch.empty(B, device=logits.device, dtype=torch.int64)
    _lib.check(_lib.load().u2_sample_f32(logits.data_ptr(), out.data_ptr(), B, V, logits.stride(0), temperature,
                                         int(top_k), float(top_p), int(seed) & ((1 << 64) - 1), _ptr(step_dev),
                                         int(step), _stream()), "u2_sample_f32")
    return out


def sample_params(device, temperature: float, top_k: int, top_p: float, seed: int,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The 24-byte u2_sample_params block (include/u2b200.h) in device memory: temperature f32, top_k i32, top_p f32,
    pad, seed u64. `out` (a block made earlier) is overwritten in place, which is how a captured decode graph gets new
    sampling parameters without a new capture."""
    import struct
    if not temperature > 0:
        raise ValueError("sample: temperature must be > 0")
    if not 0 < top_p <= 1:
        raise ValueError("sample: top_p must be in (0, 1]")
    raw = struct.pack("<fifiQ", float(temperature), int(top_k), float(top_p), 0, int(seed) & ((1 << 64) - 1))
    host = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
    if out is None:
        return host.to(device)
    out.copy_(host)
    return out


def sample_dev(logits: torch.Tensor, params: torch.Tensor, out: Optional[torch.Tensor] = None, *, step: int = 0,
               step_dev=None) -> torch.Tensor:
    """ops.sample with the parameters read from a device block made by sample_params()."""
    _need_cuda(logits, params, step_dev)
    B, V = logits.shape
    if params.dtype != torch.uint8 or params.numel() != 24:
        raise ValueError("sample_dev: params must be the 24-byte block of sample_params()")
    if out is None:
        out = torch.empty(B, device=logits.device, dtype=torch.int64)
    _lib.check(_lib.load().u2_sample_dev_f32(logits.data_ptr(), out.data_ptr(), B, V, logits.stride(0), params.data_ptr(),
                                             _ptr(step_dev), int(step), _stream()), "u2_sample_dev_f32")
    return out


def logits_proc_params(device, vocab_size: int, *, repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0,
                       min_new_tokens: int = 0, eos_token_ids=(), bad_words_ids=(),
                       out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The u2_logits_proc_params block (include/u2b200.h) in device memory, as uint8. `out` (a block made earlier) is
    overwritten in place, so a captured decode graph gets a new request's processors without a new capture.
    Raises ValueError for values the kernel cannot take (over capacity, token ids outside [0, vocab_size))."""
    import numpy as np
    p = float(repetition_penalty)
    if not p > 0:
        raise ValueError(f"repetition_penalty must be > 0, got {repetition_penalty}")
    n, k = int(no_repeat_ngram_size), int(min_new_tokens)
    if n < 0 or k < 0:
        raise ValueError("no_repeat_ngram_size and min_new_tokens must be >= 0")
    eos = [int(e) for e in eos_token_ids]
    words = [[int(x) for x in w] for w in bad_words_ids]
    if len(eos) > _lib.LP_MAX_EOS:
        raise ValueError(f"at most {_lib.LP_MAX_EOS} EOS ids, got {len(eos)}")
    if len(words) > _lib.LP_MAX_BAD_WORDS or sum(map(len, words)) > _lib.LP_MAX_BAD_TOKENS:
        raise ValueError(f"bad_words_ids holds at most {_lib.LP_MAX_BAD_WORDS} words of "
                         f"{_lib.LP_MAX_BAD_TOKENS} tokens in all")
    if any(len(w) == 0 for w in words):
        raise ValueError("bad_words_ids: every word needs at least one token")
    bad = [v for v in eos + [x for w in words for x in w] if not 0 <= v < vocab_size]
    if bad:
        raise ValueError(f"token ids {bad} outside the vocabulary [0, {vocab_size})")
    blk = _lib.LogitsProcParams()
    blk.penalty = p
    blk.inv_penalty = float(np.float32(1.0) / np.float32(p))  # fp32 reciprocal of the fp32 penalty, as torch on CUDA
    blk.ngram, blk.min_new, blk.n_eos, blk.n_bad = n, k, len(eos), len(words)
    for i, e in enumerate(eos):
        blk.eos[i] = e
    off = 0
    for i, w in enumerate(words):
        blk.bad_off[i] = off
        for x in w:
            blk.bad_tok[off] = x
            off += 1
    blk.bad_off[len(words)] = off
    host = torch.frombuffer(bytearray(bytes(blk)), dtype=torch.uint8)
    if out is None:
        return host.to(device)
    out.copy_(host)
    return out


def logits_process(logits: torch.Tensor, params: torch.Tensor, ids: torch.Tensor, hist: torch.Tensor, *,
                   step: int = 0, step_dev=None) -> torch.Tensor:
    """HF's repetition penalty -> no-repeat n-gram -> bad words -> min new tokens, in place on fp32 logits [B, V].
    ids [B] int64: the token fed to this step, appended to the history hist [B, cap] int32 at column t - 1 where
    t = *step_dev (or step) is the number of generated tokens. params: a block made by logits_proc_params()."""
    _need_cuda(logits, params, ids, hist, step_dev)
    B, V = logits.shape
    if logits.dtype != F32 or logits.stride(1) != 1:
        raise TypeError("logits_process: logits must be fp32 with unit column stride")
    if params.dtype != torch.uint8 or params.numel() != C.sizeof(_lib.LogitsProcParams):
        raise ValueError("logits_process: params must be the block of logits_proc_params()")
    if ids.dtype != torch.int64 or ids.numel() != B or not ids.is_contiguous():
        raise ValueError("logits_process: ids must be contiguous int64 [B]")
    if hist.dtype != torch.int32 or hist.dim() != 2 or hist.shape[0] != B or hist.stride(1) != 1:
        raise ValueError("logits_process: hist must be int32 [B, cap] with unit column stride")
    if step_dev is None and not 0 <= step <= hist.shape[1]:
        raise ValueError(f"logits_process: step {step} outside the history capacity {hist.shape[1]}")
    _lib.check(_lib.load().u2_logits_process_f32(logits.data_ptr(), B, V, logits.stride(0), ids.data_ptr(),
                                                 hist.data_ptr(), hist.stride(0), hist.shape[1], params.data_ptr(),
                                                 _ptr(step_dev), int(step), _stream()), "u2_logits_process_f32")
    return logits


SLOT_STATE_BYTES = C.sizeof(_lib.SlotState)


def slot_state(seeds, rows, max_new, counts=None, done=None) -> torch.Tensor:
    """u2_slot_state records (include/u2b200.h) for len(seeds) decode rows, as a CPU uint8 tensor [rows, 24]: per row
    the request's seed, its RNG row, its generated count (default 0), its max_new_tokens and its done flag (default 0)."""
    n = len(seeds)
    recs = (_lib.SlotState * n)()
    for i in range(n):
        recs[i].seed = int(seeds[i]) & ((1 << 64) - 1)
        recs[i].row, recs[i].max_new = int(rows[i]), int(max_new[i])
        recs[i].count = 0 if counts is None else int(counts[i])
        recs[i].done = 0 if done is None else int(done[i])
    return torch.frombuffer(bytearray(bytes(recs)), dtype=torch.uint8).view(n, SLOT_STATE_BYTES)


def slot_state_fields(state: torch.Tensor) -> dict:
    """The count / done / row / max_new columns of slot_state() records (any device), as int32 tensors [rows]."""
    w = state.view(torch.int32).view(-1, SLOT_STATE_BYTES // 4)
    return dict(row=w[:, 2], count=w[:, 3], max_new=w[:, 4], done=w[:, 5])


def _check_slots(slots: torch.Tensor, B: int):
    if slots.dtype != torch.uint8 or tuple(slots.shape) != (B, SLOT_STATE_BYTES) or not slots.is_contiguous():
        raise ValueError(f"slots must be the contiguous uint8 [{B}, {SLOT_STATE_BYTES}] records of slot_state()")


def slot_params(device, pad_token_id: int, eos_token_ids=(), out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The u2_slot_params block (include/u2b200.h) in device memory, as uint8: the id a finished slot feeds and the EOS
    ids that finish a slot. `out` (a block made earlier) is overwritten in place, as for sample_params()."""
    eos = [int(e) for e in eos_token_ids]
    if len(eos) > _lib.LP_MAX_EOS:
        raise ValueError(f"at most {_lib.LP_MAX_EOS} EOS ids, got {len(eos)}")
    blk = _lib.SlotParams()
    blk.pad, blk.n_eos = int(pad_token_id), len(eos)
    for i, e in enumerate(eos):
        blk.eos[i] = e
    host = torch.frombuffer(bytearray(bytes(blk)), dtype=torch.uint8)
    if out is None:
        return host.to(device)
    out.copy_(host)
    return out


def sample_slots(logits: torch.Tensor, params: torch.Tensor, slots: torch.Tensor,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """sample_dev() with the seed, RNG row and step of row b read from the slot record slots[b]."""
    _need_cuda(logits, params, slots)
    B, V = logits.shape
    if params.dtype != torch.uint8 or params.numel() != 24:
        raise ValueError("sample_slots: params must be the 24-byte block of sample_params()")
    _check_slots(slots, B)
    if out is None:
        out = torch.empty(B, device=logits.device, dtype=torch.int64)
    _lib.check(_lib.load().u2_sample_slots_f32(logits.data_ptr(), out.data_ptr(), B, V, logits.stride(0),
                                               params.data_ptr(), slots.data_ptr(), _stream()), "u2_sample_slots_f32")
    return out


def logits_process_slots(logits: torch.Tensor, params: torch.Tensor, ids: torch.Tensor, hist: torch.Tensor,
                         slots: torch.Tensor) -> torch.Tensor:
    """logits_process() with the history length of row b read from the slot record slots[b] (its generated count)."""
    _need_cuda(logits, params, ids, hist, slots)
    B, V = logits.shape
    if logits.dtype != F32 or logits.stride(1) != 1:
        raise TypeError("logits_process_slots: logits must be fp32 with unit column stride")
    if params.dtype != torch.uint8 or params.numel() != C.sizeof(_lib.LogitsProcParams):
        raise ValueError("logits_process_slots: params must be the block of logits_proc_params()")
    if ids.dtype != torch.int64 or ids.numel() != B or not ids.is_contiguous():
        raise ValueError("logits_process_slots: ids must be contiguous int64 [B]")
    if hist.dtype != torch.int32 or hist.dim() != 2 or hist.shape[0] != B or hist.stride(1) != 1:
        raise ValueError("logits_process_slots: hist must be int32 [B, cap] with unit column stride")
    _check_slots(slots, B)
    _lib.check(_lib.load().u2_logits_process_slots_f32(logits.data_ptr(), B, V, logits.stride(0), ids.data_ptr(),
                                                       hist.data_ptr(), hist.stride(0), hist.shape[1],
                                                       params.data_ptr(), slots.data_ptr(), _stream()),
               "u2_logits_process_slots_f32")
    return logits


def slot_update(ids: torch.Tensor, slots: torch.Tensor, out: torch.Tensor, params: torch.Tensor,
                length: Optional[torch.Tensor] = None, length_plus1: Optional[torch.Tensor] = None,
                lp: Optional[tuple] = None) -> None:
    """Slot bookkeeping after a pick (u2_slot_update): every decoding slot appends ids[b] to out[b] at its count,
    counts it, finishes on an EOS id or max_new_tokens and, when the cache lengths are given, advances them; every
    finished slot gets ids[b] = pad. ids int64 [B] (contiguous), out int64 [B, width], params: slot_params().
    lp (optional): (the step's log-probs fp32 [B], fp32 [B, width] like out): each live slot also appends its
    log-prob (u2_slot_update_lp)."""
    _need_cuda(ids, slots, out, params, length, length_plus1)
    B = ids.numel()
    if ids.dtype != torch.int64 or not ids.is_contiguous():
        raise ValueError("slot_update: ids must be contiguous int64 [B]")
    _check_slots(slots, B)
    if out.dtype != torch.int64 or out.dim() != 2 or out.shape[0] != B or out.stride(1) != 1:
        raise ValueError("slot_update: out must be int64 [B, width] with unit column stride")
    if params.dtype != torch.uint8 or params.numel() != C.sizeof(_lib.SlotParams):
        raise ValueError("slot_update: params must be the block of slot_params()")
    for t in (length, length_plus1):
        if t is not None and (t.dtype != torch.int32 or t.numel() != B or not t.is_contiguous()):
            raise ValueError("slot_update: length / length_plus1 must be contiguous int32 [B]")
    if lp is None:
        _lib.check(_lib.load().u2_slot_update(ids.data_ptr(), B, slots.data_ptr(), out.data_ptr(), out.stride(0),
                                              params.data_ptr(), _ptr(length), _ptr(length_plus1), _stream()),
                   "u2_slot_update")
        return
    lp_in, lp_out = lp
    _need_cuda(lp_in, lp_out)
    if lp_in.dtype != F32 or lp_in.numel() != B or not lp_in.is_contiguous():
        raise ValueError("slot_update: the step's log-probs must be contiguous fp32 [B]")
    if lp_out.dtype != F32 or lp_out.shape != out.shape or lp_out.stride() != out.stride():
        raise ValueError("slot_update: the log-prob rows must be fp32 shaped and strided like out")
    _lib.check(_lib.load().u2_slot_update_lp(ids.data_ptr(), B, slots.data_ptr(), out.data_ptr(), out.stride(0),
                                             lp_in.data_ptr(), lp_out.data_ptr(), params.data_ptr(), _ptr(length),
                                             _ptr(length_plus1), _stream()), "u2_slot_update_lp")


def row_store_params(device, dst_ptr: int, ld_step: int, ld_row: int, steps: int,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The u2_row_store_params block (include/u2b200.h) in device memory, as uint8: row r of step t goes to the fp32
    element dst_ptr + t * ld_step + r * ld_row (in elements), for 0 <= t < steps. `out` (a block made earlier) is
    overwritten in place, so a captured decode step stores into a new call's buffer without a new capture."""
    blk = _lib.RowStoreParams()
    blk.dst, blk.ld_step, blk.ld_row, blk.steps = int(dst_ptr), int(ld_step), int(ld_row), int(steps)
    host = torch.frombuffer(bytearray(bytes(blk)), dtype=torch.uint8)
    if out is None:
        return host.to(device)
    out.copy_(host)
    return out


def row_store_dst(buf: torch.Tensor) -> dict:
    """row_store_params() arguments that store step t's rows into buf[t] of an fp32 [steps, rows, V] view (unit column
    stride)."""
    if buf.dtype != F32 or buf.dim() != 3 or buf.stride(2) != 1 or not buf.is_cuda:
        raise ValueError("row store: the destination must be a CUDA fp32 [steps, rows, V] view with unit column stride")
    return dict(dst_ptr=buf.data_ptr(), ld_step=buf.stride(0), ld_row=buf.stride(1), steps=buf.shape[0])


def _check_row_store(params: Optional[torch.Tensor]):
    if params is not None and (params.dtype != torch.uint8 or params.numel() != C.sizeof(_lib.RowStoreParams)):
        raise ValueError("params must be the block of row_store_params()")


def store_rows(src: torch.Tensor, params: torch.Tensor, *, step: int = 0, step_dev=None) -> None:
    """Copies fp32 src [rows, V] to the rows of step t = *step_dev (or step) of the row_store_params() destination."""
    _need_cuda(src, params, step_dev)
    if src.dtype != F32 or src.dim() != 2 or src.stride(1) != 1:
        raise TypeError("store_rows: src must be fp32 [rows, V] with unit column stride")
    _check_row_store(params)
    _lib.check(_lib.load().u2_store_rows_f32(src.data_ptr(), src.shape[0], src.shape[1], src.stride(0),
                                             params.data_ptr(), _ptr(step_dev), int(step), _stream()),
               "u2_store_rows_f32")


def sample_out(logits: torch.Tensor, params: torch.Tensor, out: torch.Tensor, *, scores: Optional[torch.Tensor] = None,
               logprob: Optional[torch.Tensor] = None, step: int = 0, step_dev=None,
               slots: Optional[torch.Tensor] = None) -> torch.Tensor:
    """sample_dev() (or sample_slots() when `slots` is given) with the same draw, that also writes the warped scores row
    into the row_store_params() destination `scores` and the pick's log-prob into logprob fp32 [B], each when given."""
    _need_cuda(logits, params, out, scores, logprob, step_dev, slots)
    B, V = logits.shape
    if params.dtype != torch.uint8 or params.numel() != 24:
        raise ValueError("sample_out: params must be the 24-byte block of sample_params()")
    _check_row_store(scores)
    if slots is not None:
        _check_slots(slots, B)
    if logprob is not None and (logprob.dtype != F32 or logprob.numel() != B or not logprob.is_contiguous()):
        raise ValueError("sample_out: logprob must be contiguous fp32 [B]")
    _lib.check(_lib.load().u2_sample_out_f32(logits.data_ptr(), out.data_ptr(), B, V, logits.stride(0),
                                             params.data_ptr(), _ptr(step_dev), int(step), _ptr(slots), _ptr(scores),
                                             _ptr(logprob), _stream()), "u2_sample_out_f32")
    return out


def pick_logprob(logits: torch.Tensor, ids: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[b] = log_softmax(logits[b])[ids[b]], fp32 [B]."""
    _need_cuda(logits, ids, out)
    B, V = logits.shape
    if logits.dtype != F32 or logits.stride(1) != 1:
        raise TypeError("pick_logprob: logits must be fp32 with unit column stride")
    if ids.dtype != torch.int64 or ids.numel() != B or not ids.is_contiguous():
        raise ValueError("pick_logprob: ids must be contiguous int64 [B]")
    if out is None:
        out = torch.empty(B, device=logits.device, dtype=F32)
    if out.dtype != F32 or out.numel() != B or not out.is_contiguous():
        raise ValueError("pick_logprob: out must be contiguous fp32 [B]")
    _lib.check(_lib.load().u2_pick_logprob_f32(logits.data_ptr(), B, V, logits.stride(0), ids.data_ptr(),
                                               out.data_ptr(), _stream()), "u2_pick_logprob_f32")
    return out


def log_softmax(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Row-wise log_softmax of fp32 [rows, V] into `out` (a separate fp32 buffer)."""
    _need_cuda(x, out)
    if x.dtype != F32 or x.dim() != 2 or x.stride(1) != 1:
        raise TypeError("log_softmax expects fp32 rows with unit column stride")
    if out is None:
        out = torch.empty_like(x)
    if out.dtype != F32 or out.shape != x.shape or out.stride(1) != 1:
        raise ValueError("log_softmax: out must be fp32 shaped like x")
    _lib.check(_lib.load().u2_log_softmax_f32(x.data_ptr(), out.data_ptr(), x.shape[0], x.shape[1], x.stride(0),
                                              out.stride(0), _stream()), "u2_log_softmax_f32")
    return out


EARLY_STOPPING = {False: 0, True: 1, "never": 2}


def beam_params(device, *, num_beams: int, length_penalty: float = 1.0, early_stopping=False, max_new_tokens: int,
                eos_token_ids=(), out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The u2_beam_params block (include/u2b200.h) in device memory, as uint8. `out` (a block made earlier) is overwritten
    in place, so a captured decode graph gets a new request's values without a new capture. beams_to_keep is HF's
    max(2, 1 + n_eos) * num_beams."""
    K, eos = int(num_beams), [int(e) for e in eos_token_ids]
    if not 2 <= K <= _lib.BEAM_MAX_BEAMS:
        raise ValueError(f"num_beams must be in 2..{_lib.BEAM_MAX_BEAMS}, got {num_beams}")
    if len(eos) > _lib.BEAM_MAX_EOS:
        raise ValueError(f"beam search supports at most {_lib.BEAM_MAX_EOS} EOS ids, got {len(eos)}")
    if not (early_stopping is True or early_stopping is False or early_stopping == "never"):
        raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")
    if int(max_new_tokens) < 1:
        raise ValueError("max_new_tokens must be >= 1")
    blk = _lib.BeamParams()
    blk.length_penalty = float(length_penalty)
    blk.num_beams, blk.beams_to_keep = K, max(2, 1 + len(eos)) * K
    blk.early_stopping, blk.max_new_tokens, blk.n_eos = EARLY_STOPPING[early_stopping], int(max_new_tokens), len(eos)
    for i, e in enumerate(eos):
        blk.eos[i] = e
    host = torch.frombuffer(bytearray(bytes(blk)), dtype=torch.uint8)
    if out is None:
        return host.to(device)
    out.copy_(host)
    return out


def beam_topk(logprobs: torch.Tensor, running: torch.Tensor, flags: torch.Tensor, params: torch.Tensor,
              cand_val: torch.Tensor, cand_tok: torch.Tensor):
    """Per row, the top beams_to_keep of logprobs[r] + running[r] into cand_val / cand_tok [rows, BEAM_MAX_KEEP]."""
    _need_cuda(logprobs, running, flags, params, cand_val, cand_tok)
    R, V = logprobs.shape
    if logprobs.dtype != F32 or logprobs.stride(1) != 1:
        raise TypeError("beam_topk: fp32 log-probs with unit column stride")
    if cand_val.shape != (R, _lib.BEAM_MAX_KEEP) or cand_tok.shape != (R, _lib.BEAM_MAX_KEEP):
        raise ValueError(f"beam_topk: candidates must be [{R}, {_lib.BEAM_MAX_KEEP}]")
    _lib.check(_lib.load().u2_beam_topk_f32(logprobs.data_ptr(), logprobs.stride(0), R, V, running.data_ptr(),
                                            flags.data_ptr(), params.data_ptr(), cand_val.data_ptr(),
                                            cand_tok.data_ptr(), _stream()), "u2_beam_topk_f32")


def beam_step(params: torch.Tensor, st: dict, ids: torch.Tensor, kv_src: torch.Tensor, pos_dev: torch.Tensor, *,
              V: int, hist: Optional[torch.Tensor] = None, step: int = 0, step_dev=None):
    """One CTA per prompt: merge the row candidates, update the beam state `st` (tensors 'cand_val', 'cand_tok',
    'running', 'fin_score', 'fin_info', 'flags', 'rec'; see u2_beam_step_desc) and write the next ids [rows] int64,
    the reordered kv_src and (optional) processor history."""
    d = _lib.BeamStepDesc()
    d.params = params.data_ptr()
    d.prompts, d.V = st["flags"].shape[0], int(V)
    for k in ("cand_val", "cand_tok", "running", "fin_score", "fin_info", "flags"):
        _need_cuda(st[k])
        setattr(d, k, st[k].data_ptr())
    _need_cuda(ids, kv_src, pos_dev, hist, step_dev)
    if ids.dtype != torch.int64 or kv_src.dtype != torch.int32 or not kv_src.is_contiguous():
        raise ValueError("beam_step: ids int64, kv_src contiguous int32")
    d.ids = ids.data_ptr()
    d.rec, d.ld_rec, d.rec_rows = st["rec"].data_ptr(), st["rec"].stride(0), st["rec"].shape[0]
    d.kv_src, d.ld_kv_src = kv_src.data_ptr(), kv_src.stride(0)
    d.pos_dev = pos_dev.data_ptr()
    if hist is not None:
        d.hist, d.ld_hist, d.hist_cap = hist.data_ptr(), hist.stride(0), hist.shape[1]
    d.step_dev = _ptr(step_dev)
    _lib.check(_lib.load().u2_beam_step(C.byref(d), int(step), _stream()), "u2_beam_step")


def lmhead_logprob(hidden: torch.Tensor, weight: torch.Tensor, labels: torch.Tensor, *, want_lse: bool = False,
                   want_logit_sum: bool = False, nll_acc: Optional[torch.Tensor] = None, ws: Optional[torch.Tensor] = None):
    """logp[r] = log_softmax(hidden[r] @ weight.T)[labels[r]] (0 where labels[r] < 0) without materialising the logits.
    hidden [R, E] bf16, weight [V, E] bf16, labels [R] int64. Returns (logp fp32 [R], lse or None, logit_sum or None).
    nll_acc: optional fp32 [2] accumulator (+= sum(-logp), += number of labelled rows)."""
    _need_cuda(hidden, weight, labels, nll_acc, ws)
    R, E = hidden.shape
    V = weight.shape[0]
    if hidden.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16 or labels.dtype != torch.int64:
        raise TypeError("lmhead_logprob: hidden / weight must be bf16, labels int64")
    if weight.shape[1] != E or labels.shape != (R,) or hidden.stride(1) != 1 or weight.stride(1) != 1 or not labels.is_contiguous():
        raise ValueError("lmhead_logprob: shape / stride mismatch")
    lib = _lib.load()
    need = int(lib.u2_logprob_ws_bytes(R, V))
    if ws is None:
        ws = torch.empty(need, device=hidden.device, dtype=torch.uint8)
    elif ws.numel() * ws.element_size() < need:
        raise ValueError(f"lmhead_logprob: workspace of {need} bytes required")
    logp = torch.empty(R, device=hidden.device, dtype=torch.float32)
    lse = torch.empty(R, device=hidden.device, dtype=torch.float32) if want_lse else None
    lsum = torch.empty(R, device=hidden.device, dtype=torch.float32) if want_logit_sum else None
    d = _lib.LogprobDesc()
    d.R, d.V, d.E, d.ldh, d.ldw = R, V, E, hidden.stride(0), weight.stride(0)
    d.labels, d.ws, d.ws_bytes = labels.data_ptr(), ws.data_ptr(), ws.numel() * ws.element_size()
    d.lse, d.logit_sum, d.nll_acc = _ptr(lse), _ptr(lsum), _ptr(nll_acc)
    _lib.check(lib.u2_lmhead_logprob_bf16(hidden.data_ptr(), weight.data_ptr(), logp.data_ptr(), C.byref(d), _stream()),
               "u2_lmhead_logprob_bf16")
    return logp, lse, lsum


def preprocess_volume(vol: torch.Tensor, *, target: int = 256, pad_depth: int = 256, lower: float = 0.5, upper: float = 99.5,
                      ws: Optional[torch.Tensor] = None):
    """The reference's u2Transform.adaptive_resize on a device volume [D, H, W] fp32: percentile intensity scaling ->
    foreground crop -> anti-aliased trilinear resize -> zero pad. Returns (images [pad_depth / 32, 32, target, target]
    fp32, info) where info is a device byte tensor holding a ``u2_preprocess_info`` (decode with
    ``preprocess_info``; nothing is synchronised here)."""
    _need_cuda(vol, ws)
    if vol.dtype != F32 or vol.dim() != 3 or not vol.is_contiguous():
        raise TypeError("preprocess_volume expects a contiguous fp32 [D, H, W] volume")
    if pad_depth % 32:
        raise ValueError("pad_depth must be a multiple of 32 (the model consumes 32-slice chunks)")
    D, H, W = vol.shape
    lib = _lib.load()
    need = int(lib.u2_preprocess_ws_bytes(D, H, W))
    if ws is None:
        ws = torch.empty(need, device=vol.device, dtype=torch.uint8)
    elif ws.numel() * ws.element_size() < need:
        raise ValueError(f"preprocess_volume: workspace of {need} bytes required")
    out = torch.empty(pad_depth // 32, 32, target, target, device=vol.device, dtype=F32)
    info = torch.zeros(C.sizeof(_lib.PreprocessInfo), device=vol.device, dtype=torch.uint8)
    d = _lib.PreprocessDesc()
    d.D, d.H, d.W, d.target, d.pad_depth = D, H, W, target, pad_depth
    d.lower_pct, d.upper_pct = float(lower), float(upper)
    d.ws, d.ws_bytes = ws.data_ptr(), ws.numel() * ws.element_size()
    _lib.check(lib.u2_preprocess_volume_f32(vol.data_ptr(), out.data_ptr(), info.data_ptr(), C.byref(d), _stream()),
               "u2_preprocess_volume_f32")
    return out, info


def preprocess_info(info: torch.Tensor) -> dict:
    """Decode the device-side ``u2_preprocess_info`` (synchronises)."""
    raw = bytes(info.cpu().numpy().tobytes())
    s = _lib.PreprocessInfo.from_buffer_copy(raw)
    return dict(a_min=s.a_min, a_max=s.a_max, lo=list(s.lo), hi=list(s.hi), out=list(s.out), sigma=list(s.sigma),
                tail=list(s.tail), status=s.status)
