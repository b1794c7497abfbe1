// Row-wise HBM-bound kernels: LayerNorm, RMSNorm, softmax (relative-position bias / causal mask),
// SiLU*mul. One warp (or one 128-thread group) owns a row; 16-byte vector loads; the row is cached
// in registers between the statistics pass and the write pass so HBM sees each element once.
#include <cuda_bf16.h>
#include <math.h>

#include <type_traits>

#include "host_util.h"
#include "u2b200.h"

namespace u2 {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return u;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm / RMSNorm: y = norm(x [+ residual]) * gamma (+ beta); optional copy of the sum out.
// warp per row, kMaxV 16-byte vectors per lane (E <= kMaxV * 256).
// ------------------------------------------------------------------------------------------------
template <int kMaxV, bool kRms>
__global__ void __launch_bounds__(256)
norm_rows_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                 const float* __restrict__ gamma, const float* __restrict__ beta,
                 __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ sum_out, long long rows,
                 int E, long long ldx, long long ldr, long long ldy, float eps) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = E >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
  const uint4* rr = res ? reinterpret_cast<const uint4*>(res + row * ldr) : nullptr;
  float v[kMaxV][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxV; ++i) {
    const int c = i * 32 + lane;
    if (c < nvec) {
      unpack8(xr[c], v[i]);
      if (rr) {
        float r[8];
        unpack8(rr[c], r);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[i][j] += r[j];
        if (sum_out) {
          // the residual stream is kept in bf16: normalise what is actually stored
          const uint4 pk = pack8(v[i]);
          reinterpret_cast<uint4*>(sum_out + row * ldy)[c] = pk;
          unpack8(pk, v[i]);
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s += kRms ? v[i][j] * v[i][j] : v[i][j];
    }
  }
  s = warp_sum(s);
  float mean = 0.f, rstd;
  if (kRms) {
    rstd = rsqrtf(s / E + eps);
  } else {
    mean = s / E;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
      const int c = i * 32 + lane;
      if (c < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          q += d * d;
        }
      }
    }
    q = warp_sum(q);
    rstd = rsqrtf(q / E + eps);
  }
  uint4* yr = reinterpret_cast<uint4*>(y + row * ldy);
#pragma unroll
  for (int i = 0; i < kMaxV; ++i) {
    const int c = i * 32 + lane;
    if (c < nvec) {
      const float4 g0 = reinterpret_cast<const float4*>(gamma)[2 * c];
      const float4 g1 = reinterpret_cast<const float4*>(gamma)[2 * c + 1];
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      float o[8];
      if (beta) {
        const float4 b0 = reinterpret_cast<const float4*>(beta)[2 * c];
        const float4 b1 = reinterpret_cast<const float4*>(beta)[2 * c + 1];
        const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * g[j] + b[j];
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * g[j];
      }
      yr[c] = pack8(o);
    }
  }
}

template <bool kRms>
static int launch_norm(const void* x, const void* res, const float* gamma, const float* beta, void* y,
                       void* sum_out, long long rows, int E, long long ldx, long long ldr, long long ldy,
                       float eps, cudaStream_t st) {
  if (E <= 0 || (E & 7)) return set_error(U2_ERR_ARG, "norm: E must be a positive multiple of 8");
  if ((ldx & 7) || (ldy & 7) || (res && (ldr & 7))) return set_error(U2_ERR_ARG, "norm: row strides must be multiples of 8");
  if (rows <= 0) return U2_OK;
  const int nvec = E / 8;
  const int need = (nvec + 31) / 32;
  const int wpb = 8;
  const unsigned grid = (unsigned)((rows + wpb - 1) / wpb);
  auto X = reinterpret_cast<const __nv_bfloat16*>(x);
  auto R = reinterpret_cast<const __nv_bfloat16*>(res);
  auto Y = reinterpret_cast<__nv_bfloat16*>(y);
  auto S = reinterpret_cast<__nv_bfloat16*>(sum_out);
#define U2_NORM_CASE(MV)                                                                               \
  norm_rows_kernel<MV, kRms><<<grid, wpb * 32, 0, st>>>(X, R, gamma, beta, Y, S, rows, E, ldx, ldr, ldy, eps)
  if (need <= 1) U2_NORM_CASE(1);
  else if (need <= 2) U2_NORM_CASE(2);
  else if (need <= 4) U2_NORM_CASE(4);
  else if (need <= 8) U2_NORM_CASE(8);
  else if (need <= 16) U2_NORM_CASE(16);
  else if (need <= 32) U2_NORM_CASE(32);
  else return set_error(U2_ERR_UNSUPPORTED, "norm: E=%d too large (max 8192)", E);
#undef U2_NORM_CASE
  U2_CHECK_LAUNCH("norm");
  return U2_OK;
}

// ------------------------------------------------------------------------------------------------
// softmax over the last dim of fp32 score rows -> bf16 probabilities.
// rows are indexed (i0, i1, i2): i2 = query position in [0, S), i1 = head in [0, H), i0 = batch.
// ------------------------------------------------------------------------------------------------
struct SoftmaxArgs {
  const float* in;
  __nv_bfloat16* out;
  long long in_s0, in_s1, in_s2;     // element strides of (batch, head, query) for the input rows
  long long out_s0, out_s1, out_s2;  // same for the output rows
  int n0, H, S;                      // extents
  int n;                             // row length (keys)
  float scale;
  const float* rel_bias;             // [2*rel_max-1, H] or null; bias[(j - i + rel_max - 1), head]
  int rel_max;
  int causal;                        // key j visible iff j <= i + causal_off
  int causal_off;
  int zero_pad_to;                   // write zeros for columns [n, zero_pad_to)
};
// sliding window on top of the causal mask (kWin kernels): key j visible iff j > i + causal_off - window as well
// (HF masking_utils.sliding_window_overlay, masking_utils.py:90-97, used by Phi-3 through modeling_phi3.py:403).
// A separate type so that the kernels without a window keep their parameter block and code.
struct SoftmaxWinArgs : SoftmaxArgs {
  int window;
};
template <bool kWin>
using SoftmaxArgsT = std::conditional_t<kWin, SoftmaxWinArgs, SoftmaxArgs>;
template <bool kWin>
__device__ __forceinline__ int softmax_lo(const SoftmaxArgsT<kWin>& a, int i2) {
  if constexpr (kWin) return max(0, i2 + a.causal_off - a.window + 1);
  else return 0;
}

template <int kGroup, int kMaxV, bool kWin = false>
__global__ void __launch_bounds__(kGroup == 32 ? 128 : kGroup)
softmax_rows_kernel(const SoftmaxArgsT<kWin> a) {
  constexpr int kRowsPerBlock = (kGroup == 32) ? 4 : 1;
  const int gl = threadIdx.x % kGroup;  // lane within the group
  const long long row = (long long)blockIdx.x * kRowsPerBlock + threadIdx.x / kGroup;
  const long long total = (long long)a.n0 * a.H * a.S;
  __shared__ float red[8];
  const bool active = row < total;
  const long long r = active ? row : 0;
  const int i2 = (int)(r % a.S);
  const int i1 = (int)((r / a.S) % a.H);
  const long long i0 = r / ((long long)a.S * a.H);
  const float* in = a.in + i0 * a.in_s0 + i1 * a.in_s1 + i2 * a.in_s2;
  __nv_bfloat16* out = a.out + i0 * a.out_s0 + i1 * a.out_s1 + i2 * a.out_s2;
  const int limit = a.causal ? min(a.n, i2 + a.causal_off + 1) : a.n;  // keys [0, limit) are visible
  const int lo = softmax_lo<kWin>(a, i2);                                // (keys [lo, limit) with a window)

  float v[kMaxV];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < kMaxV; ++i) {
    const int j = i * kGroup + gl;
    float t = -INFINITY;
    if (active && j < limit && (!kWin || j >= lo)) {
      t = in[j] * a.scale;
      if (a.rel_bias) t += __ldg(a.rel_bias + (long long)(j - i2 + a.rel_max - 1) * a.H + i1);
    }
    v[i] = t;
    m = fmaxf(m, t);
  }
  m = warp_max(m);
  if (kGroup > 32) {
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = red[0];
#pragma unroll
    for (int w = 1; w < kGroup / 32; ++w) m = fmaxf(m, red[w]);
    __syncthreads();
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxV; ++i) {
    const float e = (v[i] == -INFINITY) ? 0.f : __expf(v[i] - m);
    v[i] = e;
    s += e;
  }
  s = warp_sum(s);
  if (kGroup > 32) {
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    s = 0.f;
#pragma unroll
    for (int w = 0; w < kGroup / 32; ++w) s += red[w];
  }
  const float inv = s > 0.f ? 1.f / s : 0.f;
  if (!active) return;
#pragma unroll
  for (int i = 0; i < kMaxV; ++i) {
    const int j = i * kGroup + gl;
    if (j < a.n) out[j] = __float2bfloat16(v[i] * inv);
    else if (j < a.zero_pad_to) out[j] = __float2bfloat16(0.f);
  }
}

// Long plain rows (the ViT's 2049 keys: no bias, no mask): one WARP per row, 16-byte vector loads, the row held in
// registers - no block-wide barriers, ~270 bytes in flight per thread (the one-CTA-per-row variant above reached
// 1.8 TB/s on these rows because every row paid two __syncthreads round trips).
template <int kMaxV4>
__global__ void __launch_bounds__(256)
softmax_warp_vec_kernel(const SoftmaxArgs a) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long total = (long long)a.n0 * a.H * a.S;
  if (row >= total) return;
  const int i2 = (int)(row % a.S);
  const int i1 = (int)((row / a.S) % a.H);
  const long long i0 = row / ((long long)a.S * a.H);
  const float4* in = reinterpret_cast<const float4*>(a.in + i0 * a.in_s0 + i1 * a.in_s1 + i2 * a.in_s2);
  __nv_bfloat16* out = a.out + i0 * a.out_s0 + i1 * a.out_s1 + i2 * a.out_s2;
  const int span = max(a.n, a.zero_pad_to);
  const int nv = (span + 3) >> 2;  // float4 groups (the padded row is readable: pads are written by the producer GEMM's ld)
  float4 v[kMaxV4];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < kMaxV4; ++i) {
    const int c = i * 32 + lane;
    if (c < nv) {
      float4 t = in[c];
      const int j = c * 4;
      t.x = j + 0 < a.n ? t.x * a.scale : -INFINITY;
      t.y = j + 1 < a.n ? t.y * a.scale : -INFINITY;
      t.z = j + 2 < a.n ? t.z * a.scale : -INFINITY;
      t.w = j + 3 < a.n ? t.w * a.scale : -INFINITY;
      v[i] = t;
      m = fmaxf(m, fmaxf(fmaxf(t.x, t.y), fmaxf(t.z, t.w)));
    }
  }
  m = warp_max(m);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxV4; ++i) {
    const int c = i * 32 + lane;
    if (c < nv) {
      v[i].x = __expf(v[i].x - m); v[i].y = __expf(v[i].y - m); v[i].z = __expf(v[i].z - m); v[i].w = __expf(v[i].w - m);
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  s = warp_sum(s);
  const float inv = s > 0.f ? 1.f / s : 0.f;
#pragma unroll
  for (int i = 0; i < kMaxV4; ++i) {
    const int c = i * 32 + lane;
    if (c < nv) {
      uint2 o;
      *reinterpret_cast<__nv_bfloat162*>(&o.x) = __floats2bfloat162_rn(v[i].x * inv, v[i].y * inv);
      *reinterpret_cast<__nv_bfloat162*>(&o.y) = __floats2bfloat162_rn(v[i].z * inv, v[i].w * inv);
      if (c * 4 + 3 < span) {
        reinterpret_cast<uint2*>(out)[c] = o;
      } else {
        const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&o);
        for (int e = 0; e < 4 && c * 4 + e < span; ++e) out[c * 4 + e] = h[e];
      }
    }
  }
}

// Rows longer than the register-resident variants hold (> 8192 keys, e.g. DiffTS over 64 frames x 256 tokens, the
// reference's own smoke shape svr.py:190-205): one CTA per row, three passes over the (L2-resident) row.
template <bool kWin = false>
__global__ void __launch_bounds__(256)
softmax_long_rows_kernel(const SoftmaxArgsT<kWin> a) {
  const long long r = blockIdx.x;
  const int i2 = (int)(r % a.S);
  const int i1 = (int)((r / a.S) % a.H);
  const long long i0 = r / ((long long)a.S * a.H);
  const float* in = a.in + i0 * a.in_s0 + i1 * a.in_s1 + i2 * a.in_s2;
  __nv_bfloat16* out = a.out + i0 * a.out_s0 + i1 * a.out_s1 + i2 * a.out_s2;
  const int limit = a.causal ? min(a.n, i2 + a.causal_off + 1) : a.n;
  const int lo = softmax_lo<kWin>(a, i2);
  __shared__ float red[8];
  auto score = [&](int j) {
    float t = in[j] * a.scale;
    if (a.rel_bias) t += __ldg(a.rel_bias + (long long)(j - i2 + a.rel_max - 1) * a.H + i1);
    return t;
  };
  auto block_reduce = [&](float v, bool is_max) {
    v = is_max ? warp_max(v) : warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = red[0];
    for (int w = 1; w < 8; ++w) t = is_max ? fmaxf(t, red[w]) : t + red[w];
    return t;
  };
  float m = -INFINITY;
  for (int j = lo + threadIdx.x; j < limit; j += 256) m = fmaxf(m, score(j));
  m = block_reduce(m, true);
  float s = 0.f;
  for (int j = lo + threadIdx.x; j < limit; j += 256) s += __expf(score(j) - m);
  s = block_reduce(s, false);
  const float inv = s > 0.f ? 1.f / s : 0.f;
  const int span = max(a.n, a.zero_pad_to);
  for (int j = threadIdx.x; j < span; j += 256)
    out[j] = __float2bfloat16(j < limit && (!kWin || j >= lo) ? __expf(score(j) - m) * inv : 0.f);
}

// ------------------------------------------------------------------------------------------------
// SiLU(gate) * up on a fused [rows, 2*I] gate|up buffer -> [rows, I]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
silu_mul_kernel(const __nv_bfloat16* __restrict__ gu, __nv_bfloat16* __restrict__ out, long long rows,
                int I, long long ldg, long long ldo, int interleaved) {
  const int nvec = I >> 3;
  const long long total = rows * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / nvec;
    const int c = (int)(idx - r * nvec);
    float g[8], u[8], o[8];
    if (interleaved) {
      float a[8], b[8];
      unpack8(reinterpret_cast<const uint4*>(gu + r * ldg)[2 * c], a);
      unpack8(reinterpret_cast<const uint4*>(gu + r * ldg)[2 * c + 1], b);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        g[j] = a[2 * j]; u[j] = a[2 * j + 1];
        g[4 + j] = b[2 * j]; u[4 + j] = b[2 * j + 1];
      }
    } else {
      unpack8(reinterpret_cast<const uint4*>(gu + r * ldg)[c], g);
      unpack8(reinterpret_cast<const uint4*>(gu + r * ldg + I)[c], u);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = __fdividef(g[j], 1.f + __expf(-g[j])) * u[j];
    reinterpret_cast<uint4*>(out + r * ldo)[c] = pack8(o);
  }
}

}  // namespace u2

using namespace u2;

extern "C" U2_API int u2_layernorm_bf16(const void* x, const void* residual, const float* gamma,
                                        const float* beta, void* y, void* sum_out, int64_t rows, int32_t E,
                                        int64_t ldx, int64_t ldr, int64_t ldy, float eps, void* stream) {
  if (!x || !gamma || !y) return set_error(U2_ERR_ARG, "layernorm: null pointer");
  return launch_norm<false>(x, residual, gamma, beta, y, sum_out, rows, E, ldx, ldr, ldy, eps,
                            reinterpret_cast<cudaStream_t>(stream));
}

extern "C" U2_API int u2_rmsnorm_bf16(const void* x, const void* residual, const float* gamma, void* y,
                                      void* sum_out, int64_t rows, int32_t E, int64_t ldx, int64_t ldr,
                                      int64_t ldy, float eps, void* stream) {
  if (!x || !gamma || !y) return set_error(U2_ERR_ARG, "rmsnorm: null pointer");
  return launch_norm<true>(x, residual, gamma, nullptr, y, sum_out, rows, E, ldx, ldr, ldy, eps,
                           reinterpret_cast<cudaStream_t>(stream));
}

extern "C" U2_API int u2_softmax_f32_bf16(const float* in, void* out, const u2_softmax_desc* d, void* stream) {
  if (!in || !out || !d) return set_error(U2_ERR_ARG, "softmax: null pointer");
  if (d->n <= 0 || d->n0 <= 0 || d->H <= 0 || d->S <= 0) return set_error(U2_ERR_ARG, "softmax: bad extents");
  if (d->rel_bias && (d->n > d->rel_max || d->S > d->rel_max))
    return set_error(U2_ERR_ARG, "softmax: sequence length %d/%d exceeds the relative-bias table (%d)", d->S, d->n, d->rel_max);
  if (d->window < 0 || (d->window > 0 && !d->causal))
    return set_error(U2_ERR_ARG, "softmax: window %d needs causal != 0 (and >= 0)", d->window);
  SoftmaxWinArgs a;
  a.in = in;
  a.out = reinterpret_cast<__nv_bfloat16*>(out);
  a.in_s0 = d->in_s0; a.in_s1 = d->in_s1; a.in_s2 = d->in_s2;
  a.out_s0 = d->out_s0; a.out_s1 = d->out_s1; a.out_s2 = d->out_s2;
  a.n0 = d->n0; a.H = d->H; a.S = d->S; a.n = d->n;
  a.scale = d->scale;
  a.rel_bias = d->rel_bias; a.rel_max = d->rel_max;
  a.causal = d->causal; a.causal_off = d->causal_off;
  a.zero_pad_to = d->zero_pad_to;
  a.window = d->window;
  const bool win = d->window > 0;
  const SoftmaxArgs& a0 = a;
  const int span = d->n > d->zero_pad_to ? d->n : d->zero_pad_to;
  const long long rows = (long long)d->n0 * d->H * d->S;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define U2_SM_GRID(G) (unsigned)((rows + ((G) == 32 ? 4 : 1) - 1) / ((G) == 32 ? 4 : 1)), (G) == 32 ? 128 : (G), 0, st
#define U2_SM_CASE(G, MV)                                           \
  do {                                                              \
    if (win) softmax_rows_kernel<G, MV, true><<<U2_SM_GRID(G)>>>(a); \
    else softmax_rows_kernel<G, MV><<<U2_SM_GRID(G)>>>(a0);          \
  } while (0)
  // long plain rows: warp-per-row vector variant (needs 16-byte aligned fp32 rows, 8-byte aligned bf16 rows, a span that
  // is a whole number of float4 groups - the callers pad rows to 8 elements)
  const bool vec_ok = !d->rel_bias && !d->causal && span > 1024 && span <= 2560 && (span & 3) == 0 &&
                      (d->in_s0 & 3) == 0 && (d->in_s1 & 3) == 0 && (d->in_s2 & 3) == 0 && (d->out_s0 & 3) == 0 &&
                      (d->out_s1 & 3) == 0 && (d->out_s2 & 3) == 0 && (reinterpret_cast<uintptr_t>(in) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(out) & 7) == 0 && d->zero_pad_to >= d->n;
  if (vec_ok) {
    softmax_warp_vec_kernel<20><<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(a0);
    U2_CHECK_LAUNCH("softmax");
    return U2_OK;
  }
  if (span <= 32) U2_SM_CASE(32, 1);
  else if (span <= 64) U2_SM_CASE(32, 2);
  else if (span <= 128) U2_SM_CASE(32, 4);
  else if (span <= 256) U2_SM_CASE(32, 8);
  else if (span <= 512) U2_SM_CASE(32, 16);
  else if (span <= 1024) U2_SM_CASE(128, 8);
  else if (span <= 2048) U2_SM_CASE(128, 16);
  else if (span <= 4096) U2_SM_CASE(256, 16);
  else if (span <= 8192) U2_SM_CASE(256, 32);
  else if (rows <= 0x7fffffffLL && win) softmax_long_rows_kernel<true><<<(unsigned)rows, 256, 0, st>>>(a);
  else if (rows <= 0x7fffffffLL) softmax_long_rows_kernel<<<(unsigned)rows, 256, 0, st>>>(a0);
  else return set_error(U2_ERR_UNSUPPORTED, "softmax: %lld rows of length %d", rows, span);
#undef U2_SM_CASE
#undef U2_SM_GRID
  U2_CHECK_LAUNCH("softmax");
  return U2_OK;
}

extern "C" U2_API int u2_silu_mul_bf16(const void* gate_up, void* out, int64_t rows, int32_t I, int64_t ldg,
                                       int64_t ldo, int32_t interleaved, void* stream) {
  if (!gate_up || !out) return set_error(U2_ERR_ARG, "silu_mul: null pointer");
  if (I <= 0 || (I & 7) || (ldg & 7) || (ldo & 7)) return set_error(U2_ERR_ARG, "silu_mul: I/ld must be multiples of 8");
  if (rows <= 0) return U2_OK;
  const long long total = rows * (I / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 16) blocks = 132LL * 16;
  silu_mul_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(gate_up), reinterpret_cast<__nv_bfloat16*>(out), rows, I, ldg, ldo, interleaved);
  U2_CHECK_LAUNCH("silu_mul");
  return U2_OK;
}
