// Decode-step linear layers: Y[b, n] = sum_k X[b, k] * W[n, k] for a handful of sequences (b <= 8).
// This regime streams every weight exactly once per generated token, so it is HBM-bound
// (15.1 GB per step for Qwen3-8B in bf16); the tensor cores are irrelevant here.
//
// Each warp owns kRows consecutive output rows and walks K with 16-byte loads (8 bf16 per lane per
// row); the activation vectors are re-used across the kRows rows from registers, so L1 traffic for X
// stays at 1/kRows of the weight stream. fp32 accumulation, warp-shuffle reduction at the end.
// Optional fusions: RMSNorm of X on the way in (rstd computed per CTA, gamma applied per element),
// residual add, SiLU(gate)*up pairing, fp32 or bf16 output.
//
// Reference call sites: the HF decoder Linears executed with q_len == 1 inside generate()
// (reference u2llama.py:123-126 -> HF GenerationMixin._sample).
#include <cuda_bf16.h>
#include <math.h>

#include "host_util.h"
#include "u2b200.h"

namespace u2 {

constexpr int kMaxB = 8;

__device__ __forceinline__ void unpack8g(const uint4& u, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

struct GemvArgs {
  const __nv_bfloat16* x;   // [B, K], row stride ldx
  const __nv_bfloat16* w;   // [N, K], row stride ldw
  void* y;                  // [B, N] (bf16 or fp32), row stride ldy
  const __nv_bfloat16* residual;  // [B, N] bf16 or null, row stride ldr
  const float* norm_gamma;  // [K] or null: x is RMS-normalised on the fly (fused input norm)
  float norm_eps;
  int B, N, K;
  long long ldx, ldw, ldy, ldr;
  int y_dtype;
  int silu_pair;            // rows (2j, 2j+1) are (gate_j, up_j): y[b, j] = silu(g_j) * u_j, N/2 outputs
};

template <int kB, int kRows>
__global__ void __launch_bounds__(128)
gemv_kernel(const GemvArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int n_out = a.silu_pair ? a.N / 2 : a.N;

  // fused RMSNorm: every CTA recomputes the (tiny) per-sequence statistics
  __shared__ float s_rstd[kMaxB];
  if (a.norm_gamma) {
    __shared__ float s_part[kMaxB][4];
    float ss[kB];
#pragma unroll
    for (int b = 0; b < kB; ++b) ss[b] = 0.f;
    for (int v = threadIdx.x; v < (a.K >> 3); v += blockDim.x) {
#pragma unroll
      for (int b = 0; b < kB; ++b) {
        float f[8];
        unpack8g(reinterpret_cast<const uint4*>(a.x + b * a.ldx)[v], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) ss[b] += f[j] * f[j];
      }
    }
#pragma unroll
    for (int b = 0; b < kB; ++b) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss[b] += __shfl_xor_sync(0xffffffffu, ss[b], o);
      if (lane == 0) s_part[b][warp] = ss[b];
    }
    __syncthreads();
    if (threadIdx.x < kB) {
      float t = 0.f;
      for (int w = 0; w < warps_per_block; ++w) t += s_part[threadIdx.x][w];
      s_rstd[threadIdx.x] = rsqrtf(t / a.K + a.norm_eps);
    }
    __syncthreads();
  }

  const int row0 = (blockIdx.x * warps_per_block + warp) * kRows;
  if (row0 >= n_out) return;
  constexpr int kW = kRows;  // weight rows handled per pass ("gate" rows; "up" rows in a second set)
  const int nsets = a.silu_pair ? 2 : 1;
  float acc[2][kW][kB];
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int r = 0; r < kW; ++r)
#pragma unroll
      for (int b = 0; b < kB; ++b) acc[s][r][b] = 0.f;

  const int nvec = a.K >> 3;
  for (int v = lane; v < nvec; v += 32) {
    float xf[kB][8];
#pragma unroll
    for (int b = 0; b < kB; ++b) unpack8g(reinterpret_cast<const uint4*>(a.x + b * a.ldx)[v], xf[b]);
    if (a.norm_gamma) {
      const float4 g0 = reinterpret_cast<const float4*>(a.norm_gamma)[2 * v];
      const float4 g1 = reinterpret_cast<const float4*>(a.norm_gamma)[2 * v + 1];
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
      for (int b = 0; b < kB; ++b) {
        const float rs = s_rstd[b];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          // match the unfused path: the normalised activation is rounded to bf16 before the GEMV
          xf[b][j] = __bfloat162float(__float2bfloat16(xf[b][j] * rs * g[j]));
        }
      }
    }
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      if (s < nsets) {
        uint4 wv[kW];
#pragma unroll
        for (int r = 0; r < kW; ++r) {
          // silu_pair: weight rows are interleaved (gate_j, up_j) = rows (2j, 2j+1)
          const int rb = (row0 + r < n_out) ? (row0 + r) : (n_out - 1);
          const int rr = a.silu_pair ? 2 * rb + s : rb;
          wv[r] = ldg_stream(reinterpret_cast<const uint4*>(a.w + (long long)rr * a.ldw) + v);
        }
#pragma unroll
        for (int r = 0; r < kW; ++r) {
          float wf[8];
          unpack8g(wv[r], wf);
#pragma unroll
          for (int b = 0; b < kB; ++b) {
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[s][r][b] += wf[j] * xf[b][j];
          }
        }
      }
    }
  }
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int r = 0; r < kW; ++r)
#pragma unroll
      for (int b = 0; b < kB; ++b) {
        if (s < nsets) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) acc[s][r][b] += __shfl_xor_sync(0xffffffffu, acc[s][r][b], o);
        }
      }
  if (lane == 0) {
#pragma unroll
    for (int r = 0; r < kW; ++r) {
      const int n = row0 + r;
      if (n < n_out) {
#pragma unroll
        for (int b = 0; b < kB; ++b) {
          float v = acc[0][r][b];
          if (a.silu_pair) {
            // unfused path rounds gate/up to bf16 before the activation: keep the same rounding points
            const float g = __bfloat162float(__float2bfloat16(v));
            const float u = __bfloat162float(__float2bfloat16(acc[1][r][b]));
            v = __fdividef(g, 1.f + __expf(-g)) * u;
          }
          if (a.residual) v += __bfloat162float(a.residual[b * a.ldr + n]);
          if (a.y_dtype == U2_DT_BF16) reinterpret_cast<__nv_bfloat16*>(a.y)[b * a.ldy + n] = __float2bfloat16(v);
          else reinterpret_cast<float*>(a.y)[b * a.ldy + n] = v;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// argmax over fp32 logits [B, V] -> int64 ids [B] (first index among equal maxima, like torch.argmax).
// Two tiny launches: (1) every CTA reduces a slice of a row and folds its (value, index) candidate into a
// 64-bit packed atomicMax per row; (2) one CTA unpacks the winners and clears the scratch for the next call.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long pack_candidate(float v, int idx) {
  unsigned int u = __float_as_uint(v);
  if (u == 0x80000000u) u = 0u;                            // -0.0 == +0.0
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);          // order-preserving float -> uint
  return ((unsigned long long)u << 32) | (unsigned int)(0xffffffffu - (unsigned int)idx);  // ties -> lower index
}

__global__ void __launch_bounds__(256)
argmax_partial_kernel(const float* __restrict__ logits, unsigned long long* __restrict__ scratch, int V, long long ld) {
  const int b = blockIdx.y;
  const float* p = logits + b * ld;
  const int per = (V + gridDim.x - 1) / gridDim.x;
  const int i0 = blockIdx.x * per;
  const int i1 = min(V, i0 + per);
  unsigned long long best = 0ull;
  for (int i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
    const unsigned long long c = pack_candidate(p[i], i);
    best = c > best ? c : best;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other > best ? other : best;
  }
  __shared__ unsigned long long sb[8];
  if ((threadIdx.x & 31) == 0) sb[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) best = sb[w] > best ? sb[w] : best;
    if (best) atomicMax(scratch + b, best);
  }
}

__global__ void argmax_final_kernel(unsigned long long* __restrict__ scratch, long long* __restrict__ out, int B) {
  const int b = threadIdx.x;
  if (b < B) {
    out[b] = (long long)(0xffffffffu - (unsigned int)(scratch[b] & 0xffffffffull));
    scratch[b] = 0ull;
  }
}

// ------------------------------------------------------------------------------------------------
// Generation scores inside the captured decode step. A captured graph keeps its pointers, so the destination of a
// step's row store is read from a device block (u2_row_store_params) and the step from *step_dev: one capture serves
// every step, chunk and call. Grid (slices, rows); each CTA copies one slice of a row, coalesced.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
store_rows_kernel(const float* __restrict__ src, long long ld_src, int V, const u2_row_store_params* __restrict__ p,
                  const int* __restrict__ step_dev, int step_host) {
  const long long t = step_dev ? *step_dev : step_host;
  if (t < 0 || t >= p->steps) return;
  const int r = blockIdx.y;
  const float* s = src + r * ld_src;
  float* d = p->dst + t * p->ld_step + r * p->ld_row;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < V; i += gridDim.x * blockDim.x) d[i] = s[i];
}

// logprob[b] = logits[b, ids[b]] - logsumexp(logits[b]): one CTA per row, an online (max, sum of exp) per thread
// merged across the block. Rows may hold -inf entries (logits processors); a row that is all -inf yields NaN.
__global__ void __launch_bounds__(512)
pick_logprob_kernel(const float* __restrict__ logits, long long ld, int V, const long long* __restrict__ ids,
                    float* __restrict__ logprob) {
  const int b = blockIdx.x;
  const float* l = logits + b * ld;
  float m = -INFINITY, s = 0.f;
  for (int i = threadIdx.x; i < V; i += blockDim.x) {
    const float x = l[i];
    if (x > m) {
      s = s * expf(m - x) + 1.f;
      m = x;
    } else if (x > -INFINITY) {
      s += expf(x - m);
    }
  }
  __shared__ float sm[16], ss[16];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const float mm = fmaxf(m, m2);
    s = (m == -INFINITY ? 0.f : s * expf(m - mm)) + (m2 == -INFINITY ? 0.f : s2 * expf(m2 - mm));
    m = mm;
  }
  if ((threadIdx.x & 31) == 0) { sm[threadIdx.x >> 5] = m; ss[threadIdx.x >> 5] = s; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float M = -INFINITY, S = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
      const float mm = fmaxf(M, sm[w]);
      S = (M == -INFINITY ? 0.f : S * expf(M - mm)) + (sm[w] == -INFINITY ? 0.f : ss[w] * expf(sm[w] - mm));
      M = mm;
    }
    logprob[b] = (l[ids[b]] - M) - logf(S);
  }
}

template <int kB>
static int launch_gemv(const GemvArgs& a, cudaStream_t st) {
  const int n_out = a.silu_pair ? a.N / 2 : a.N;
  const int wpb = 4;
  // 4 rows per warp when there are plenty of rows, else 2 / 1 so that the grid still fills 132 SMs
  if (!a.silu_pair && n_out >= 132 * 4 * wpb * 4) {
    const int rpb = wpb * 4;
    gemv_kernel<kB, 4><<<(n_out + rpb - 1) / rpb, wpb * 32, 0, st>>>(a);
  } else if (n_out >= 132 * 2 * wpb * 2) {
    const int rpb = wpb * 2;
    gemv_kernel<kB, 2><<<(n_out + rpb - 1) / rpb, wpb * 32, 0, st>>>(a);
  } else {
    const int rpb = wpb;
    gemv_kernel<kB, 1><<<(n_out + rpb - 1) / rpb, wpb * 32, 0, st>>>(a);
  }
  U2_CHECK_LAUNCH("gemv");
  return U2_OK;
}

}  // namespace u2

using namespace u2;

extern "C" U2_API int u2_gemv_bf16(const void* x, const void* w, void* y, const u2_gemv_desc* d, void* stream) {
  if (!x || !w || !y || !d) return set_error(U2_ERR_ARG, "gemv: null pointer");
  if (d->B < 1 || d->B > kMaxB) return set_error(U2_ERR_UNSUPPORTED, "gemv: 1 <= B <= %d (got %d)", kMaxB, d->B);
  if (d->N <= 0 || d->K <= 0 || (d->K & 7) || (d->ldx & 7) || (d->ldw & 7))
    return set_error(U2_ERR_ARG, "gemv: K, ldx, ldw must be positive multiples of 8");
  if (d->silu_pair && (d->N & 1)) return set_error(U2_ERR_ARG, "gemv: silu_pair needs an even N");
  GemvArgs a;
  a.x = reinterpret_cast<const __nv_bfloat16*>(x);
  a.w = reinterpret_cast<const __nv_bfloat16*>(w);
  a.y = y;
  a.residual = reinterpret_cast<const __nv_bfloat16*>(d->residual);
  a.norm_gamma = d->norm_gamma;
  a.norm_eps = d->norm_eps;
  a.B = d->B; a.N = d->N; a.K = d->K;
  a.ldx = d->ldx; a.ldw = d->ldw; a.ldy = d->ldy; a.ldr = d->ldr;
  a.y_dtype = d->y_dtype;
  a.silu_pair = d->silu_pair;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (d->B) {
    case 1: return launch_gemv<1>(a, st);
    case 2: return launch_gemv<2>(a, st);
    case 3: return launch_gemv<3>(a, st);
    case 4: return launch_gemv<4>(a, st);
    case 5: return launch_gemv<5>(a, st);
    case 6: return launch_gemv<6>(a, st);
    case 7: return launch_gemv<7>(a, st);
    default: return launch_gemv<8>(a, st);
  }
}

extern "C" U2_API int u2_argmax_f32(const float* logits, int64_t* out, uint64_t* scratch, int32_t B, int32_t V,
                                    int64_t ld, void* stream) {
  if (!logits || !out || !scratch) return set_error(U2_ERR_ARG, "argmax: null pointer");
  if (B <= 0 || V <= 0) return U2_OK;
  if (B > 1024) return set_error(U2_ERR_UNSUPPORTED, "argmax: B <= 1024");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int chunks = (V + 4095) / 4096;
  if (chunks > 64) chunks = 64;
  dim3 grid((unsigned)chunks, (unsigned)B);
  argmax_partial_kernel<<<grid, 256, 0, st>>>(logits, reinterpret_cast<unsigned long long*>(scratch), V, ld);
  U2_CHECK_LAUNCH("argmax partial");
  argmax_final_kernel<<<1, 1024, 0, st>>>(reinterpret_cast<unsigned long long*>(scratch), reinterpret_cast<long long*>(out), B);
  U2_CHECK_LAUNCH("argmax final");
  return U2_OK;
}

extern "C" U2_API int u2_store_rows_f32(const float* src, int32_t rows, int32_t V, int64_t ld_src,
                                        const u2_row_store_params* params_dev, const int32_t* step_dev, int32_t step,
                                        void* stream) {
  if (!src || !params_dev) return set_error(U2_ERR_ARG, "store_rows: null pointer");
  if (rows <= 0 || V <= 0) return U2_OK;
  if (rows > 65535) return set_error(U2_ERR_UNSUPPORTED, "store_rows: rows <= 65535");
  int slices = (V + 4095) / 4096;
  if (slices > 64) slices = 64;
  store_rows_kernel<<<dim3((unsigned)slices, (unsigned)rows), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src, ld_src, V, params_dev, step_dev, step);
  U2_CHECK_LAUNCH("store_rows");
  return U2_OK;
}

extern "C" U2_API int u2_pick_logprob_f32(const float* logits, int32_t B, int32_t V, int64_t ld, const int64_t* ids,
                                          float* logprob, void* stream) {
  if (!logits || !ids || !logprob) return set_error(U2_ERR_ARG, "pick_logprob: null pointer");
  if (B <= 0 || V <= 0) return U2_OK;
  pick_logprob_kernel<<<B, 512, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, ld, V, reinterpret_cast<const long long*>(ids), logprob);
  U2_CHECK_LAUNCH("pick_logprob");
  return U2_OK;
}
