// Training-side kernels (everything of the backward pass that is not a GEMM): HBM-bound row-wise / elementwise
// work, 16-byte vector accesses, fp32 statistics, fp32 accumulators for the small parameter gradients.
// The contractions (dgrad, wgrad, dP, dQ, dK, dV) run on gemm_wgmma.cu with its MN-major operand flags.
// Declared in include/u2b200_train.h; reference call sites: HF Trainer backward over the modules of src/model
// (train_stage1.py:244-250), DeepSpeed ZeRO-1 optimizer step (config/ds_config.json:27-39).
#include <cuda_bf16.h>
#include <math.h>

#include "host_util.h"
#include "u2b200_train.h"

namespace u2 {

#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)

__device__ __forceinline__ float t_wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float t_wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ void t_unpack8(const uint4& u, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 t_pack8(const float (&f)[8]) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return u;
}
__device__ __forceinline__ void t_load8f(const float* p, float (&f)[8]) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
static inline unsigned t_grid(long long total, int threads, long long cap = 132LL * 16) {
  long long b = (total + threads - 1) / threads;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

// ------------------------------------------------------------------------------------------------
// batched 2-D transpose (32 x 32 tiles through shared memory)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
transpose_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int rows, int cols,
                 long long ld_in, long long ld_out, long long in_bs, long long out_bs) {
  __shared__ __nv_bfloat16 tile[32][34];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const long long b = blockIdx.z;
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int r = r0 + ty + 8 * k, c = c0 + tx;
    if (r < rows && c < cols) tile[ty + 8 * k][tx] = in[b * in_bs + (long long)r * ld_in + c];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = c0 + ty + 8 * k, r = r0 + tx;
    if (c < cols && r < rows) out[b * out_bs + (long long)c * ld_out + r] = tile[tx][ty + 8 * k];
  }
}

// ------------------------------------------------------------------------------------------------
// column sums: out[c] += sum_r x[r, c]
// block = 32 column vectors (256 columns) x 8 row lanes; grid (column blocks, row chunks)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, long long rows, long long cols,
              long long ld, long long rows_per_block) {
  __shared__ float red[8][32][8];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const long long cv = (long long)blockIdx.x * 32 + tx;
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const bool ok = cv * 8 < cols;
  if (ok) {
    for (long long r = r0 + ty; r < r1; r += 8) {
      float v[8];
      t_unpack8(*reinterpret_cast<const uint4*>(x + r * ld + cv * 8), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[ty][tx][j] = acc[j];
  __syncthreads();
  if (ty == 0 && ok) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += red[w][tx][j];
      atomicAdd(out + cv * 8 + j, s);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// GELU (erf) forward / backward, SiLU*mul backward
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gelu_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long nvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float v[8], o[8];
    t_unpack8(reinterpret_cast<const uint4*>(x)[i], v);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = 0.5f * v[j] * (1.f + erff(v[j] * 0.70710678118654752440f));
    reinterpret_cast<uint4*>(y)[i] = t_pack8(o);
  }
}

__global__ void __launch_bounds__(256)
gelu_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx,
                long long nvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float v[8], g[8], o[8];
    t_unpack8(reinterpret_cast<const uint4*>(x)[i], v);
    t_unpack8(reinterpret_cast<const uint4*>(dy)[i], g);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float cdf = 0.5f * (1.f + erff(v[j] * 0.70710678118654752440f));
      const float pdf = 0.39894228040143267794f * __expf(-0.5f * v[j] * v[j]);
      o[j] = g[j] * (cdf + v[j] * pdf);
    }
    reinterpret_cast<uint4*>(dx)[i] = t_pack8(o);
  }
}

__global__ void __launch_bounds__(256)
silu_mul_bwd_kernel(const __nv_bfloat16* __restrict__ gu, const __nv_bfloat16* __restrict__ dact,
                    __nv_bfloat16* __restrict__ dgu, long long rows, int I, long long ldg, long long ldd) {
  const int nvec = I >> 3;
  const long long total = rows * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / nvec;
    const int c = (int)(idx - r * nvec);
    float g[8], u[8], d[8], dg[8], du[8];
    t_unpack8(reinterpret_cast<const uint4*>(gu + r * ldg)[c], g);
    t_unpack8(reinterpret_cast<const uint4*>(gu + r * ldg + I)[c], u);
    t_unpack8(reinterpret_cast<const uint4*>(dact + r * ldd)[c], d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float s = __fdividef(1.f, 1.f + __expf(-g[j]));
      dg[j] = d[j] * u[j] * s * (1.f + g[j] * (1.f - s));
      du[j] = d[j] * g[j] * s;
    }
    reinterpret_cast<uint4*>(dgu + r * ldg)[c] = t_pack8(dg);
    reinterpret_cast<uint4*>(dgu + r * ldg + I)[c] = t_pack8(du);
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm / RMSNorm backward: warp per row (x held in registers), rows strided over the grid;
// dgamma / dbeta accumulate in shared memory (fp32 atomics) and are flushed once per block.
// ------------------------------------------------------------------------------------------------
template <int kMaxV, bool kRms>
__global__ void __launch_bounds__(256)
norm_bwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma, const __nv_bfloat16* __restrict__ dy,
                const __nv_bfloat16* dres, __nv_bfloat16* dx, float* __restrict__ dgamma, float* __restrict__ dbeta,
                long long rows, int E, long long ldx, long long ldy, long long ldr, long long ldo, float eps) {
  extern __shared__ float s_acc[];  // [E] dgamma, then [E] dbeta
  float* s_dg = s_acc;
  float* s_db = s_acc + E;
  const bool want_dg = dgamma != nullptr;
  if (want_dg) {
    for (int i = threadIdx.x; i < (kRms ? E : 2 * E); i += blockDim.x) s_acc[i] = 0.f;
    __syncthreads();
  }
  const int lane = threadIdx.x & 31;
  const int nvec = E >> 3;
  const float invE = 1.f / E;
  for (long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); row < rows; row += (long long)gridDim.x * 8) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
    const uint4* gr = reinterpret_cast<const uint4*>(dy + row * ldy);
    float v[kMaxV][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
      const int c = i * 32 + lane;
      if (c < nvec) {
        t_unpack8(xr[c], v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += kRms ? v[i][j] * v[i][j] : v[i][j];
      }
    }
    s = t_wsum(s);
    float mean = 0.f, rstd;
    if (kRms) {
      rstd = rsqrtf(s * invE + eps);
    } else {
      mean = s * invE;
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
      q = t_wsum(q);
      rstd = rsqrtf(q * invE + eps);
    }
    // xhat in place; sums of dy*gamma and dy*gamma*xhat
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
      const int c = i * 32 + lane;
      if (c < nvec) {
        float g[8], w[8];
        t_unpack8(gr[c], g);
        t_load8f(gamma + c * 8, w);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (v[i][j] - mean) * rstd;
          v[i][j] = xh;
          const float gw = g[j] * w[j];
          s1 += gw;
          s2 += gw * xh;
          if (want_dg) {
            atomicAdd(&s_dg[c * 8 + j], g[j] * xh);
            if (!kRms) atomicAdd(&s_db[c * 8 + j], g[j]);
          }
        }
      }
    }
    s1 = kRms ? 0.f : t_wsum(s1) * invE;
    s2 = t_wsum(s2) * invE;
    const uint4* rr = dres ? reinterpret_cast<const uint4*>(dres + row * ldr) : nullptr;
    uint4* outr = reinterpret_cast<uint4*>(dx + row * ldo);
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
      const int c = i * 32 + lane;
      if (c < nvec) {
        float g[8], w[8], o[8];
        t_unpack8(gr[c], g);
        t_load8f(gamma + c * 8, w);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (g[j] * w[j] - s1 - v[i][j] * s2);
        if (rr) {
          float r[8];
          t_unpack8(rr[c], r);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r[j];
        }
        outr[c] = t_pack8(o);
      }
    }
  }
  if (want_dg) {
    __syncthreads();
    for (int i = threadIdx.x; i < E; i += blockDim.x) {
      atomicAdd(dgamma + i, s_dg[i]);
      if (!kRms && dbeta) atomicAdd(dbeta + i, s_db[i]);
    }
  }
}

template <bool kRms>
static int launch_norm_bwd(const void* x, const float* gamma, const void* dy, const void* dres, void* dx, float* dgamma,
                           float* dbeta, long long rows, int E, long long ldx, long long ldy, long long ldr, long long ldo,
                           float eps, cudaStream_t st) {
  if (!x || !gamma || !dy || !dx) return set_error(U2_ERR_ARG, "norm_bwd: null pointer");
  if (E <= 0 || (E & 7)) return set_error(U2_ERR_ARG, "norm_bwd: E must be a positive multiple of 8");
  if ((ldx & 7) || (ldy & 7) || (ldo & 7) || (dres && (ldr & 7))) return set_error(U2_ERR_ARG, "norm_bwd: row strides must be multiples of 8");
  if (rows <= 0) return U2_OK;
  const int need = (E / 8 + 31) / 32;
  long long blocks = (rows + 7) / 8;
  if (blocks > 132 * 2) blocks = 132 * 2;
  const size_t smem = dgamma ? (size_t)(kRms ? E : 2 * E) * sizeof(float) : 0;
#define U2_NB_CASE(MV)                                                                                                 \
  do {                                                                                                                 \
    if (smem > 48 * 1024) {                                                                                            \
      cudaError_t e = cudaFuncSetAttribute(norm_bwd_kernel<MV, kRms>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
      if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "norm_bwd smem: %s", cudaGetErrorString(e));                 \
    }                                                                                                                  \
    norm_bwd_kernel<MV, kRms><<<(unsigned)blocks, 256, smem, st>>>(CBF(x), gamma, CBF(dy), CBF(dres), BF(dx), dgamma, dbeta, \
                                                                   rows, E, ldx, ldy, ldr, ldo, eps);                  \
  } while (0)
  if (need <= 1) U2_NB_CASE(1);
  else if (need <= 2) U2_NB_CASE(2);
  else if (need <= 4) U2_NB_CASE(4);
  else if (need <= 8) U2_NB_CASE(8);
  else if (need <= 16) U2_NB_CASE(16);
  else if (need <= 32) U2_NB_CASE(32);
  else return set_error(U2_ERR_UNSUPPORTED, "norm_bwd: E=%d too large (max 8192)", E);
#undef U2_NB_CASE
  U2_CHECK_LAUNCH("norm_bwd");
  return U2_OK;
}

// ------------------------------------------------------------------------------------------------
// softmax backward: dS = P * (dP - sum(dP * P)) per row
// ------------------------------------------------------------------------------------------------
struct SmBwdArgs {
  const __nv_bfloat16* P;
  const float* dP;
  __nv_bfloat16* dS;
  long long p_s0, p_s1, p_s2, dp_s0, dp_s1, dp_s2, ds_s0, ds_s1, ds_s2;
  int n0, H, S, n, zero_pad_to;
};

template <int kGroup, int kMaxV>
__global__ void __launch_bounds__(kGroup == 32 ? 128 : kGroup)
softmax_bwd_kernel(const SmBwdArgs a) {
  constexpr int kRowsPerBlock = (kGroup == 32) ? 4 : 1;
  const int gl = threadIdx.x % kGroup;
  const long long row = (long long)blockIdx.x * kRowsPerBlock + threadIdx.x / kGroup;
  const long long total = (long long)a.n0 * a.H * a.S;
  __shared__ float red[8];
  const bool active = row < total;
  const long long r = active ? row : 0;
  const int i2 = (int)(r % a.S);
  const int i1 = (int)((r / a.S) % a.H);
  const long long i0 = r / ((long long)a.S * a.H);
  const __nv_bfloat16* P = a.P + i0 * a.p_s0 + i1 * a.p_s1 + i2 * a.p_s2;
  const float* dP = a.dP + i0 * a.dp_s0 + i1 * a.dp_s1 + i2 * a.dp_s2;
  __nv_bfloat16* dS = a.dS + i0 * a.ds_s0 + i1 * a.ds_s1 + i2 * a.ds_s2;
  float p[kMaxV], g[kMaxV];
  float dot = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxV; ++i) {
    const int j = i * kGroup + gl;
    p[i] = 0.f;
    g[i] = 0.f;
    if (active && j < a.n) {
      p[i] = __bfloat162float(P[j]);
      g[i] = dP[j];
    }
    dot += p[i] * g[i];
  }
  dot = t_wsum(dot);
  if (kGroup > 32) {
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dot;
    __syncthreads();
    dot = 0.f;
#pragma unroll
    for (int w = 0; w < kGroup / 32; ++w) dot += red[w];
  }
  if (!active) return;
#pragma unroll
  for (int i = 0; i < kMaxV; ++i) {
    const int j = i * kGroup + gl;
    if (j < a.n) dS[j] = __float2bfloat16(p[i] * (g[i] - dot));
    else if (j < a.zero_pad_to) dS[j] = __float2bfloat16(0.f);
  }
}

// long plain rows (ViT, 2049 keys): one warp per row, 16-byte vector loads of P (8 bf16) and dP (2 x float4)
template <int kMaxV8>
__global__ void __launch_bounds__(256)
softmax_bwd_warp_vec_kernel(const SmBwdArgs a) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long total = (long long)a.n0 * a.H * a.S;
  if (row >= total) return;
  const int i2 = (int)(row % a.S);
  const int i1 = (int)((row / a.S) % a.H);
  const long long i0 = row / ((long long)a.S * a.H);
  const uint4* P = reinterpret_cast<const uint4*>(a.P + i0 * a.p_s0 + i1 * a.p_s1 + i2 * a.p_s2);
  const float4* dP = reinterpret_cast<const float4*>(a.dP + i0 * a.dp_s0 + i1 * a.dp_s1 + i2 * a.dp_s2);
  uint4* dS = reinterpret_cast<uint4*>(a.dS + i0 * a.ds_s0 + i1 * a.ds_s1 + i2 * a.ds_s2);
  const int span = max(a.n, a.zero_pad_to);
  const int nv = span >> 3;  // groups of 8 (span % 8 == 0 checked by the host)
  float p[kMaxV8][8], g[kMaxV8][8];
  float dot = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxV8; ++i) {
    const int c = i * 32 + lane;
    if (c < nv) {
      t_unpack8(P[c], p[i]);
      const float4 g0 = dP[2 * c], g1 = dP[2 * c + 1];
      g[i][0] = g0.x; g[i][1] = g0.y; g[i][2] = g0.z; g[i][3] = g0.w;
      g[i][4] = g1.x; g[i][5] = g1.y; g[i][6] = g1.z; g[i][7] = g1.w;
#pragma unroll
      for (int j = 0; j < 8; ++j) dot += (c * 8 + j < a.n) ? p[i][j] * g[i][j] : 0.f;
    }
  }
  dot = t_wsum(dot);
#pragma unroll
  for (int i = 0; i < kMaxV8; ++i) {
    const int c = i * 32 + lane;
    if (c < nv) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (c * 8 + j < a.n) ? p[i][j] * (g[i][j] - dot) : 0.f;
      dS[c] = t_pack8(o);
    }
  }
}

// rows longer than 8192 (DiffTS over many frames): one CTA per row, two passes
__global__ void __launch_bounds__(256)
softmax_bwd_long_kernel(const SmBwdArgs a) {
  const long long r = blockIdx.x;
  const int i2 = (int)(r % a.S);
  const int i1 = (int)((r / a.S) % a.H);
  const long long i0 = r / ((long long)a.S * a.H);
  const __nv_bfloat16* P = a.P + i0 * a.p_s0 + i1 * a.p_s1 + i2 * a.p_s2;
  const float* dP = a.dP + i0 * a.dp_s0 + i1 * a.dp_s1 + i2 * a.dp_s2;
  __nv_bfloat16* dS = a.dS + i0 * a.ds_s0 + i1 * a.ds_s1 + i2 * a.ds_s2;
  __shared__ float red[8];
  float dot = 0.f;
  for (int j = threadIdx.x; j < a.n; j += 256) dot += __bfloat162float(P[j]) * dP[j];
  dot = t_wsum(dot);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dot;
  __syncthreads();
  dot = 0.f;
  for (int w = 0; w < 8; ++w) dot += red[w];
  const int span = max(a.n, a.zero_pad_to);
  for (int j = threadIdx.x; j < span; j += 256)
    dS[j] = __float2bfloat16(j < a.n ? __bfloat162float(P[j]) * (dP[j] - dot) : 0.f);
}

// relative-bias gradient: one CTA per (batch, head); diagonal sums in shared memory first
__global__ void __launch_bounds__(256)
relbias_grad_kernel(const __nv_bfloat16* __restrict__ dS, float* __restrict__ drel, int H, int S, int n, long long s0,
                    long long s1, long long s2, int rel_max) {
  extern __shared__ float tab[];  // [S + n - 1]
  const int i1 = blockIdx.x;
  const long long i0 = blockIdx.y;
  const int nd = S + n - 1;
  for (int d = threadIdx.x; d < nd; d += blockDim.x) tab[d] = 0.f;
  __syncthreads();
  const __nv_bfloat16* base = dS + i0 * s0 + i1 * s1;
  for (int i2 = 0; i2 < S; ++i2)
    for (int j = threadIdx.x; j < n; j += blockDim.x)
      atomicAdd(&tab[j - i2 + S - 1], __bfloat162float(base[i2 * s2 + j]));
  __syncthreads();
  for (int d = threadIdx.x; d < nd; d += blockDim.x)
    atomicAdd(drel + (long long)(d - (S - 1) + rel_max - 1) * H + i1, tab[d]);
}

// ------------------------------------------------------------------------------------------------
// D[b, h, s] = sum_d a[b, s, h, d] * c[b, s, h, d]  (rowsum(dO * O) of the attention backward); warp per (b, s, h)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
rowdot_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ c, float* __restrict__ out, int B, int S,
              int H, int dh, long long a_sb, long long a_ss, long long a_sh, long long c_sb, long long c_ss, long long c_sh) {
  const int lane = threadIdx.x & 31;
  const long long total = (long long)B * S * H;
  for (long long item = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); item < total; item += (long long)gridDim.x * 8) {
    const int h = (int)(item % H);
    const int s = (int)((item / H) % S);
    const long long b = item / ((long long)H * S);
    const __nv_bfloat16* pa = a + b * a_sb + s * a_ss + h * a_sh;
    const __nv_bfloat16* pc = c + b * c_sb + s * c_ss + h * c_sh;
    float d = 0.f;
    for (int e = lane * 2; e < dh; e += 64) {
      const float2 x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(pa + e));
      const float2 y = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(pc + e));
      d += x.x * y.x + x.y * y.y;
    }
    d = t_wsum(d);
    if (lane == 0) out[(b * H + h) * S + s] = d;
  }
}

// ------------------------------------------------------------------------------------------------
// temporal attention backward: one CTA per (head, token, batch); everything of the C x C problem in smem
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
temporal_attention_bwd_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ dout,
                              __nv_bfloat16* __restrict__ dqkv, int C, int N, int H, int dh, long long ld_qkv,
                              long long ld_dout, long long ld_dqkv, float scale, const float* __restrict__ rel_bias,
                              float* __restrict__ drel, int rel_max) {
  extern __shared__ __align__(16) unsigned char t_sm[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(t_sm);
  __nv_bfloat16* sK = sQ + (size_t)C * dh;
  __nv_bfloat16* sV = sK + (size_t)C * dh;
  __nv_bfloat16* sG = sV + (size_t)C * dh;           // dout rows
  float* sP = reinterpret_cast<float*>(sG + (size_t)C * dh);  // [C][C]
  float* sD = sP + (size_t)C * C;                              // dS [C][C]
  const int h = blockIdx.x, n = blockIdx.y, b = blockIdx.z;
  const int E = H * dh;
  const int nvec = dh >> 3;
  for (int i = threadIdx.x; i < C * nvec; i += blockDim.x) {
    const int c = i / nvec, v = i - c * nvec;
    const long long row = ((long long)b * C + c) * N + n;
    const __nv_bfloat16* base = qkv + row * ld_qkv + h * dh;
    reinterpret_cast<uint4*>(sQ + (size_t)c * dh)[v] = reinterpret_cast<const uint4*>(base)[v];
    reinterpret_cast<uint4*>(sK + (size_t)c * dh)[v] = reinterpret_cast<const uint4*>(base + E)[v];
    reinterpret_cast<uint4*>(sV + (size_t)c * dh)[v] = reinterpret_cast<const uint4*>(base + 2 * E)[v];
    reinterpret_cast<uint4*>(sG + (size_t)c * dh)[v] = reinterpret_cast<const uint4*>(dout + row * ld_dout + h * dh)[v];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  // phase 1: P and dS rows (warp per query frame c)
  for (int c = warp; c < C; c += nw) {
    float mx = -INFINITY;
    for (int j = 0; j < C; ++j) {
      float d = 0.f, g = 0.f;
      for (int e = lane * 2; e < dh; e += 64) {
        const float2 qq = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sQ + (size_t)c * dh + e));
        const float2 kk = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sK + (size_t)j * dh + e));
        const float2 gg = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sG + (size_t)c * dh + e));
        const float2 vv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sV + (size_t)j * dh + e));
        d += qq.x * kk.x + qq.y * kk.y;
        g += gg.x * vv.x + gg.y * vv.y;
      }
      d = t_wsum(d) * scale;
      g = t_wsum(g);
      if (rel_bias) d += __ldg(rel_bias + (long long)(j - c + rel_max - 1) * H + h);
      if (lane == 0) {
        sP[c * C + j] = d;
        sD[c * C + j] = g;  // dP for now
      }
      mx = fmaxf(mx, d);
    }
    __syncwarp();
    float ssum = 0.f;
    for (int j = lane; j < C; j += 32) {
      const float e = __expf(sP[c * C + j] - mx);
      sP[c * C + j] = e;
      ssum += e;
    }
    ssum = t_wsum(ssum);
    const float inv = 1.f / ssum;
    float dot = 0.f;
    for (int j = lane; j < C; j += 32) {
      const float p = sP[c * C + j] * inv;
      sP[c * C + j] = p;
      dot += p * sD[c * C + j];
    }
    dot = t_wsum(dot);
    for (int j = lane; j < C; j += 32) sD[c * C + j] = sP[c * C + j] * (sD[c * C + j] - dot);
  }
  __syncthreads();
  // phase 2: dq_c = scale * sum_j dS[c][j] k_j ; dk_j = scale * sum_c dS[c][j] q_c ; dv_j = sum_c P[c][j] dO_c
  for (int t = warp; t < C; t += nw) {
    const long long row = ((long long)b * C + t) * N + n;
    __nv_bfloat16* o = dqkv + row * ld_dqkv + h * dh;
    for (int e = lane * 2; e < dh; e += 64) {
      float qx = 0.f, qy = 0.f, kx = 0.f, ky = 0.f, vx = 0.f, vy = 0.f;
      for (int u = 0; u < C; ++u) {
        const float ds_tu = sD[t * C + u], ds_ut = sD[u * C + t], p_ut = sP[u * C + t];
        const float2 kk = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sK + (size_t)u * dh + e));
        const float2 qq = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sQ + (size_t)u * dh + e));
        const float2 gg = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sG + (size_t)u * dh + e));
        qx += ds_tu * kk.x; qy += ds_tu * kk.y;
        kx += ds_ut * qq.x; ky += ds_ut * qq.y;
        vx += p_ut * gg.x;  vy += p_ut * gg.y;
      }
      *reinterpret_cast<__nv_bfloat162*>(o + e) = __floats2bfloat162_rn(qx * scale, qy * scale);
      *reinterpret_cast<__nv_bfloat162*>(o + E + e) = __floats2bfloat162_rn(kx * scale, ky * scale);
      *reinterpret_cast<__nv_bfloat162*>(o + 2 * E + e) = __floats2bfloat162_rn(vx, vy);
    }
  }
  // relative-bias gradient: diagonal sums of dS
  if (drel) {
    for (int d = threadIdx.x; d < 2 * C - 1; d += blockDim.x) {
      const int off = d - (C - 1);  // j - c
      float s = 0.f;
      for (int c = max(0, -off); c < min(C, C - off); ++c) s += sD[c * C + c + off];
      atomicAdd(drel + (long long)(off + rel_max - 1) * H + h, s);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// RoPE (+ per-head RMSNorm) backward, in place on the gradient buffer; warp per (row, head)
// ------------------------------------------------------------------------------------------------
struct RopeBwdArgs {
  __nv_bfloat16* dx;
  const __nv_bfloat16* x_raw;
  long long rows, ld;
  int dh, n_q_heads, n_k_heads;
  const float* q_norm_w;
  const float* k_norm_w;
  float eps;
  const float* inv_freq;
  int pos0, pos_div, pos_mod;
  float* dq_norm_w;
  float* dk_norm_w;
};

__global__ void __launch_bounds__(256)
rope_bwd_kernel(const RopeBwdArgs a) {
  extern __shared__ float s_dw[];  // [2][dh] when a norm weight is trained
  const bool any_dw = a.dq_norm_w || a.dk_norm_w;
  if (any_dw) {
    for (int i = threadIdx.x; i < 2 * a.dh; i += blockDim.x) s_dw[i] = 0.f;
    __syncthreads();
  }
  const int heads = a.n_q_heads + a.n_k_heads;
  const int lane = threadIdx.x & 31;
  const int half = a.dh >> 1;
  for (long long item = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); item < a.rows * heads; item += (long long)gridDim.x * 8) {
    const long long row = item / heads;
    const int head = (int)(item - row * heads);
    __nv_bfloat16* g = a.dx + row * a.ld + (long long)head * a.dh;
    const int pos = a.pos0 + (int)((row / a.pos_div) % a.pos_mod);
    const bool is_q = head < a.n_q_heads;
    const float* nw = is_q ? a.q_norm_w : a.k_norm_w;
    float* sdw = s_dw + (is_q ? 0 : a.dh);
    const bool want_dw = is_q ? (a.dq_norm_w != nullptr) : (a.dk_norm_w != nullptr);
    const __nv_bfloat16* xr = a.x_raw ? a.x_raw + row * a.ld + (long long)head * a.dh : nullptr;
    float rstd = 1.f;
    if (nw) {
      float ss = 0.f;
      for (int e = lane; e < a.dh; e += 32) {
        const float v = __bfloat162float(xr[e]);
        ss += v * v;
      }
      rstd = rsqrtf(t_wsum(ss) / a.dh + a.eps);
    }
    // un-rotate, then (optionally) the RMSNorm backward; two passes because the norm needs sum(g * w * x)
    float dot = 0.f;
    for (int i = lane; i < half; i += 32) {
      const float d1 = __bfloat162float(g[i]), d2 = __bfloat162float(g[i + half]);
      float sn, cs;
      sincosf((float)pos * a.inv_freq[i], &sn, &cs);
      const float n1 = d1 * cs + d2 * sn, n2 = d2 * cs - d1 * sn;
      if (nw) {
        const float x1 = __bfloat162float(xr[i]), x2 = __bfloat162float(xr[i + half]);
        dot += n1 * nw[i] * x1 + n2 * nw[i + half] * x2;
        if (want_dw) {
          atomicAdd(&sdw[i], n1 * x1 * rstd);
          atomicAdd(&sdw[i + half], n2 * x2 * rstd);
        }
      }
      // keep the un-rotated gradient in place for the second pass (bf16 rounding here matches an unfused chain)
      g[i] = __float2bfloat16(n1);
      g[i + half] = __float2bfloat16(n2);
    }
    if (nw) {
      dot = t_wsum(dot);
      const float k = dot * rstd * rstd * rstd / a.dh;
      __syncwarp();
      for (int e = lane; e < a.dh; e += 32) {
        const float n = __bfloat162float(g[e]);
        g[e] = __float2bfloat16(rstd * n * nw[e] - __bfloat162float(xr[e]) * k);
      }
    }
  }
  if (any_dw) {
    __syncthreads();
    for (int i = threadIdx.x; i < a.dh; i += blockDim.x) {
      if (a.dq_norm_w) atomicAdd(a.dq_norm_w + i, s_dw[i]);
      if (a.dk_norm_w) atomicAdd(a.dk_norm_w + i, s_dw[a.dh + i]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// pooling backward
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
spp_pool_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx, long long frames, int g0, int g1,
                    int g2, int ps, int E, long long in_frame_stride, long long in_off, long long ldx,
                    long long rows_per_frame, int sequence) {
  const int nvec = E >> 3;
  const long long total = frames * rows_per_frame * nvec;
  const int o0 = g0 / ps, o1 = g1 / ps, o2 = g2 / ps;
  const long long ntok = (long long)g0 * g1 * g2;
  const int k = ps * ps * ps;
  const long long n_out = sequence ? ntok / k : (long long)o0 * o1 * o2;
  const float inv = 1.f / k;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % nvec);
    const long long t = idx / nvec;
    const long long r = t % rows_per_frame;
    const long long f = t / rows_per_frame;
    const long long tok = r - in_off;
    float o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (tok >= 0 && tok < ntok) {
      long long po = -1;
      if (sequence) {
        if (tok / k < n_out) po = tok / k;
      } else {
        const int a2 = (int)(tok % g2), a1 = (int)((tok / g2) % g1), a0 = (int)(tok / ((long long)g1 * g2));
        if (a0 / ps < o0 && a1 / ps < o1 && a2 / ps < o2) po = ((long long)(a0 / ps) * o1 + a1 / ps) * o2 + a2 / ps;
      }
      if (po >= 0) {
        t_unpack8(reinterpret_cast<const uint4*>(dy + (f * n_out + po) * E)[c], o);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] *= inv;
      }
    }
    reinterpret_cast<uint4*>(dx + (f * in_frame_stride + r) * ldx)[c] = t_pack8(o);
  }
}

// multi-scale pooling backward, pass 1 (dynamic gate only): ws[b][k] += sum dy_k . pool_k(x)  (k = 0, 1, 2)
__global__ void __launch_bounds__(256)
msp_bwd_dot_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, float* __restrict__ ws, int K,
                   int E, int rows_per_block) {
  const int b = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(K, r0 + rows_per_block);
  const int nvec = E >> 3;
  const int k2 = (K >= 2) ? K / 2 : 0, k4 = (K >= 4) ? K / 4 : 0;
  const int n_out = K + k2 + k4;
  float p[3] = {0.f, 0.f, 0.f};
  for (int c = threadIdx.x; c < nvec; c += blockDim.x) {
    for (int r = r0; r < r1; ++r) {
      float v[8], g[8];
      t_unpack8(reinterpret_cast<const uint4*>(x + ((long long)b * K + r) * E)[c], v);
      t_unpack8(reinterpret_cast<const uint4*>(dy + ((long long)b * n_out + r) * E)[c], g);
      float d = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) d += v[j] * g[j];
      p[0] += d;
      if (r < k2 * 2) {
        t_unpack8(reinterpret_cast<const uint4*>(dy + ((long long)b * n_out + K + r / 2) * E)[c], g);
        d = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) d += v[j] * g[j];
        p[1] += 0.5f * d;
      }
      if (r < k4 * 4) {
        t_unpack8(reinterpret_cast<const uint4*>(dy + ((long long)b * n_out + K + k2 + r / 4) * E)[c], g);
        d = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) d += v[j] * g[j];
        p[2] += 0.25f * d;
      }
    }
  }
  __shared__ float red[3][8];
#pragma unroll
  for (int k = 0; k < 3; ++k) p[k] = t_wsum(p[k]);
  if ((threadIdx.x & 31) == 0)
    for (int k = 0; k < 3; ++k) red[k][threadIdx.x >> 5] = p[k];
  __syncthreads();
  if (threadIdx.x < 3) {
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[threadIdx.x][w];
    atomicAdd(&ws[b * 8 + threadIdx.x], s);
  }
}

// pass 2: dx rows (+ gate_w gradient)
__global__ void __launch_bounds__(256)
msp_bwd_write_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx,
                     const float* __restrict__ gate_w, const float* __restrict__ logits, const float* __restrict__ ws,
                     float* __restrict__ dgate_w, int K, int E, int dynamic, int rows_per_block) {
  const int b = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(K, r0 + rows_per_block);
  const int nvec = E >> 3;
  const int k2 = (K >= 2) ? K / 2 : 0, k4 = (K >= 4) ? K / 4 : 0;
  const int n_out = K + k2 + k4;
  const int n2 = k2 * 2, n4 = k4 * 4;
  float w[3] = {1.f, 1.f, 1.f}, dl[3] = {0.f, 0.f, 0.f};
  if (dynamic) {
    const float l0 = logits[b * 3 + 0], l1 = k2 ? logits[b * 3 + 1] : -INFINITY, l2 = k4 ? logits[b * 3 + 2] : -INFINITY;
    const float m = fmaxf(l0, fmaxf(l1, l2));
    const float e0 = __expf(l0 - m), e1 = k2 ? __expf(l1 - m) : 0.f, e2 = k4 ? __expf(l2 - m) : 0.f;
    const float inv = 1.f / (e0 + e1 + e2);
    w[0] = e0 * inv; w[1] = e1 * inv; w[2] = e2 * inv;
    const float dw0 = ws[b * 8 + 0], dw1 = ws[b * 8 + 1], dw2 = ws[b * 8 + 2];
    const float dot = w[0] * dw0 + w[1] * dw1 + w[2] * dw2;
    dl[0] = w[0] * (dw0 - dot);
    dl[1] = w[1] * (dw1 - dot);
    dl[2] = w[2] * (dw2 - dot);
  }
  // d(logit_k)/dx_r = gate_w / n_k for r < n_k ; d(logit_k)/d(gate_w) = sum_{r < n_k} x_r / n_k
  const float c0 = dl[0] / K, c1 = n2 ? dl[1] / n2 : 0.f, c2 = n4 ? dl[2] / n4 : 0.f;
  for (int c = threadIdx.x; c < nvec; c += blockDim.x) {
    float gw[8] = {0, 0, 0, 0, 0, 0, 0, 0}, dgw[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (dynamic) t_load8f(gate_w + c * 8, gw);
    for (int r = r0; r < r1; ++r) {
      float g[8], o[8];
      t_unpack8(reinterpret_cast<const uint4*>(dy + ((long long)b * n_out + r) * E)[c], g);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = w[0] * g[j];
      float coef = c0;
      if (r < n2) {
        t_unpack8(reinterpret_cast<const uint4*>(dy + ((long long)b * n_out + K + r / 2) * E)[c], g);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += 0.5f * w[1] * g[j];
        coef += c1;
      }
      if (r < n4) {
        t_unpack8(reinterpret_cast<const uint4*>(dy + ((long long)b * n_out + K + k2 + r / 4) * E)[c], g);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += 0.25f * w[2] * g[j];
        coef += c2;
      }
      if (dynamic) {
        float v[8];
        t_unpack8(reinterpret_cast<const uint4*>(x + ((long long)b * K + r) * E)[c], v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          o[j] += coef * gw[j];
          dgw[j] += coef * v[j];
        }
      }
      reinterpret_cast<uint4*>(dx + ((long long)b * K + r) * E)[c] = t_pack8(o);
    }
    if (dynamic && dgate_w) {
#pragma unroll
      for (int j = 0; j < 8; ++j) atomicAdd(dgate_w + c * 8 + j, dgw[j]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// embedding / selection scatter-add, GQA group sum
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
embed_scatter_add_kernel(const long long* __restrict__ ids, const __nv_bfloat16* __restrict__ drows, __nv_bfloat16* dtable,
                         __nv_bfloat16* dvis, int B, int L, int E, int n_vis, long long vocab) {
  const int nvec = E >> 3;
  const long long total = (long long)B * L * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % nvec);
    const long long bl = idx / nvec;
    const int l = (int)(bl % L);
    const int b = (int)(bl / L);
    const uint4 v = reinterpret_cast<const uint4*>(drows + bl * E)[c];
    if (dvis && l >= 1 && l <= n_vis) {
      reinterpret_cast<uint4*>(dvis + ((long long)b * n_vis + (l - 1)) * E)[c] = v;
    } else if (dtable) {
      long long id = ids[bl];
      if (id < 0) id = 0;
      if (id >= vocab) id = vocab - 1;
      __nv_bfloat162* dst = reinterpret_cast<__nv_bfloat162*>(dtable + id * E + c * 8);
      const __nv_bfloat162* src = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) atomicAdd(dst + j, src[j]);
    }
  }
}

__global__ void __launch_bounds__(256)
group_sum_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, long long rows, int heads, int G,
                 int dh, long long ld_in, long long ld_out) {
  const int nvec = dh >> 3;
  const long long total = rows * heads * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % nvec);
    const long long t = idx / nvec;
    const int h = (int)(t % heads);
    const long long r = t / heads;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int g = 0; g < G; ++g) {
      float v[8];
      t_unpack8(reinterpret_cast<const uint4*>(in + r * ld_in + (long long)(h * G + g) * dh)[c], v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
    reinterpret_cast<uint4*>(out + r * ld_out + (long long)h * dh)[c] = t_pack8(acc);
  }
}

// ------------------------------------------------------------------------------------------------
// loss heads
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ce_bwd_kernel(const float* __restrict__ logits, __nv_bfloat16* __restrict__ dlogits, const float* __restrict__ lse,
              const long long* __restrict__ labels, const float* __restrict__ coef, long long R, int V, long long ld_in,
              long long ld_out) {
  const int nvec = V >> 3;
  const long long total = R * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / nvec;
    const int c = (int)(idx - r * nvec);
    const float cf = coef[r];
    float o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (cf != 0.f) {
      float v[8];
      t_load8f(logits + r * ld_in + c * 8, v);
      const float l = lse[r];
      const long long lab = labels[r] - (long long)c * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = cf * (__expf(v[j] - l) - (lab == j ? 1.f : 0.f));
    }
    reinterpret_cast<uint4*>(dlogits + r * ld_out)[c] = t_pack8(o);
  }
}

__global__ void __launch_bounds__(1024)
dpo_loss_kernel(const float* __restrict__ per_tok, const float* __restrict__ ref_sum, const uint8_t* __restrict__ mask,
                float* __restrict__ out, float* __restrict__ coef, int P, int L, float beta) {
  __shared__ float s_loss[32], s_acc[32], s_mar[32];
  const int p = threadIdx.x;
  float loss = 0.f, acc = 0.f, mar = 0.f;
  if (p < P) {
    float pc = 0.f, pr = 0.f;
    for (int l = 0; l < L; ++l) {
      if (mask[(long long)p * L + l]) pc += per_tok[(long long)p * L + l];
      if (mask[(long long)(P + p) * L + l]) pr += per_tok[(long long)(P + p) * L + l];
    }
    const float rc = ref_sum[p], rr = ref_sum[P + p];
    const float x = beta * ((pc - pr) - (rc - rr));
    // -logsigmoid(x) = softplus(-x)
    loss = (x > 0.f ? 0.f : -x) + log1pf(__expf(-fabsf(x)));
    const float sg = 1.f / (1.f + __expf(x));  // sigmoid(-x) = -dloss/dx
    const float cchosen = beta * sg / P;       // -dloss/dlogp on chosen tokens
    for (int l = 0; l < L; ++l) {
      coef[(long long)p * L + l] = mask[(long long)p * L + l] ? cchosen : 0.f;
      coef[(long long)(P + p) * L + l] = mask[(long long)(P + p) * L + l] ? -cchosen : 0.f;
    }
    const float rwc = beta * (pc - rc), rwr = beta * (pr - rr);
    acc = rwc > rwr ? 1.f : 0.f;
    mar = rwc - rwr;
  }
  loss = t_wsum(loss); acc = t_wsum(acc); mar = t_wsum(mar);
  if ((threadIdx.x & 31) == 0) { s_loss[threadIdx.x >> 5] = loss; s_acc[threadIdx.x >> 5] = acc; s_mar[threadIdx.x >> 5] = mar; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f, c = 0.f;
    for (int w = 0; w < (int)((blockDim.x + 31) >> 5); ++w) { a += s_loss[w]; b += s_acc[w]; c += s_mar[w]; }
    out[0] = a / P; out[1] = b / P; out[2] = c / P;
  }
}

// ------------------------------------------------------------------------------------------------
// optimizer: fused AdamW on a flat shard, gradient norm, casts
// ------------------------------------------------------------------------------------------------
struct AdamArgs {
  float lr, beta1, beta2, eps, wd, bc1, bc2_rsqrt;
  const float* grad_scale;
  uint32_t sr_key;      // stochastic rounding of bf16 moments: hash key of (seed, step)
  long long index0;     // global index of element 0 of this call
};

// MurmurHash3's fmix32 finaliser: the counter-based hash of the LoRA dropout masks (lora.cu)
__host__ __device__ __forceinline__ uint32_t adam_fmix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}

// bf16 bits of x rounded stochastically with the 16 random bits r: up (away from zero) with probability
// (|x| - |trunc(x)|) / ulp, so E[SR(x)] = x. Round-to-nearest would make a moment stall whenever its update is below half
// a bf16 ulp (v + (1 - beta2)(g^2 - v) with beta2 = 0.999 needs g^2 > ~3 v to move v at all). Inf / NaN round to nearest.
__device__ __forceinline__ uint32_t bf16_sr_bits(float x, uint32_t r) {
  const uint32_t u = __float_as_uint(x);
  if ((u & 0x7F800000u) == 0x7F800000u) return __bfloat16_as_ushort(__float2bfloat16_rn(x));
  return (u + (r & 0xFFFFu)) >> 16;
}

__device__ __forceinline__ void ld4(const float* p, long long i, float (&o)[4]) {
  const float4 t = reinterpret_cast<const float4*>(p)[i];
  o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w;
}
__device__ __forceinline__ void ld4(const __nv_bfloat16* p, long long i, float (&o)[4]) {
  const uint2 t = reinterpret_cast<const uint2*>(p)[i];
  const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.x));
  const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.y));
  o[0] = lo.x; o[1] = lo.y; o[2] = hi.x; o[3] = hi.y;
}
__device__ __forceinline__ void st4(float* p, long long i, const float (&o)[4]) {
  reinterpret_cast<float4*>(p)[i] = make_float4(o[0], o[1], o[2], o[3]);
}
__device__ __forceinline__ void st4(__nv_bfloat16* p, long long i, const float (&o)[4]) {
  uint2 t;
  *reinterpret_cast<__nv_bfloat162*>(&t.x) = __floats2bfloat162_rn(o[0], o[1]);
  *reinterpret_cast<__nv_bfloat162*>(&t.y) = __floats2bfloat162_rn(o[2], o[3]);
  reinterpret_cast<uint2*>(p)[i] = t;
}

// fp32 master + bf16 moments (the single-GPU memory mode: 8 instead of 12 bytes of optimizer state per parameter).
// m and v are stored with stochastic rounding; the random bits of element e are fmix32(fmix32(key ^ lo32(e)) ^ hi32(e))
// with e the GLOBAL index (index0 + local index): its low half rounds m, its high half rounds v. They depend on (seed,
// step, e) only, so any split of the buffer into calls (ZeRO-1 slices, buckets) stores the same bits.
__global__ void __launch_bounds__(256)
adamw_mom16_kernel(float* __restrict__ master, __nv_bfloat16* __restrict__ m, __nv_bfloat16* __restrict__ v,
                   const __nv_bfloat16* __restrict__ grad, __nv_bfloat16* __restrict__ p_bf16, long long n, const AdamArgs a) {
  const float gs = a.grad_scale ? *a.grad_scale : 1.f;
  const long long nvec = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float g[4], w[4], mm[4], vv[4];
    uint32_t mb[4], vb[4];
    ld4(grad, i, g); ld4(master, i, w); ld4(m, i, mm); ld4(v, i, vv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gj = g[j] * gs;
      mm[j] = a.beta1 * mm[j] + (1.f - a.beta1) * gj;
      vv[j] = a.beta2 * vv[j] + (1.f - a.beta2) * gj * gj;
      const float denom = sqrtf(vv[j]) * a.bc2_rsqrt + a.eps;
      w[j] = w[j] * (1.f - a.lr * a.wd) - (a.lr / a.bc1) * (mm[j] / denom);
      const unsigned long long e = (unsigned long long)(a.index0 + 4 * i + j);
      const uint32_t h = adam_fmix32(adam_fmix32(a.sr_key ^ (uint32_t)e) ^ (uint32_t)(e >> 32));
      mb[j] = bf16_sr_bits(mm[j], h);
      vb[j] = bf16_sr_bits(vv[j], h >> 16);
    }
    st4(master, i, w);
    reinterpret_cast<uint2*>(m)[i] = make_uint2(mb[0] | (mb[1] << 16), mb[2] | (mb[3] << 16));
    reinterpret_cast<uint2*>(v)[i] = make_uint2(vb[0] | (vb[1] << 16), vb[2] | (vb[3] << 16));
    if (p_bf16) st4(p_bf16, i, w);
  }
}

template <bool kGradF32>
__global__ void __launch_bounds__(256)
adamw_kernel(float* __restrict__ master, float* __restrict__ m, float* __restrict__ v, const void* __restrict__ grad,
             __nv_bfloat16* __restrict__ p_bf16, float* __restrict__ p_f32, long long n, const AdamArgs a) {
  const float gs = a.grad_scale ? *a.grad_scale : 1.f;
  const long long nvec = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float g[4];
    if (kGradF32) {
      const float4 t = reinterpret_cast<const float4*>(grad)[i];
      g[0] = t.x; g[1] = t.y; g[2] = t.z; g[3] = t.w;
    } else {
      const uint2 t = reinterpret_cast<const uint2*>(grad)[i];
      const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.x));
      const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.y));
      g[0] = lo.x; g[1] = lo.y; g[2] = hi.x; g[3] = hi.y;
    }
    float4 w4 = reinterpret_cast<float4*>(master)[i], m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i];
    float w[4] = {w4.x, w4.y, w4.z, w4.w}, mm[4] = {m4.x, m4.y, m4.z, m4.w}, vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gj = g[j] * gs;
      mm[j] = a.beta1 * mm[j] + (1.f - a.beta1) * gj;
      vv[j] = a.beta2 * vv[j] + (1.f - a.beta2) * gj * gj;
      const float denom = sqrtf(vv[j]) * a.bc2_rsqrt + a.eps;
      w[j] = w[j] * (1.f - a.lr * a.wd) - (a.lr / a.bc1) * (mm[j] / denom);
    }
    reinterpret_cast<float4*>(master)[i] = make_float4(w[0], w[1], w[2], w[3]);
    reinterpret_cast<float4*>(m)[i] = make_float4(mm[0], mm[1], mm[2], mm[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    if (p_bf16) {
      uint2 o;
      *reinterpret_cast<__nv_bfloat162*>(&o.x) = __floats2bfloat162_rn(w[0], w[1]);
      *reinterpret_cast<__nv_bfloat162*>(&o.y) = __floats2bfloat162_rn(w[2], w[3]);
      reinterpret_cast<uint2*>(p_bf16)[i] = o;
    }
    if (p_f32) {
      // vector parameters are kept bf16-VALUED in their fp32 mirrors (what the bf16 module parameter holds)
      reinterpret_cast<float4*>(p_f32)[i] =
          make_float4(__bfloat162float(__float2bfloat16(w[0])), __bfloat162float(__float2bfloat16(w[1])),
                      __bfloat162float(__float2bfloat16(w[2])), __bfloat162float(__float2bfloat16(w[3])));
    }
  }
}

template <bool kF32>
__global__ void __launch_bounds__(256)
sumsq_kernel(const void* __restrict__ x, float* __restrict__ out, long long n) {
  float s = 0.f;
  if (kF32) {
    const long long nvec = n >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
      const float4 t = reinterpret_cast<const float4*>(x)[i];
      s += t.x * t.x + t.y * t.y + t.z * t.z + t.w * t.w;
    }
  } else {
    const long long nvec = n >> 3;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
      float v[8];
      t_unpack8(reinterpret_cast<const uint4*>(x)[i], v);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[j] * v[j];
    }
  }
  __shared__ float red[8];
  s = t_wsum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    atomicAdd(out, t);
  }
}

__global__ void __launch_bounds__(256)
add_bf16_kernel(__nv_bfloat16* __restrict__ dst, const __nv_bfloat16* __restrict__ src, long long nvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8];
    t_unpack8(reinterpret_cast<const uint4*>(dst)[i], a);
    t_unpack8(reinterpret_cast<const uint4*>(src)[i], b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    reinterpret_cast<uint4*>(dst)[i] = t_pack8(a);
  }
}

__global__ void __launch_bounds__(256)
cast_f32_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = __float2bfloat16(in[i]);
}
__global__ void __launch_bounds__(256)
cast_bf16_f32_kernel(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = __bfloat162float(in[i]);
}

}  // namespace u2

using namespace u2;

extern "C" U2_API int u2_transpose_bf16(const void* in, void* out, int32_t rows, int32_t cols, int64_t ld_in, int64_t ld_out,
                                        int32_t batch, int64_t in_bs, int64_t out_bs, void* stream) {
  if (!in || !out) return set_error(U2_ERR_ARG, "transpose: null pointer");
  if (rows <= 0 || cols <= 0 || batch <= 0) return U2_OK;
  if (batch > 65535 || (rows + 31) / 32 > 65535) return set_error(U2_ERR_UNSUPPORTED, "transpose: grid too large");
  dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32), (unsigned)batch);
  transpose_kernel<<<grid, 256, 0, ST(stream)>>>(CBF(in), BF(out), rows, cols, ld_in, ld_out, in_bs, out_bs);
  U2_CHECK_LAUNCH("transpose");
  return U2_OK;
}

extern "C" U2_API int u2_colsum_bf16(const void* x, float* out, int64_t rows, int64_t cols, int64_t ld, void* stream) {
  if (!x || !out) return set_error(U2_ERR_ARG, "colsum: null pointer");
  if (cols <= 0 || (cols & 7) || (ld & 7)) return set_error(U2_ERR_ARG, "colsum: cols / ld must be multiples of 8");
  if (rows <= 0) return U2_OK;
  const long long gx = (cols + 255) / 256;
  long long gy = (132LL * 4 + gx - 1) / gx;
  long long rpb = (rows + gy - 1) / gy;
  if (rpb < 64) rpb = 64;
  gy = (rows + rpb - 1) / rpb;
  if (gx > 0x7fffffffLL || gy > 65535) return set_error(U2_ERR_UNSUPPORTED, "colsum: grid too large");
  colsum_kernel<<<dim3((unsigned)gx, (unsigned)gy), 256, 0, ST(stream)>>>(CBF(x), out, rows, cols, ld, rpb);
  U2_CHECK_LAUNCH("colsum");
  return U2_OK;
}

extern "C" U2_API int u2_gelu_bf16(const void* x, void* y, int64_t n, void* stream) {
  if (!x || !y) return set_error(U2_ERR_ARG, "gelu: null pointer");
  if (n & 7) return set_error(U2_ERR_ARG, "gelu: n must be a multiple of 8");
  if (n <= 0) return U2_OK;
  gelu_kernel<<<t_grid(n / 8, 256), 256, 0, ST(stream)>>>(CBF(x), BF(y), n / 8);
  U2_CHECK_LAUNCH("gelu");
  return U2_OK;
}

extern "C" U2_API int u2_gelu_bwd_bf16(const void* x_pre, const void* dy, void* dx, int64_t n, void* stream) {
  if (!x_pre || !dy || !dx) return set_error(U2_ERR_ARG, "gelu_bwd: null pointer");
  if (n & 7) return set_error(U2_ERR_ARG, "gelu_bwd: n must be a multiple of 8");
  if (n <= 0) return U2_OK;
  gelu_bwd_kernel<<<t_grid(n / 8, 256), 256, 0, ST(stream)>>>(CBF(x_pre), CBF(dy), BF(dx), n / 8);
  U2_CHECK_LAUNCH("gelu_bwd");
  return U2_OK;
}

extern "C" U2_API int u2_silu_mul_bwd_bf16(const void* gate_up, const void* dact, void* dgu, int64_t rows, int32_t I,
                                           int64_t ldg, int64_t ldd, void* stream) {
  if (!gate_up || !dact || !dgu) return set_error(U2_ERR_ARG, "silu_mul_bwd: null pointer");
  if (I <= 0 || (I & 7) || (ldg & 7) || (ldd & 7)) return set_error(U2_ERR_ARG, "silu_mul_bwd: I / ld must be multiples of 8");
  if (rows <= 0) return U2_OK;
  silu_mul_bwd_kernel<<<t_grid(rows * (I / 8), 256), 256, 0, ST(stream)>>>(CBF(gate_up), CBF(dact), BF(dgu), rows, I, ldg, ldd);
  U2_CHECK_LAUNCH("silu_mul_bwd");
  return U2_OK;
}

extern "C" U2_API int u2_layernorm_bwd_bf16(const void* x, const float* gamma, const void* dy, const void* dres, void* dx_out,
                                            float* dgamma, float* dbeta, int64_t rows, int32_t E, int64_t ldx, int64_t ldy,
                                            int64_t ldr, int64_t ldo, float eps, void* stream) {
  if (dgamma && !dbeta) return set_error(U2_ERR_ARG, "layernorm_bwd: dgamma and dbeta go together");
  return launch_norm_bwd<false>(x, gamma, dy, dres, dx_out, dgamma, dbeta, rows, E, ldx, ldy, ldr, ldo, eps, ST(stream));
}

extern "C" U2_API int u2_rmsnorm_bwd_bf16(const void* x, const float* gamma, const void* dy, const void* dres, void* dx_out,
                                          float* dgamma, int64_t rows, int32_t E, int64_t ldx, int64_t ldy, int64_t ldr,
                                          int64_t ldo, float eps, void* stream) {
  return launch_norm_bwd<true>(x, gamma, dy, dres, dx_out, dgamma, nullptr, rows, E, ldx, ldy, ldr, ldo, eps, ST(stream));
}

extern "C" U2_API int u2_softmax_bwd_bf16(const void* P, const float* dP, void* dS, const u2_softmax_bwd_desc* d, void* stream) {
  if (!P || !dP || !dS || !d) return set_error(U2_ERR_ARG, "softmax_bwd: null pointer");
  if (d->n <= 0 || d->n0 <= 0 || d->H <= 0 || d->S <= 0) return set_error(U2_ERR_ARG, "softmax_bwd: bad extents");
  SmBwdArgs a;
  a.P = CBF(P); a.dP = dP; a.dS = BF(dS);
  a.p_s0 = d->p_s0; a.p_s1 = d->p_s1; a.p_s2 = d->p_s2;
  a.dp_s0 = d->dp_s0; a.dp_s1 = d->dp_s1; a.dp_s2 = d->dp_s2;
  a.ds_s0 = d->ds_s0; a.ds_s1 = d->ds_s1; a.ds_s2 = d->ds_s2;
  a.n0 = d->n0; a.H = d->H; a.S = d->S; a.n = d->n; a.zero_pad_to = d->zero_pad_to;
  const int span = d->n > d->zero_pad_to ? d->n : d->zero_pad_to;
  const long long rows = (long long)d->n0 * d->H * d->S;
  cudaStream_t st = ST(stream);
  const bool vec_ok = span > 1024 && span <= 2304 && (span & 7) == 0 && d->zero_pad_to >= d->n &&
                      ((d->p_s0 | d->p_s1 | d->p_s2 | d->ds_s0 | d->ds_s1 | d->ds_s2) & 7) == 0 &&
                      ((d->dp_s0 | d->dp_s1 | d->dp_s2) & 3) == 0 && (reinterpret_cast<uintptr_t>(P) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(dP) & 15) == 0 && (reinterpret_cast<uintptr_t>(dS) & 15) == 0;
  if (vec_ok) {
    softmax_bwd_warp_vec_kernel<9><<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(a);
    U2_CHECK_LAUNCH("softmax_bwd");
    return U2_OK;
  }
#define U2_SB_CASE(G, MV)                                                                        \
  softmax_bwd_kernel<G, MV><<<(unsigned)((rows + ((G) == 32 ? 4 : 1) - 1) / ((G) == 32 ? 4 : 1)), \
                              (G) == 32 ? 128 : (G), 0, st>>>(a)
  if (span <= 32) U2_SB_CASE(32, 1);
  else if (span <= 64) U2_SB_CASE(32, 2);
  else if (span <= 128) U2_SB_CASE(32, 4);
  else if (span <= 256) U2_SB_CASE(32, 8);
  else if (span <= 512) U2_SB_CASE(32, 16);
  else if (span <= 1024) U2_SB_CASE(128, 8);
  else if (span <= 2048) U2_SB_CASE(128, 16);
  else if (span <= 4096) U2_SB_CASE(256, 16);
  else if (span <= 8192) U2_SB_CASE(256, 32);
  else if (rows <= 0x7fffffffLL) softmax_bwd_long_kernel<<<(unsigned)rows, 256, 0, st>>>(a);
  else return set_error(U2_ERR_UNSUPPORTED, "softmax_bwd: %lld rows of length %d", rows, span);
#undef U2_SB_CASE
  U2_CHECK_LAUNCH("softmax_bwd");
  return U2_OK;
}

extern "C" U2_API int u2_relbias_grad_bf16(const void* dS, float* drel, int32_t n0, int32_t H, int32_t S, int32_t n, int64_t s0,
                                           int64_t s1, int64_t s2, int32_t rel_max, void* stream) {
  if (!dS || !drel) return set_error(U2_ERR_ARG, "relbias_grad: null pointer");
  if (S > rel_max || n > rel_max) return set_error(U2_ERR_ARG, "relbias_grad: sequence exceeds the bias table");
  if (n0 <= 0 || H <= 0 || S <= 0 || n <= 0) return U2_OK;
  if (n0 > 65535) return set_error(U2_ERR_UNSUPPORTED, "relbias_grad: batch too large");
  relbias_grad_kernel<<<dim3((unsigned)H, (unsigned)n0), 256, (size_t)(S + n) * sizeof(float), ST(stream)>>>(
      CBF(dS), drel, H, S, n, s0, s1, s2, rel_max);
  U2_CHECK_LAUNCH("relbias_grad");
  return U2_OK;
}

extern "C" U2_API int u2_rowdot_bf16(const void* a, const void* c, float* out, int32_t B, int32_t S, int32_t H, int32_t dh,
                                     int64_t a_sb, int64_t a_ss, int64_t a_sh, int64_t c_sb, int64_t c_ss, int64_t c_sh,
                                     void* stream) {
  if (!a || !c || !out) return set_error(U2_ERR_ARG, "rowdot: null pointer");
  if ((dh & 1) || ((a_sb | a_ss | a_sh | c_sb | c_ss | c_sh) & 1)) return set_error(U2_ERR_ARG, "rowdot: dh / strides must be even");
  if (B <= 0 || S <= 0 || H <= 0) return U2_OK;
  long long blocks = ((long long)B * S * H + 7) / 8;
  if (blocks > 132 * 16) blocks = 132 * 16;
  rowdot_kernel<<<(unsigned)blocks, 256, 0, ST(stream)>>>(CBF(a), CBF(c), out, B, S, H, dh, a_sb, a_ss, a_sh, c_sb, c_ss, c_sh);
  U2_CHECK_LAUNCH("rowdot");
  return U2_OK;
}

extern "C" U2_API int u2_temporal_attention_bwd_bf16(const void* qkv, const void* dout, void* dqkv, int32_t B, int32_t C,
                                                     int32_t N, int32_t H, int32_t dh, int64_t ld_qkv, int64_t ld_dout,
                                                     int64_t ld_dqkv, float scale, const float* rel_bias, float* drel,
                                                     int32_t rel_max, void* stream) {
  if (!qkv || !dout || !dqkv) return set_error(U2_ERR_ARG, "temporal_attention_bwd: null pointer");
  if (C <= 0 || C > 128) return set_error(U2_ERR_UNSUPPORTED, "temporal_attention_bwd: C=%d (1..128)", C);
  if ((dh & 7) || (ld_qkv & 7) || (ld_dout & 7) || (ld_dqkv & 7)) return set_error(U2_ERR_ARG, "temporal_attention_bwd: dh / ld must be multiples of 8");
  if (rel_bias && C > rel_max) return set_error(U2_ERR_ARG, "temporal_attention_bwd: C exceeds the bias table");
  if (N > 65535 || B > 65535) return set_error(U2_ERR_UNSUPPORTED, "temporal_attention_bwd: grid too large");
  const size_t smem = (size_t)4 * C * dh * 2 + (size_t)2 * C * C * 4;
  if (smem > 220 * 1024) return set_error(U2_ERR_UNSUPPORTED, "temporal_attention_bwd: C=%d, head_dim=%d needs %zu bytes of shared memory", C, dh, smem);
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(temporal_attention_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "temporal_attention_bwd smem: %s", cudaGetErrorString(e));
    configured = smem;
  }
  dim3 grid((unsigned)H, (unsigned)N, (unsigned)B);
  temporal_attention_bwd_kernel<<<grid, 128, smem, ST(stream)>>>(CBF(qkv), CBF(dout), BF(dqkv), C, N, H, dh, ld_qkv, ld_dout,
                                                                ld_dqkv, scale, rel_bias, drel, rel_max);
  U2_CHECK_LAUNCH("temporal_attention_bwd");
  return U2_OK;
}

extern "C" U2_API int u2_rope_bwd_bf16(void* dx, const void* x_raw, const u2_rope_desc* d, float* dq_norm_w, float* dk_norm_w,
                                       void* stream) {
  if (!dx || !d || !d->inv_freq) return set_error(U2_ERR_ARG, "rope_bwd: null pointer");
  if (d->dh <= 0 || (d->dh & 1) || (d->ld & 1)) return set_error(U2_ERR_ARG, "rope_bwd: head_dim and ld must be even");
  if ((d->q_norm_w || d->k_norm_w) && !x_raw) return set_error(U2_ERR_ARG, "rope_bwd: the per-head norm backward needs the raw projections");
  if (d->pos0_per_batch) return set_error(U2_ERR_UNSUPPORTED, "rope_bwd: per-batch positions are a decode-only feature");
  if (d->rows <= 0) return U2_OK;
  RopeBwdArgs a;
  a.dx = BF(dx); a.x_raw = CBF(x_raw);
  a.rows = d->rows; a.ld = d->ld; a.dh = d->dh;
  a.n_q_heads = d->n_q_heads; a.n_k_heads = d->n_k_heads;
  a.q_norm_w = d->q_norm_w; a.k_norm_w = d->k_norm_w; a.eps = d->eps;
  a.inv_freq = d->inv_freq;
  a.pos0 = d->pos0; a.pos_div = d->pos_div > 0 ? d->pos_div : 1; a.pos_mod = d->pos_mod > 0 ? d->pos_mod : 1;
  a.dq_norm_w = d->q_norm_w ? dq_norm_w : nullptr;
  a.dk_norm_w = d->k_norm_w ? dk_norm_w : nullptr;
  const long long items = d->rows * (long long)(a.n_q_heads + a.n_k_heads);
  long long blocks = (items + 7) / 8;
  if (blocks > 132 * 8) blocks = 132 * 8;
  const size_t smem = (a.dq_norm_w || a.dk_norm_w) ? (size_t)2 * a.dh * sizeof(float) : 0;
  rope_bwd_kernel<<<(unsigned)blocks, 256, smem, ST(stream)>>>(a);
  U2_CHECK_LAUNCH("rope_bwd");
  return U2_OK;
}

extern "C" U2_API int u2_spp_pool_bwd_bf16(const void* dy, void* dx, int64_t frames, int32_t g0, int32_t g1, int32_t g2,
                                           int32_t ps, int32_t E, int64_t in_frame_stride, int64_t in_off, int64_t ldx,
                                           int64_t rows_per_frame, int32_t sequence, void* stream) {
  if (!dy || !dx) return set_error(U2_ERR_ARG, "spp_pool_bwd: null pointer");
  if ((E & 7) || (ldx & 7) || ps <= 0) return set_error(U2_ERR_ARG, "spp_pool_bwd: E / ldx must be multiples of 8");
  if (frames <= 0) return U2_OK;
  spp_pool_bwd_kernel<<<t_grid(frames * rows_per_frame * (E / 8), 256, 132LL * 32), 256, 0, ST(stream)>>>(
      CBF(dy), BF(dx), frames, g0, g1, g2, ps, E, in_frame_stride, in_off, ldx, rows_per_frame, sequence);
  U2_CHECK_LAUNCH("spp_pool_bwd");
  return U2_OK;
}

extern "C" U2_API int u2_multiscale_pool_bwd_bf16(const void* x, const void* dy, void* dx, const float* gate_w,
                                                  const float* logits, float* dgate_w, float* ws, int32_t B, int32_t K,
                                                  int32_t E, int32_t dynamic, void* stream) {
  if (!x || !dy || !dx) return set_error(U2_ERR_ARG, "multiscale_pool_bwd: null pointer");
  if (dynamic && (!gate_w || !logits || !ws)) return set_error(U2_ERR_ARG, "multiscale_pool_bwd: the dynamic gate needs gate_w, logits and ws");
  if (E & 7) return set_error(U2_ERR_ARG, "multiscale_pool_bwd: E must be a multiple of 8");
  if (B <= 0 || K <= 0) return U2_OK;
  const int rpb = 8;
  dim3 grid((unsigned)((K + rpb - 1) / rpb), (unsigned)B);
  if (dynamic) {
    cudaError_t e = cudaMemsetAsync(ws, 0, (size_t)B * 8 * sizeof(float), ST(stream));
    if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "multiscale_pool_bwd memset: %s", cudaGetErrorString(e));
    msp_bwd_dot_kernel<<<grid, 256, 0, ST(stream)>>>(CBF(x), CBF(dy), ws, K, E, rpb);
    U2_CHECK_LAUNCH("multiscale_pool_bwd dot");
  }
  msp_bwd_write_kernel<<<grid, 256, 0, ST(stream)>>>(CBF(x), CBF(dy), BF(dx), gate_w, logits, ws, dgate_w, K, E, dynamic, rpb);
  U2_CHECK_LAUNCH("multiscale_pool_bwd write");
  return U2_OK;
}

extern "C" U2_API int u2_embed_scatter_add_bf16(const int64_t* ids, const void* drows, void* dtable, void* dvis, int32_t B,
                                                int32_t L, int32_t E, int32_t n_vis, int64_t vocab, void* stream) {
  if (!ids || !drows) return set_error(U2_ERR_ARG, "embed_scatter_add: null pointer");
  if (E & 7) return set_error(U2_ERR_ARG, "embed_scatter_add: E must be a multiple of 8");
  if (B <= 0 || L <= 0) return U2_OK;
  embed_scatter_add_kernel<<<t_grid((long long)B * L * (E / 8), 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const long long*>(ids), CBF(drows), BF(dtable), BF(dvis), B, L, E, n_vis, vocab);
  U2_CHECK_LAUNCH("embed_scatter_add");
  return U2_OK;
}

extern "C" U2_API int u2_group_sum_bf16(const void* in, void* out, int64_t rows, int32_t heads, int32_t G, int32_t dh,
                                        int64_t ld_in, int64_t ld_out, void* stream) {
  if (!in || !out) return set_error(U2_ERR_ARG, "group_sum: null pointer");
  if ((dh & 7) || (ld_in & 7) || (ld_out & 7)) return set_error(U2_ERR_ARG, "group_sum: dh / ld must be multiples of 8");
  if (rows <= 0) return U2_OK;
  group_sum_kernel<<<t_grid(rows * heads * (dh / 8), 256), 256, 0, ST(stream)>>>(CBF(in), BF(out), rows, heads, G, dh, ld_in, ld_out);
  U2_CHECK_LAUNCH("group_sum");
  return U2_OK;
}

extern "C" U2_API int u2_ce_bwd_f32_bf16(const float* logits, void* dlogits, const float* lse, const int64_t* labels,
                                         const float* coef, int64_t R, int32_t V, int64_t ld_in, int64_t ld_out, void* stream) {
  if (!logits || !dlogits || !lse || !labels || !coef) return set_error(U2_ERR_ARG, "ce_bwd: null pointer");
  if ((V & 7) || (ld_in & 3) || (ld_out & 7)) return set_error(U2_ERR_ARG, "ce_bwd: V / ld must be multiples of 8");
  if (R <= 0) return U2_OK;
  ce_bwd_kernel<<<t_grid(R * (V / 8), 256, 132LL * 32), 256, 0, ST(stream)>>>(logits, BF(dlogits), lse,
                                                                            reinterpret_cast<const long long*>(labels), coef, R, V, ld_in, ld_out);
  U2_CHECK_LAUNCH("ce_bwd");
  return U2_OK;
}

extern "C" U2_API int u2_dpo_loss_f32(const float* per_tok, const float* ref_sum, const uint8_t* mask, float* out, float* coef,
                                      int32_t P, int32_t L, float beta, void* stream) {
  if (!per_tok || !ref_sum || !mask || !out || !coef) return set_error(U2_ERR_ARG, "dpo_loss: null pointer");
  if (P <= 0 || P > 1024 || L <= 0) return set_error(U2_ERR_ARG, "dpo_loss: 1 <= P <= 1024 pairs");
  const int threads = ((P + 31) / 32) * 32;
  dpo_loss_kernel<<<1, threads, 0, ST(stream)>>>(per_tok, ref_sum, mask, out, coef, P, L, beta);
  U2_CHECK_LAUNCH("dpo_loss");
  return U2_OK;
}

static int adam_args(const u2_adamw_desc* d, AdamArgs* a) {
  if (!d || d->step < 1) return set_error(U2_ERR_ARG, "adamw: descriptor / step >= 1");
  if (d->index_offset < 0) return set_error(U2_ERR_ARG, "adamw: index_offset >= 0");
  a->lr = d->lr; a->beta1 = d->beta1; a->beta2 = d->beta2; a->eps = d->eps; a->wd = d->weight_decay;
  a->bc1 = 1.f - powf(d->beta1, (float)d->step);
  a->bc2_rsqrt = 1.f / sqrtf(1.f - powf(d->beta2, (float)d->step));
  a->grad_scale = d->grad_scale;
  // the LoRA mask's key schedule with the step in place of the stream id
  a->sr_key = adam_fmix32((uint32_t)d->seed ^ adam_fmix32((uint32_t)(d->seed >> 32) + (uint32_t)d->step * 0x9E3779B9u));
  a->index0 = d->index_offset;
  return U2_OK;
}

extern "C" U2_API int u2_adamw_bf16(float* master, float* m, float* v, const void* grad, void* param_out, int64_t n,
                                    const u2_adamw_desc* desc, void* stream) {
  if (!master || !m || !v || !grad) return set_error(U2_ERR_ARG, "adamw: null pointer");
  if (n & 3) return set_error(U2_ERR_ARG, "adamw: n must be a multiple of 4");
  AdamArgs a;
  int rc = adam_args(desc, &a);
  if (rc) return rc;
  if (n <= 0) return U2_OK;
  adamw_kernel<false><<<t_grid(n / 4, 256, 132LL * 16), 256, 0, ST(stream)>>>(master, m, v, grad, BF(param_out), nullptr, n, a);
  U2_CHECK_LAUNCH("adamw");
  return U2_OK;
}

extern "C" U2_API int u2_adamw_bf16_mom16(float* master, void* m, void* v, const void* grad, void* param_out, int64_t n,
                                          const u2_adamw_desc* desc, void* stream) {
  if (!master || !m || !v || !grad) return set_error(U2_ERR_ARG, "adamw: null pointer");
  if (n & 3) return set_error(U2_ERR_ARG, "adamw: n must be a multiple of 4");
  AdamArgs a;
  int rc = adam_args(desc, &a);
  if (rc) return rc;
  if (n <= 0) return U2_OK;
  adamw_mom16_kernel<<<t_grid(n / 4, 256, 132LL * 16), 256, 0, ST(stream)>>>(master, BF(m), BF(v), CBF(grad), BF(param_out), n, a);
  U2_CHECK_LAUNCH("adamw");
  return U2_OK;
}

extern "C" U2_API int u2_adamw_f32grad(float* master, float* m, float* v, const float* grad, void* param_out_bf16,
                                       float* param_out_f32, int64_t n, const u2_adamw_desc* desc, void* stream) {
  if (!master || !m || !v || !grad) return set_error(U2_ERR_ARG, "adamw: null pointer");
  if (n & 3) return set_error(U2_ERR_ARG, "adamw: n must be a multiple of 4");
  AdamArgs a;
  int rc = adam_args(desc, &a);
  if (rc) return rc;
  if (n <= 0) return U2_OK;
  adamw_kernel<true><<<t_grid(n / 4, 256, 132LL * 16), 256, 0, ST(stream)>>>(master, m, v, grad, BF(param_out_bf16), param_out_f32, n, a);
  U2_CHECK_LAUNCH("adamw");
  return U2_OK;
}

extern "C" U2_API int u2_sumsq_bf16(const void* x, float* out, int64_t n, void* stream) {
  if (!x || !out) return set_error(U2_ERR_ARG, "sumsq: null pointer");
  if (n & 7) return set_error(U2_ERR_ARG, "sumsq: n must be a multiple of 8");
  if (n <= 0) return U2_OK;
  sumsq_kernel<false><<<t_grid(n / 8, 256, 132LL * 8), 256, 0, ST(stream)>>>(x, out, n);
  U2_CHECK_LAUNCH("sumsq");
  return U2_OK;
}

extern "C" U2_API int u2_sumsq_f32(const float* x, float* out, int64_t n, void* stream) {
  if (!x || !out) return set_error(U2_ERR_ARG, "sumsq: null pointer");
  if (n & 3) return set_error(U2_ERR_ARG, "sumsq: n must be a multiple of 4");
  if (n <= 0) return U2_OK;
  sumsq_kernel<true><<<t_grid(n / 4, 256, 132LL * 8), 256, 0, ST(stream)>>>(x, out, n);
  U2_CHECK_LAUNCH("sumsq");
  return U2_OK;
}

extern "C" U2_API int u2_add_bf16(void* dst, const void* src, int64_t n, void* stream) {
  if (!dst || !src) return set_error(U2_ERR_ARG, "add: null pointer");
  if (n & 7) return set_error(U2_ERR_ARG, "add: n must be a multiple of 8");
  if (n <= 0) return U2_OK;
  add_bf16_kernel<<<t_grid(n / 8, 256), 256, 0, ST(stream)>>>(BF(dst), CBF(src), n / 8);
  U2_CHECK_LAUNCH("add");
  return U2_OK;
}

extern "C" U2_API int u2_cast_f32_bf16(const float* in, void* out, int64_t n, void* stream) {
  if (!in || !out) return set_error(U2_ERR_ARG, "cast: null pointer");
  if (n <= 0) return U2_OK;
  cast_f32_bf16_kernel<<<t_grid(n, 256), 256, 0, ST(stream)>>>(in, BF(out), n);
  U2_CHECK_LAUNCH("cast");
  return U2_OK;
}

extern "C" U2_API int u2_cast_bf16_f32(const void* in, float* out, int64_t n, void* stream) {
  if (!in || !out) return set_error(U2_ERR_ARG, "cast: null pointer");
  if (n <= 0) return U2_OK;
  cast_bf16_f32_kernel<<<t_grid(n, 256), 256, 0, ST(stream)>>>(CBF(in), out, n);
  U2_CHECK_LAUNCH("cast");
  return U2_OK;
}
