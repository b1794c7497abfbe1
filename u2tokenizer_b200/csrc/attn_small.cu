// Small-sequence attention pieces that do not belong on the tensor cores:
//   temporal_attention  RMA / RoPE attention across the <= 128 frames of one spatial token
//                       (reference svr.py:33-36 + rma.py:60-73); one CTA per (batch, token, head)
//   rope / qk_norm_rope rotate-half RoPE (optionally per-head RMSNorm first: Qwen3) applied in place
//                       on a fused QKV buffer, and the KV-cache append of the decoder
//   decode_attention    one query token against the KV cache (HBM-bound, GQA)
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <math.h>

#include <type_traits>

#include "host_util.h"
#include "u2b200.h"

namespace u2 {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------------
// temporal attention. qkv rows are (b, c, n) -> row = (b*C + c)*N + n, columns [q | k | v] each E wide.
// out[(b*C + c)*N + n][h*dh + d] = sum_c' softmax_c'(q_c . k_c' * scale + bias[c'-c+rel_max-1][h]) v_c'[d]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
temporal_attention_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int C, int N,
                          int H, int dh, long long ld_qkv, long long ld_out, float scale,
                          const float* __restrict__ rel_bias, int rel_max) {
  extern __shared__ __nv_bfloat16 sm[];  // K [C][dh] then V [C][dh]
  __nv_bfloat16* sK = sm;
  __nv_bfloat16* sV = sm + (size_t)C * dh;
  const int h = blockIdx.x, n = blockIdx.y, b = blockIdx.z;
  const int E = H * dh;
  const int nvec = dh >> 3;
  for (int i = threadIdx.x; i < C * nvec; i += blockDim.x) {
    const int c = i / nvec, v = i - c * nvec;
    const long long row = ((long long)b * C + c) * N + n;
    const __nv_bfloat16* base = qkv + row * ld_qkv + h * dh;
    reinterpret_cast<uint4*>(sK + (size_t)c * dh)[v] = reinterpret_cast<const uint4*>(base + E)[v];
    reinterpret_cast<uint4*>(sV + (size_t)c * dh)[v] = reinterpret_cast<const uint4*>(base + 2 * E)[v];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int c = warp; c < C; c += (blockDim.x >> 5)) {
    const long long row = ((long long)b * C + c) * N + n;
    const __nv_bfloat16* q = qkv + row * ld_qkv + h * dh;
    // scores: lane l keeps the scores of key frames l, l + 32, l + 64, l + 96
    float my[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
#pragma unroll
    for (int jb = 0; jb < 4; ++jb) {
      if (jb * 32 >= C) break;
      const int jn = min(32, C - jb * 32);
      for (int jj = 0; jj < jn; ++jj) {
        const int j = jb * 32 + jj;
        float d = 0.f;
        for (int e = lane * 2; e < dh; e += 64) {
          const float2 qq = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(q + e));
          const float2 kk = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sK + (size_t)j * dh + e));
          d += qq.x * kk.x + qq.y * kk.y;
        }
        d = wsum(d) * scale;
        if (rel_bias) d += __ldg(rel_bias + (long long)(j - c + rel_max - 1) * H + h);
        if (lane == jj) my[jb] = d;
      }
    }
    const float m = wmax(fmaxf(fmaxf(my[0], my[1]), fmaxf(my[2], my[3])));
    float pr[4], ssum = 0.f;
#pragma unroll
    for (int jb = 0; jb < 4; ++jb) {
      pr[jb] = (jb * 32 + lane < C) ? __expf(my[jb] - m) : 0.f;
      ssum += pr[jb];
    }
    const float inv = 1.f / wsum(ssum);
    __nv_bfloat16* o = out + row * ld_out + h * dh;
    for (int eb = 0; eb < dh; eb += 64) {  // warp-uniform trip count: the shuffles below need every lane
      const int e0 = eb + lane * 2;
      const bool own = e0 < dh;
      float ax = 0.f, ay = 0.f;
#pragma unroll
      for (int jb = 0; jb < 4; ++jb) {
        if (jb * 32 >= C) break;
        const int jn = min(32, C - jb * 32);
        for (int jj = 0; jj < jn; ++jj) {
          const float pj = __shfl_sync(0xffffffffu, pr[jb], jj);
          if (own) {
            const float2 vv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sV + (size_t)(jb * 32 + jj) * dh + e0));
            ax += pj * vv.x;
            ay += pj * vv.y;
          }
        }
      }
      if (own) *reinterpret_cast<__nv_bfloat162*>(o + e0) = __floats2bfloat162_rn(ax * inv, ay * inv);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// (optional per-head RMSNorm) + rotate-half RoPE, in place on `n_rot_heads` heads of every row of a
// fused buffer; optional KV-cache append. One warp per (row, head).
//   position(row) = pos0 + (row / pos_div) % pos_mod
// ------------------------------------------------------------------------------------------------
struct RopeArgs {
  __nv_bfloat16* x;          // [rows, ld]
  long long rows, ld;
  int dh;
  int n_q_heads;             // heads [0, n_q_heads) use q_norm_w
  int n_k_heads;             // heads [n_q_heads, n_q_heads + n_k_heads) use k_norm_w
  int n_v_heads;             // heads after that are V (no rope): only copied to the cache
  const float* q_norm_w;     // [dh] or null
  const float* k_norm_w;     // [dh] or null
  float eps;
  const float* inv_freq;     // [dh/2]
  int pos0, pos_div, pos_mod;
  const int* pos0_dev;       // when set, pos0 is read from the device (CUDA-graph friendly decode)
  __nv_bfloat16* k_cache;    // [B, n_k_heads, Tmax, dh] or null
  __nv_bfloat16* v_cache;
  int Tmax, rows_per_batch;  // batch index = row / rows_per_batch, cache position = position(row)
  int pos0_per_batch;        // pos0 = pos0_dev[batch index] instead of pos0_dev[0]
};

__global__ void __launch_bounds__(256)
rope_kernel(const RopeArgs a) {
  const int heads = a.n_q_heads + a.n_k_heads + a.n_v_heads;
  const long long item = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (item >= a.rows * heads) return;
  const int lane = threadIdx.x & 31;
  const long long row = item / heads;
  const int head = (int)(item - row * heads);
  __nv_bfloat16* p = a.x + row * a.ld + (long long)head * a.dh;
  const int b = (int)(row / a.rows_per_batch);
  const int pos0 = a.pos0_dev ? a.pos0_dev[a.pos0_per_batch ? b : 0] : a.pos0;
  const int pos = pos0 + (int)((row / a.pos_div) % a.pos_mod);
  const int half = a.dh >> 1;
  const bool is_q = head < a.n_q_heads;
  const bool is_k = !is_q && head < a.n_q_heads + a.n_k_heads;
  if (!is_q && !is_k) {
    if (a.v_cache) {
      const int hv = head - a.n_q_heads - a.n_k_heads;
      __nv_bfloat16* dst = a.v_cache + (((long long)b * a.n_v_heads + hv) * a.Tmax + pos) * a.dh;
      for (int e = lane * 2; e < a.dh; e += 64)
        *reinterpret_cast<uint32_t*>(dst + e) = *reinterpret_cast<const uint32_t*>(p + e);
    }
    return;
  }
  const float* nw = is_q ? a.q_norm_w : a.k_norm_w;
  float rstd = 1.f;
  if (nw) {
    float ss = 0.f;
    for (int e = lane; e < a.dh; e += 32) {
      const float v = __bfloat162float(p[e]);
      ss += v * v;
    }
    ss = wsum(ss);
    rstd = rsqrtf(ss / a.dh + a.eps);
  }
  __nv_bfloat16* kdst = nullptr;
  if (is_k && a.k_cache)
    kdst = a.k_cache + (((long long)b * a.n_k_heads + (head - a.n_q_heads)) * a.Tmax + pos) * a.dh;
  for (int i = lane; i < half; i += 32) {
    float x1 = __bfloat162float(p[i]), x2 = __bfloat162float(p[i + half]);
    if (nw) {
      x1 = x1 * rstd * nw[i];
      x2 = x2 * rstd * nw[i + half];
    }
    float sn, cs;
    sincosf((float)pos * a.inv_freq[i], &sn, &cs);
    const __nv_bfloat16 o1 = __float2bfloat16(x1 * cs - x2 * sn);
    const __nv_bfloat16 o2 = __float2bfloat16(x2 * cs + x1 * sn);
    p[i] = o1;
    p[i + half] = o2;
    if (kdst) {
      kdst[i] = o1;
      kdst[i + half] = o2;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// decode attention: one query token per sequence against the KV cache.
//   q   [B, Hq, dh] (row stride ldq), caches [B, Hkv, Tmax, dh], T valid keys, out [B, Hq*dh]
// grid (Hq, B), 8 warps split the keys; online softmax per warp, merged through smem.
// ------------------------------------------------------------------------------------------------
template <int kEpl>
__device__ __forceinline__ void load_epl(const __nv_bfloat16* p, float (&f)[kEpl]) {
  if constexpr (kEpl == 1) {
    f[0] = __bfloat162float(p[0]);
  } else if constexpr (kEpl == 2) {
    const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
    f[0] = t.x; f[1] = t.y;
  } else {
    static_assert(kEpl == 4, "kEpl in {1,2,4}");
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
  }
}

// Beam-indirect cache (kInd): sequence b reads the key / value of position t from cache row kv_src[b * ld_src + t]
// (FasterTransformer's "cache indirection"); its own newest position (t == pos) always comes from row b. Returns the
// element offset from row b's slot to the source row's slot. kInd == false compiles to nothing.
template <bool kInd>
__device__ __forceinline__ long long kv_src_delta(const int* __restrict__ kv_src, long long ld_src, int b, int t,
                                                  int pos, long long row_elems) {
  if constexpr (kInd) {
    const int r = t == pos ? b : __ldg(kv_src + (long long)b * ld_src + t);
    return (long long)(r - b) * row_elems;
  } else {
    return 0;
  }
}

// dh = kEpl * kLanes: lane < kLanes owns elements [lane*kEpl, lane*kEpl + kEpl). dh 96 runs 24 lanes x 4 elements
// (8-byte accesses; 3 elements per lane would put lanes on 6-byte boundaries); lanes >= kLanes load the last owned
// slice again, contribute a zero query to the dot products and store nothing.
// kWin: sliding window of `window` keys (window > 0): only keys [max(0, T - window), T) are read.
template <int kEpl, bool kInd, bool kWin = false, int kLanes = 32>
__global__ void __launch_bounds__(256)
decode_attention_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kc,
                        const __nv_bfloat16* __restrict__ vc, __nv_bfloat16* __restrict__ out, int Hq, int Hkv,
                        int Tmax, int T_host, const int* __restrict__ T_dev, long long ldq, long long ldo,
                        float scale, int T_per_seq, const int* __restrict__ kv_src, long long ld_src, int window) {
  constexpr int dh = kEpl * kLanes;
  const int h = blockIdx.x, b = blockIdx.y;
  const int T = T_dev ? min(T_dev[T_per_seq ? b : 0], Tmax) : T_host;
  const int hk = h / (Hq / Hkv);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool own = kLanes == 32 || lane < kLanes;
  const int le = kLanes == 32 ? lane : min(lane, kLanes - 1);
  const __nv_bfloat16* qp = q + (long long)b * ldq + (long long)h * dh + le * kEpl;
  const __nv_bfloat16* kp = kc + ((long long)b * Hkv + hk) * Tmax * dh + le * kEpl;
  const __nv_bfloat16* vp = vc + ((long long)b * Hkv + hk) * Tmax * dh + le * kEpl;
  float qv[kEpl];
  load_epl<kEpl>(qp, qv);
  const float qs = own ? scale : 0.f;
#pragma unroll
  for (int i = 0; i < kEpl; ++i) qv[i] *= qs;
  float m = -INFINITY, l = 0.f;
  float acc[kEpl];
#pragma unroll
  for (int i = 0; i < kEpl; ++i) acc[i] = 0.f;
  int t_lo = 0;
  if constexpr (kWin) t_lo = window > 0 ? max(0, T - window) : 0;
  for (int t = t_lo + warp; t < T; t += 8) {
    float kk[kEpl], vv[kEpl];
    const long long off = (long long)t * dh + kv_src_delta<kInd>(kv_src, ld_src, b, t, T - 1, (long long)Hkv * Tmax * dh);
    load_epl<kEpl>(kp + off, kk);
    load_epl<kEpl>(vp + off, vv);
    float d = 0.f;
#pragma unroll
    for (int i = 0; i < kEpl; ++i) d += qv[i] * kk[i];
    d = wsum(d);
    const float mn = fmaxf(m, d);
    const float corr = __expf(m - mn);
    const float pe = __expf(d - mn);
    l = l * corr + pe;
#pragma unroll
    for (int i = 0; i < kEpl; ++i) acc[i] = acc[i] * corr + pe * vv[i];
    m = mn;
  }
  __shared__ float s_m[8], s_l[8];
  __shared__ float s_acc[8][dh];
  if (lane == 0) {
    s_m[warp] = m;
    s_l[warp] = l;
  }
  if (own) {
#pragma unroll
    for (int i = 0; i < kEpl; ++i) s_acc[warp][lane * kEpl + i] = acc[i];
  }
  __syncthreads();
  float gm = -INFINITY;
#pragma unroll
  for (int w = 0; w < 8; ++w) gm = fmaxf(gm, s_m[w]);
  float gl = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) gl += (s_m[w] == -INFINITY) ? 0.f : s_l[w] * __expf(s_m[w] - gm);
  for (int e = threadIdx.x; e < dh; e += blockDim.x) {
    float o = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w)
      if (s_m[w] != -INFINITY) o += s_acc[w][e] * __expf(s_m[w] - gm);
    out[(long long)b * ldo + (long long)h * dh + e] = __float2bfloat16(o / gl);
  }
}

}  // namespace u2

using namespace u2;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)

extern "C" U2_API int u2_temporal_attention_bf16(const void* qkv, void* out, int32_t B, int32_t C, int32_t N,
                                                 int32_t H, int32_t dh, int64_t ld_qkv, int64_t ld_out,
                                                 float scale, const float* rel_bias, int32_t rel_max,
                                                 void* stream) {
  if (!qkv || !out) return set_error(U2_ERR_ARG, "temporal_attention: null pointer");
  if (C <= 0 || C > 128) return set_error(U2_ERR_UNSUPPORTED, "temporal_attention: 1 <= frames <= 128 (got %d)", C);
  if ((size_t)2 * C * dh * sizeof(__nv_bfloat16) > 200 * 1024)
    return set_error(U2_ERR_UNSUPPORTED, "temporal_attention: frames * head_dim = %d exceeds the shared-memory staging (51200)", C * dh);
  if ((dh & 7) || (ld_qkv & 7) || (ld_out & 1)) return set_error(U2_ERR_ARG, "temporal_attention: dh/ld alignment");
  if (rel_bias && C > rel_max) return set_error(U2_ERR_ARG, "temporal_attention: frames exceed relative-bias table");
  if (B <= 0 || N <= 0) return U2_OK;
  if (N > 65535 || B > 65535) return set_error(U2_ERR_ARG, "temporal_attention: N,B must be <= 65535");
  const size_t smem = (size_t)2 * C * dh * sizeof(__nv_bfloat16);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(temporal_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "temporal_attention smem: %s", cudaGetErrorString(e));
  }
  dim3 grid((unsigned)H, (unsigned)N, (unsigned)B);
  temporal_attention_kernel<<<grid, 128, smem, ST(stream)>>>(CBF(qkv), BF(out), C, N, H, dh, ld_qkv, ld_out, scale, rel_bias, rel_max);
  U2_CHECK_LAUNCH("temporal_attention");
  return U2_OK;
}

extern "C" U2_API int u2_rope_bf16(void* x, const u2_rope_desc* d, void* stream) {
  if (!x || !d || !d->inv_freq) return set_error(U2_ERR_ARG, "rope: null pointer");
  if (d->dh <= 0 || (d->dh & 1) || (d->ld & 1)) return set_error(U2_ERR_ARG, "rope: head_dim and ld must be even");
  if (d->rows <= 0) return U2_OK;
  if ((d->k_cache || d->v_cache) && (d->Tmax <= 0 || d->rows_per_batch <= 0))
    return set_error(U2_ERR_ARG, "rope: cache append needs Tmax and rows_per_batch");
  if (d->k_cache && !d->pos0_dev && d->pos0 + d->pos_mod > d->Tmax)
    return set_error(U2_ERR_ARG, "rope: cache overflow (pos0 %d + %d > Tmax %d)", d->pos0, d->pos_mod, d->Tmax);
  if (d->pos0_per_batch && !d->pos0_dev) return set_error(U2_ERR_ARG, "rope: pos0_per_batch needs pos0_dev");
  RopeArgs a;
  a.x = BF(x);
  a.rows = d->rows; a.ld = d->ld; a.dh = d->dh;
  a.n_q_heads = d->n_q_heads; a.n_k_heads = d->n_k_heads; a.n_v_heads = d->n_v_heads;
  a.q_norm_w = d->q_norm_w; a.k_norm_w = d->k_norm_w; a.eps = d->eps;
  a.inv_freq = d->inv_freq;
  a.pos0_dev = d->pos0_dev;
  a.pos0 = d->pos0; a.pos_div = d->pos_div > 0 ? d->pos_div : 1; a.pos_mod = d->pos_mod > 0 ? d->pos_mod : 1;
  a.k_cache = BF(d->k_cache); a.v_cache = BF(d->v_cache);
  a.Tmax = d->Tmax; a.rows_per_batch = d->rows_per_batch > 0 ? d->rows_per_batch : 1;
  a.pos0_per_batch = d->pos0_per_batch != 0;
  const long long items = d->rows * (long long)(a.n_q_heads + a.n_k_heads + a.n_v_heads);
  rope_kernel<<<(unsigned)((items + 7) / 8), 256, 0, ST(stream)>>>(a);
  U2_CHECK_LAUNCH("rope");
  return U2_OK;
}

static int decode_attention_launch(const void* q, const void* k_cache, const void* v_cache, void* out, int32_t B,
                                   int32_t Hq, int32_t Hkv, int32_t dh, int32_t Tmax, int32_t T, const int32_t* T_dev,
                                   int64_t ldq, int64_t ldo, float scale, int32_t T_per_seq, const int32_t* kv_src,
                                   int64_t ld_kv_src, int32_t window, void* stream) {
  if (!q || !k_cache || !v_cache || !out) return set_error(U2_ERR_ARG, "decode_attention: null pointer");
  if (Hkv <= 0 || Hq % Hkv) return set_error(U2_ERR_ARG, "decode_attention: Hq must be a multiple of Hkv");
  if (!T_dev && (T <= 0 || T > Tmax)) return set_error(U2_ERR_ARG, "decode_attention: need 0 < T <= Tmax");
  if (T_per_seq && !T_dev) return set_error(U2_ERR_ARG, "decode_attention: T_per_seq needs T_dev");
  if (kv_src && ld_kv_src < Tmax) return set_error(U2_ERR_ARG, "decode_attention: kv_src row stride < Tmax");
  if (window < 0) return set_error(U2_ERR_ARG, "decode_attention: window %d < 0", window);
  dim3 grid((unsigned)Hq, (unsigned)B);
#define U2_DA(EPL, IND, WIN, LN) decode_attention_kernel<EPL, IND, WIN, LN><<<grid, 256, 0, ST(stream)>>>(CBF(q), CBF(k_cache), CBF(v_cache), BF(out), Hq, Hkv, Tmax, T, T_dev, ldq, ldo, scale, T_per_seq != 0, kv_src, ld_kv_src, window)
#define U2_DA2(EPL, LN)                                        \
  if (window > 0) {                                            \
    if (kv_src) U2_DA(EPL, true, true, LN);                    \
    else U2_DA(EPL, false, true, LN);                          \
  } else if (kv_src) U2_DA(EPL, true, false, LN);              \
  else U2_DA(EPL, false, false, LN)
  switch (dh) {
    case 32: U2_DA2(1, 32); break;
    case 64: U2_DA2(2, 32); break;
    case 96: U2_DA2(4, 24); break;
    case 128: U2_DA2(4, 32); break;
    default: return set_error(U2_ERR_UNSUPPORTED, "decode_attention: head_dim %d (supported: 32, 64, 96, 128)", dh);
  }
#undef U2_DA2
#undef U2_DA
  U2_CHECK_LAUNCH("decode_attention");
  return U2_OK;
}

extern "C" U2_API int u2_decode_attention_bf16(const void* q, const void* k_cache, const void* v_cache, void* out,
                                               int32_t B, int32_t Hq, int32_t Hkv, int32_t dh, int32_t Tmax,
                                               int32_t T, const int32_t* T_dev, int64_t ldq, int64_t ldo,
                                               float scale, int32_t T_per_seq, const int32_t* kv_src,
                                               int64_t ld_kv_src, void* stream) {
  return decode_attention_launch(q, k_cache, v_cache, out, B, Hq, Hkv, dh, Tmax, T, T_dev, ldq, ldo, scale, T_per_seq,
                                 kv_src, ld_kv_src, 0, stream);
}

extern "C" U2_API int u2_decode_attention_window_bf16(const void* q, const void* k_cache, const void* v_cache,
                                                      void* out, int32_t B, int32_t Hq, int32_t Hkv, int32_t dh,
                                                      int32_t Tmax, int32_t T, const int32_t* T_dev, int64_t ldq,
                                                      int64_t ldo, float scale, int32_t T_per_seq,
                                                      const int32_t* kv_src, int64_t ld_kv_src, int32_t window,
                                                      void* stream) {
  return decode_attention_launch(q, k_cache, v_cache, out, B, Hq, Hkv, dh, Tmax, T, T_dev, ldq, ldo, scale, T_per_seq,
                                 kv_src, ld_kv_src, window, stream);
}

// ------------------------------------------------------------------------------------------------
// Fused decode-step attention: per-head RMSNorm (Qwen3) + RoPE of the new q/k, KV-cache append and the
// attention of the G = Hq/Hkv query heads of one KV head against the cache - one launch per layer.
// One CTA per (sequence, KV head): the K/V rows are read once and shared by the G query heads.
//   QK^T : lane == key (no shuffles; q broadcast from shared memory)
//   PV   : lane == slice of head_dim (coalesced V rows; probabilities broadcast by shuffle)
// ------------------------------------------------------------------------------------------------
namespace u2 {

constexpr int kFaMaxG = 8;
// 16 warps (512 threads): <= 512 cached keys are covered in a single 32-keys-per-warp round; 8 warps where the
// per-warp accumulator staging would not fit the 48 KB static shared memory
template <int kDh, int kG>
struct FaCfg {
  static constexpr int kWarps = (kG * kDh * 16 * 4 > 40 * 1024) ? 8 : 16;
};

struct FusedDecodeArgs {
  const __nv_bfloat16* qkv;  // [B, (Hq + 2 Hkv) * dh]
  long long ldq;
  __nv_bfloat16* kc;         // [B, Hkv, Tmax, dh]
  __nv_bfloat16* vc;
  __nv_bfloat16* out;        // [B, Hq * dh]
  long long ldo;
  int Hq, Hkv, Tmax;
  const int* pos_dev;        // position of the new token (device); T = pos + 1
  int pos_per_seq;           // pos = pos_dev[sequence] instead of pos_dev[0]
  int pos_host;
  const float* q_norm_w;     // [dh] or null
  const float* k_norm_w;
  float eps;
  const float* inv_freq;     // [dh/2]
  float scale;
};
// beam search: the cache row of every position, int32 [B, ld_src]. A separate type, so that the kernels without the
// table keep the parameter block (and the code) they had before it existed
struct FusedDecodeIndArgs : FusedDecodeArgs {
  const int* kv_src;
  long long ld_src;
};
// sliding window (kWin kernels only, with or without the table): keys [max(0, pos - window + 1), pos]
struct FusedDecodeWinArgs : FusedDecodeIndArgs {
  int window;
};
template <bool kInd, bool kWin = false>
using FusedArgsT = std::conditional_t<kWin, FusedDecodeWinArgs, std::conditional_t<kInd, FusedDecodeIndArgs, FusedDecodeArgs>>;
// first visible key of the window (0 without one)
template <bool kWin>
__device__ __forceinline__ int window_lo(const FusedArgsT<false, kWin>& a, int pos) {
  if constexpr (kWin) return a.window > 0 ? max(0, pos - a.window + 1) : 0;
  else return 0;
}
// head_dim elements per lane in the PV phase and the lanes that own them: dh / 32 on 32 lanes, except dh 96 = 24 lanes x
// 4 elements (8-byte aligned slices); lanes >= kLanes load the last owned slice again and store nothing
template <int kDh>
struct PvMap {
  static constexpr int kEpl = kDh == 96 ? 4 : kDh / 32;
  static constexpr int kLanes = kDh / kEpl;
};
template <bool kInd>
__device__ __forceinline__ long long kv_src_delta(const FusedArgsT<kInd>& a, int b, int t, int pos, long long row_elems) {
  if constexpr (kInd) return kv_src_delta<true>(a.kv_src, a.ld_src, b, t, pos, row_elems);
  else return 0;
}

template <int kDh>
__device__ __forceinline__ void norm_rope_head(const __nv_bfloat16* src, const float* nw, float eps,
                                               const float* inv_freq, int pos, float mul, float* dst_f32,
                                               __nv_bfloat16* dst_bf16, int lane) {
  // one warp; element i pairs with i + dh/2 (rotate-half)
  constexpr int half = kDh / 2;
  float rstd = 1.f;
  if (nw) {
    float ss = 0.f;
    for (int e = lane; e < kDh; e += 32) {
      const float v = __bfloat162float(src[e]);
      ss += v * v;
    }
    ss = wsum(ss);
    rstd = rsqrtf(ss / kDh + eps);
  }
  for (int i = lane; i < half; i += 32) {
    float x1 = __bfloat162float(src[i]), x2 = __bfloat162float(src[i + half]);
    if (nw) {
      x1 = x1 * rstd * nw[i];
      x2 = x2 * rstd * nw[i + half];
    }
    float sn, cs;
    sincosf((float)pos * inv_freq[i], &sn, &cs);
    // round to bf16 exactly where the unfused path stores q / k
    const __nv_bfloat16 o1 = __float2bfloat16(x1 * cs - x2 * sn);
    const __nv_bfloat16 o2 = __float2bfloat16(x2 * cs + x1 * sn);
    if (dst_bf16) {
      dst_bf16[i] = o1;
      dst_bf16[i + half] = o2;
    }
    if (dst_f32) {
      dst_f32[i] = __bfloat162float(o1) * mul;
      dst_f32[i + half] = __bfloat162float(o2) * mul;
    }
  }
}

template <int kDh, int kG, bool kInd, bool kWin = false>
__global__ void __launch_bounds__(FaCfg<kDh, kG>::kWarps * 32)
fused_decode_attention_kernel(const FusedArgsT<kInd, kWin> a) {
  constexpr int kFaWarps = FaCfg<kDh, kG>::kWarps;
  constexpr int kEpl = PvMap<kDh>::kEpl;  // head_dim elements per lane in the PV phase
  constexpr int kLanes = PvMap<kDh>::kLanes;
  constexpr int kPf = 16;         // V rows prefetched per batch (memory-level parallelism in the PV loop)
  const int hk = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int le = kLanes == 32 ? lane : min(lane, kLanes - 1);
  asm volatile("griddepcontrol.wait;" ::: "memory");  // PDL: the QKV projection must have landed
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // o_proj may start prefetching its weights
  const int pos = a.pos_dev ? a.pos_dev[a.pos_per_seq ? b : 0] : a.pos_host;
  const int T = min(pos + 1, a.Tmax);
  const int lo = window_lo<kWin>(a, pos);  // every 32-key group from lo's group on holds at least one visible key
  __shared__ __align__(16) float s_q[kG][kDh];
  __shared__ float s_m[kFaWarps][kG], s_l[kFaWarps][kG];
  __shared__ float s_acc[kFaWarps][kG][kDh];

  const __nv_bfloat16* row = a.qkv + (long long)b * a.ldq;
  __nv_bfloat16* kbase = a.kc + ((long long)b * a.Hkv + hk) * a.Tmax * kDh;
  __nv_bfloat16* vbase = a.vc + ((long long)b * a.Hkv + hk) * a.Tmax * kDh;
  // ---- phase A: new k (norm + rope -> cache), new v (-> cache), G query heads (norm + rope -> smem)
  for (int job = warp; job < kG + 2; job += kFaWarps) {
    if (job == 0) {
      norm_rope_head<kDh>(row + (long long)(a.Hq + hk) * kDh, a.k_norm_w, a.eps, a.inv_freq, pos, 1.f, nullptr,
                          kbase + (long long)pos * kDh, lane);
    } else if (job == 1) {
      const __nv_bfloat16* v = row + (long long)(a.Hq + a.Hkv + hk) * kDh;
      for (int e = lane; e < kDh; e += 32) vbase[(long long)pos * kDh + e] = v[e];
    } else {
      const int g = job - 2;
      norm_rope_head<kDh>(row + (long long)(hk * kG + g) * kDh, a.q_norm_w, a.eps, a.inv_freq, pos, a.scale, s_q[g],
                          nullptr, lane);
    }
  }
  __syncthreads();

  // ---- phase B: online-softmax attention, 32 keys per warp iteration
  float m[kG], l[kG], acc[kG][kEpl];
#pragma unroll
  for (int g = 0; g < kG; ++g) {
    m[g] = -INFINITY;
    l[g] = 0.f;
#pragma unroll
    for (int i = 0; i < kEpl; ++i) acc[g][i] = 0.f;
  }
  const long long row_elems = (long long)a.Hkv * a.Tmax * kDh;
  for (int t0 = (lo & ~31) + warp * 32; t0 < T; t0 += kFaWarps * 32) {
    const int t = t0 + lane;
    const bool vis = t < T && (!kWin || t >= lo);
    // lane's key row (clamped like the V rows below); the V loop takes the other lanes' offsets by shuffle
    const long long dsrc = kv_src_delta<kInd>(a, b, min(t, T - 1), pos, row_elems);
    float s[kG];
#pragma unroll
    for (int g = 0; g < kG; ++g) s[g] = 0.f;
    if (vis) {
      const uint4* kr = reinterpret_cast<const uint4*>(kbase + (long long)t * kDh + dsrc);
      // the whole K row of this lane's key in one burst of independent 16-byte loads (one L2 round trip)
      uint4 u[kDh / 8];
#pragma unroll
      for (int c = 0; c < kDh / 8; ++c) u[c] = kr[c];
#pragma unroll
      for (int c0 = 0; c0 < kDh / 8; c0 += 4) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&u[c0 + c]);
          float kf[8];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f2 = __bfloat1622float2(h2[j]);
            kf[2 * j] = f2.x;
            kf[2 * j + 1] = f2.y;
          }
#pragma unroll
          for (int g = 0; g < kG; ++g) {
            const float4 q0 = *reinterpret_cast<const float4*>(&s_q[g][(c0 + c) * 8]);
            const float4 q1 = *reinterpret_cast<const float4*>(&s_q[g][(c0 + c) * 8 + 4]);
            s[g] += kf[0] * q0.x + kf[1] * q0.y + kf[2] * q0.z + kf[3] * q0.w + kf[4] * q1.x + kf[5] * q1.y +
                    kf[6] * q1.z + kf[7] * q1.w;
          }
        }
      }
    } else {
#pragma unroll
      for (int g = 0; g < kG; ++g) s[g] = -INFINITY;
    }
    float p[kG];
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      const float mx = fmaxf(m[g], wmax(s[g]));
      const float corr = __expf(m[g] - mx);
      p[g] = vis ? __expf(s[g] - mx) : 0.f;
      l[g] = l[g] * corr + wsum(p[g]);
#pragma unroll
      for (int i = 0; i < kEpl; ++i) acc[g][i] *= corr;
      m[g] = mx;
    }
    const int nk = min(32, T - t0);
    for (int j0 = 0; j0 < nk; j0 += kPf) {
      float vv[kPf][kEpl];
#pragma unroll
      for (int jj = 0; jj < kPf; ++jj) {
        const int tj = min(t0 + j0 + jj, T - 1);  // clamped rows (and rows below the window) carry probability 0
        long long dj = 0;
        if constexpr (kInd) dj = __shfl_sync(0xffffffffu, dsrc, tj - t0);
        load_epl<kEpl>(vbase + (long long)tj * kDh + dj + le * kEpl, vv[jj]);
      }
#pragma unroll
      for (int jj = 0; jj < kPf; ++jj) {
#pragma unroll
        for (int g = 0; g < kG; ++g) {
          const float pj = __shfl_sync(0xffffffffu, p[g], (j0 + jj) & 31);
#pragma unroll
          for (int i = 0; i < kEpl; ++i) acc[g][i] += pj * vv[jj][i];
        }
      }
    }
  }
  // ---- merge the 8 warps
#pragma unroll
  for (int g = 0; g < kG; ++g) {
    if (lane == 0) {
      s_m[warp][g] = m[g];
      s_l[warp][g] = l[g];
    }
    if (kLanes == 32 || lane < kLanes) {
#pragma unroll
      for (int i = 0; i < kEpl; ++i) s_acc[warp][g][lane * kEpl + i] = acc[g][i];
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < kG * kDh; idx += blockDim.x) {
    const int g = idx / kDh, e = idx - g * kDh;
    float gm = -INFINITY;
#pragma unroll
    for (int w = 0; w < kFaWarps; ++w) gm = fmaxf(gm, s_m[w][g]);
    float gl = 0.f, o = 0.f;
#pragma unroll
    for (int w = 0; w < kFaWarps; ++w) {
      if (s_m[w][g] != -INFINITY) {
        const float f = __expf(s_m[w][g] - gm);
        gl += s_l[w][g] * f;
        o += s_acc[w][g][e] * f;
      }
    }
    a.out[(long long)b * a.ldo + (long long)(hk * kG + g) * kDh + e] = __float2bfloat16(o / gl);
  }
}

// ------------------------------------------------------------------------------------------------
// Split-KV variant: a cluster of S CTAs shares one (sequence, KV head); the 32-key groups of the cache are dealt
// round-robin to the S x 8 warps, so that for up to S*256 cached keys every warp owns ONE group and the whole K/V
// read is a single round trip. The group's K row (lane == key) and V slices (lane == head-dim slice, all 32 rows)
// are requested BEFORE the new token's norm / RoPE work, which depends on nothing in the cache; the new token's own
// k / v never go through global memory (every CTA recomputes them into shared memory, rank 0 appends them to the
// cache). CTA partials (m, l, o) are merged by rank 0 over distributed shared memory.
// ------------------------------------------------------------------------------------------------
template <int kDh, int kG, bool kInd, bool kWin = false>
__global__ void __launch_bounds__(256)
fused_decode_attention_split_kernel(const FusedArgsT<kInd, kWin> a) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  constexpr int kW = 8;
  constexpr int kEpl = PvMap<kDh>::kEpl;   // head_dim elements per lane in the PV phase
  constexpr int kLanes = PvMap<kDh>::kLanes;
  constexpr int kVw = (kEpl + 1) / 2;      // 32-bit words holding one V row slice
  const int S = (int)gridDim.z, rank = (int)blockIdx.z;  // the cluster spans the grid's z extent
  const int hk = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int le = kLanes == 32 ? lane : min(lane, kLanes - 1);
  // PDL: the kernel behind us (the next chained decode-linear launch) may start its prologue and weight prefetch
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // the position is advanced at the end of the previous decode step, several fully serialised launches ago: safe to
  // read before the dependency wait, like the cache rows below the new position. b is uniform over the cluster (it
  // spans z only), so every CTA of a cluster sees the same T
  const int pos = a.pos_dev ? a.pos_dev[a.pos_per_seq ? b : 0] : a.pos_host;
  const int T = min(pos + 1, a.Tmax);
  // a window deals only its own key groups (from lo's group on) to the cluster: the bytes read are bounded by it
  const int lo = window_lo<kWin>(a, pos);
  __shared__ __align__(16) float s_q[kG][kDh];
  __shared__ __align__(16) __nv_bfloat16 s_knew[kDh];
  __shared__ __align__(16) __nv_bfloat16 s_vnew[kDh];
  __shared__ float s_m[kW][kG], s_l[kW][kG];
  __shared__ float s_acc[kW][kG][kDh];
  __shared__ float c_m[kG], c_l[kG];
  __shared__ __align__(16) float c_o[kG][kDh];

  const __nv_bfloat16* row = a.qkv + (long long)b * a.ldq;
  __nv_bfloat16* kbase = a.kc + ((long long)b * a.Hkv + hk) * a.Tmax * kDh;
  __nv_bfloat16* vbase = a.vc + ((long long)b * a.Hkv + hk) * a.Tmax * kDh;

  // ---- request this warp's first key group (rows >= pos are stale: they are replaced from shared memory below).
  // A beam-indirection table is written by the previous step's beam kernel, like the positions: safe to read here
  uint4 ku[kDh / 8];
  uint32_t vw[32][kVw];
  int t0 = (lo & ~31) + (warp * S + rank) * 32;
  const long long row_elems = (long long)a.Hkv * a.Tmax * kDh;
  auto request = [&](int base) {
    const int t = min(base + lane, T - 1);
    const long long dsrc = kv_src_delta<kInd>(a, b, t, pos, row_elems);
    const uint4* kr = reinterpret_cast<const uint4*>(kbase + (long long)t * kDh + dsrc);
#pragma unroll
    for (int c = 0; c < kDh / 8; ++c) ku[c] = kr[c];
#pragma unroll
    for (int jj = 0; jj < 32; ++jj) {
      const int tj = min(base + jj, T - 1);
      long long dj = 0;
      if constexpr (kInd) dj = __shfl_sync(0xffffffffu, dsrc, tj - base);
      const __nv_bfloat16* vp = vbase + (long long)tj * kDh + dj + le * kEpl;
      if constexpr (kEpl == 4) {
        const uint2 u = *reinterpret_cast<const uint2*>(vp);
        vw[jj][0] = u.x;
        vw[jj][1] = u.y;
      } else if constexpr (kEpl == 2) {
        vw[jj][0] = *reinterpret_cast<const uint32_t*>(vp);
      } else {
        vw[jj][0] = *reinterpret_cast<const unsigned short*>(vp);
      }
    }
  };
  if (t0 < T) request(t0);
  // PDL: everything above overlaps the tail of the kernel in front of us; the QKV projection must have landed now
  asm volatile("griddepcontrol.wait;" ::: "memory");

  // ---- phase A: G query heads (norm + rope -> smem), new k (norm + rope) and new v -> smem (+ cache on rank 0)
  for (int job = warp; job < kG + 2; job += kW) {
    if (job == kG) {
      norm_rope_head<kDh>(row + (long long)(a.Hq + hk) * kDh, a.k_norm_w, a.eps, a.inv_freq, pos, 1.f, nullptr, s_knew, lane);
      __syncwarp();
      if (rank == 0)
        for (int e = lane; e < kDh; e += 32) kbase[(long long)pos * kDh + e] = s_knew[e];
    } else if (job == kG + 1) {
      const __nv_bfloat16* v = row + (long long)(a.Hq + a.Hkv + hk) * kDh;
      for (int e = lane; e < kDh; e += 32) {
        const __nv_bfloat16 x = v[e];
        s_vnew[e] = x;
        if (rank == 0) vbase[(long long)pos * kDh + e] = x;
      }
    } else {
      norm_rope_head<kDh>(row + (long long)(hk * kG + job) * kDh, a.q_norm_w, a.eps, a.inv_freq, pos, a.scale, s_q[job],
                          nullptr, lane);
    }
  }
  __syncthreads();

  // ---- phase B: online softmax over this warp's groups
  float m[kG], l[kG], acc[kG][kEpl];
#pragma unroll
  for (int g = 0; g < kG; ++g) {
    m[g] = -INFINITY;
    l[g] = 0.f;
#pragma unroll
    for (int i = 0; i < kEpl; ++i) acc[g][i] = 0.f;
  }
  while (t0 < T) {
    const int t = t0 + lane;
    if (t == pos) {  // the new token's key: from shared memory, not from the cache
#pragma unroll
      for (int c = 0; c < kDh / 8; ++c) ku[c] = reinterpret_cast<const uint4*>(s_knew)[c];
    }
    float s[kG];
#pragma unroll
    for (int g = 0; g < kG; ++g) s[g] = 0.f;
#pragma unroll
    for (int c = 0; c < kDh / 8; ++c) {
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&ku[c]);
      float kf[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f2 = __bfloat1622float2(h2[j]);
        kf[2 * j] = f2.x;
        kf[2 * j + 1] = f2.y;
      }
#pragma unroll
      for (int g = 0; g < kG; ++g) {
        const float4 q0 = *reinterpret_cast<const float4*>(&s_q[g][c * 8]);
        const float4 q1 = *reinterpret_cast<const float4*>(&s_q[g][c * 8 + 4]);
        s[g] += kf[0] * q0.x + kf[1] * q0.y + kf[2] * q0.z + kf[3] * q0.w + kf[4] * q1.x + kf[5] * q1.y + kf[6] * q1.z +
                kf[7] * q1.w;
      }
    }
    float p[kG];
    const bool vis = t < T && (!kWin || t >= lo);
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      if (!vis) s[g] = -INFINITY;
      // lane 0 of every group is a valid key (with a window: lane lo & 31 of lo's group): mx is finite
      const float mx = fmaxf(m[g], wmax(s[g]));
      const float corr = __expf(m[g] - mx);
      p[g] = vis ? __expf(s[g] - mx) : 0.f;
      l[g] = l[g] * corr + wsum(p[g]);
#pragma unroll
      for (int i = 0; i < kEpl; ++i) acc[g][i] *= corr;
      m[g] = mx;
    }
#pragma unroll
    for (int jj = 0; jj < 32; ++jj) {
      float vf[kEpl];
      if (t0 + jj == pos) {  // warp-uniform
#pragma unroll
        for (int i = 0; i < kEpl; ++i) vf[i] = __bfloat162float(s_vnew[le * kEpl + i]);
      } else if constexpr (kEpl == 4) {
        const float2 x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&vw[jj][0]));
        const float2 y = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&vw[jj][1]));
        vf[0] = x.x; vf[1] = x.y; vf[2] = y.x; vf[3] = y.y;
      } else if constexpr (kEpl == 2) {
        const float2 x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&vw[jj][0]));
        vf[0] = x.x; vf[1] = x.y;
      } else {
        vf[0] = __uint_as_float(vw[jj][0] << 16);
      }
#pragma unroll
      for (int g = 0; g < kG; ++g) {
        const float pj = __shfl_sync(0xffffffffu, p[g], jj);  // rows past T carry probability 0
#pragma unroll
        for (int i = 0; i < kEpl; ++i) acc[g][i] += pj * vf[i];
      }
    }
    t0 += S * kW * 32;
    if (t0 < T) request(t0);
  }
  // ---- merge the warps of this CTA
#pragma unroll
  for (int g = 0; g < kG; ++g) {
    if (lane == 0) {
      s_m[warp][g] = m[g];
      s_l[warp][g] = l[g];
    }
    if (kLanes == 32 || lane < kLanes) {
#pragma unroll
      for (int i = 0; i < kEpl; ++i) s_acc[warp][g][lane * kEpl + i] = acc[g][i];
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < kG * kDh; idx += blockDim.x) {
    const int g = idx / kDh, e = idx - g * kDh;
    float gm = -INFINITY;
#pragma unroll
    for (int w = 0; w < kW; ++w) gm = fmaxf(gm, s_m[w][g]);
    float gl = 0.f, o = 0.f;
#pragma unroll
    for (int w = 0; w < kW; ++w) {
      if (s_m[w][g] != -INFINITY) {
        const float f = __expf(s_m[w][g] - gm);
        gl += s_l[w][g] * f;
        o += s_acc[w][g][e] * f;
      }
    }
    c_o[g][e] = o;
    if (e == 0) {
      c_m[g] = gm;
      c_l[g] = gl;
    }
  }
  // ---- merge the CTAs of the cluster on rank 0 (distributed shared memory)
  cluster.sync();
  if (rank == 0) {
    for (int idx = threadIdx.x; idx < kG * kDh; idx += blockDim.x) {
      const int g = idx / kDh, e = idx - g * kDh;
      float gm = -INFINITY;
      for (int r = 0; r < S; ++r) gm = fmaxf(gm, *cluster.map_shared_rank(&c_m[g], r));
      float gl = 0.f, o = 0.f;
      for (int r = 0; r < S; ++r) {
        const float mr = *cluster.map_shared_rank(&c_m[g], r);
        if (mr != -INFINITY) {
          const float f = __expf(mr - gm);
          gl += *cluster.map_shared_rank(&c_l[g], r) * f;
          o += *cluster.map_shared_rank(&c_o[g][e], r) * f;
        }
      }
      a.out[(long long)b * a.ldo + (long long)(hk * kG + g) * kDh + e] = __float2bfloat16(o / gl);
    }
  }
  cluster.sync();  // the other ranks' shared memory must outlive rank 0's reads
}

template <int kDh, int kG, bool kInd, bool kWin>
static int launch_fused_decode_split(const FusedArgsT<kInd, kWin>& a, dim3 grid, bool pdl, cudaStream_t st) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = grid.z;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 2 : 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, fused_decode_attention_split_kernel<kDh, kG, kInd, kWin>, a);
  if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "decode_attention_fused (split-KV) launch: %s", cudaGetErrorString(e));
  return U2_OK;
}

template <int kDh, bool kInd, bool kWin = false>
static int launch_fused_decode(const FusedArgsT<kInd, kWin>& a, int G, dim3 grid, bool pdl, cudaStream_t st) {
  if (grid.z > 1) {
    switch (G) {
      case 1: return launch_fused_decode_split<kDh, 1, kInd, kWin>(a, grid, pdl, st);
      case 2: return launch_fused_decode_split<kDh, 2, kInd, kWin>(a, grid, pdl, st);
      case 4: return launch_fused_decode_split<kDh, 4, kInd, kWin>(a, grid, pdl, st);
      case 8: return launch_fused_decode_split<kDh, 8, kInd, kWin>(a, grid, pdl, st);
      default: return set_error(U2_ERR_UNSUPPORTED, "decode_attention_fused: Hq/Hkv = %d (supported 1, 2, 4, 8)", G);
    }
  }
  switch (G) {
    case 1: fused_decode_attention_kernel<kDh, 1, kInd, kWin><<<grid, FaCfg<kDh, 1>::kWarps * 32, 0, st>>>(a); break;
    case 2: fused_decode_attention_kernel<kDh, 2, kInd, kWin><<<grid, FaCfg<kDh, 2>::kWarps * 32, 0, st>>>(a); break;
    case 4: fused_decode_attention_kernel<kDh, 4, kInd, kWin><<<grid, FaCfg<kDh, 4>::kWarps * 32, 0, st>>>(a); break;
    case 8: fused_decode_attention_kernel<kDh, 8, kInd, kWin><<<grid, FaCfg<kDh, 8>::kWarps * 32, 0, st>>>(a); break;
    default: return set_error(U2_ERR_UNSUPPORTED, "decode_attention_fused: Hq/Hkv = %d (supported 1, 2, 4, 8)", G);
  }
  return U2_OK;
}

template <int kDh>
static int launch_fused_decode(const FusedDecodeWinArgs& a, int G, dim3 grid, bool pdl, cudaStream_t st) {
  if (a.window > 0) {
    if (a.kv_src) return launch_fused_decode<kDh, true, true>(a, G, grid, pdl, st);
    return launch_fused_decode<kDh, false, true>(a, G, grid, pdl, st);
  }
  if (a.kv_src) return launch_fused_decode<kDh, true>(static_cast<const FusedDecodeIndArgs&>(a), G, grid, pdl, st);
  return launch_fused_decode<kDh, false>(static_cast<const FusedDecodeArgs&>(a), G, grid, pdl, st);
}

}  // namespace u2

extern "C" U2_API int u2_decode_attention_fused_bf16(const void* qkv, void* k_cache, void* v_cache, void* out,
                                                     const u2_fused_decode_desc* d, void* stream) {
  using namespace u2;
  if (!qkv || !k_cache || !v_cache || !out || !d || !d->inv_freq) return set_error(U2_ERR_ARG, "decode_attention_fused: null pointer");
  if (d->Hkv <= 0 || d->Hq % d->Hkv || d->Hq / d->Hkv > kFaMaxG)
    return set_error(U2_ERR_UNSUPPORTED, "decode_attention_fused: Hq/Hkv must be an integer <= %d", kFaMaxG);
  if (!d->pos_dev && (d->pos < 0 || d->pos >= d->Tmax)) return set_error(U2_ERR_ARG, "decode_attention_fused: position outside the cache");
  if (d->pos_per_seq && !d->pos_dev) return set_error(U2_ERR_ARG, "decode_attention_fused: pos_per_seq needs pos_dev");
  if (d->window < 0) return set_error(U2_ERR_ARG, "decode_attention_fused: window %d < 0", d->window);
  FusedDecodeWinArgs a;
  a.qkv = CBF(qkv); a.ldq = d->ldq;
  a.kc = BF(k_cache); a.vc = BF(v_cache);
  a.out = BF(out); a.ldo = d->ldo;
  a.Hq = d->Hq; a.Hkv = d->Hkv; a.Tmax = d->Tmax;
  a.pos_dev = d->pos_dev; a.pos_per_seq = d->pos_per_seq != 0; a.pos_host = d->pos;
  a.q_norm_w = d->q_norm_w; a.k_norm_w = d->k_norm_w; a.eps = d->eps;
  a.inv_freq = d->inv_freq; a.scale = d->scale;
  a.kv_src = d->kv_src; a.ld_src = d->ld_kv_src;
  a.window = d->window;
  if (a.kv_src && a.ld_src < d->Tmax) return set_error(U2_ERR_ARG, "decode_attention_fused: kv_src row stride < Tmax");
  const int splits = d->kv_splits > 1 ? d->kv_splits : 1;
  if (splits != 1 && splits != 2 && splits != 4 && splits != 8)
    return set_error(U2_ERR_ARG, "decode_attention_fused: kv_splits must be 0/1, 2, 4 or 8 (portable cluster sizes)");
  dim3 grid((unsigned)d->Hkv, (unsigned)d->B, (unsigned)splits);
  const int G = d->Hq / d->Hkv;
  int rc;
  switch (d->dh) {
    case 32: rc = launch_fused_decode<32>(a, G, grid, d->pdl != 0, ST(stream)); break;
    case 64: rc = launch_fused_decode<64>(a, G, grid, d->pdl != 0, ST(stream)); break;
    case 96: rc = launch_fused_decode<96>(a, G, grid, d->pdl != 0, ST(stream)); break;
    case 128: rc = launch_fused_decode<128>(a, G, grid, d->pdl != 0, ST(stream)); break;
    default: return set_error(U2_ERR_UNSUPPORTED, "decode_attention_fused: head_dim %d (supported 32/64/96/128)", d->dh);
  }
  if (rc) return rc;
  U2_CHECK_LAUNCH("decode_attention_fused");
  return U2_OK;
}
