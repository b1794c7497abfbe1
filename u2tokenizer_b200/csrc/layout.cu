// Data-movement kernels of the vision front and the mu2-tokenizer (all HBM-bound):
//   patchify        CT volume bricks (4x16x16 voxels) -> K-major patch rows (the im2col of the 3-D
//                   patch embedding), fp32 -> bf16
//   set_rows        broadcast a vector into selected rows (cls token)
//   transpose_heads [b, S, h, dh] -> [b, h, dh, S_pad]  (V^T for the PV contraction; X^T for DiffTS)
//   spp_pool        [frames, grid] tokens -> 2x2x2 average pooled tokens
//   multiscale_pool token-dim pooling at scales 1/2/4 with the dynamic (gated) weighting
//   embed_splice    token embedding gather + splice of the visual tokens
#include <cuda_bf16.h>
#include <math.h>

#include "host_util.h"
#include "ptx.cuh"
#include "u2b200.h"

namespace u2 {

__device__ __forceinline__ void unpack8l(const uint4& u, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8l(const float (&f)[8]) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return u;
}

// ------------------------------------------------------------------------------------------------
// patchify: vol fp32 [F, D0, D1, D2] (single channel) -> rows bf16 [F * n_patches, p0*p1*p2]
// feature order inside a patch (p0 p1 p2), token order (g0 g1 g2): MONAI "perceptron" rearrange
// "b c (h p1) (w p2) (d p3) -> b (h w d) (p1 p2 p3 c)" with c == 1.
// One thread moves 4 consecutive voxels (16 B fp32 in -> 8 B bf16 out); consecutive threads walk the
// innermost image axis so global reads are fully coalesced 128-byte lines.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
patchify_kernel(const float* __restrict__ vol, __nv_bfloat16* __restrict__ rows, long long frames, int D0,
                int D1, int D2, int p0, int p1, int p2) {
  const int q2 = D2 >> 2;  // float4 per innermost line
  const long long total = frames * D0 * D1 * q2;
  const int g1 = D1 / p1, g2 = D2 / p2;
  const int pd = p0 * p1 * p2;
  const long long npatch = (long long)(D0 / p0) * g1 * g2;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x2 = (int)(idx % q2) * 4;
    long long t = idx / q2;
    const int x1 = (int)(t % D1);
    t /= D1;
    const int x0 = (int)(t % D0);
    const long long f = t / D0;
    const float4 v = reinterpret_cast<const float4*>(vol)[idx];
    const int a0 = x0 / p0, b0 = x0 - a0 * p0;
    const int a1 = x1 / p1, b1 = x1 - a1 * p1;
    const int a2 = x2 / p2, b2 = x2 - a2 * p2;
    const long long row = f * npatch + ((long long)a0 * g1 + a1) * g2 + a2;
    const int col = (b0 * p1 + b1) * p2 + b2;
    __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&lo);
    o.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(rows + row * pd + col) = o;
  }
}

// TMA-staged variant (the default when the brick slab fits shared memory): one CTA per (frame, a0, a1) loads the
// [p0][p1][D2] fp32 slab that holds the g2 patches of one patch row with a single 3-D bulk tensor copy
// (fully coalesced 1 KB lines), converts to bf16 and writes the g2 consecutive output rows (g2 * pd * 2 bytes,
// one contiguous span) with 16-byte stores that are consecutive across the warp: both directions move whole lines.
__global__ void __launch_bounds__(256)
patchify_tma_kernel(const __grid_constant__ CUtensorMap tmap, __nv_bfloat16* __restrict__ rows, int D0, int g1,
                    int g2, int p0, int p1, int p2, int D2) {
  extern __shared__ __align__(128) float slab[];  // [p0][p1][D2]
  __shared__ uint64_t bar;
  const int a1 = blockIdx.x, a0 = blockIdx.y, f = blockIdx.z;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bar, (uint32_t)(p0 * p1 * D2 * sizeof(float)));
    tma_load_3d(slab, &tmap, &bar, 0, a1 * p1, f * D0 + a0 * p0);
  }
  mbar_wait(&bar, 0);
  const int pd = p0 * p1 * p2;
  const int cpp = pd >> 3;  // 16-byte output chunks per patch
  const long long row0 = ((long long)f * (D0 / p0) * g1 + (long long)a0 * g1 + a1) * g2;
  __nv_bfloat16* dst = rows + row0 * pd;
  for (int c = threadIdx.x; c < g2 * cpp; c += blockDim.x) {
    const int a2 = c / cpp;
    const int col = (c - a2 * cpp) << 3;
    const int b0 = col / (p1 * p2);
    const int b1 = (col / p2) % p1;
    const int b2 = col % p2;
    const float* sp = slab + ((b0 * p1 + b1) * D2 + a2 * p2 + b2);
    const float4 v0 = *reinterpret_cast<const float4*>(sp);
    const float4 v1 = *reinterpret_cast<const float4*>(sp + 4);
    uint4 o;
    __nv_bfloat162* h2 = reinterpret_cast<__nv_bfloat162*>(&o);
    h2[0] = __floats2bfloat162_rn(v0.x, v0.y);
    h2[1] = __floats2bfloat162_rn(v0.z, v0.w);
    h2[2] = __floats2bfloat162_rn(v1.x, v1.y);
    h2[3] = __floats2bfloat162_rn(v1.z, v1.w);
    *reinterpret_cast<uint4*>(dst + (long long)a2 * pd + col) = o;
  }
}

__global__ void set_rows_kernel(__nv_bfloat16* __restrict__ dst, const __nv_bfloat16* __restrict__ vec,
                                long long n_rows, long long row_stride, long long row_off, int E) {
  const long long total = n_rows * E;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / E;
    const int c = (int)(idx - r * E);
    dst[(r * row_stride + row_off) * E + c] = vec[c];
  }
}

// ViT sequence buffer [frames][Sp][E]: row 0 of every frame = cls token, rows [S, Sp) (the 16-byte alignment padding) = 0.
// One launch replaces zero-filling the whole buffer: rows 1..S-1 are written by the patch-embed GEMM's epilogue.
__global__ void vit_frame_rows_kernel(__nv_bfloat16* __restrict__ dst, const __nv_bfloat16* __restrict__ cls, long long frames,
                                      int Sp, int S, int E) {
  const int per = 1 + (Sp - S);
  const long long total = frames * per * E;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % E);
    const long long t = idx / E;
    const int k = (int)(t % per);
    const long long f = t / per;
    const int row = k == 0 ? 0 : S + k - 1;
    dst[(f * Sp + row) * E + c] = k == 0 ? cls[c] : __float2bfloat16(0.f);
  }
}

// ------------------------------------------------------------------------------------------------
// transpose_heads: in[b][s][h][d] (strides given) -> out[b][h][d][s], s padded to ld_out.
// 32x32 smem tiles, bf16.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
transpose_heads_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int S, int H,
                       int Dh, long long in_sb, long long in_ss, long long in_sh, long long out_sb,
                       long long out_sh, long long ld_out) {
  __shared__ __nv_bfloat16 tile[32][34];
  const int bh = blockIdx.z;
  const int b = bh / H, h = bh - b * H;
  const int s0 = blockIdx.x * 32, d0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const __nv_bfloat16* src = in + b * in_sb + h * in_sh;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int s = s0 + ty + k * 8, d = d0 + tx;
    tile[ty + k * 8][tx] = (s < S && d < Dh) ? src[(long long)s * in_ss + d] : __float2bfloat16(0.f);
  }
  __syncthreads();
  __nv_bfloat16* dst = out + b * out_sb + h * out_sh;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int d = d0 + ty + k * 8, s = s0 + tx;
    if (d < Dh && s < ld_out) dst[(long long)d * ld_out + s] = tile[tx][ty + k * 8];  // zeros beyond S
  }
}

// ------------------------------------------------------------------------------------------------
// spp_pool: x [F, in_row_stride rows..., E] with token (a0,a1,a2) at row in_off + (a0*g1+a1)*g2+a2
//   -> out [F, (g0/ps)(g1/ps)(g2/ps), E] mean over ps^3 neighbours (avg_pool3d, stride = kernel).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
spp_pool_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out, long long frames,
                int g0, int g1, int g2, int ps, int E, long long in_frame_stride, long long in_off,
                long long ldx) {
  const int o0 = g0 / ps, o1 = g1 / ps, o2 = g2 / ps;
  const int nvec = E >> 3;
  const long long total = frames * o0 * o1 * o2 * nvec;
  const float inv = 1.f / (ps * ps * ps);
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % nvec);
    long long t = idx / nvec;
    const int c2 = (int)(t % o2);
    t /= o2;
    const int c1 = (int)(t % o1);
    t /= o1;
    const int c0 = (int)(t % o0);
    const long long f = t / o0;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i0 = 0; i0 < ps; ++i0)
      for (int i1 = 0; i1 < ps; ++i1)
        for (int i2 = 0; i2 < ps; ++i2) {
          const long long tok = ((long long)(c0 * ps + i0) * g1 + (c1 * ps + i1)) * g2 + (c2 * ps + i2);
          float v[8];
          unpack8l(reinterpret_cast<const uint4*>(x + (f * in_frame_stride + in_off + tok) * ldx)[c], v);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += v[j];
        }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
    const long long orow = ((f * o0 + c0) * o1 + c1) * o2 + c2;
    reinterpret_cast<uint4*>(out + orow * E)[c] = pack8l(acc);
  }
}

// sequence pooling variant (avg_pool1d over ps^3 consecutive tokens)
__global__ void __launch_bounds__(256)
seq_pool_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out, long long frames,
                int n_out, int k, int E, long long in_frame_stride, long long in_off, long long ldx) {
  const int nvec = E >> 3;
  const long long total = frames * n_out * nvec;
  const float inv = 1.f / k;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % nvec);
    long long t = idx / nvec;
    const int o = (int)(t % n_out);
    const long long f = t / n_out;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < k; ++i) {
      float v[8];
      unpack8l(reinterpret_cast<const uint4*>(x + (f * in_frame_stride + in_off + (long long)o * k + i) * ldx)[c], v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
    reinterpret_cast<uint4*>(out + (f * n_out + o) * E)[c] = pack8l(acc);
  }
}

// ------------------------------------------------------------------------------------------------
// multi-scale pooling (scales 1, 2, 4 over the token dim) with the dynamic gate:
//   pass 1 (gate): part[b][blk][k] = sum over the block's rows of sum_e w[e] * pool_k(x)[e] / covered rows
//   pass 1b:       logits[b][k] = sum_blk part[b][blk][k], in block order (the same bits on every run; float
//                  atomics would add the blocks in the order they happen to finish)
//   pass 2 (write): out[b] = cat_k softmax(logits[b] + bias)[k] * pool_k(x[b])
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
msp_gate_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gate_w, float* __restrict__ part,
                int K, int E, int rows_per_block) {
  // grid: (ceil(K / rows_per_block), B); each thread owns E/8-vector columns strided by blockDim
  const int b = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(K, r0 + rows_per_block);
  const int nvec = E >> 3;
  const int n2 = (K / 2) * 2, n4 = (K / 4) * 4;  // avg_pool1d drops the ragged tail
  float p1 = 0.f, p2 = 0.f, p4 = 0.f;
  for (int c = threadIdx.x; c < nvec; c += blockDim.x) {
    const float4 w0 = reinterpret_cast<const float4*>(gate_w)[2 * c];
    const float4 w1 = reinterpret_cast<const float4*>(gate_w)[2 * c + 1];
    const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    for (int r = r0; r < r1; ++r) {
      float v[8];
      unpack8l(reinterpret_cast<const uint4*>(x + ((long long)b * K + r) * E)[c], v);
      float d = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) d += v[j] * w[j];
      p1 += d;
      if (r < n2) p2 += d;
      if (r < n4) p4 += d;
    }
  }
  __shared__ float red[3][8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    p1 += __shfl_xor_sync(0xffffffffu, p1, o);
    p2 += __shfl_xor_sync(0xffffffffu, p2, o);
    p4 += __shfl_xor_sync(0xffffffffu, p4, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = p1;
    red[1][threadIdx.x >> 5] = p2;
    red[2][threadIdx.x >> 5] = p4;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[threadIdx.x][w];
    // mean over the pooled tokens of scale k == sum over the covered input rows / covered rows
    const int denom = threadIdx.x == 0 ? K : (threadIdx.x == 1 ? n2 : n4);
    part[((long long)b * gridDim.x + blockIdx.x) * 3 + threadIdx.x] = denom > 0 ? s / denom : 0.f;
  }
}

__global__ void __launch_bounds__(256)
msp_gate_sum_kernel(const float* __restrict__ part, float* __restrict__ logits, int B, int nblk) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 3 * B; i += gridDim.x * blockDim.x) {
    const int b = i / 3, k = i - 3 * b;
    float s = 0.f;
    for (int j = 0; j < nblk; ++j) s += part[((long long)b * nblk + j) * 3 + k];
    logits[i] = s;
  }
}

__global__ void __launch_bounds__(256)
msp_write_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ logits, float gate_bias,
                 int dynamic, __nv_bfloat16* __restrict__ out, int B, int K, int E) {
  const int nvec = E >> 3;
  const int k1 = K, k2 = (K >= 2) ? K / 2 : 0, k4 = (K >= 4) ? K / 4 : 0;
  const int n_out = k1 + k2 + k4;
  const long long total = (long long)B * n_out * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % nvec);
    long long t = idx / nvec;
    const int o = (int)(t % n_out);
    const int b = (int)(t / n_out);
    int scale, first, sidx;
    if (o < k1) { scale = 1; first = o; sidx = 0; }
    else if (o < k1 + k2) { scale = 2; first = (o - k1) * 2; sidx = 1; }
    else { scale = 4; first = (o - k1 - k2) * 4; sidx = 2; }
    float wgt = 1.f;
    if (dynamic) {
      // softmax over the scales that exist
      float l[3] = {logits[b * 3 + 0] + gate_bias, k2 ? logits[b * 3 + 1] + gate_bias : -INFINITY,
                    k4 ? logits[b * 3 + 2] + gate_bias : -INFINITY};
      const float m = fmaxf(l[0], fmaxf(l[1], l[2]));
      const float e0 = __expf(l[0] - m), e1 = k2 ? __expf(l[1] - m) : 0.f, e2 = k4 ? __expf(l[2] - m) : 0.f;
      const float es[3] = {e0, e1, e2};
      wgt = es[sidx] / (e0 + e1 + e2);
    }
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < scale; ++i) {
      float v[8];
      unpack8l(reinterpret_cast<const uint4*>(x + ((long long)b * K + first + i) * E)[c], v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
    const float f = wgt / scale;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= f;
    reinterpret_cast<uint4*>(out + ((long long)b * n_out + o) * E)[c] = pack8l(acc);
  }
}

// ------------------------------------------------------------------------------------------------
// embed_splice: out[b][l] = (1 <= l <= n_vis && vis) ? vis[b][l-1] : table[ids[b][l]]
// (reference u2_arch.py:118-121: the visual tokens overwrite positions 1..n_vis)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
embed_splice_kernel(const long long* __restrict__ ids, const __nv_bfloat16* __restrict__ table,
                    const __nv_bfloat16* __restrict__ vis, __nv_bfloat16* __restrict__ out, int B, int L,
                    int E, int n_vis, long long vocab) {
  const int nvec = E >> 3;
  const long long total = (long long)B * L * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % nvec);
    const long long bl = idx / nvec;
    const int l = (int)(bl % L);
    const int b = (int)(bl / L);
    uint4 v;
    if (vis && l >= 1 && l <= n_vis) {
      v = reinterpret_cast<const uint4*>(vis + ((long long)b * n_vis + (l - 1)) * E)[c];
    } else {
      long long id = ids[bl];
      if (id < 0) id = 0;
      if (id >= vocab) id = vocab - 1;
      v = reinterpret_cast<const uint4*>(table + id * E)[c];
    }
    reinterpret_cast<uint4*>(out + bl * E)[c] = v;
  }
}

static inline unsigned grid_for(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = 132LL * 32;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

}  // namespace u2

using namespace u2;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)

extern "C" U2_API int u2_patchify_f32_bf16(const float* vol, void* rows, int64_t frames, int32_t d0, int32_t d1,
                                           int32_t d2, int32_t p0, int32_t p1, int32_t p2, void* stream) {
  if (!vol || !rows) return set_error(U2_ERR_ARG, "patchify: null pointer");
  if (p0 <= 0 || p1 <= 0 || p2 <= 0 || d0 % p0 || d1 % p1 || d2 % p2 || (p2 & 3) || (d2 & 3))
    return set_error(U2_ERR_ARG, "patchify: image dims must be multiples of the patch dims and p2 %% 4 == 0");
  if (reinterpret_cast<uintptr_t>(vol) & 15) return set_error(U2_ERR_ARG, "patchify: volume must be 16-byte aligned");
  const long long total = (long long)frames * d0 * d1 * (d2 / 4);
  if (total <= 0) return U2_OK;
  const size_t slab_bytes = (size_t)p0 * p1 * d2 * sizeof(float);
  const bool tma_ok = d2 <= 256 && p1 <= 256 && p0 <= 256 && (p2 % 8) == 0 && slab_bytes <= 96 * 1024 &&
                      frames <= 65535 && (d0 / p0) <= 65535 && (long long)frames * d0 < (1LL << 31);
  if (tma_ok) {
    CUtensorMap tm;
    int rc = make_tmap_f32_3d(&tm, vol, d2, d1, (int64_t)frames * d0, d2, (int64_t)d1 * d2, d2, p1, p0);
    if (rc) return rc;
    static size_t configured = 0;
    if (slab_bytes > 48 * 1024 && slab_bytes > configured) {
      cudaError_t e = cudaFuncSetAttribute(patchify_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)slab_bytes);
      if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "patchify smem: %s", cudaGetErrorString(e));
      configured = slab_bytes;
    }
    dim3 grid((unsigned)(d1 / p1), (unsigned)(d0 / p0), (unsigned)frames);
    patchify_tma_kernel<<<grid, 256, slab_bytes, ST(stream)>>>(tm, BF(rows), d0, d1 / p1, d2 / p2, p0, p1, p2, d2);
  } else {
    patchify_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(vol, BF(rows), frames, d0, d1, d2, p0, p1, p2);
  }
  U2_CHECK_LAUNCH("patchify");
  return U2_OK;
}

extern "C" U2_API int u2_set_rows_bf16(void* dst, const void* vec, int64_t n_rows, int64_t row_stride,
                                       int64_t row_off, int32_t E, void* stream) {
  if (!dst || !vec) return set_error(U2_ERR_ARG, "set_rows: null pointer");
  if (n_rows <= 0 || E <= 0) return U2_OK;
  set_rows_kernel<<<grid_for(n_rows * E, 256), 256, 0, ST(stream)>>>(BF(dst), CBF(vec), n_rows, row_stride, row_off, E);
  U2_CHECK_LAUNCH("set_rows");
  return U2_OK;
}

extern "C" U2_API int u2_vit_frame_rows_bf16(void* dst, const void* cls, int64_t frames, int32_t Sp, int32_t S, int32_t E,
                                             void* stream) {
  if (!dst || !cls) return set_error(U2_ERR_ARG, "vit_frame_rows: null pointer");
  if (frames <= 0 || E <= 0 || S <= 0 || Sp < S) return set_error(U2_ERR_ARG, "vit_frame_rows: bad extents");
  vit_frame_rows_kernel<<<grid_for(frames * (1 + Sp - S) * E, 256), 256, 0, ST(stream)>>>(BF(dst), CBF(cls), frames, Sp, S, E);
  U2_CHECK_LAUNCH("vit_frame_rows");
  return U2_OK;
}

extern "C" U2_API int u2_transpose_heads_bf16(const void* in, void* out, int32_t B, int32_t S, int32_t H,
                                              int32_t Dh, int64_t in_sb, int64_t in_ss, int64_t in_sh,
                                              int64_t out_sb, int64_t out_sh, int64_t ld_out, void* stream) {
  if (!in || !out) return set_error(U2_ERR_ARG, "transpose_heads: null pointer");
  if (B <= 0 || S <= 0 || H <= 0 || Dh <= 0) return U2_OK;
  if (ld_out < S) return set_error(U2_ERR_ARG, "transpose_heads: ld_out < S");
  if ((long long)B * H > 65535) return set_error(U2_ERR_ARG, "transpose_heads: B*H > 65535");
  dim3 grid((unsigned)((ld_out + 31) / 32), (unsigned)((Dh + 31) / 32), (unsigned)(B * H));
  transpose_heads_kernel<<<grid, 256, 0, ST(stream)>>>(CBF(in), BF(out), S, H, Dh, in_sb, in_ss, in_sh, out_sb,
                                                      out_sh, ld_out);
  U2_CHECK_LAUNCH("transpose_heads");
  return U2_OK;
}

extern "C" U2_API int u2_spp_pool_bf16(const void* x, void* out, int64_t frames, int32_t g0, int32_t g1, int32_t g2,
                                       int32_t ps, int32_t E, int64_t in_frame_stride, int64_t in_off, int64_t ldx,
                                       int32_t sequence, void* stream) {
  if (!x || !out) return set_error(U2_ERR_ARG, "spp_pool: null pointer");
  if ((E & 7) || (ldx & 7) || ps <= 0) return set_error(U2_ERR_ARG, "spp_pool: E/ldx must be multiples of 8");
  if (sequence) {
    const int k = ps * ps * ps;
    const int n_out = (g0 * g1 * g2) / k;
    const long long total = frames * n_out * (E / 8);
    if (total <= 0) return U2_OK;
    seq_pool_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(CBF(x), BF(out), frames, n_out, k, E, in_frame_stride, in_off, ldx);
  } else {
    const long long total = frames * (g0 / ps) * (g1 / ps) * (g2 / ps) * (E / 8);
    if (total <= 0) return U2_OK;
    spp_pool_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(CBF(x), BF(out), frames, g0, g1, g2, ps, E, in_frame_stride, in_off, ldx);
  }
  U2_CHECK_LAUNCH("spp_pool");
  return U2_OK;
}

constexpr int kMspRowsPerBlock = 16;

extern "C" U2_API int64_t u2_multiscale_pool_ws_elems(int32_t B, int32_t K) {
  if (B <= 0 || K <= 0) return 0;
  return 3LL * B * (1 + (K + kMspRowsPerBlock - 1) / kMspRowsPerBlock);
}

extern "C" U2_API int u2_multiscale_pool_bf16(const void* x, void* out, const float* gate_w, float gate_bias,
                                              float* logits_ws, int32_t B, int32_t K, int32_t E, int32_t dynamic,
                                              void* stream) {
  if (!x || !out) return set_error(U2_ERR_ARG, "multiscale_pool: null pointer");
  if (E & 7) return set_error(U2_ERR_ARG, "multiscale_pool: E must be a multiple of 8");
  if (B <= 0 || K <= 0) return U2_OK;
  if (dynamic) {
    if (!gate_w || !logits_ws)
      return set_error(U2_ERR_ARG, "multiscale_pool: dynamic gate needs gate_w and a u2_multiscale_pool_ws_elems(B, K) fp32 workspace");
    const int nblk = (K + kMspRowsPerBlock - 1) / kMspRowsPerBlock;
    float* part = logits_ws + 3 * B;
    dim3 grid((unsigned)nblk, (unsigned)B);
    msp_gate_kernel<<<grid, 256, 0, ST(stream)>>>(CBF(x), gate_w, part, K, E, kMspRowsPerBlock);
    U2_CHECK_LAUNCH("multiscale_pool gate");
    msp_gate_sum_kernel<<<(unsigned)((3 * B + 255) / 256), 256, 0, ST(stream)>>>(part, logits_ws, B, nblk);
    U2_CHECK_LAUNCH("multiscale_pool gate sum");
  }
  const int n_out = K + (K >= 2 ? K / 2 : 0) + (K >= 4 ? K / 4 : 0);
  const long long total = (long long)B * n_out * (E / 8);
  msp_write_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(CBF(x), logits_ws, gate_bias, dynamic, BF(out), B, K, E);
  U2_CHECK_LAUNCH("multiscale_pool write");
  return U2_OK;
}

extern "C" U2_API int u2_embed_splice_bf16(const int64_t* ids, const void* table, const void* vis, void* out,
                                           int32_t B, int32_t L, int32_t E, int32_t n_vis, int64_t vocab,
                                           void* stream) {
  if (!ids || !table || !out) return set_error(U2_ERR_ARG, "embed_splice: null pointer");
  if (E & 7) return set_error(U2_ERR_ARG, "embed_splice: E must be a multiple of 8");
  if (vis && n_vis + 1 > L) return set_error(U2_ERR_ARG, "embed_splice: prompt shorter than n_vis + 1");
  const long long total = (long long)B * L * (E / 8);
  if (total <= 0) return U2_OK;
  embed_splice_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(reinterpret_cast<const long long*>(ids), CBF(table), CBF(vis), BF(out), B, L, E, n_vis, vocab);
  U2_CHECK_LAUNCH("embed_splice");
  return U2_OK;
}

// ------------------------------------------------------------------------------------------------
// top-k over rows of fp32 scores (hard TokenSelection, reference svr.py:75-91: torch.topk sorted descending).
// One CTA per row: bitonic sort of 64-bit keys (score descending, index ascending on ties) in shared memory.
// ------------------------------------------------------------------------------------------------
namespace u2 {

__global__ void __launch_bounds__(1024)
topk_rows_kernel(const float* __restrict__ scores, long long ld, int T, int K, long long* __restrict__ out_idx,
                 long long idx_offset_per_row, int n_pad) {
  extern __shared__ unsigned long long keys[];
  const int row = blockIdx.x;
  const float* s = scores + (long long)row * ld;
  for (int i = threadIdx.x; i < n_pad; i += blockDim.x) {
    unsigned long long k = ~0ull;
    if (i < T) {
      unsigned int u = __float_as_uint(s[i]);
      if (u == 0x80000000u) u = 0u;  // -0.0 == +0.0
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // order-preserving map float -> uint
      k = ((unsigned long long)(~u) << 32) | (unsigned int)i;  // ascending key == descending score, then index
    }
    keys[i] = k;
  }
  __syncthreads();
  for (int k = 2; k <= n_pad; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n_pad; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = keys[i], b = keys[l];
          const bool up = ((i & k) == 0);
          if ((a > b) == up) {
            keys[i] = b;
            keys[l] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < K; i += blockDim.x)
    out_idx[(long long)row * K + i] = (long long)(keys[i] & 0xffffffffull) + (long long)row * idx_offset_per_row;
}

}  // namespace u2

extern "C" U2_API int u2_topk_rows_f32(const float* scores, int64_t* out_idx, int32_t rows, int32_t T, int32_t K,
                                       int64_t ld, int64_t idx_offset_per_row, void* stream) {
  using namespace u2;
  if (!scores || !out_idx) return set_error(U2_ERR_ARG, "topk: null pointer");
  if (K <= 0 || K > T) return set_error(U2_ERR_ARG, "topk: need 0 < K <= T (reference torch.topk raises too)");
  if (T > 16384) return set_error(U2_ERR_UNSUPPORTED, "topk: T=%d > 16384 (keys are sorted in shared memory)", T);
  if (rows <= 0) return U2_OK;
  int n_pad = 1;
  while (n_pad < T) n_pad <<= 1;
  const size_t smem = (size_t)n_pad * sizeof(unsigned long long);
  static bool cfgd = false;
  if (!cfgd) {
    cudaError_t e = cudaFuncSetAttribute(topk_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 8);
    if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "topk smem: %s", cudaGetErrorString(e));
    cfgd = true;
  }
  topk_rows_kernel<<<rows, 1024, smem, ST(stream)>>>(scores, ld, T, K, reinterpret_cast<long long*>(out_idx),
                                                    idx_offset_per_row, n_pad);
  U2_CHECK_LAUNCH("topk");
  return U2_OK;
}
