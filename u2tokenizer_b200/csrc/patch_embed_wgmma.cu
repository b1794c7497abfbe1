// Fused 3-D patch embedding (K1 / K2 of SURVEY.md section 2d): fp32 CT volume -> bf16 ViT tokens in ONE kernel.
//
//   x[f, 1 + t, :] = bf16( patch(f, t) [1024 fp32 voxels] . W^T + bias + pos[t] )      t = (h, w, d) over the 8 x 16 x 16 grid
//
// The einops gather "b c (h p1) (w p2) (d p3) -> b (h w d) (p1 p2 p3 c)" of MONAI's PatchEmbeddingBlock (reference
// src/model/multimodal_encoder/vit.py:90-99,115) never materialises: a 128-token M tile is the 8 (w) x 16 (d) tokens of one
// (frame, h) slab, and k-block kb = (p1, 4 consecutive p2, 16 p3) of those tokens is ONE 5-D TMA box
// {256 (D2), 4 (p2), 8 (w), 1 (D0 = 4 h + p1), 1 (frame)} = 32 KB of fp32 that lands in shared memory as
// [w][p2][256]. A converter warp-group (thread = token) rewrites it as the 128 x 64 bf16 K-major SWIZZLE_128B A tile the
// tensor core wants (bank-conflict-free: the four 16-byte pieces of a thread's 64-byte segment are read in an order
// rotated by the token index), the MMA warpgroup accumulates with wgmma in registers and its epilogue adds bias + position
// embedding and stores the rows behind the cls row. The unfused path wrote and re-read 134 MB of bf16 im2col rows per 4
// volumes; here the volume is read once (the N tiles of an M tile run on neighbouring CTAs in the same time window, so the
// later reads of a slab hit L2).
//
// Warp roles (384 threads, 1 CTA / SM, persistent over (m tile, n tile)):
//   warp 0      TMA producer: fp32 slabs -> 3-stage staging ring (96 KB in flight)
//   warp 1      TMA producer: W tiles (128 x 64 bf16) -> 2-stage ring
//   warps 4-7   converter warp-group (fp32 staging -> swizzled bf16 A ring, 2 stages)
//   warps 8-11  MMA warpgroup: 128 x 128 x 16 per k step as wgmma 64 x 64 x 16 pieces, fp32 accumulators in registers,
//               then the bias + position epilogue straight from the accumulator fragment
#include <cuda_bf16.h>
#include <stdlib.h>

#include "host_util.h"
#include "ptx.cuh"
#include "u2b200.h"

namespace u2 {

constexpr int kPeM = 128, kPeN = 128, kPeK = 64;
constexpr int kPeStg = 3, kPeA = 2, kPeB = 2;
constexpr int kPeStgBytes = 128 * 64 * 4;   // 32 KB fp32 slab
constexpr int kPeABytes = kPeM * kPeK * 2;  // 16 KB
constexpr int kPeBBytes = kPeN * kPeK * 2;  // 16 KB
constexpr int kPeSmem = kPeA * kPeABytes + kPeB * kPeBBytes + kPeStg * kPeStgBytes + 1024 + 256;
constexpr int kPeThreads = 384;
constexpr int kPeConvWarp0 = 4, kPeMmaWarp0 = 8;

struct PeArgs {
  int frames, g0, g1, g2;   // token grid per frame (8, 16, 16)
  int p0, p1;               // patch extents along D0, D1 (4, 16); the extent along D2 is 16
  int N;                    // hidden size (768)
  int P, Sp;                // tokens per frame, padded rows per frame of the output buffer
  const float* bias;        // [N]
  const __nv_bfloat16* pos; // [P, N]
  __nv_bfloat16* out;       // [frames, Sp, N]; token t goes to row 1 + t
  int dbg;                  // timing experiments only (U2_PE_DBG): 1 no proxy fence, 2 no staging reads, 4 no A-tile stores
};

// 5-D tiled load (fp32 slab of the volume)
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
        "r"(c4)
      : "memory");
}

__global__ void __launch_bounds__(kPeThreads, 1)
patch_embed_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_vol, const __grid_constant__ CUtensorMap tmap_w,
                           const PeArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = sA + kPeA * kPeABytes;
  uint8_t* sStg = sB + kPeB * kPeBBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStg + kPeStg * kPeStgBytes);
  uint64_t* stg_full = bars;                 // [kPeStg]
  uint64_t* stg_empty = stg_full + kPeStg;   // [kPeStg]
  uint64_t* a_full = stg_empty + kPeStg;     // [kPeA]
  uint64_t* a_empty = a_full + kPeA;         // [kPeA]
  uint64_t* b_full = a_empty + kPeA;         // [kPeB]
  uint64_t* b_empty = b_full + kPeB;         // [kPeB]

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int w_tiles = p.g1 / 8;                                // M tiles per (frame, h)
  const int num_m = p.frames * p.g0 * w_tiles;
  const int num_n = (p.N + kPeN - 1) / kPeN;
  const int num_tiles = num_m * num_n;
  const int kb_per_p0 = p.p1 / 4;
  const int num_kb = p.p0 * kb_per_p0;                          // 16

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_vol);
    tma_prefetch_desc(&tmap_w);
  }
  if (warp_idx == 1 && lane == 0) {
    // consumer barriers count WARPS, not threads: 128 mbarrier.arrive on one barrier serialise (~10 ns each) - with per-thread
    // arrivals on a_full and stg_empty every k-block cost 2.5 us whatever the converter did (first version: 419 us per pass)
    for (int s = 0; s < kPeStg; ++s) { mbar_init(&stg_full[s], 1); mbar_init(&stg_empty[s], 4); }
    for (int s = 0; s < kPeA; ++s) { mbar_init(&a_full[s], 4); mbar_init(&a_empty[s], 4); }
    for (int s = 0; s < kPeB; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp_idx == 0) {
    // ===================== TMA producer 1: fp32 volume slabs =====================
    // (separate from the weight-tile producer: with one thread feeding both rings the slab prefetch depth was tied to the
    //  2-stage weight ring and every other k-block paid a full HBM latency)
    if (lane == 0) {
      int ss = 0;
      uint32_t sph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / num_n;
        const int wt = m_blk % w_tiles;
        const int fh = m_blk / w_tiles;
        const int h = fh % p.g0, f = fh / p.g0;
        for (int kb = 0; kb < num_kb; ++kb) {
          const int q0 = kb / kb_per_p0, q1 = (kb - q0 * kb_per_p0) * 4;
          mbar_wait(&stg_empty[ss], sph ^ 1);
          mbar_arrive_expect_tx(&stg_full[ss], kPeStgBytes);
          tma_load_5d(sStg + ss * kPeStgBytes, &tmap_vol, &stg_full[ss], 0, q1, wt * 8, h * p.p0 + q0, f);
          if (++ss == kPeStg) { ss = 0; sph ^= 1; }
        }
      }
    }
  } else if (warp_idx == 1) {
    // ===================== TMA producer 2: weight tiles =====================
    if (lane == 0) {
      int bs = 0;
      uint32_t bph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n_blk = tile % num_n;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&b_empty[bs], bph ^ 1);
          mbar_arrive_expect_tx(&b_full[bs], kPeBBytes);
          tma_load_4d(sB + bs * kPeBBytes, &tmap_w, &b_full[bs], kb * kPeK, n_blk * kPeN, 0, 0);
          if (++bs == kPeB) { bs = 0; bph ^= 1; }
        }
      }
    }
  } else if (warp_idx >= kPeConvWarp0 && warp_idx < kPeMmaWarp0) {
    // ===================== converter: fp32 [w][p2][256] slab -> bf16 K-major SW128 A tile =====================
    // A staging row (w, p2) holds 16 tokens (d) x 16 fp32 (p3) = 1 KB: a warp reads it with two fully coalesced 16-byte
    // loads per lane (lane l -> token d = l / 4 (+ 8), p3 quarter l % 4), converts and writes 8 bytes into row
    // r = 16 w + d of the A tile at chunk (2 p2 + quarter / 2) ^ (r & 7): 32 lanes x 8 B cover every bank exactly twice.
    // All register indices are static (the first version routed pieces with data-dependent selects, which the compiler
    // turned into divergent branch trees: 819 instructions per warp and k-block, 2.5 us per k-block).
    const int cw = warp_idx - kPeConvWarp0;   // this warp converts w = 2 cw, 2 cw + 1
    const int dq = lane >> 2, quarter = lane & 3;
    int ss = 0, as = 0;
    uint32_t sph = 0, aph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&stg_full[ss], sph);
        mbar_wait(&a_empty[as], aph ^ 1);
        const uint32_t src0 = smem_u32(sStg) + ss * kPeStgBytes + lane * 16;
        const uint32_t dst0 = smem_u32(sA) + as * kPeABytes + (quarter & 1) * 8;
#pragma unroll
        for (int wi = 0; wi < 2; ++wi) {
          const int w = 2 * cw + wi;
#pragma unroll
          for (int q = 0; q < 4; ++q) {      // p2 offset inside the k-block
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const float4 v = (p.dbg & 2) ? make_float4(1.f, 2.f, 3.f, 4.f)
                                           : lds128_f32(src0 + (w * 4 + q) * 1024 + half * 512);
              const int r = w * 16 + half * 8 + dq;
              const int chunk = 2 * q + (quarter >> 1);
              __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
              if (!(p.dbg & 4))
                sts64(dst0 + r * 128 + ((chunk ^ (r & 7)) << 4), *reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
            }
          }
        }
        if (!(p.dbg & 1)) fence_proxy_async_smem();  // generic-proxy stores -> visible to the tensor core's async-proxy reads
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&a_full[as]);
          mbar_arrive(&stg_empty[ss]);
        }
        if (++ss == kPeStg) { ss = 0; sph ^= 1; }
        if (++as == kPeA) { as = 0; aph ^= 1; }
      }
    }
  } else if (warp_idx >= kPeMmaWarp0) {
    // ===================== MMA warpgroup + epilogue =====================
    const int w = warp_idx - kPeMmaWarp0;
    int as = 0, bs = 0;
    uint32_t aph = 0, bph = 0;
    float acc[2][2][32];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile / num_n, n_blk = tile - m_blk * num_n;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&a_full[as], aph);
        mbar_wait(&b_full[bs], bph);
        const uint64_t a_desc = gmma_desc_sw128(smem_u32(sA + as * kPeABytes));
        const uint64_t b_desc = gmma_desc_sw128(smem_u32(sB + bs * kPeBBytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kPeK / 16; ++k) {
#pragma unroll
          for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
            for (int nc = 0; nc < 2; ++nc)  // tokens / W rows 64..127 start 8 KB further
              wgmma_m64n64k16_ss<0, 0>(acc[mh][nc], a_desc + 512 * mh + 2 * k, b_desc + 512 * nc + 2 * k, (kb | k) != 0);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (lane == 0) {
          mbar_arrive(&a_empty[as]);
          mbar_arrive(&b_empty[bs]);
        }
        if (++as == kPeA) { as = 0; aph ^= 1; }
        if (++bs == kPeB) { bs = 0; bph ^= 1; }
      }
      // ---- epilogue: + bias + position embedding, bf16 pairs straight from the fragment
#pragma unroll
      for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const long long grow = (long long)m_blk * kPeM + mh * 64 + w * 16 + (lane >> 2) + 8 * hr;  // frame * P + t
          const int t = (int)(grow % p.P);
          const long long orow = (grow / p.P) * p.Sp + 1 + t;
          const __nv_bfloat16* prow = p.pos + (long long)t * p.N;
#pragma unroll
          for (int nc = 0; nc < 2; ++nc) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int col = n_blk * kPeN + nc * 64 + 8 * i + 2 * (lane & 3);
              if (col < p.N) {
                const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                const float2 pp = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(prow + col));
                *reinterpret_cast<__nv_bfloat162*>(p.out + orow * p.N + col) = __floats2bfloat162_rn(
                    acc[mh][nc][4 * i + 2 * hr] + bb.x + pp.x, acc[mh][nc][4 * i + 2 * hr + 1] + bb.y + pp.y);
              }
            }
          }
        }
      }
    }
  }
}

}  // namespace u2

extern "C" U2_API int u2_patch_embed_f32_bf16(const float* vol, const void* W, const float* bias, const void* pos, void* out,
                                              int64_t frames, int32_t d0, int32_t d1, int32_t d2, int32_t p0, int32_t p1,
                                              int32_t p2, int32_t N, int64_t out_frame_rows, void* stream) {
  using namespace u2;
  if (!vol || !W || !bias || !pos || !out) return set_error(U2_ERR_ARG, "patch_embed: null pointer");
  if (p0 <= 0 || p1 <= 0 || p2 <= 0 || d0 % p0 || d1 % p1 || d2 % p2) return set_error(U2_ERR_ARG, "patch_embed: image not divisible by the patch");
  const int g0 = d0 / p0, g1 = d1 / p1, g2 = d2 / p2;
  // the fused tiling: 16-voxel patch rows along D2, 16 tokens along D2 per (h, w) and groups of 8 w per M tile
  if (p2 != 16 || g2 != 16 || (p1 & 3) || (g1 & 7) || d2 > 256 || (N & 31))
    return set_error(U2_ERR_UNSUPPORTED, "patch_embed: fused kernel covers patch (*, 4k, 16) on a (*, 8m, 16) token grid with D2 <= 256 "
                                         "(got patch %d x %d x %d, grid %d x %d x %d); use u2_patchify_f32_bf16 + u2_gemm_bf16", p0, p1, p2, g0, g1, g2);
  const long long P = (long long)g0 * g1 * g2;
  if (out_frame_rows < P + 1) return set_error(U2_ERR_ARG, "patch_embed: out_frame_rows must be >= tokens + 1 (cls row)");
  if ((reinterpret_cast<uintptr_t>(vol) & 15) || (reinterpret_cast<uintptr_t>(W) & 15) || (reinterpret_cast<uintptr_t>(out) & 15) ||
      (reinterpret_cast<uintptr_t>(pos) & 15) || (reinterpret_cast<uintptr_t>(bias) & 15))
    return set_error(U2_ERR_ARG, "patch_embed: pointers must be 16-byte aligned");
  if (frames <= 0) return U2_OK;
  const int K = p0 * p1 * p2;
  CUtensorMap tv, tw;
  {
    // volume [frames][D0][D1 = (w, p2)][D2] fp32 as a 5-D map {D2, p2, w, D0, frame}; box {D2, 4, 8, 1, 1}
    const int64_t dims[5] = {d2, p1, g1, d0, frames};
    const int64_t strides[4] = {(int64_t)d2 * 4, (int64_t)p1 * d2 * 4, (int64_t)d1 * d2 * 4, (int64_t)d0 * d1 * d2 * 4};
    const int box[5] = {d2, 4, 8, 1, 1};
    int rc = make_tmap_f32_nd(&tv, vol, 5, dims, strides, box);
    if (rc) return rc;
  }
  int rc = make_tmap_bf16_4d(&tw, W, K, N, 1, 1, K, 0, 0, kPeK, kPeN);
  if (rc) return rc;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(patch_embed_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPeSmem);
    if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "patch_embed: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  PeArgs a;
  a.frames = (int)frames; a.g0 = g0; a.g1 = g1; a.g2 = g2; a.p0 = p0; a.p1 = p1; a.N = N;
  a.P = (int)P; a.Sp = (int)out_frame_rows;
  a.dbg = getenv("U2_PE_DBG") ? atoi(getenv("U2_PE_DBG")) : 0;
  a.bias = bias; a.pos = reinterpret_cast<const __nv_bfloat16*>(pos); a.out = reinterpret_cast<__nv_bfloat16*>(out);
  const long long tiles = (long long)frames * g0 * (g1 / 8) * ((N + kPeN - 1) / kPeN);
  const int sms = num_sms();
  const int grid = (int)(tiles < sms ? tiles : sms);
  patch_embed_wgmma_kernel<<<grid, kPeThreads, kPeSmem, reinterpret_cast<cudaStream_t>(stream)>>>(tv, tw, a);
  U2_CHECK_LAUNCH("patch_embed");
  return U2_OK;
}
