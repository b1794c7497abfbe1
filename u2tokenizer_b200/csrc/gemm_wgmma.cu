// bf16 x bf16 -> fp32-accumulate GEMM on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
//   for every batch z = (zo, zi):   C[z] = epilogue( alpha * A[z] (M x K)  *  B[z'] (N x K)^T )
//
// Both operands are K-major (the natural layout of torch.nn.Linear: activations [rows, K],
// weights [out, K]); the same kernel serves every Linear on the hot path (ViT qkv / out_proj /
// MLP, projector, the mu2-tokenizer wq/wk/wv/dense, decoder q/k/v/o/gate/up/down, lm_head) and,
// through the 4-D batch coordinates, the QK^T and PV contractions of the attention blocks.
//
// Structure (persistent, warp specialised, 1 CTA per SM, 3 warpgroups):
//   warp 0    : TMA producer  - 4-D tiled loads of A/B k-blocks into a kStages-deep smem ring
//   warps 4-7 : MMA warpgroup - wgmma 64 x 64 x 16 (two row halves x BLOCK_N / 64 column chunks per k step), fp32
//                               accumulators in registers; a finished tile is parked in a shared-memory accumulator
//                               tile, so the next tile's mainloop overlaps the epilogue of this one
//   warps 8-11: epilogue      - thread == output row: accumulator row segments from shared memory -> registers,
//                               alpha/bias/activation/residual, store
//
// Reference call sites this replaces: every nn.Linear / torch.matmul on the path, e.g.
// src/model/u2tokenizer/rma.py:52-58,60-73 and tta.py:42-69 (reference repo paths).
#include <cuda_bf16.h>
#include <math.h>
#include <stdlib.h>

#include "host_util.h"
#include "ptx.cuh"
#include "u2b200.h"

namespace u2 {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // 64 bf16 = 128 bytes = one swizzle-128B row
constexpr int kMmaK = 16;
constexpr int kNumThreads = 384;   // producer warpgroup, MMA warpgroup, epilogue warpgroup
constexpr int kMmaWarp0 = 4;
constexpr int kEpiWarp0 = 8;
constexpr int kEpiWarps = 4;       // one warp per 32 accumulator rows, each drains all of the tile's columns
#ifndef U2_GEMM_TMA_STORE_DEFAULT
#define U2_GEMM_TMA_STORE_DEFAULT 1
#endif

// The widest tile is 128 columns: the parked accumulator tile (128 x 132 fp32) and a 4-deep operand ring must share
// the 227 KB of shared memory an H100 block may use.
template <int kBlockN>
struct GemmCfg {
  static constexpr int kStages = (kBlockN == 128) ? 4 : 6;
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = kBlockN * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccLd = kBlockN + 4;  // fp32 pitch of the parked accumulator: conflict-free 16-byte row reads
  static constexpr int kAccBytes = kBlockM * kAccLd * 4;
  static constexpr int kEpiStageBytes = kEpiWarps * 4096;  // one 32 x 32 fp32 staging tile per epilogue warp (coalesced stores)
  static constexpr int kSmemBytes = kStages * kStageBytes + kAccBytes + kEpiStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

// 32 consecutive fp32 accumulator values of one row of the parked tile (16-byte shared loads)
__device__ __forceinline__ void acc_ld32(uint32_t addr, uint32_t (&v)[32]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint4 x = lds128(addr + 16 * j);
    v[4 * j] = x.x; v[4 * j + 1] = x.y; v[4 * j + 2] = x.z; v[4 * j + 3] = x.w;
  }
}

struct GemmDev {
  int M, N, K;
  int zi, zo, b_zi_div;
  long long ldc, c_stride_zi, c_stride_zo;
  int c_dtype;
  float alpha;
  const float* bias;
  int act;
  const __nv_bfloat16* residual;
  long long ldr;
  int res_row_mod;
  int row_div, row_stride, row_off;
  void* C;
  int m_major;                // tile order inside a batch (see tile_coords)
  int tma_store;              // C goes out through TMA bulk stores of the staged 32 x 32 blocks (tmap_c valid)
  int epi_op;                 // U2_EPI_*
  const float* rowvec;
  long long rv_zi, rv_zo;
  const __nv_bfloat16* mul;
  // kMode 1 (fused lm_head + log-softmax statistics): nothing of the N-wide result is stored
  const long long* labels;  // [M], label column per row (< 0: none)
  float4* part;             // [num_n_blocks][part_ld]: (running max, sum exp(x - max), sum x, -) per row and tile
  float* lab_logit;         // [part_ld]: the logit at the label column
  long long part_ld;
};

// erf-based GELU (nn.GELU() default, MONAI MLPBlock / the projector MLP) with erf from Abramowitz & Stegun 7.1.26
// (|error| <= 1.5e-7, far below the bf16 rounding of the result), written branch-free: erff, IEEE division and
// __frcp_rn all compile to a fast path plus a guarded call per ELEMENT (BSSY/BSYNC), which serialises the 32 values a
// thread holds and made the bias+GELU epilogue of the K = 768 ViT GEMMs 3x longer than their mainloop.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));  // rcp.approx: no IEEE slow-path call, keeps the 32 elements independent
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = __expf(-z * z);
  const float erf_abs = fmaf(-p * t, e, 1.0f);
  const float hx = 0.5f * x;
  return fmaf(hx, copysignf(erf_abs, x), hx);
}

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == U2_ACT_GELU) return gelu_erf(x);
  if (act == U2_ACT_SILU) return __fdividef(x, 1.0f + __expf(-x));  // branch-free (IEEE '/' compiles to a guarded slow-path call)
  return x;
}

// kMajor bit 0: A is MN-major (stored [K][M], the contraction index is the slow one), bit 1: same for B. An MN-major
// operand tile is loaded as 64-wide MN chunks x 64 k-rows (one TMA box each, 8 KB, 128-byte swizzle): exactly the
// canonical wgmma "MN-major, SWIZZLE_128B" layout ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units with LBO = 8192 B
// between chunks and SBO = 1024 B between groups of 8 k-rows. dgrad (dY * W) and wgrad (dY^T * X) of every Linear,
// P^T dO / dS^T Q of the attention backward and the DiffTS products run through this without transposed copies.
// Tile order inside a batch. n-major (default): consecutive tiles share the B tile, A streams - right when A (the
// activations) fits L2 or N is one tile wide. m-major: the num_n tiles of one M block run back to back on neighbouring CTAs,
// so a tall A (ViT / patch-embed activations: 100-400 MB) is read from HBM ONCE while the small weight matrix stays
// L2-resident; with the n-major order the ncu capture of the patch-embed GEMM showed 403 MB of DRAM reads for 134 MB of A.
__device__ __forceinline__ void tile_coords(int t, int num_m_blocks, int num_n_blocks, int m_major, int& m_blk, int& n_blk) {
  if (m_major) {
    m_blk = t / num_n_blocks;
    n_blk = t - m_blk * num_n_blocks;
  } else {
    n_blk = t / num_m_blocks;
    m_blk = t - n_blk * num_m_blocks;
  }
}

template <int kBlockN, int kMode = 0, int kMajor = 0>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                       const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_c, const GemmDev p) {
  using Cfg = GemmCfg<kBlockN>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kNC = kBlockN / 64;  // 64-column wgmma chunks per tile

  extern __shared__ uint8_t smem_raw[];
  // swizzle-128B operand tiles need 1024-byte alignment
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * Cfg::kABytes;
  float* smem_acc = reinterpret_cast<float*>(smem + kStages * Cfg::kStageBytes);  // [kBlockM][kAccLd] parked accumulator
  // 4 x 4 KB staging tiles, one per epilogue warp, 1024-byte aligned: sources of swizzled TMA stores
  uint8_t* smem_epi = smem + kStages * Cfg::kStageBytes + Cfg::kAccBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_epi + Cfg::kEpiStageBytes);
  uint64_t* full_bar = bars;                  // [kStages]
  uint64_t* empty_bar = bars + kStages;       // [kStages]
  uint64_t* acc_full_bar = bars + 2 * kStages;      // parked accumulator written
  uint64_t* acc_empty_bar = bars + 2 * kStages + 1;  // parked accumulator drained

  const int warp_idx = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;

  const int num_m_blocks = (p.M + kBlockM - 1) / kBlockM;
  const int num_n_blocks = (p.N + kBlockN - 1) / kBlockN;
  const int num_k_blocks = (p.K + kBlockK - 1) / kBlockK;
  const int tiles_per_batch = num_m_blocks * num_n_blocks;
  const int num_tiles = tiles_per_batch * p.zi * p.zo;

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (p.tma_store) tma_prefetch_desc(&tmap_c);
  }
  if (warp_idx == 1 && lane == 0) {
    // consumer barriers count WARPS: one arrival per MMA / epilogue warp (per-thread arrivals on one barrier serialise)
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);
    }
    mbar_init(acc_full_bar, 4);
    mbar_init(acc_empty_bar, kEpiWarps);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp_idx == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int z = tile / tiles_per_batch;
        const int t = tile - z * tiles_per_batch;
        int m_blk, n_blk;
        tile_coords(t, num_m_blocks, num_n_blocks, p.m_major, m_blk, n_blk);
        const int zo_i = z / p.zi;
        const int zi_i = z - zo_i * p.zi;
        const int zi_b = zi_i / p.b_zi_div;
        for (int kb = 0; kb < num_k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if constexpr (kMajor & 1) {
#pragma unroll
            for (int c = 0; c < kBlockM / 64; ++c)
              tma_load_4d(smem_a + stage * Cfg::kABytes + c * (64 * kBlockK * 2), &tmap_a, &full_bar[stage],
                          m_blk * kBlockM + c * 64, kb * kBlockK, zi_i, zo_i);
          } else {
            tma_load_4d(smem_a + stage * Cfg::kABytes, &tmap_a, &full_bar[stage], kb * kBlockK,
                        m_blk * kBlockM, zi_i, zo_i);
          }
          if constexpr (kMajor & 2) {
#pragma unroll
            for (int c = 0; c < kBlockN / 64; ++c)
              tma_load_4d(smem_b + stage * Cfg::kBBytes + c * (64 * kBlockK * 2), &tmap_b, &full_bar[stage],
                          n_blk * kBlockN + c * 64, kb * kBlockK, zi_b, zo_i);
          } else {
            tma_load_4d(smem_b + stage * Cfg::kBBytes, &tmap_b, &full_bar[stage], kb * kBlockK,
                        n_blk * kBlockN, zi_b, zo_i);
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else if (warp_idx >= kMmaWarp0 && warp_idx < kEpiWarp0) {
    // ===================== MMA warpgroup =====================
    // descriptor start-address step (16-byte units) per 16 contraction indices: 32 B inside the swizzle row for a
    // K-major tile, two 1024-byte groups of 8 k-rows for an MN-major one. Rows 64..127 of A and columns 64c.. of B
    // start 8 KB further in either layout (64 rows of 128 B, or the next 64-wide MN chunk).
    constexpr uint32_t a_kstep = (kMajor & 1) ? 128 : 2, b_kstep = (kMajor & 2) ? 128 : 2;
    const int w = warp_idx - kMmaWarp0;
    float acc[2][kNC][32];
    int stage = 0;
    uint32_t phase = 0;
    uint32_t acc_phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int prev_stage = -1;
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t a_desc = gmma_desc_sw128(smem_u32(smem_a + stage * Cfg::kABytes), 64 * kBlockK * 2);
        const uint64_t b_desc = gmma_desc_sw128(smem_u32(smem_b + stage * Cfg::kBBytes), 64 * kBlockK * 2);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kMmaK; ++k) {
#pragma unroll
          for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
            for (int nc = 0; nc < kNC; ++nc)
              wgmma_m64n64k16_ss<(kMajor & 1), (kMajor >> 1)>(acc[mh][nc], a_desc + 512 * mh + a_kstep * k,
                                                              b_desc + 512 * nc + b_kstep * k, (kb | k) != 0);
          }
        }
        wgmma_commit();
        // the previous k-block's MMAs are complete: its smem slot goes back to the producer
        wgmma_wait<1>();
        if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      // park the accumulator once the epilogue has drained the previous tile
      mbar_wait(acc_empty_bar, acc_phase ^ 1);
#pragma unroll
      for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float* dst = smem_acc + (mh * 64 + w * 16 + (lane >> 2) + 8 * h) * Cfg::kAccLd + 2 * (lane & 3);
#pragma unroll
          for (int nc = 0; nc < kNC; ++nc) {
#pragma unroll
            for (int i = 0; i < 8; ++i)
              *reinterpret_cast<float2*>(dst + nc * 64 + 8 * i) = make_float2(acc[mh][nc][4 * i + 2 * h], acc[mh][nc][4 * i + 2 * h + 1]);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(acc_full_bar);
      acc_phase ^= 1;
    }
  } else if (warp_idx >= kEpiWarp0) {
    // ===================== epilogue: parked accumulator -> registers -> global =====================
    const int q = warp_idx - kEpiWarp0;  // this warp's 32 rows of the tile
    uint32_t acc_phase = 0;
    uint32_t n_st = 0;  // TMA stores issued by this warp (bf16: two 2 KB staging buffers used alternately)
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int z = tile / tiles_per_batch;
      const int t = tile - z * tiles_per_batch;
      int m_blk, n_blk;
      tile_coords(t, num_m_blocks, num_n_blocks, p.m_major, m_blk, n_blk);
      const int zo_i = z / p.zi;
      const int zi_i = z - zo_i * p.zi;

      const int row = m_blk * kBlockM + q * 32 + lane;  // row of the logical (M x N) output
      const bool row_ok = row < p.M;
      long long out_row = row;
      if (p.row_div > 0) out_row = (long long)(row / p.row_div) * p.row_stride + p.row_off + row % p.row_div;
      const long long zoff = (long long)zo_i * p.c_stride_zo + (long long)zi_i * p.c_stride_zi;
      const long long c_off = zoff + out_row * p.ldc;
      const long long res_row = p.res_row_mod > 0 ? (long long)(row % p.res_row_mod) : out_row;
      const __nv_bfloat16* res_ptr =
          p.residual ? p.residual + (p.res_row_mod > 0 ? 0 : zoff) + res_row * p.ldr : nullptr;

      const uint32_t arow = smem_u32(smem_acc + (q * 32 + lane) * Cfg::kAccLd);  // this thread's row of the parked tile
      if constexpr (kMode == 1) {
        mbar_wait(acc_full_bar, acc_phase);
        // log-softmax statistics of this thread's row over the tile's columns; the logits never leave
        // the SM (reference dpo_u2trainer.py:289-300 materialises [rows, vocab] logits and log-softmaxes them)
        const long long lab = row_ok ? p.labels[row] : -1;
        float mx = -INFINITY, se = 0.f, sx = 0.f;
#pragma unroll 1
        for (int c0 = 0; c0 < kBlockN; c0 += 32) {
          const int col0 = n_blk * kBlockN + c0;
          if (col0 >= p.N) break;  // warp-uniform
          uint32_t v[32];
          acc_ld32(arow + 4 * c0, v);
          const int nv = min(32, p.N - col0);
          float cm = -INFINITY;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float x = __uint_as_float(v[j]) * p.alpha;
            v[j] = __float_as_uint(x);
            if (j < nv) cm = fmaxf(cm, x);
          }
          const float nm = fmaxf(mx, cm);
          const long long ljl = lab - col0;
          const uint32_t hit = (ljl >= 0 && ljl < nv) ? (1u << (int)ljl) : 0u;  // one-hot of the label column
          float acc_e = 0.f, acc_x = 0.f, pick = 0.f;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float x = __uint_as_float(v[j]);
            if (j < nv) {
              acc_e += __expf(x - nm);
              acc_x += x;
            }
            pick += (hit >> j) & 1u ? x : 0.f;
          }
          se = se * __expf(mx - nm) + acc_e;  // mx == -inf on the first chunk: exp(-inf) == 0
          sx += acc_x;
          mx = nm;
          if (hit) p.lab_logit[row] = pick;
        }
        if (row_ok) p.part[(long long)n_blk * p.part_ld + row] = make_float4(mx, se, sx, 0.f);
        // hand the parked accumulator back to the MMA warpgroup
        __syncwarp();
        if (lane == 0) mbar_arrive(acc_empty_bar);
      } else {
        // ---- drain of this warp's 32 rows x kBlockN columns in 32-column chunks. A short-K GEMM (attention scores / dP
        // with K = 64: ONE k-block per tile) is nothing but this loop, so
        //   * everything that does not depend on the accumulator (row vector, the first chunk's residual / P segment)
        //     is requested BEFORE the wait for the MMA,
        //   * chunk c + 1's residual / P loads are issued as soon as chunk c's are consumed, so they fly while chunk c
        //     is computed and stored,
        //   * the parked accumulator goes back to the MMA warpgroup as soon as the last chunk has been read.
        constexpr int kChunks = kBlockN / 32;
        const int colb = n_blk * kBlockN;
        const bool ds_vec_ok = p.epi_op == U2_EPI_DS_ROW && (((p.ldc | zoff) & 7) == 0);
        const bool res_vec_ok = res_ptr && p.epi_op != U2_EPI_DS_ROW && ((p.ldr & 7) == 0);
        // 2: the P ("mul") segment is prefetched, 1: the residual segment is prefetched, 0: nothing / element-wise tail path
        auto side_kind = [&](int col0) -> int {
          if (!row_ok || col0 + 32 > p.N) return 0;
          return ds_vec_ok ? 2 : (res_vec_ok ? 1 : 0);
        };
        auto side_load = [&](int col0, int kind, uint4 (&sd)[4]) {
          if (kind == 0) return;
          const __nv_bfloat16* src = (kind == 2) ? (p.mul + c_off + col0) : (res_ptr + col0);
#pragma unroll
          for (int j = 0; j < 4; ++j) sd[j] = *reinterpret_cast<const uint4*>(src + 8 * j);
        };
        const uint32_t st = smem_u32(smem_epi) + (warp_idx - kEpiWarp0) * 4096;
        const int row0 = m_blk * kBlockM + q * 32;

        uint32_t v[32];
        uint4 sd[4];   // residual / P segment of the chunk in flight (requested as soon as the previous one is consumed)
        int kind = 0;
        const bool any = colb < p.N;  // warp-uniform
        float rv = 0.f;
        if (row_ok && p.epi_op != U2_EPI_NONE)
          rv = __ldg(p.rowvec + (long long)zo_i * p.rv_zo + (long long)zi_i * p.rv_zi + row);
        if (any) {
          kind = side_kind(colb);
          side_load(colb, kind, sd);
        }
        mbar_wait(acc_full_bar, acc_phase);
        bool released = false;
        // the loop stays ROLLED (one copy of the body in the instruction cache)
#pragma unroll 1
        for (int c = 0; c < kChunks; ++c) {
          const int col0 = colb + 32 * c;
          if (col0 < p.N) {  // warp-uniform
            acc_ld32(arow + 4 * 32 * c, v);
            float f[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(v[j]) * p.alpha;
            const bool more = (c + 1 < kChunks) && (col0 + 32 < p.N);
            if (!more) {
              // every accumulator value of this warp has been read: hand the parked tile back to the MMA warpgroup
              __syncwarp();
              if (lane == 0) mbar_arrive(acc_empty_bar);
              released = true;
            }
            const int kd = kind;
            const bool full = (col0 + 32 <= p.N);
            if (row_ok && p.epi_op != U2_EPI_NONE) {
              // attention backward: probabilities rebuilt from the row log-sum-exp / dS formed against the stored P
              if (p.epi_op == U2_EPI_EXP_ROW) {
#pragma unroll
                for (int j = 0; j < 32; ++j) f[j] = __expf(f[j] - rv);
              } else if (kd == 2) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const __nv_bfloat162* r2 = reinterpret_cast<const __nv_bfloat162*>(&sd[j]);
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float2 rf = __bfloat1622float2(r2[e]);
                    f[8 * j + 2 * e] = rf.x * (f[8 * j + 2 * e] - rv);
                    f[8 * j + 2 * e + 1] = rf.y * (f[8 * j + 2 * e + 1] - rv);
                  }
                }
              } else {
                const __nv_bfloat16* mp = p.mul + c_off + col0;
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  f[j] = (col0 + j < p.N) ? __bfloat162float(mp[j]) * (f[j] - rv) : 0.f;
              }
            }
            if (row_ok) {
              if (p.bias) {
                if (full && ((reinterpret_cast<uintptr_t>(p.bias) & 15) == 0)) {
#pragma unroll
                  for (int j = 0; j < 32; j += 4) {
                    const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + j));
                    f[j] += b4.x; f[j + 1] += b4.y; f[j + 2] += b4.z; f[j + 3] += b4.w;
                  }
                } else {
#pragma unroll
                  for (int j = 0; j < 32; ++j)
                    if (full || col0 + j < p.N) f[j] += __ldg(p.bias + col0 + j);
                }
              }
              if (p.act != U2_ACT_NONE) {
#pragma unroll
                for (int j = 0; j < 32; ++j) f[j] = apply_act(f[j], p.act);
              }
              if (kd == 1) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const __nv_bfloat162* r2 = reinterpret_cast<const __nv_bfloat162*>(&sd[j]);
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float2 rf = __bfloat1622float2(r2[e]);
                    f[8 * j + 2 * e] += rf.x;
                    f[8 * j + 2 * e + 1] += rf.y;
                  }
                }
              } else if (res_ptr) {
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  if (col0 + j < p.N) f[j] += __bfloat162float(res_ptr[col0 + j]);
              }
            }
            if (more) {  // the side operands of chunk c are consumed: request chunk c + 1's (in flight during the store below)
              kind = side_kind(col0 + 32);
              side_load(col0 + 32, kind, sd);
            }
            // ---- store. Fast path: the warp's 32 x 32 block goes through a swizzled shared-memory tile so that every
            // store instruction writes whole 128-byte (fp32) / 64-byte (bf16) row segments; the thread-per-row pattern it
            // replaces touched 32 half-used sectors per request, which bounded every short-K GEMM by its epilogue.
            const bool fast = full &&
                              (p.c_dtype == U2_DT_BF16 ? (((p.ldc | zoff) & 7) == 0) : (((p.ldc | zoff) & 3) == 0));
            if (p.tma_store) {
              // ---- TMA path: the same swizzled 32 x 32 image (it IS the 64-byte / 128-byte TMA swizzle of a box of 32
              // rows) leaves through ONE bulk tensor store issued by lane 0: no read-back, no per-row address arithmetic,
              // rows >= M and columns >= N are clipped by the tensor map. bf16 blocks are 2 KB, so the warp's 4 KB
              // staging area double-buffers them: block c is filled while the copy engine still reads block c - 1.
              if (p.c_dtype == U2_DT_BF16) {
                const uint32_t sb = st + (n_st & 1) * 2048;
                if (lane == 0) bulk_wait_group_read<1>();
                __syncwarp();
#pragma unroll
                for (int cc = 0; cc < 4; ++cc) {
                  uint4 o;
                  __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
                  for (int e = 0; e < 4; ++e) o2[e] = __floats2bfloat162_rn(f[8 * cc + 2 * e], f[8 * cc + 2 * e + 1]);
                  sts128(sb + lane * 64 + ((cc ^ ((lane >> 1) & 3)) << 4), o);
                }
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) {
                  tma_store_4d(&tmap_c, sb, col0, row0, zi_i, zo_i);
                  bulk_commit_group();
                }
              } else {
                if (lane == 0) bulk_wait_group_read<0>();
                __syncwarp();
#pragma unroll
                for (int cc = 0; cc < 8; ++cc)
                  sts128(st + lane * 128 + ((cc ^ (lane & 7)) << 4),
                         make_uint4(__float_as_uint(f[4 * cc]), __float_as_uint(f[4 * cc + 1]), __float_as_uint(f[4 * cc + 2]),
                                    __float_as_uint(f[4 * cc + 3])));
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) {
                  tma_store_4d(&tmap_c, st, col0, row0, zi_i, zo_i);
                  bulk_commit_group();
                }
              }
              ++n_st;
            } else if (fast) {
              __syncwarp();  // the previous chunk's read-back is complete
              if (p.c_dtype == U2_DT_BF16) {
#pragma unroll
                for (int cc = 0; cc < 4; ++cc) {
                  uint4 o;
                  __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
                  for (int e = 0; e < 4; ++e) o2[e] = __floats2bfloat162_rn(f[8 * cc + 2 * e], f[8 * cc + 2 * e + 1]);
                  sts128(st + lane * 64 + ((cc ^ ((lane >> 1) & 3)) << 4), o);
                }
                __syncwarp();
#pragma unroll
                for (int it = 0; it < 4; ++it) {
                  const int rr = it * 8 + (lane >> 2), ch = lane & 3;
                  const uint4 o = lds128(st + rr * 64 + ((ch ^ ((rr >> 1) & 3)) << 4));
                  const int grow = row0 + rr;
                  if (grow < p.M) {
                    long long orow = grow;
                    if (p.row_div > 0) orow = (long long)(grow / p.row_div) * p.row_stride + p.row_off + grow % p.row_div;
                    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.C) + zoff + orow * p.ldc + col0 + ch * 8) = o;
                  }
                }
              } else {
#pragma unroll
                for (int cc = 0; cc < 8; ++cc)
                  sts128(st + lane * 128 + ((cc ^ (lane & 7)) << 4),
                         make_uint4(__float_as_uint(f[4 * cc]), __float_as_uint(f[4 * cc + 1]), __float_as_uint(f[4 * cc + 2]),
                                    __float_as_uint(f[4 * cc + 3])));
                __syncwarp();
#pragma unroll
                for (int it = 0; it < 8; ++it) {
                  const int rr = it * 4 + (lane >> 3), ch = lane & 7;
                  const float4 o = lds128_f32(st + rr * 128 + ((ch ^ (rr & 7)) << 4));
                  const int grow = row0 + rr;
                  if (grow < p.M) {
                    long long orow = grow;
                    if (p.row_div > 0) orow = (long long)(grow / p.row_div) * p.row_stride + p.row_off + grow % p.row_div;
                    *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.C) + zoff + orow * p.ldc + col0 + ch * 4) = o;
                  }
                }
              }
            } else if (row_ok) {
              if (p.c_dtype == U2_DT_BF16) {
                __nv_bfloat16* cp = reinterpret_cast<__nv_bfloat16*>(p.C) + c_off + col0;
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  if (col0 + j < p.N) cp[j] = __float2bfloat16(f[j]);
              } else {
                float* cp = reinterpret_cast<float*>(p.C) + c_off + col0;
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  if (col0 + j < p.N) cp[j] = f[j];
              }
            }
          }
        }
        if (!released) {  // defensive: every tile has at least one column < N
          __syncwarp();
          if (lane == 0) mbar_arrive(acc_empty_bar);
        }
      }  // kMode
      acc_phase ^= 1;
    }
    // outstanding bulk stores read this CTA's shared memory: they must be complete before the CTA retires
    if (p.tma_store && lane == 0) bulk_wait_group<0>();
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
template <int kBlockN, int kMode = 0, int kMajor = 0>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const GemmDev& p, int num_sms,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<kBlockN>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<kBlockN, kMode, kMajor>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "gemm: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  const int num_m = (p.M + kBlockM - 1) / kBlockM;
  const int num_n = (p.N + kBlockN - 1) / kBlockN;
  const long long tiles = (long long)num_m * num_n * p.zi * p.zo;
  const int grid = (int)(tiles < num_sms ? tiles : num_sms);
  gemm_bf16_wgmma_kernel<kBlockN, kMode, kMajor><<<grid, kNumThreads, Cfg::kSmemBytes, stream>>>(ta, tb, tc, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "gemm launch: %s", cudaGetErrorString(e));
  return U2_OK;
}

// Merge of the per-tile statistics: one thread per (row, partial group), 8 groups per row.
//   lse = m + log(sum_p s_p * exp(m_p - m)),  logp = logit[label] - lse
__global__ void __launch_bounds__(256) logprob_merge_kernel(const float4* __restrict__ part, const float* __restrict__ lab_logit,
                                                            const long long* __restrict__ labels, int R, int P, long long part_ld,
                                                            float* __restrict__ logp, float* __restrict__ lse_out,
                                                            float* __restrict__ logit_sum, float* __restrict__ nll_acc) {
  __shared__ float s_m[8][32], s_s[8][32], s_x[8][32];
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int r = blockIdx.x * 32 + lane;
  float m = -INFINITY, s = 0.f, x = 0.f;
  if (r < R) {
    for (int pi = grp; pi < P; pi += 8) {
      const float4 v = __ldcs(part + (long long)pi * part_ld + r);
      if (v.x == -INFINITY) continue;  // a row without valid columns
      const float nm = fmaxf(m, v.x);
      s = s * __expf(m - nm) + v.y * __expf(v.x - nm);
      x += v.z;
      m = nm;
    }
  }
  s_m[grp][lane] = m;
  s_s[grp][lane] = s;
  s_x[grp][lane] = x;
  __syncthreads();
  if (grp == 0 && r < R) {
    float gm = -INFINITY;
#pragma unroll
    for (int g = 0; g < 8; ++g) gm = fmaxf(gm, s_m[g][lane]);
    float gs = 0.f, gx = 0.f;
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      if (s_m[g][lane] != -INFINITY) gs += s_s[g][lane] * __expf(s_m[g][lane] - gm);
      gx += s_x[g][lane];
    }
    const float lse = gm + logf(gs);
    const bool has = labels[r] >= 0;
    const float lp = has ? lab_logit[r] - lse : 0.f;
    logp[r] = lp;
    if (lse_out) lse_out[r] = lse;
    if (logit_sum) logit_sum[r] = gx;
    if (nll_acc && has) {
      atomicAdd(nll_acc, -lp);
      atomicAdd(nll_acc + 1, 1.f);
    }
  }
}

}  // namespace u2

extern "C" U2_API int64_t u2_logprob_ws_bytes(int32_t R, int32_t V) {
  if (R <= 0 || V <= 0) return 0;
  const long long r_pad = ((long long)R + 127) / 128 * 128;
  const long long P = (V + 127) / 128;  // one partial per 128-column tile
  return P * r_pad * 16 + r_pad * 4;
}

extern "C" U2_API int u2_lmhead_logprob_bf16(const void* hidden, const void* W, float* logp, const u2_logprob_desc* d,
                                             void* stream) {
  using namespace u2;
  if (!hidden || !W || !logp || !d || !d->labels || !d->ws) return set_error(U2_ERR_ARG, "lmhead_logprob: null pointer");
  if (d->R <= 0 || d->V <= 0 || d->E <= 0) return set_error(U2_ERR_ARG, "lmhead_logprob: R, V, E must be > 0");
  if ((d->ldh & 7) || (d->ldw & 7)) return set_error(U2_ERR_ARG, "lmhead_logprob: row strides must be multiples of 8 elements (16 B, TMA)");
  if ((reinterpret_cast<uintptr_t>(hidden) & 15) || (reinterpret_cast<uintptr_t>(W) & 15) || (reinterpret_cast<uintptr_t>(d->ws) & 15))
    return set_error(U2_ERR_ARG, "lmhead_logprob: hidden / W / ws must be 16-byte aligned");
  if (d->ws_bytes < u2_logprob_ws_bytes(d->R, d->V))
    return set_error(U2_ERR_ARG, "lmhead_logprob: workspace too small (%lld < %lld bytes)", (long long)d->ws_bytes,
                     (long long)u2_logprob_ws_bytes(d->R, d->V));
  constexpr int kBn = 128;
  CUtensorMap ta, tb;
  int rc = make_tmap_bf16_4d(&ta, hidden, d->E, d->R, 1, 1, d->ldh, 0, 0, kBlockK, kBlockM);
  if (rc) return rc;
  rc = make_tmap_bf16_4d(&tb, W, d->E, d->V, 1, 1, d->ldw, 0, 0, kBlockK, kBn);
  if (rc) return rc;
  const long long r_pad = ((long long)d->R + 127) / 128 * 128;
  const int P = (d->V + kBn - 1) / kBn;
  GemmDev p = {};
  p.M = d->R; p.N = d->V; p.K = d->E;
  p.zi = 1; p.zo = 1; p.b_zi_div = 1;
  p.alpha = 1.f;
  p.labels = reinterpret_cast<const long long*>(d->labels);
  p.part = reinterpret_cast<float4*>(d->ws);
  p.lab_logit = reinterpret_cast<float*>(reinterpret_cast<char*>(d->ws) + (long long)P * r_pad * 16);
  p.part_ld = r_pad;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  rc = launch_gemm<kBn, 1>(ta, tb, ta /* no C tensor map: nothing of the logits is stored */, p, num_sms(), s);
  if (rc) return rc;
  logprob_merge_kernel<<<(unsigned)((d->R + 31) / 32), 256, 0, s>>>(p.part, p.lab_logit, p.labels, d->R, P, r_pad, logp, d->lse,
                                                                    d->logit_sum, d->nll_acc);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "lmhead_logprob merge launch: %s", cudaGetErrorString(e));
  return U2_OK;
}

extern "C" U2_API int u2_gemm_bf16(const void* A, const void* B, void* C, const u2_gemm_desc* d, void* stream) {
  using namespace u2;
  if (!A || !B || !C || !d) return set_error(U2_ERR_ARG, "gemm: null pointer");
  if (d->M <= 0 || d->N <= 0 || d->K <= 0) return set_error(U2_ERR_ARG, "gemm: M,N,K must be > 0");
  const int zi = d->zi > 0 ? d->zi : 1, zo = d->zo > 0 ? d->zo : 1;
  const int bdiv = d->b_zi_div > 0 ? d->b_zi_div : 1;
  if ((d->lda & 7) || (d->ldb & 7)) return set_error(U2_ERR_ARG, "gemm: lda/ldb must be multiples of 8 elements (16 B, TMA)");
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15))
    return set_error(U2_ERR_ARG, "gemm: A/B must be 16-byte aligned");
  if (zi > 1 && ((d->a_stride_zi & 7) || (d->b_stride_zi & 7))) return set_error(U2_ERR_ARG, "gemm: inner batch strides must be multiples of 8 elements");
  if (zo > 1 && ((d->a_stride_zo & 7) || (d->b_stride_zo & 7))) return set_error(U2_ERR_ARG, "gemm: outer batch strides must be multiples of 8 elements");

  int block_n = d->block_n;
  if (block_n != 0 && block_n != 64 && block_n != 128 && block_n != 256) return set_error(U2_ERR_ARG, "gemm: block_n must be 0/64/128/256");
  // 0 / 256: the widest tile this kernel has (128 columns, see GemmCfg); 64 only where N fits in it
  if (block_n == 0 || block_n == 256) block_n = d->N <= 64 ? 64 : 128;

  CUtensorMap ta, tb;
  const int zi_b = (zi + bdiv - 1) / bdiv;
  const int major = (d->a_mn ? 1 : 0) | (d->b_mn ? 2 : 0);
  int rc;
  if (d->a_mn)  // stored [K][M]: inner dim = M, rows = K, boxes of 64 (M) x 64 (K)
    rc = make_tmap_bf16_4d(&ta, A, d->M, d->K, zi, zo, d->lda, zi > 1 ? d->a_stride_zi : 0, zo > 1 ? d->a_stride_zo : 0, 64, kBlockK);
  else
    rc = make_tmap_bf16_4d(&ta, A, d->K, d->M, zi, zo, d->lda, zi > 1 ? d->a_stride_zi : 0, zo > 1 ? d->a_stride_zo : 0, kBlockK, kBlockM);
  if (rc) return rc;
  if (d->b_mn)
    rc = make_tmap_bf16_4d(&tb, B, d->N, d->K, zi_b, zo, d->ldb, zi_b > 1 ? d->b_stride_zi : 0, zo > 1 ? d->b_stride_zo : 0, 64, kBlockK);
  else
    rc = make_tmap_bf16_4d(&tb, B, d->K, d->N, zi_b, zo, d->ldb, zi_b > 1 ? d->b_stride_zi : 0, zo > 1 ? d->b_stride_zo : 0, kBlockK, block_n);
  if (rc) return rc;

  GemmDev p = {};
  p.M = d->M; p.N = d->N; p.K = d->K;
  p.zi = zi; p.zo = zo; p.b_zi_div = bdiv;
  p.ldc = d->ldc; p.c_stride_zi = d->c_stride_zi; p.c_stride_zo = d->c_stride_zo;
  p.c_dtype = d->c_dtype;
  p.alpha = d->alpha;
  p.bias = d->bias;
  p.act = d->act;
  p.residual = reinterpret_cast<const __nv_bfloat16*>(d->residual);
  p.ldr = d->ldr;
  p.res_row_mod = d->res_row_mod;
  p.row_div = d->row_div; p.row_stride = d->row_stride; p.row_off = d->row_off;
  p.C = C;
  {
    // tall activations x small weights: walk the N tiles of an M block back to back (A read from HBM once)
    const long long a_bytes = (long long)d->M * d->K * 2, b_bytes = (long long)d->N * d->K * 2;
    const int num_n = (d->N + block_n - 1) / block_n;
    p.m_major = (num_n > 1 && b_bytes <= (48LL << 20) && a_bytes > b_bytes && a_bytes > (32LL << 20)) ? 1 : 0;
    if (const char* e = getenv("U2_GEMM_ORDER")) p.m_major = (e[0] == 'm');
  }
  p.epi_op = d->epi_op;
  p.rowvec = d->rowvec; p.rv_zi = d->rv_stride_zi; p.rv_zo = d->rv_stride_zo;
  p.mul = reinterpret_cast<const __nv_bfloat16*>(d->mul);
  if (p.epi_op != U2_EPI_NONE) {
    if (!p.rowvec) return set_error(U2_ERR_ARG, "gemm: the fused attention epilogue needs rowvec");
    if (p.epi_op == U2_EPI_DS_ROW && (!p.mul || d->c_dtype != U2_DT_BF16)) return set_error(U2_ERR_ARG, "gemm: U2_EPI_DS_ROW needs mul and a bf16 C");
    if (p.row_div > 0) return set_error(U2_ERR_ARG, "gemm: the fused attention epilogue does not combine with row remapping");
  }
  // C through TMA bulk stores (staged 32 x 32 blocks, clipped at the matrix edges) when its layout allows a tensor map:
  // 16-byte aligned base / row pitch / batch strides and no row remapping. U2_GEMM_TMA_STORE=0 keeps the ld.shared +
  // st.global read-back path. The dS epilogue, which reads P from the buffer it overwrites, keeps the read-back path.
  CUtensorMap tc = ta;
  {
    static const int want = [] {
      const char* e = getenv("U2_GEMM_TMA_STORE");
      return e ? atoi(e) : U2_GEMM_TMA_STORE_DEFAULT;
    }();
    const long long es = (d->c_dtype == U2_DT_BF16) ? 2 : 4;
    const bool ok = want && p.row_div <= 0 && p.epi_op != U2_EPI_DS_ROW && (d->c_dtype == U2_DT_BF16 || d->c_dtype == U2_DT_F32) &&
                    (reinterpret_cast<uintptr_t>(C) & 15) == 0 && ((d->ldc * es) & 15) == 0 &&
                    (zi == 1 || ((d->c_stride_zi * es) & 15) == 0) && (zo == 1 || ((d->c_stride_zo * es) & 15) == 0) &&
                    d->ldc >= d->N;
    // a layout the driver refuses to encode simply keeps the read-back path
    if (ok && make_tmap_store_4d(&tc, C, (int)es, d->N, d->M, zi, zo, d->ldc, d->c_stride_zi, d->c_stride_zo, 32, 32) == U2_OK)
      p.tma_store = 1;
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
#define U2_GEMM_BN(MAJ)                                                        \
  switch (block_n) {                                                          \
    case 64: return launch_gemm<64, 0, MAJ>(ta, tb, tc, p, num_sms(), s);     \
    default: return launch_gemm<128, 0, MAJ>(ta, tb, tc, p, num_sms(), s);   \
  }
  switch (major) {
    case 0: U2_GEMM_BN(0)
    case 1: U2_GEMM_BN(1)
    case 2: U2_GEMM_BN(2)
    default: U2_GEMM_BN(3)
  }
#undef U2_GEMM_BN
}
