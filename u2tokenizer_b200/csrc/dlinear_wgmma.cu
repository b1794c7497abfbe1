// Decode-step linear layers on wgmma with a TMA weight stream ("skinny GEMM", swap-AB + stream-K).
//
//   y[b, n] = epilogue( sum_k W[n, k] * x[b, k] ),   b < B <= 16,  one generated token per sequence
//
// Every weight byte is read exactly once per token, so the kernel is HBM-bound; the design goal is to
// keep one deep TMA pipeline per SM pulling 16 KB weight tiles back to back:
//   * swap-AB: the weight rows are the MMA M dimension (128 per tile), the <= 16 sequences are N = 16,
//     so the tensor-core cost per 64-wide k-block is 8 tiny wgmmas (64 x 16 x 16) - the tensor pipe idles,
//     the TMA engine and HBM do the work;
//   * stream-K: the (tile, k-block) space is cut into one equal contiguous range per CTA (grid = #SMs),
//     so narrow layers (o_proj, down_proj: 32 row tiles) still occupy every SM;
//   * partial sums meet in an fp32 workspace through red.global.add; the CTA that completes a tile
//     (per-tile k-block counter) runs the fused epilogue and re-zeroes workspace + counter, so the
//     workspace is self-cleaning and one kernel launch per linear suffices;
//   * fused epilogues: RMSNorm scale (x is pre-multiplied by gamma, the per-sequence 1/rms is applied to
//     the result), residual add, SiLU(gate)*up on row-interleaved [gate_j, up_j] weights, and the
//     "prepare the next norm" outputs (x * gamma_next in bf16, sum of squares per sequence).
//
// Warp roles: warp 0 TMA producer, warps 4-7 epilogue, warps 8-11 the MMA warpgroup (accumulators in registers,
// handed to the epilogue through a double-buffered fp32 tile in shared memory). Replaces the HF decoder Linears at q_len == 1 inside generate()
// (reference src/model/language_model/u2llama.py:123-126 -> HF GenerationMixin._sample).
#include <cuda_bf16.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include "host_util.h"
#include "ptx.cuh"
#include "u2b200.h"

namespace u2 {

constexpr int kDlN = 16;       // padded batch (wgmma N)
constexpr int kDlK = 64;       // k-block: 64 bf16 = one 128-byte swizzle row
constexpr int kDlBBytes = kDlN * kDlK * 2;   // 2 KB
constexpr int kDlThreads = 384;
constexpr int kDlMmaWarp0 = 8;
constexpr int kDlAccLd = 20;   // fp32 pitch of a handed-over accumulator row (16 used): conflict-free 16-byte reads

// Two schedules:
//   kM = 128, stream-K : (tile, k-block) units cut into equal contiguous ranges per CTA; partial tiles meet in
//                        the fp32 workspace (atomics + per-tile counter + last-arriver epilogue)
//   kM =  64, tiles    : every CTA owns whole 64-row tiles (round robin) and streams their full K range: no
//                        inter-CTA reduction at all, so an op ends ~1 us after its last MMA. 64 rows x K is
//                        still >= 0.5 MB per tile, and 64..96 active SMs already saturate HBM because one SM
//                        can ingest far more than 1/132 of the HBM bandwidth through TMA.
//
// Packed weights (kPacked, kM = 128 only): one 128 x 64 unit is stored losslessly in 13 bits per weight, 13 328 B instead
// of 16 KB, and streamed with one 1-D bulk copy. Per unit, base = max(emax - 31, 0) (emax: largest bf16 exponent field of
// the unit); a weight's exponent e is coded as c = 0 when e = 0 (zeros, subnormals) and c = e - base (1..31) otherwise.
// Layout (every plane in wgmma A-fragment order, interleaved [16-byte chunk][MMA thread] for conflict-free 16-byte loads;
// thread t of the warpgroup owns 32 bf16x2 fragment words R = 16 mh + 4 ks + r, see unpack_word):
//   [0, 16)          header: u32 base, 12 spare bytes
//   [16, 8208)       s << 7 | m bytes: byte 2R + h of thread t at 16 + ((2R + h) / 16 * 128 + t) * 16 + (2R + h) % 16
//   [8208, 12304)    low 4 code bits: word q = R / 4 of thread t holds word R's codes at bits 4 (R % 4) (column c) and
//                    16 + 4 (R % 4) (column c + 1); word q at 8208 + (q / 4 * 128 + t) * 16 + 4 (q % 4)
//   [12304, 13328)   high code bit: word u = R / 16 of thread t (at 12304 + 8 t + 4 u) holds bits R % 16 and 16 + R % 16
// Units are stored tile-major ((tile * kblocks + kb) * 13 328 B), the order in which a CTA's stream-K range walks them.
constexpr int kPkUnitBytes = 13328;
constexpr int kPkSmOff = 16, kPkNibOff = 16 + 8192, kPkHiOff = 16 + 8192 + 4096;

template <int kM, bool kPacked = false>
struct DlCfg {
  static constexpr int kABytes = kPacked ? kPkUnitBytes : kM * kDlK * 2;  // 13 328 B / 16 KB / 8 KB
  static constexpr int kStageBytes = kABytes + kDlBBytes;
#ifndef U2_DL_STAGES128
#define U2_DL_STAGES128 10
#endif
  // <= ~180 KB of weight tiles in flight per SM (packed: 13 units of 13 328 B fill the same shared memory)
  static constexpr int kStages = kPacked ? 13 : (kM == 128) ? U2_DL_STAGES128 : 18;
  static constexpr int kBOff = (kStages * kABytes + 1023) & ~1023;  // B tiles 1024-byte aligned (128-byte swizzle)
  static constexpr int kAccOff = kBOff + kStages * kDlBBytes;
  static constexpr int kAccBytes = 2 * kM * kDlAccLd * 4;      // double-buffered accumulator hand-over
  static constexpr int kBarOff = kAccOff + kAccBytes;
  static constexpr int kSmem = kBarOff + 512 + 1024;
  static_assert(!kPacked || kM == 128, "packed weights use the 128-row stream-K schedule");
};

__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t sel) {  // prmt.b32 (selector bit 3: replicate the sign)
  uint32_t r;
  asm("prmt.b32 %0, %1, 0, %2;" : "=r"(r) : "r"(a), "r"(sel));
  return r;
}

// Fragment word R of a packed unit as the bf16x2 wgmma A operand. sm: the 32-bit word of s<<7|m bytes holding word R's
// two bytes (bytes 0-1 for even R, 2-3 for odd R); nib / hi: this thread's code words covering R; b7 = (base << 7) in
// both 16-bit halves. Every step works on both halves at once; no half carries into the other.
template <int R>
__device__ __forceinline__ uint32_t unpack_word(uint32_t sm, uint32_t nib, uint32_t hi, uint32_t b7) {
  constexpr int i = R & 3, j = R & 15;
  const uint32_t ns = (i < 2) ? (nib << (7 - 4 * i)) : (nib >> (4 * i - 7));
  const uint32_t hs = (j <= 11) ? (hi << (11 - j)) : (hi >> (j - 11));
  const uint32_t c7 = (ns & 0x07800780u) | (hs & 0x08000800u);  // code << 7 per half
  // all-ones half where the code is not 0: bit 15 of (c7 + 0x7f80) is set iff c7 >= 0x80, replicated by byte permute
  const uint32_t nz = prmt(c7 + 0x7f807f80u, 0xBB99u);
  const uint32_t e7 = c7 + (nz & b7);                           // exponent field << 7
  const uint32_t z = prmt(sm, (R & 1) ? 0x3322u : 0x1100u);  // byte b in both bytes of its half
  return (z & 0x807f807fu) | e7;                                // sign (bit 7 of the high copy) | mantissa | exponent
}

struct DlinArgs {
  int B, N, K;                 // sequences, output rows of W, reduction length
  int num_tiles, kblocks;      // ceil(N/kM), K/64
  const uint8_t* wpk;          // packed weight units (kPacked launches; the tensor map is unused then)
  float* ws;                   // [num_tiles][max_slots][kM][16] fp32 partial-sum slots (stream-K schedule only);
                               // every word holds the sentinel 0xffffffff between uses
  int max_slots;
  int* counters;               // [num_tiles] int32 arrival counters, zero between launches
  // epilogue
  const float* ssq_in;         // [16] sum of squares of the (un-normalised) input rows, or null
  float inv_norm_dim, eps;     // rstd = rsqrt(ssq_in[b] * inv_norm_dim + eps)
  const __nv_bfloat16* residual;  // [B, N] (ldr) or null
  long long ldr;
  void* y;                     // [B, N_out] bf16 / fp32 (ldy); N_out = N/2 when silu_pair
  long long ldy;
  int y_dtype;
  int silu_pair;               // rows (2j, 2j+1) = (gate_j, up_j) -> y[b, j] = silu(gate) * up
  const float* gamma_next;     // [N] or null: also write xg[b, n] = bf16(y * gamma_next[n]) ...
  __nv_bfloat16* xg;           // ... here (ldxg)
  long long ldxg;
  float* ssq_out;              // [16] += sum_n y^2 (of the bf16-rounded y), or null
  float* ssq_part;             // [num_tiles][16] per-tile sums of squares (tail of ws), used with ssq_out
  int* ssq_ticket;             // counters[ceil(N / 64)]: finalised tiles of this op, zero between launches
  float* ssq_zero;             // [16] buffer to reset (the one the *next* producer accumulates into), or null
  // fine-grained dataflow inside a multi-op launch (all optional):
  const int* dep_flags;        // per-tile "finalised in step s" flags of the op that PRODUCES our x (same launch)
  int dep_shift;               // our k-block kb needs producer tile (kb >> dep_shift)
  int* out_flags;              // our own per-tile flags (consumed by the next op of the launch)
  unsigned long long* dbg;     // optional [gridDim][8] globaltimer stamps (tuning aid)
};

constexpr int kDlMaxOps = 4;

struct DlinMulti {
  CUtensorMap tw[kDlMaxOps];
  CUtensorMap tx[kDlMaxOps];
  DlinArgs op[kDlMaxOps];
  int n_ops;
  unsigned int* gridbar;      // [kDlMaxOps] monotonically increasing arrival counters (grid barriers between ops)
  const int* step_dev;        // barrier target = *step_dev * gridDim.x (step counter bumped once per decode step)
  unsigned long long* dbg;    // optional [gridDim][kDlMaxOps][8] globaltimer stamps (tuning aid)
  // L2 look-ahead: weights of the linear(s) the NEXT launch will stream (they only depend on the model):
  // issued when this launch has nothing left to load, so HBM keeps working through our tail, the launch gap
  // and the attention kernel in between.
  CUtensorMap tnext[2];
  const uint8_t* next_pk[2];  // packed next weights (else null: tnext)
  int next_tiles[2], next_kblocks[2], next_units[2];  // next_units: how many leading units per CTA to prefetch
  int n_next;
  int pre_stages;             // ring stages filled with the next op's weights before its dependency resolves
  int lookahead_units;        // per-CTA L2 prefetch depth beyond the smem ring at an in-launch op boundary
};

#define U2_STAMP(op, i)                                                                  \
  do {                                                                                   \
    if (mp.dbg) {                                                                        \
      unsigned long long t__;                                                            \
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t__));                           \
      mp.dbg[(blockIdx.x * kDlMaxOps + (op)) * 8 + (i)] = t__;                           \
    }                                                                                    \
  } while (0)

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// polling load: volatile asm so that the compiler re-issues it on every sweep (a plain __ldcg is loop-invariant)
__device__ __forceinline__ float4 ld_relaxed_f4(const float4* p) {
  float4 v;
  asm volatile("ld.relaxed.gpu.global.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

// single-thread poll (relaxed loads: one L2 round trip each), acquire fence once the target is reached
// The barrier needs every CTA of the grid to be resident (grid = #SMs, one CTA per SM: checked on the host against
// the occupancy calculator). If something outside this library takes SMs away for good (an MPS active-thread limit,
// a kernel of another context that never ends), the missing CTAs never arrive: after ~2^24 L2 round trips (seconds;
// a healthy wait is tens of microseconds) the poller traps, so the step fails loudly instead of hanging the GPU.
// No printf here: any function call in the kernel makes ptxas serialize every wgmma (C7510: a wait after each one),
// which made the MMA warpgroup, not HBM, set the pace of the weight stream.
__device__ __forceinline__ void grid_barrier_wait(const unsigned int* bar, unsigned int target) {
  unsigned int v, spins = 0;
  do {
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
    if (++spins == (1u << 24)) __trap();  // CTAs of the launch are not co-resident
  } while (v < target);
  asm volatile("fence.acq_rel.gpu;" ::: "memory");
}

// Work enumeration of one CTA inside one op: an incremental (tile, k-block) cursor - the producer thread is
// on the critical path of the weight stream, so no 64-bit divisions inside the loops.
struct UnitIter {
  int tile, kb, kblocks, tile_step;
  int left;  // units remaining, including the current one
  __device__ __forceinline__ void next() {
    if (++kb == kblocks) {
      kb = 0;
      tile += tile_step;
    }
    --left;
  }
  // units of the current tile that belong to this CTA, starting at the cursor
  __device__ __forceinline__ int seg_len() const {
    const int r = kblocks - kb;
    return r < left ? r : left;
  }
};

__device__ __forceinline__ UnitIter make_iter(int num_tiles, int kblocks, bool tiles) {
  UnitIter it;
  it.kblocks = kblocks;
  if (tiles) {
    const int mine = (num_tiles > (int)blockIdx.x) ? (num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    it.tile = blockIdx.x;
    it.kb = 0;
    it.tile_step = gridDim.x;
    it.left = mine * kblocks;
  } else {
    // stream-K over G = min(#CTAs, #units) CTAs, so that every participating CTA owns >= 1 unit
    const long long units = (long long)num_tiles * kblocks;
    const long long G = units < (long long)gridDim.x ? units : (long long)gridDim.x;
    it.tile_step = 1;
    if ((long long)blockIdx.x >= G) {
      it.tile = 0;
      it.kb = 0;
      it.left = 0;
    } else {
      const long long base = units * blockIdx.x / G;
      const long long end = units * (blockIdx.x + 1) / G;
      it.tile = (int)(base / kblocks);
      it.kb = (int)(base - (long long)it.tile * kblocks);
      it.left = (int)(end - base);
    }
  }
  return it;
}

// Producer-thread helper: block until producer tile `t` carries this step's flag. Flags are fetched four at a
// time (one 16-byte L2 round trip covers 8 k-blocks of activations), results cached in shared memory.
__device__ __forceinline__ void wait_tile_flag(const int* flags, int t, int step, unsigned char* ready, int tag) {
  if (ready[t] == (unsigned char)tag) return;
  const int t4 = t & ~3;
  for (;;) {
    int4 f;
    asm volatile("ld.relaxed.gpu.global.v4.s32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(f.x), "=r"(f.y), "=r"(f.z), "=r"(f.w)
                 : "l"(flags + t4)
                 : "memory");
    if (f.x >= step) ready[t4] = (unsigned char)tag;
    if (f.y >= step) ready[t4 + 1] = (unsigned char)tag;
    if (f.z >= step) ready[t4 + 2] = (unsigned char)tag;
    if (f.w >= step) ready[t4 + 3] = (unsigned char)tag;
    if (ready[t] == (unsigned char)tag) break;
  }
  asm volatile("fence.acq_rel.gpu;" ::: "memory");
  asm volatile("fence.proxy.async;" ::: "memory");  // other CTAs' generic-proxy stores -> our TMA reads
}

// One launch executes up to four dependent decode linears back to back (o_proj -> gate|up -> down -> next
// layer's qkv): between two linears all CTAs meet at a software grid barrier, but the TMA producer keeps
// the smem ring full with the NEXT linear's weight tiles while the current one drains and finalises, so the
// HBM stream barely pauses at the dependency.
template <int kM, bool kPacked>
__global__ void __launch_bounds__(kDlThreads, 1)
dlinear_wgmma_kernel(const __grid_constant__ DlinMulti mp) {
  using Cfg = DlCfg<kM, kPacked>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kABytes = Cfg::kABytes;
  constexpr int kStageBytes = Cfg::kStageBytes;
  constexpr bool kTiles = (kM == 64);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kBOff;
  float* smem_acc = reinterpret_cast<float*>(smem + Cfg::kAccOff);  // [2][kM][kDlAccLd]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kBarOff);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;
  uint64_t* acc_full_bar = bars + 2 * kStages;
  uint64_t* acc_empty_bar = bars + 2 * kStages + 2;
  __shared__ unsigned char s_ready[1024];  // producer-thread private: producer tile t known finalised for op (value)
  if (threadIdx.x < 256) reinterpret_cast<unsigned int*>(s_ready)[threadIdx.x] = 0u;

  const int warp_idx = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  const int n_ops = mp.n_ops;

  if (warp_idx == 0 && lane == 0) {
    for (int i = 0; i < n_ops; ++i) {
      if (!kPacked) tma_prefetch_desc(&mp.tw[i]);
      tma_prefetch_desc(&mp.tx[i]);
    }
  }
  if (warp_idx == 1 && lane == 0) {
    // one arrival per MMA / epilogue warp (128 per-thread arrivals on one mbarrier serialise)
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);
    }
    for (int s = 0; s < 2; ++s) {
      mbar_init(&acc_full_bar[s], 4);
      mbar_init(&acc_empty_bar[s], 4);
    }
    fence_barrier_init();
  }
  __syncthreads();
  // Programmatic dependent launch: the next kernel may start its prologue as soon as SMs free up; it
  // still waits (griddepcontrol.wait) for this grid to complete before touching anything we write.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp_idx == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      // every weight byte is read once per token: weight tiles are the first lines L2 gives up, so the streamed weights
      // do not push out what is read again (activations, split-tile slots, counters, the attention's KV cache)
      const uint64_t pol_w = l2_policy_evict_first();
      // weight half of a stage: one packed unit (1-D bulk copy) or one 128B-swizzled bf16 tile (tensor map)
      auto load_w = [&](int st, const DlinArgs& p, int oi, const UnitIter& u) {
        if constexpr (kPacked)
          bulk_load_hint(smem_a + st * kABytes, p.wpk + ((long long)u.tile * u.kblocks + u.kb) * kPkUnitBytes,
                         kPkUnitBytes, &full_bar[st], pol_w);
        else
          tma_load_4d_hint(smem_a + st * kABytes, &mp.tw[oi], &full_bar[st], u.kb * kDlK, u.tile * kM, 0, 0, pol_w);
      };
      int stage = 0;
      uint32_t phase = 0;
      unsigned int target = 0;
      int step = 0;
      for (int oi = 0; oi < n_ops; ++oi) {
        const DlinArgs& p = mp.op[oi];
        UnitIter it = make_iter(p.num_tiles, p.kblocks, kTiles);
        // stages of weight tiles requested BEFORE the dependency is satisfied (first op: all; later ops: tunable -
        // a full-ring burst queues the dependency's control traffic behind 24 MB of bulk loads)
        const int pre_cap = (oi == 0 || mp.pre_stages <= 0 || mp.pre_stages > kStages) ? kStages : mp.pre_stages;
        const int npre = it.left < pre_cap ? it.left : pre_cap;
        // (1) weights never depend on earlier kernels / ops: refill the ring with this op's W tiles as
        //     soon as the previous op's MMAs release the slots ...
        int st = stage;
        uint32_t ph = phase;
        UnitIter pre = it;
        for (int j = 0; j < npre; ++j) {
          mbar_wait(&empty_bar[st], ph ^ 1);
          mbar_arrive_expect_tx(&full_bar[st], kStageBytes);
          load_w(st, p, oi, pre);
          pre.next();
          if (++st == kStages) {
            st = 0;
            ph ^= 1;
          }
        }
        // ... and keep HBM busy while we wait for the dependency: L2 prefetch of the tiles after the ring
        {
          UnitIter la = pre;
          for (int j = 0; j < mp.lookahead_units && la.left > 0; ++j) {
            if constexpr (kPacked)
              bulk_prefetch_l2(p.wpk + ((long long)la.tile * la.kblocks + la.kb) * kPkUnitBytes, kPkUnitBytes);
            else
              tma_prefetch_l2_4d(&mp.tw[oi], la.kb * kDlK, la.tile * kM, 0, 0);
            la.next();
          }
        }
        U2_STAMP(oi, 0);  // W prefetch issued
        // (2) ... then wait until the activations exist: the previous kernel (first op), the producing tiles of
        //     the previous op (per-tile flags: no grid-wide wait on the critical path), or the grid barrier
        if (oi == 0) {
          asm volatile("griddepcontrol.wait;" ::: "memory");
          step = *reinterpret_cast<const volatile int*>(mp.step_dev);
          target = (unsigned int)step * gridDim.x;
        } else if (!p.dep_flags) {
          grid_barrier_wait(mp.gridbar + (oi - 1), target);
          asm volatile("fence.proxy.async;" ::: "memory");  // generic-proxy writes of other CTAs -> our TMA reads
        }
        U2_STAMP(oi, 1);  // dependency satisfied
        // (3) add the activation tiles of the prefetched stages
        for (int j = 0; j < npre; ++j) {
          if (oi > 0 && p.dep_flags) wait_tile_flag(p.dep_flags, it.kb >> p.dep_shift, step, s_ready, oi);
          tma_load_4d(smem_b + stage * kDlBBytes, &mp.tx[oi], &full_bar[stage], it.kb * kDlK, 0, 0, 0);
          it.next();
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
        // (4) steady state
        while (it.left > 0) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          load_w(stage, p, oi, it);
          if (oi > 0 && p.dep_flags) wait_tile_flag(p.dep_flags, it.kb >> p.dep_shift, step, s_ready, oi);
          tma_load_4d(smem_b + stage * kDlBBytes, &mp.tx[oi], &full_bar[stage], it.kb * kDlK, 0, 0, 0);
          it.next();
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
      // nothing left to load for this launch: warm L2 with the next launch's leading weight tiles
      for (int jn = 0; jn < mp.n_next; ++jn) {
        UnitIter la = make_iter(mp.next_tiles[jn], mp.next_kblocks[jn], kTiles);
        for (int j = 0; j < mp.next_units[jn] && la.left > 0; ++j) {
          if (mp.next_pk[jn])
            bulk_prefetch_l2(mp.next_pk[jn] + ((long long)la.tile * la.kblocks + la.kb) * kPkUnitBytes, kPkUnitBytes);
          else
            tma_prefetch_l2_4d(&mp.tnext[jn], la.kb * kDlK, la.tile * kM, 0, 0);
          la.next();
        }
      }
    }
  } else if (warp_idx >= kDlMmaWarp0) {
    // ===================== MMA warpgroup =====================
    const int w = warp_idx - kDlMmaWarp0;
    int stage = 0;
    uint32_t phase = 0;
    int acc = 0;
    uint32_t acc_phase = 0;
    for (int oi = 0; oi < n_ops; ++oi) {
      UnitIter it = make_iter(mp.op[oi].num_tiles, mp.op[oi].kblocks, kTiles);
      bool first_unit = true;
      while (it.left > 0) {
        const int seg = it.seg_len();
        float d[kM / 64][8];
        for (int j = 0; j < seg; ++j) {
          mbar_wait(&full_bar[stage], phase);
          if (first_unit) {
            if (threadIdx.x == kDlMmaWarp0 * 32) U2_STAMP(oi, 2);  // first stage of the op landed
            first_unit = false;
          }
          const uint64_t b_desc = gmma_desc_sw128(smem_u32(smem_b + stage * kDlBBytes));
          if constexpr (kPacked) {
            // this thread's 104 bytes of the unit -> its 32 bf16x2 A-fragment words (bit-identical to the bf16 weights)
            const uint32_t ua = smem_u32(smem_a + stage * kABytes);
            const uint32_t t16 = (threadIdx.x - kDlMmaWarp0 * 32) * 16;
            uint32_t smw[16], nib[8], hi[2];
            const uint32_t base = lds128(ua).x;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const uint4 v = lds128(ua + kPkSmOff + c * 2048 + t16);
              smw[4 * c] = v.x; smw[4 * c + 1] = v.y; smw[4 * c + 2] = v.z; smw[4 * c + 3] = v.w;
            }
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const uint4 v = lds128(ua + kPkNibOff + c * 2048 + t16);
              nib[4 * c] = v.x; nib[4 * c + 1] = v.y; nib[4 * c + 2] = v.z; nib[4 * c + 3] = v.w;
            }
            {
              uint2 v;
              asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(ua + kPkHiOff + t16 / 2));
              hi[0] = v.x; hi[1] = v.y;
            }
            const uint32_t b7 = (base << 7) * 0x10001u;
            uint32_t a[8][4];  // [mh * 4 + ks][r]
#define U2_PK_W(R) a[(R) >> 2][(R) & 3] = unpack_word<R>(smw[(R) >> 1], nib[(R) >> 2], hi[(R) >> 4], b7)
            U2_PK_W(0); U2_PK_W(1); U2_PK_W(2); U2_PK_W(3); U2_PK_W(4); U2_PK_W(5); U2_PK_W(6); U2_PK_W(7);
            U2_PK_W(8); U2_PK_W(9); U2_PK_W(10); U2_PK_W(11); U2_PK_W(12); U2_PK_W(13); U2_PK_W(14); U2_PK_W(15);
            U2_PK_W(16); U2_PK_W(17); U2_PK_W(18); U2_PK_W(19); U2_PK_W(20); U2_PK_W(21); U2_PK_W(22); U2_PK_W(23);
            U2_PK_W(24); U2_PK_W(25); U2_PK_W(26); U2_PK_W(27); U2_PK_W(28); U2_PK_W(29); U2_PK_W(30); U2_PK_W(31);
#undef U2_PK_W
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kDlK / 16; ++k) {
#pragma unroll
              for (int mh = 0; mh < kM / 64; ++mh)
                wgmma_m64n16k16_rs(d[mh], a[mh * 4 + k], b_desc + 2 * k, (j == 0 && k == 0) ? 0u : 1u);
            }
          } else {
            const uint64_t a_desc = gmma_desc_sw128(smem_u32(smem_a + stage * kABytes));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kDlK / 16; ++k) {
#pragma unroll
              for (int mh = 0; mh < kM / 64; ++mh)  // weight rows 64..127 start 8 KB further
                wgmma_m64n16k16_ss(d[mh], a_desc + 512 * mh + 2 * k, b_desc + 2 * k, (j == 0 && k == 0) ? 0u : 1u);
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
          it.next();
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
        // hand the accumulator to the epilogue: row n of the tile, column b = sequence
        mbar_wait(&acc_empty_bar[acc], acc_phase ^ 1);
        float* dst = smem_acc + acc * (kM * kDlAccLd);
#pragma unroll
        for (int mh = 0; mh < kM / 64; ++mh) {
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int r = mh * 64 + w * 16 + (lane >> 2) + 8 * ((e >> 1) & 1);
            dst[r * kDlAccLd + 8 * (e >> 2) + 2 * (lane & 3) + (e & 1)] = d[mh][e];
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&acc_full_bar[acc]);
        if (it.left == 0 && threadIdx.x == kDlMmaWarp0 * 32) U2_STAMP(oi, 3);  // last MMA of the op done
        if (++acc == 2) {
          acc = 0;
          acc_phase ^= 1;
        }
      }
    }
  } else if (warp_idx >= 4) {
    // ===================== epilogue (warps 4-7) =====================
    const int q = warp_idx - 4;
    const int et = threadIdx.x - 128;  // 0..127
    // accumulator row held by this thread: M = 128 -> thread == row; M = 64 -> rows 16q .. 16q+15 go to lanes
    // 0 .. 15 of warp q (the upper 16 lanes of every warp are unused)
    const int trow = (kM == 128) ? et : (q * 16 + (lane & 15));
    const bool tvalid = (kM == 128) ? true : (lane < 16);
    asm volatile("griddepcontrol.wait;" ::: "memory");  // workspace / residual / ssq come from earlier kernels
    const unsigned int target = (unsigned int)(*reinterpret_cast<const volatile int*>(mp.step_dev)) * gridDim.x;
    int acc = 0;
    uint32_t acc_phase = 0;
    for (int oi = 0; oi < n_ops; ++oi) {
      const DlinArgs& p = mp.op[oi];
      UnitIter it = make_iter(p.num_tiles, p.kblocks, kTiles);
      bool prev_done = (oi == 0);  // "every tile of the previous op is finalised" already observed by this CTA?
      if (oi > 0 && !p.dep_flags) {
        // coarse mode: previous op fully finalised everywhere? one poller per CTA, the CTA barrier fans it out
        if (et == 0) grid_barrier_wait(mp.gridbar + (oi - 1), target);
        asm volatile("bar.sync 1, 128;" ::: "memory");
        prev_done = true;
      }
      while (it.left > 0) {
        const int tile = it.tile;
        const int seg_kb = it.seg_len();
        // advance the cursor past this segment (always ends at a tile boundary or at the end of the range)
        it.left -= seg_kb;
        it.kb += seg_kb;
        if (it.kb == it.kblocks) {
          it.kb = 0;
          it.tile += it.tile_step;
        }

        // ---- role of this CTA for the tile, and the epilogue operands that do not depend on any partial sum: both
        //      are resolved BEFORE waiting for the accumulator, so their L2 round trips hide behind the weight stream
        const int row = tile * kM + trow;  // output row n of W
        const bool whole = (seg_kb == p.kblocks);  // this CTA sees the entire K range of the tile
        // Split tile (stream-K only). The CTA whose range contains k-block 0 of the tile finalises it - that
        // segment is the LAST one of its range - while the CTAs holding the later k-blocks meet the tile as
        // their FIRST segment: they drop their partial sums into a private slot and move on.
        int gf = (int)blockIdx.x, n_contrib = 0;
        if (!whole) {
          const long long units = (long long)p.num_tiles * p.kblocks;
          const long long G = units < (long long)gridDim.x ? units : (long long)gridDim.x;
          const long long u0 = (long long)tile * p.kblocks;
          gf = (int)(((u0 + 1) * G + units - 1) / units) - 1;
          n_contrib = (int)(((u0 + p.kblocks) * G + units - 1) / units) - 1 - gf;
        }
        const bool finalizer = (gf == (int)blockIdx.x);
        const int nvec = (p.B + 3) >> 2;
        const bool row_ok = tvalid && row < p.N;
        unsigned short res_raw[16];
        float rs[16];
        float gam = 0.f;
        if (finalizer) {
          if (!prev_done) {
            // fine-grained mode: ssq / residual / ssq_zero need the WHOLE previous op (long since finished)
            if (et == 0) grid_barrier_wait(mp.gridbar + (oi - 1), target);
            asm volatile("bar.sync 1, 128;" ::: "memory");
            prev_done = true;
          }
#pragma unroll
          for (int b = 0; b < 16; ++b) {
            res_raw[b] = 0;
            rs[b] = 1.f;
            if (b < p.B) {
              if (p.residual && !p.silu_pair && row_ok)
                res_raw[b] = __ldcg(reinterpret_cast<const unsigned short*>(p.residual) + (long long)b * p.ldr + row);
              if (p.ssq_in) rs[b] = __ldcg(p.ssq_in + b);
            }
          }
          if (p.gamma_next && row_ok) gam = __ldg(p.gamma_next + row);
        }

        mbar_wait(&acc_full_bar[acc], acc_phase);
        if (et == 0 && it.left == 0) U2_STAMP(oi, 4);  // last accumulator of the op available
        uint32_t v[16];
        {
          const uint32_t src = smem_u32(smem_acc + acc * (kM * kDlAccLd) + trow * kDlAccLd);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const uint4 x = lds128(src + 16 * c);
            v[4 * c] = x.x; v[4 * c + 1] = x.y; v[4 * c + 2] = x.z; v[4 * c + 3] = x.w;
          }
        }
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(&acc_empty_bar[acc]);  // accumulator buffer is free again
        if (++acc == 2) {
          acc = 0;
          acc_phase ^= 1;
        }

        float f[16];
#pragma unroll
        for (int b = 0; b < 16; ++b) f[b] = __uint_as_float(v[b]);
        if (!finalizer) {
          const int slot = (int)blockIdx.x - gf - 1;
          float4* dst = reinterpret_cast<float4*>(p.ws + (((long long)tile * p.max_slots + slot) * kM + trow) * kDlN);
          // self-validating slots: every 4-byte word of a slot holds either the sentinel (all ones, a NaN pattern no
          // fp32 sum produces) or a final partial sum, so the finaliser polls the DATA - no flag, no fence, no RMW
          if (tvalid) {
#pragma unroll
            for (int c = 0; c < 4; ++c)
              if (c < nvec) __stcg(dst + c, make_float4(f[4 * c], f[4 * c + 1], f[4 * c + 2], f[4 * c + 3]));
          }
        } else {
          // ---------------- this CTA finalises the tile ----------------
          if (et == 0) U2_STAMP(oi, 6);  // finaliser: start waiting for the contributors
          if (n_contrib > 0 && tvalid) {
            // poll the contributors' slots of this row (independent loads, one L2 round trip per sweep); a slot is
            // complete when none of its words is the sentinel; consumed slots are handed back as sentinels
            const long long slot_stride = (long long)kM * kDlN / 4;  // in float4
            float4* src0 = reinterpret_cast<float4*>(p.ws + (((long long)tile * p.max_slots) * kM + trow) * kDlN);
            const float4 sent = make_float4(__uint_as_float(0xffffffffu), __uint_as_float(0xffffffffu),
                                            __uint_as_float(0xffffffffu), __uint_as_float(0xffffffffu));
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              if (c >= nvec) break;
              constexpr int kMaxSlots = 8;
              for (int s0 = 0; s0 < n_contrib; s0 += kMaxSlots) {
                float4 t[kMaxSlots];
                bool ok;
                unsigned int spins = 0;
                do {
                  ok = true;
#pragma unroll
                  for (int sl = 0; sl < kMaxSlots; ++sl)
                    if (s0 + sl < n_contrib) t[sl] = ld_relaxed_f4(src0 + (s0 + sl) * slot_stride + c);
#pragma unroll
                  for (int sl = 0; sl < kMaxSlots; ++sl)
                    if (s0 + sl < n_contrib) {
                      ok = ok && (__float_as_uint(t[sl].x) != 0xffffffffu) && (__float_as_uint(t[sl].y) != 0xffffffffu) &&
                           (__float_as_uint(t[sl].z) != 0xffffffffu) && (__float_as_uint(t[sl].w) != 0xffffffffu);
                    }
                } while (!ok && ++spins < (1u << 22));  // bounded: a lost contributor must not hang the GPU
#pragma unroll
                for (int sl = 0; sl < kMaxSlots; ++sl)
                  if (s0 + sl < n_contrib) {
                    f[4 * c] += t[sl].x; f[4 * c + 1] += t[sl].y; f[4 * c + 2] += t[sl].z; f[4 * c + 3] += t[sl].w;
                    __stcg(src0 + (s0 + sl) * slot_stride + c, sent);
                  }
              }
            }
          }
          if (et == 0) U2_STAMP(oi, 7);  // finaliser: all partial sums in
          // ---------------- fused epilogue for the finished tile ----------------
          if (p.ssq_zero && tile == 0 && et < 16) p.ssq_zero[et] = 0.f;
          float sq[16];
#pragma unroll
          for (int b = 0; b < 16; ++b) {
            sq[b] = 0.f;
            if (b < p.B) {
              float val = f[b];
              if (p.ssq_in) val *= rsqrtf(rs[b] * p.inv_norm_dim + p.eps);
              if (p.silu_pair) {
                // rounding points of the unfused path: gate/up are bf16 before the activation
                const float me = __bfloat162float(__float2bfloat16(val));
                const float other = __shfl_down_sync(0xffffffffu, me, 1);
                if (row_ok && (trow & 1) == 0) {
                  const float o = __fdividef(me, 1.f + __expf(-me)) * other;
                  reinterpret_cast<__nv_bfloat16*>(p.y)[(long long)b * p.ldy + (row >> 1)] = __float2bfloat16(o);
                }
              } else if (row_ok) {
                val += __bfloat162float(__ushort_as_bfloat16(res_raw[b]));
                if (p.y_dtype == U2_DT_BF16) {
                  const __nv_bfloat16 o = __float2bfloat16(val);
                  reinterpret_cast<__nv_bfloat16*>(p.y)[(long long)b * p.ldy + row] = o;
                  val = __bfloat162float(o);
                } else {
                  reinterpret_cast<float*>(p.y)[(long long)b * p.ldy + row] = val;
                }
                if (p.gamma_next) p.xg[(long long)b * p.ldxg + row] = __float2bfloat16(val * gam);
                sq[b] = val * val;
              }
            }
          }
          if (p.ssq_out) {
            // run-to-run identical sums (the next op's RMSNorm scale depends on them): the tile's sum per sequence is
            // formed in a fixed order and stored; the CTA that finalises the op's last tile adds the stored sums up in
            // tile order. Float atomics would make the result depend on the order in which tiles finish.
            __shared__ float s_sq[4][16];
            __shared__ int s_last;
#pragma unroll
            for (int b = 0; b < 16; ++b) {
              float s = sq[b];
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
              if (lane == 0) s_sq[q][b] = s;
            }
            asm volatile("bar.sync 1, 128;" ::: "memory");
            if (et < 16) {
              __stcg(p.ssq_part + (long long)tile * 16 + et, ((s_sq[0][et] + s_sq[1][et]) + s_sq[2][et]) + s_sq[3][et]);
              __threadfence();
            }
            asm volatile("bar.sync 1, 128;" ::: "memory");
            if (et == 0) s_last = (atomicAdd(p.ssq_ticket, 1) == p.num_tiles - 1);
            asm volatile("bar.sync 1, 128;" ::: "memory");
            if (s_last) {
              // 8 groups of 16 threads (one per sequence) each sum the tiles g, g + 8, g + 16, ... with their loads in
              // flight together, then the group sums are added in group order. The stored sums are re-armed with the
              // sentinel: another op of the launch that shares this ws may use these words as split-tile slots, which
              // must read "empty" until written.
              __shared__ float s_grp[8][16];
              __threadfence();
              const int col = et & 15, grp = et >> 4;
              float t = 0.f;
              for (int i0 = grp; i0 < p.num_tiles; i0 += 32) {
                float v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                  const int i = i0 + 8 * u;
                  v[u] = (i < p.num_tiles) ? __ldcg(p.ssq_part + (long long)i * 16 + col) : 0.f;
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                  const int i = i0 + 8 * u;
                  if (i < p.num_tiles) {
                    t += v[u];
                    __stcg(p.ssq_part + (long long)i * 16 + col, __uint_as_float(0xffffffffu));
                  }
                }
              }
              s_grp[grp][col] = t;
              asm volatile("bar.sync 1, 128;" ::: "memory");
              if (et < p.B) {
                float tot = 0.f;
#pragma unroll
                for (int g = 0; g < 8; ++g) tot += s_grp[g][et];
                p.ssq_out[et] += tot;
              }
              if (et == 0) *p.ssq_ticket = 0;  // zero again for the next launch
            }
          }
          if (p.out_flags) {
            // publish "tile finalised in this step" for the consumers of the next op (release after the CTA barrier
            // covers all 128 threads' output stores)
            asm volatile("bar.sync 1, 128;" ::: "memory");
            if (et == 0) {
              const int stepv = (int)(target / gridDim.x);
              asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p.out_flags + tile), "r"(stepv) : "memory");
            }
          }
        }
      }
      if (et == 0) U2_STAMP(oi, 5);  // epilogue of the op done
      // this CTA's share of op `oi` is complete (partials published / tiles finalised): arrive at the grid
      // barrier that gates the next op (release covers the whole epilogue warp-group through the CTA barrier)
      if (oi + 1 < n_ops) {
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (et == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(mp.gridbar + oi) : "memory");
      }
    }
  }
}

// embed gather for the decode step + preparation of the first layer's fused norm:
// x[b] = table[ids[b]], xg[b] = bf16(x * gamma), ssq[b] = sum x^2 ; also resets ssq_zero.
__global__ void __launch_bounds__(256)
decode_embed_kernel(const long long* __restrict__ ids, const __nv_bfloat16* __restrict__ table,
                    const float* __restrict__ gamma, __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ xg,
                    float* __restrict__ ssq, float* __restrict__ ssq_zero, int* __restrict__ step_counter, int E,
                    long long vocab) {
  const int b = blockIdx.x;
  if (b == 0 && threadIdx.x == 0 && step_counter) *step_counter += 1;  // grid-barrier epoch of this decode step
  long long id = ids[b];
  if (id < 0) id = 0;
  if (id >= vocab) id = vocab - 1;
  const __nv_bfloat16* src = table + id * E;
  float s = 0.f;
  for (int i = threadIdx.x; i < E; i += blockDim.x) {
    const __nv_bfloat16 v = src[i];
    const float f = __bfloat162float(v);
    x[(long long)b * E + i] = v;
    xg[(long long)b * E + i] = __float2bfloat16(f * gamma[i]);
    s += f * f;
  }
  __shared__ float red[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    ssq[b] = t;
    if (ssq_zero) ssq_zero[b] = 0.f;
  }
}

// Packs one 128 x 64 unit per CTA (128 threads, thread t = the MMA thread that will unpack its 64 weights) into the
// layout described at kPkUnitBytes. A unit whose exponents do not fit the code (a nonzero exponent at or below base)
// is counted in *bad; its bytes are then meaningless and the caller keeps the bf16 weights.
__global__ void __launch_bounds__(128)
dlinear_pack_kernel(const uint16_t* __restrict__ w, long long ldw, int N, int kblocks, uint8_t* __restrict__ out,
                    int* __restrict__ bad) {
  const int unit = blockIdx.x, tile = unit / kblocks, kb = unit - tile * kblocks;
  const int t = threadIdx.x, wq = t >> 5, l = t & 31;
  uint32_t v[32];  // fragment word R: (column c, column c + 1) bf16 pair
  int emax = 0;
#pragma unroll
  for (int R = 0; R < 32; ++R) {
    const int mh = R >> 4, ks = (R >> 2) & 3, r = R & 3;
    const int row = tile * 128 + mh * 64 + wq * 16 + (l >> 2) + 8 * (r & 1);
    const int col = kb * kDlK + ks * 16 + 2 * (l & 3) + 8 * (r >> 1);
    v[R] = row < N ? *reinterpret_cast<const uint32_t*>(w + (long long)row * ldw + col) : 0u;
    emax = max(emax, (int)max((v[R] >> 7) & 0xff, (v[R] >> 23) & 0xff));
  }
  __shared__ int s_max[4];
  __shared__ int s_bad;
  emax = __reduce_max_sync(0xffffffffu, emax);
  if (l == 0) s_max[wq] = emax;
  if (t == 0) s_bad = 0;
  __syncthreads();
  emax = max(max(s_max[0], s_max[1]), max(s_max[2], s_max[3]));
  const int base = emax > 31 ? emax - 31 : 0;
  uint32_t smw[16] = {}, nib[8] = {}, hi[2] = {};
  bool fits = true;
#pragma unroll
  for (int R = 0; R < 32; ++R) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t x = (v[R] >> (16 * h)) & 0xffffu;
      const int e = (x >> 7) & 0xff;
      fits = fits && (e == 0 || e > base);
      const uint32_t c = e == 0 ? 0u : (uint32_t)(e - base) & 31u;
      smw[R >> 1] |= (((x >> 8) & 0x80u) | (x & 0x7fu)) << (8 * (2 * (R & 1) + h));
      nib[R >> 2] |= (c & 15u) << (4 * (R & 3) + 16 * h);
      hi[R >> 4] |= (c >> 4) << ((R & 15) + 16 * h);
    }
  }
  if (!fits) s_bad = 1;
  uint8_t* u = out + (long long)unit * kPkUnitBytes;
  if (t == 0) *reinterpret_cast<uint4*>(u) = make_uint4((uint32_t)base, 0u, 0u, 0u);
#pragma unroll
  for (int c = 0; c < 4; ++c)
    *reinterpret_cast<uint4*>(u + kPkSmOff + (c * 128 + t) * 16) =
        make_uint4(smw[4 * c], smw[4 * c + 1], smw[4 * c + 2], smw[4 * c + 3]);
#pragma unroll
  for (int c = 0; c < 2; ++c)
    *reinterpret_cast<uint4*>(u + kPkNibOff + (c * 128 + t) * 16) =
        make_uint4(nib[4 * c], nib[4 * c + 1], nib[4 * c + 2], nib[4 * c + 3]);
  *reinterpret_cast<uint2*>(u + kPkHiOff + t * 8) = make_uint2(hi[0], hi[1]);
  __syncthreads();
  if (t == 0 && s_bad) atomicAdd(bad, 1);
}

}  // namespace u2

using namespace u2;

static int fill_op(const void* x, const void* w, void* y, const u2_dlinear_desc* d, DlinArgs* p, CUtensorMap* tw,
                   CUtensorMap* tx, int kM) {
  if (!x || !w || !y || !d || !d->ws || !d->counters) return set_error(U2_ERR_ARG, "dlinear: null pointer");
  if (d->B < 1 || d->B > kDlN) return set_error(U2_ERR_UNSUPPORTED, "dlinear: 1 <= B <= 16 (got %d)", d->B);
  if (d->N <= 0 || d->K <= 0 || (d->K % kDlK)) return set_error(U2_ERR_ARG, "dlinear: K must be a positive multiple of 64");
  const bool packed = d->w_format == U2_DLIN_W_PACKED13;
  if (!packed && d->w_format != U2_DLIN_W_BF16) return set_error(U2_ERR_ARG, "dlinear: unknown w_format %d", d->w_format);
  if (packed && kM != 128) return set_error(U2_ERR_UNSUPPORTED, "dlinear: packed weights need the stream-K schedule");
  if (packed && (reinterpret_cast<uintptr_t>(w) & 15)) return set_error(U2_ERR_ARG, "dlinear: packed weights must be 16-byte aligned");
  if ((d->ldx & 7) || (!packed && (d->ldw & 7))) return set_error(U2_ERR_ARG, "dlinear: ldx/ldw must be multiples of 8");
  if (d->silu_pair && (d->N & 1)) return set_error(U2_ERR_ARG, "dlinear: silu_pair needs an even N");
  if (d->gamma_next && !d->xg) return set_error(U2_ERR_ARG, "dlinear: gamma_next needs xg");
  p->B = d->B; p->N = d->N; p->K = d->K;
  p->num_tiles = (d->N + kM - 1) / kM;
  p->kblocks = d->K / kDlK;
  p->wpk = packed ? reinterpret_cast<const uint8_t*>(w) : nullptr;
  p->ws = d->ws; p->counters = d->counters;
  p->max_slots = 1;
  if (kM == 128) {
    // contributors per split tile <= ceil(kblocks / shortest CTA range) + 1
    const long long units = (long long)p->num_tiles * p->kblocks;
    int g = num_sms();
    if (g <= 0) g = 132;
    long long rmin = units / g;
    if (rmin < 1) rmin = 1;
    const long long cmax = (p->kblocks + rmin - 1) / rmin + 1;
    p->max_slots = (int)cmax;
    if ((long long)p->num_tiles * cmax * kM * kDlN > d->ws_elems)
      return set_error(U2_ERR_ARG, "dlinear: workspace too small (%lld fp32 needed for N=%d K=%d)",
                       (long long)p->num_tiles * cmax * kM * kDlN, d->N, d->K);
  }
  p->ssq_in = d->ssq_in;
  p->inv_norm_dim = 1.0f / (float)d->K;
  p->eps = d->eps;
  p->residual = reinterpret_cast<const __nv_bfloat16*>(d->residual);
  p->ldr = d->ldr;
  p->y = y; p->ldy = d->ldy; p->y_dtype = d->y_dtype;
  p->silu_pair = d->silu_pair;
  p->gamma_next = d->gamma_next;
  p->xg = reinterpret_cast<__nv_bfloat16*>(d->xg);
  p->ldxg = d->ldxg;
  p->ssq_out = d->ssq_out;
  p->ssq_part = nullptr;
  p->ssq_ticket = nullptr;
  if (d->ssq_out) {
    // the per-tile sums of squares live behind the split-tile slots of ws; the op's tile ticket behind the counters
    const long long slots = (kM == 128) ? (long long)p->num_tiles * p->max_slots * kM * kDlN : 0;
    if (slots + (long long)p->num_tiles * kDlN > d->ws_elems)
      return set_error(U2_ERR_ARG, "dlinear: workspace too small for the sums of squares (%lld fp32 needed for N=%d K=%d)",
                       slots + (long long)p->num_tiles * kDlN, d->N, d->K);
    p->ssq_part = d->ws + slots;
    p->ssq_ticket = d->counters + (d->N + 63) / 64;
  }
  p->ssq_zero = d->ssq_zero;
  p->dep_flags = d->dep_flags;
  p->dep_shift = d->dep_shift;
  p->out_flags = d->out_flags;
  p->dbg = nullptr;
  if (!packed) {
    int rc = make_tmap_bf16_4d(tw, w, d->K, d->N, 1, 1, d->ldw, 0, 0, kDlK, kM);
    if (rc) return rc;
  }
  return make_tmap_bf16_4d(tx, x, d->K, d->B, 1, 1, d->ldx, 0, 0, kDlK, kDlN);
}

template <int kM, bool kPacked>
static int launch_multi_t(DlinMulti& mp, int pdl, cudaStream_t stream) {
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(dlinear_wgmma_kernel<kM, kPacked>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         DlCfg<kM, kPacked>::kSmem);
    if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "dlinear: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    // the software grid barrier between the chained linears needs grid <= resident CTA capacity
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dlinear_wgmma_kernel<kM, kPacked>, kDlThreads,
                                                      DlCfg<kM, kPacked>::kSmem);
    if (e != cudaSuccess || per_sm < 1)
      return set_error(U2_ERR_CUDA, "dlinear: kernel cannot be resident on an SM (%s, %d CTA/SM): set U2_MULTI_OP=0",
                       cudaGetErrorString(e), per_sm);
    configured = true;
  }
  int grid = num_sms();
  if (grid <= 0) return set_error(U2_ERR_CUDA, "dlinear: cannot query SM count");
  if (mp.n_ops == 1) {
    const long long work = (kM == 64) ? mp.op[0].num_tiles : (long long)mp.op[0].num_tiles * mp.op[0].kblocks;
    if (work < grid) grid = (int)work;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kDlThreads);
  cfg.dynamicSmemBytes = DlCfg<kM, kPacked>::kSmem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, dlinear_wgmma_kernel<kM, kPacked>, mp);
  if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "dlinear launch: %s", cudaGetErrorString(e));
  return U2_OK;
}

static int launch_multi(DlinMulti& mp, int kM, bool packed, int pdl, cudaStream_t stream) {
  if (packed) return launch_multi_t<128, true>(mp, pdl, stream);
  return kM == 64 ? launch_multi_t<64, false>(mp, pdl, stream) : launch_multi_t<128, false>(mp, pdl, stream);
}

static inline int tile_m_of(const u2_dlinear_desc* d) { return d->sched == U2_DLIN_TILES64 ? 64 : 128; }


extern "C" U2_API int64_t u2_dlinear_ws_elems(int32_t N, int32_t K) {
  if (N <= 0 || K <= 0) return 0;
  const long long tiles = (N + 127) / 128, kblocks = (K + kDlK - 1) / kDlK;
  int g = num_sms();
  if (g <= 0) g = 132;
  long long rmin = tiles * kblocks / g;
  if (rmin < 1) rmin = 1;
  const long long cmax = (kblocks + rmin - 1) / rmin + 1;
  return tiles * cmax * 128 * kDlN + (N + 63) / 64 * kDlN;  // split-tile slots + per-tile sums of squares
}

extern "C" U2_API int u2_dlinear_bf16(const void* x, const void* w, void* y, const u2_dlinear_desc* d, void* stream) {
  static DlinMulti mp;  // large (tensor maps): keep off the stack; single-threaded use per the ABI contract
  mp.n_ops = 1;
  if (!d) return set_error(U2_ERR_ARG, "dlinear: null descriptor");
  const int kM = tile_m_of(d);
  int rc = fill_op(x, w, y, d, &mp.op[0], &mp.tw[0], &mp.tx[0], kM);
  if (rc) return rc;
  mp.gridbar = nullptr;
  mp.n_next = 0;
  mp.lookahead_units = 0;
  mp.pre_stages = 0;
  mp.dbg = reinterpret_cast<unsigned long long*>(d->dbg);
  // single op: the step counter is only read to form a barrier target that is never used; point it at any
  // valid device int (the tile counters are zero between launches)
  mp.step_dev = d->counters;
  return launch_multi(mp, kM, d->w_format == U2_DLIN_W_PACKED13, d->pdl, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" U2_API int u2_dlinear_multi_bf16(const void* const* x, const void* const* w, void* const* y,
                                            const u2_dlinear_desc* descs, int32_t n_ops, uint32_t* gridbar,
                                            const int32_t* step_dev, int32_t pdl, const u2_dlinear_next* next,
                                            void* stream) {
  if (!x || !w || !y || !descs) return set_error(U2_ERR_ARG, "dlinear_multi: null pointer");
  if (n_ops < 1 || n_ops > kDlMaxOps) return set_error(U2_ERR_ARG, "dlinear_multi: 1 <= n_ops <= %d", kDlMaxOps);
  if (n_ops > 1 && (!gridbar || !step_dev)) return set_error(U2_ERR_ARG, "dlinear_multi: gridbar / step_dev required");
  static DlinMulti mp;
  mp.n_ops = n_ops;
  const int kM = tile_m_of(&descs[0]);
  const int32_t fmt = descs[0].w_format;
  for (int i = 0; i < n_ops; ++i) {
    if (tile_m_of(&descs[i]) != kM) return set_error(U2_ERR_ARG, "dlinear_multi: all ops of a launch must share one schedule");
    if (descs[i].w_format != fmt) return set_error(U2_ERR_ARG, "dlinear_multi: all ops of a launch must share one weight format");
    int rc = fill_op(x[i], w[i], y[i], &descs[i], &mp.op[i], &mp.tw[i], &mp.tx[i], kM);
    if (rc) return rc;
  }
  mp.gridbar = gridbar;
  mp.lookahead_units = next ? next->lookahead_units : 0;
  mp.pre_stages = next ? next->pre_stages : 0;
  mp.n_next = 0;
  if (next) {
    for (int j = 0; j < 2 && j < next->n; ++j) {
      if (!next->w[j] || next->K[j] % kDlK || next->N[j] <= 0) return set_error(U2_ERR_ARG, "dlinear_multi: bad look-ahead weight");
      mp.next_pk[j] = nullptr;
      if (next->w_format[j] == U2_DLIN_W_PACKED13) {
        if (kM != 128) return set_error(U2_ERR_UNSUPPORTED, "dlinear_multi: packed look-ahead needs the stream-K schedule");
        mp.next_pk[j] = reinterpret_cast<const uint8_t*>(next->w[j]);
      } else {
        int rc = make_tmap_bf16_4d(&mp.tnext[j], next->w[j], next->K[j], next->N[j], 1, 1, next->ldw[j], 0, 0, kDlK, kM);
        if (rc) return rc;
      }
      mp.next_tiles[j] = (next->N[j] + kM - 1) / kM;
      mp.next_kblocks[j] = next->K[j] / kDlK;
      mp.next_units[j] = next->units[j];
      mp.n_next = j + 1;
    }
  }
  mp.dbg = reinterpret_cast<unsigned long long*>(descs[0].dbg);
  mp.step_dev = step_dev ? step_dev : descs[0].counters;
  return launch_multi(mp, kM, fmt == U2_DLIN_W_PACKED13, pdl, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" U2_API int u2_dlinear_pack_bf16(const void* w, int32_t N, int32_t K, int64_t ldw, void* out, int32_t* bad,
                                           void* stream) {
  if (!w || !out || !bad) return set_error(U2_ERR_ARG, "dlinear_pack: null pointer");
  if (N <= 0 || K <= 0 || K % kDlK) return set_error(U2_ERR_ARG, "dlinear_pack: K must be a positive multiple of 64");
  if (ldw < K || (ldw & 1) || (reinterpret_cast<uintptr_t>(w) & 3) || (reinterpret_cast<uintptr_t>(out) & 15))
    return set_error(U2_ERR_ARG, "dlinear_pack: ldw >= K and even, w 4-byte and out 16-byte aligned");
  const long long units = (long long)((N + 127) / 128) * (K / kDlK);
  dlinear_pack_kernel<<<(unsigned)units, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint16_t*>(w), ldw, N, K / kDlK, reinterpret_cast<uint8_t*>(out), bad);
  U2_CHECK_LAUNCH("dlinear_pack");
  return U2_OK;
}

extern "C" U2_API int u2_decode_embed_bf16(const int64_t* ids, const void* table, const float* gamma, void* x,
                                           void* xg, float* ssq, float* ssq_zero, int32_t* step_counter, int32_t B,
                                           int32_t E, int64_t vocab, void* stream) {
  if (!ids || !table || !gamma || !x || !xg || !ssq) return set_error(U2_ERR_ARG, "decode_embed: null pointer");
  if (B < 1 || B > kDlN) return set_error(U2_ERR_UNSUPPORTED, "decode_embed: 1 <= B <= 16");
  decode_embed_kernel<<<B, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(ids), reinterpret_cast<const __nv_bfloat16*>(table), gamma,
      reinterpret_cast<__nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(xg), ssq, ssq_zero, step_counter, E, vocab);
  U2_CHECK_LAUNCH("decode_embed");
  return U2_OK;
}
