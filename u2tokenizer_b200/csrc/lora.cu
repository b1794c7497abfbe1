// LoRA adapters of the decoder linears on the training path (PEFT LoraLayer: y = W x + s * B A dropout(x)).
//
//   u2_lora_down_bf16   U[:, j r:(j+1) r] = s * (D_j o X) A_j^T       wgmma, X tiles by TMA, mask applied to the register A operand
//   u2_lora_wgrad_bf16  dA_j (+)= s * dU_j^T (D_j o X)                 fp32 over all M rows, one CTA per (64 columns, adapter)
//   u2_lora_dgrad_bf16  dX += sum_j D_j o (s * dU_j A_j)               one pass over dX
//
// The up-projection (y += U_j B_j^T), dB_j = dY_j^T U_j and dU_j = dY_j B_j run on u2_gemm_bf16. The dropout masks D_j are
// never stored: every kernel recomputes them from the counter hash documented in include/u2b200_train.h.
#include <cuda_bf16.h>
#include <math.h>

#include "host_util.h"
#include "ptx.cuh"
#include "u2b200_train.h"

namespace u2 {

__device__ __forceinline__ uint32_t lora_fmix32(uint32_t h) {
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h;
}

struct LoraMask {
  uint32_t key[3];  // per adapter: fmix32(lo(seed) ^ fmix32(hi(seed) + stream * 0x9E3779B9))
  uint32_t thr;     // an element is dropped when its hash is below thr = floor(p * 2^32)
  float keep;       // 1 / (1 - p)
  int on;           // p > 0
};

__device__ __forceinline__ uint32_t lora_row_key(const LoraMask& mk, int j, uint32_t row) {
  return lora_fmix32(mk.key[j] ^ row);
}
// D_j(row, col) given the row key of (j, row)
__device__ __forceinline__ float lora_mask(const LoraMask& mk, uint32_t row_key, uint32_t col) {
  return lora_fmix32(row_key ^ col) < mk.thr ? 0.f : mk.keep;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// ---- wgmma m64nNk16 with the A operand (64 x 16 bf16) in registers, B (N x 16) K-major in shared memory, D += A B^T --
template <int N>
struct WgmmaRS;

template <>
struct WgmmaRS<8> {
  static __device__ __forceinline__ void run(float (&d)[4], const uint32_t (&a)[4], uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0, %1, %2, %3}, {%4, %5, %6, %7}, %8, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
  }
};
template <>
struct WgmmaRS<16> {
  static __device__ __forceinline__ void run(float (&d)[8], const uint32_t (&a)[4], uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, "
        "1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
  }
};
template <>
struct WgmmaRS<32> {
  static __device__ __forceinline__ void run(float (&d)[16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, "
        "%14, %15}, {%16, %17, %18, %19}, %20, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
  }
};
template <>
struct WgmmaRS<64> {
  static __device__ __forceinline__ void run(float (&d)[32], const uint32_t (&a)[4], uint64_t b) {
    wgmma_m64n64k16_rs<0>(d, a, b);
  }
};

constexpr int kLoraRows = 64;    // rows of X per CTA (one warpgroup, one m64 wgmma row block)
constexpr int kLoraK = 64;       // contraction block: one 128-byte swizzle row of bf16
constexpr int kLoraStages = 2;
constexpr int kLoraMaxAdapters = 3;

template <int R>
struct LoraDownCfg {
  static constexpr int kXBytes = kLoraRows * kLoraK * 2;
  static constexpr int kABytes = kLoraMaxAdapters * R * kLoraK * 2;
  static constexpr int kStageBytes = kXBytes + kABytes;
  static constexpr int kSmemBytes = kLoraStages * kStageBytes + 1024 /*align slack*/ + 64 /*barriers*/;
};

// nA (adapters) is a template parameter: a data-dependent branch between the wgmma issues makes ptxas serialise them
template <int R, int nA>
__global__ void __launch_bounds__(128, 1)
lora_down_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_a,
                 __nv_bfloat16* __restrict__ U, long long ldu, int M, int K, float s, LoraMask mk) {
  using Cfg = LoraDownCfg<R>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kLoraStages * Cfg::kStageBytes);
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
  const int m0 = blockIdx.x * kLoraRows;
  const int nk = (K + kLoraK - 1) / kLoraK;
  const uint32_t tx_bytes = Cfg::kXBytes + nA * R * kLoraK * 2;
  if (tid == 0) {
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_a);
    for (int st = 0; st < kLoraStages; ++st) mbar_init(&full[st], 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto issue = [&](int kb) {
    const int st = kb % kLoraStages;
    uint8_t* base = smem + st * Cfg::kStageBytes;
    mbar_arrive_expect_tx(&full[st], tx_bytes);
    tma_load_4d(base, &tmap_x, &full[st], kb * kLoraK, m0, 0, 0);
#pragma unroll
    for (int j = 0; j < nA; ++j)
      tma_load_4d(base + Cfg::kXBytes + j * R * kLoraK * 2, &tmap_a, &full[st], kb * kLoraK, j * R, 0, 0);
  };
  if (tid == 0) {
    for (int kb = 0; kb < kLoraStages && kb < nk; ++kb) issue(kb);
  }
  // this thread's two rows of the A fragment (rows g and g + 8 of warp w's 16)
  const int r0 = w * 16 + g, r1 = r0 + 8;
  uint32_t rk[nA][2];
#pragma unroll
  for (int j = 0; j < nA; ++j) {
    rk[j][0] = lora_row_key(mk, j, (uint32_t)(m0 + r0));
    rk[j][1] = lora_row_key(mk, j, (uint32_t)(m0 + r1));
  }
  float acc[nA][R / 2];
#pragma unroll
  for (int j = 0; j < nA; ++j)
#pragma unroll
    for (int i = 0; i < R / 2; ++i) acc[j][i] = 0.f;

  for (int kb = 0; kb < nk; ++kb) {
    const int st = kb % kLoraStages;
    mbar_wait(&full[st], (kb / kLoraStages) & 1);
    const uint8_t* xs = smem + st * Cfg::kStageBytes;
    const uint32_t xa = smem_u32(xs);
    // A fragments of the four k16 steps for every adapter: element (row, col) of the swizzled 64 x 64 tile sits at byte
    // row * 128 + ((col / 8) ^ (row % 8)) * 16 + (col % 8) * 2
    uint32_t frag[nA][4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t raw[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int row = (q & 1) ? r1 : r0;
        const int chunk = 2 * kk + (q >> 1);
        const uint32_t addr = xa + row * 128 + ((chunk ^ (row & 7)) << 4) + c * 4;
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(raw[q]) : "r"(addr));
      }
#pragma unroll
      for (int j = 0; j < nA; ++j) {
        if (!mk.on) {
#pragma unroll
          for (int q = 0; q < 4; ++q) frag[j][kk][q] = raw[q];
          continue;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t col = (uint32_t)(kb * kLoraK + kk * 16 + 8 * (q >> 1) + 2 * c);
          const uint32_t key = rk[j][q & 1];
          const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&raw[q]);
          const float2 f = __bfloat1622float2(v);
          frag[j][kk][q] = pack_bf16x2(f.x * lora_mask(mk, key, col), f.y * lora_mask(mk, key, col + 1));
        }
      }
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int j = 0; j < nA; ++j) {
        const uint64_t bd = gmma_desc_sw128(xa + Cfg::kXBytes + j * R * kLoraK * 2) + 2 * kk;
        WgmmaRS<R>::run(acc[j], frag[j][kk], bd);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();  // every thread is done with this stage: it may be refilled
    if (tid == 0 && kb + kLoraStages < nk) issue(kb + kLoraStages);
  }
  // accumulator fragment: element i of this thread is row 16 w + g + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 c + (i & 1)
#pragma unroll
  for (int j = 0; j < nA; ++j) {
#pragma unroll
    for (int i = 0; i < R / 2; i += 2) {
      const int row = m0 + w * 16 + g + 8 * ((i >> 1) & 1);
      const int col = j * R + 8 * (i >> 2) + 2 * c;
      if (row < M)
        *reinterpret_cast<__nv_bfloat162*>(U + (long long)row * ldu + col) = __floats2bfloat162_rn(s * acc[j][i], s * acc[j][i + 1]);
    }
  }
}

// dA_j[k, col] (+)= s * sum_m dU[m, j R + k] * bf16(D_j(m, col) * X[m, col]); CTA = 64 columns of one adapter
template <int R>
__global__ void __launch_bounds__(256)
lora_wgrad_kernel(const __nv_bfloat16* __restrict__ dU, long long ldu, const __nv_bfloat16* __restrict__ X, long long ldx,
                  __nv_bfloat16* __restrict__ dA, int M, int K, float s, int accumulate, LoraMask mk) {
  constexpr int kRows = 32;
  __shared__ float sU[kRows][R];
  __shared__ float sX[kRows][64];
  const int t = threadIdx.x, cc = t & 63, rg = t >> 6;
  const int j = blockIdx.y;
  const int col0 = blockIdx.x * 64;
  float acc[R / 4];
#pragma unroll
  for (int i = 0; i < R / 4; ++i) acc[i] = 0.f;
  for (int m0 = 0; m0 < M; m0 += kRows) {
    for (int e = t; e < kRows * R; e += 256) {
      const int r = e / R, k = e % R;
      sU[r][k] = (m0 + r < M) ? __bfloat162float(dU[(long long)(m0 + r) * ldu + j * R + k]) : 0.f;
    }
#pragma unroll
    for (int q = 0; q < kRows * 64 / 256; ++q) {
      const int e = t + 256 * q, r = e >> 6, c = e & 63;
      const int row = m0 + r, col = col0 + c;
      float v = 0.f;
      if (row < M && col < K) {
        v = __bfloat162float(X[(long long)row * ldx + col]);
        if (mk.on) v = __bfloat162float(__float2bfloat16(v * lora_mask(mk, lora_row_key(mk, j, (uint32_t)row), (uint32_t)col)));
      }
      sX[r][c] = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int m = 0; m < kRows; ++m) {
      const float xv = sX[m][cc];
#pragma unroll
      for (int i = 0; i < R / 4; ++i) acc[i] = fmaf(sU[m][rg + 4 * i], xv, acc[i]);
    }
    __syncthreads();
  }
  const int col = col0 + cc;
  if (col >= K) return;
#pragma unroll
  for (int i = 0; i < R / 4; ++i) {
    __nv_bfloat16* p = dA + (long long)(j * R + rg + 4 * i) * K + col;
    float v = s * acc[i];
    if (accumulate) v += __bfloat162float(*p);
    *p = __float2bfloat16(v);
  }
}

// dX[m, col] += sum_j D_j(m, col) * s * sum_k dU[m, j R + k] A_j[k, col]; CTA = 16 rows x 64 columns
template <int R>
__global__ void __launch_bounds__(256)
lora_dgrad_kernel(const __nv_bfloat16* __restrict__ dU, long long ldu, const __nv_bfloat16* __restrict__ A,
                  __nv_bfloat16* __restrict__ dX, long long ldx, int M, int K, int nA, float s, LoraMask mk) {
  constexpr int kRows = 16;
  __shared__ __nv_bfloat16 sA[kLoraMaxAdapters * R][64];
  __shared__ float sU[kRows][kLoraMaxAdapters * R];
  const int t = threadIdx.x, cc = t & 63, rg = t >> 6;
  const int col0 = blockIdx.x * 64, m0 = blockIdx.y * kRows;
  const int col = col0 + cc;
  for (int e = t; e < nA * R * 64; e += 256) {
    const int k = e >> 6, c = e & 63;
    sA[k][c] = (col0 + c < K) ? A[(long long)k * K + col0 + c] : __float2bfloat16(0.f);
  }
  for (int e = t; e < kRows * nA * R; e += 256) {
    const int r = e / (nA * R), k = e % (nA * R);
    sU[r][k] = (m0 + r < M) ? __bfloat162float(dU[(long long)(m0 + r) * ldu + k]) : 0.f;
  }
  __syncthreads();
  if (col >= K) return;
#pragma unroll 1
  for (int i = 0; i < kRows / 4; ++i) {
    const int r = rg + 4 * i, row = m0 + r;
    if (row >= M) break;
    float out = 0.f;
    for (int j = 0; j < nA; ++j) {
      const float d = mk.on ? lora_mask(mk, lora_row_key(mk, j, (uint32_t)row), (uint32_t)col) : 1.f;
      if (d == 0.f) continue;
      float sum = 0.f;
#pragma unroll
      for (int k = 0; k < R; ++k) sum = fmaf(sU[r][j * R + k], __bfloat162float(sA[j * R + k][cc]), sum);
      out = fmaf(d, s * sum, out);
    }
    __nv_bfloat16* p = dX + (long long)row * ldx + col;
    *p = __float2bfloat16(__bfloat162float(*p) + out);
  }
}

static int lora_check(const u2_lora_desc* d, const char* what) {
  if (!d) return set_error(U2_ERR_ARG, "%s: null descriptor", what);
  if (d->M <= 0 || d->K <= 0) return set_error(U2_ERR_ARG, "%s: M and K must be > 0", what);
  if (d->r != 8 && d->r != 16 && d->r != 32 && d->r != 64) return set_error(U2_ERR_ARG, "%s: r must be 8, 16, 32 or 64 (got %d)", what, d->r);
  if (d->n_adapters < 1 || d->n_adapters > kLoraMaxAdapters) return set_error(U2_ERR_ARG, "%s: 1 to 3 adapters (got %d)", what, d->n_adapters);
  if (!(d->p >= 0.f && d->p < 1.f)) return set_error(U2_ERR_ARG, "%s: dropout probability must lie in [0, 1)", what);
  if (d->ldu < (long long)d->n_adapters * d->r || d->ldx < d->K) return set_error(U2_ERR_ARG, "%s: row strides too small", what);
  return U2_OK;
}

static LoraMask lora_mask_params(const u2_lora_desc* d) {
  LoraMask mk = {};
  const uint32_t lo = (uint32_t)d->seed, hi = (uint32_t)(d->seed >> 32);
  auto fmix = [](uint32_t h) {
    h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
    return h;
  };
  for (int j = 0; j < kLoraMaxAdapters; ++j) mk.key[j] = fmix(lo ^ fmix(hi + (uint32_t)d->stream[j] * 0x9E3779B9u));
  const double thr = floor((double)d->p * 4294967296.0);
  mk.thr = thr >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)thr;
  mk.keep = 1.0f / (1.0f - d->p);
  mk.on = mk.thr != 0;
  return mk;
}

template <int R, int nA>
static int launch_lora_down(const CUtensorMap& tx, const CUtensorMap& ta, void* U, const u2_lora_desc* d, const LoraMask& mk,
                            cudaStream_t s) {
  using Cfg = LoraDownCfg<R>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(lora_down_kernel<R, nA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "lora_down: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  const unsigned grid = (unsigned)((d->M + kLoraRows - 1) / kLoraRows);
  lora_down_kernel<R, nA><<<grid, 128, Cfg::kSmemBytes, s>>>(tx, ta, reinterpret_cast<__nv_bfloat16*>(U), d->ldu, d->M, d->K,
                                                              d->scale, mk);
  U2_CHECK_LAUNCH("lora_down launch");
  return U2_OK;
}

template <int R>
static int launch_lora_down_r(const CUtensorMap& tx, const CUtensorMap& ta, void* U, const u2_lora_desc* d, const LoraMask& mk,
                              cudaStream_t s) {
  switch (d->n_adapters) {
    case 1: return launch_lora_down<R, 1>(tx, ta, U, d, mk, s);
    case 2: return launch_lora_down<R, 2>(tx, ta, U, d, mk, s);
    default: return launch_lora_down<R, 3>(tx, ta, U, d, mk, s);
  }
}

}  // namespace u2

extern "C" U2_API int u2_lora_down_bf16(const void* X, const void* A, void* U, const u2_lora_desc* d, void* stream) {
  using namespace u2;
  int rc = lora_check(d, "lora_down");
  if (rc) return rc;
  if (!X || !A || !U) return set_error(U2_ERR_ARG, "lora_down: null pointer");
  if ((d->ldx & 7) || (d->K & 7)) return set_error(U2_ERR_ARG, "lora_down: K and ldx must be multiples of 8 (16 B, TMA)");
  if ((reinterpret_cast<uintptr_t>(X) & 15) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(U) & 3) ||
      (d->ldu & 1))
    return set_error(U2_ERR_ARG, "lora_down: X / A must be 16-byte aligned, U 4-byte aligned with an even row stride");
  CUtensorMap tx, ta;
  rc = make_tmap_bf16_4d(&tx, X, d->K, d->M, 1, 1, d->ldx, 0, 0, kLoraK, kLoraRows);
  if (rc) return rc;
  rc = make_tmap_bf16_4d(&ta, A, d->K, (int64_t)d->n_adapters * d->r, 1, 1, d->K, 0, 0, kLoraK, d->r);
  if (rc) return rc;
  const LoraMask mk = lora_mask_params(d);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  switch (d->r) {
    case 8: return launch_lora_down_r<8>(tx, ta, U, d, mk, s);
    case 16: return launch_lora_down_r<16>(tx, ta, U, d, mk, s);
    case 32: return launch_lora_down_r<32>(tx, ta, U, d, mk, s);
    default: return launch_lora_down_r<64>(tx, ta, U, d, mk, s);
  }
}

extern "C" U2_API int u2_lora_wgrad_bf16(const void* dU, const void* X, void* dA, const u2_lora_desc* d, void* stream) {
  using namespace u2;
  int rc = lora_check(d, "lora_wgrad");
  if (rc) return rc;
  if (!dU || !X || !dA) return set_error(U2_ERR_ARG, "lora_wgrad: null pointer");
  const LoraMask mk = lora_mask_params(d);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid((unsigned)((d->K + 63) / 64), (unsigned)d->n_adapters);
  const auto* u = reinterpret_cast<const __nv_bfloat16*>(dU);
  const auto* x = reinterpret_cast<const __nv_bfloat16*>(X);
  auto* a = reinterpret_cast<__nv_bfloat16*>(dA);
  switch (d->r) {
    case 8: lora_wgrad_kernel<8><<<grid, 256, 0, s>>>(u, d->ldu, x, d->ldx, a, d->M, d->K, d->scale, d->accumulate, mk); break;
    case 16: lora_wgrad_kernel<16><<<grid, 256, 0, s>>>(u, d->ldu, x, d->ldx, a, d->M, d->K, d->scale, d->accumulate, mk); break;
    case 32: lora_wgrad_kernel<32><<<grid, 256, 0, s>>>(u, d->ldu, x, d->ldx, a, d->M, d->K, d->scale, d->accumulate, mk); break;
    default: lora_wgrad_kernel<64><<<grid, 256, 0, s>>>(u, d->ldu, x, d->ldx, a, d->M, d->K, d->scale, d->accumulate, mk); break;
  }
  U2_CHECK_LAUNCH("lora_wgrad launch");
  return U2_OK;
}

extern "C" U2_API int u2_lora_dgrad_bf16(const void* dU, const void* A, void* dX, const u2_lora_desc* d, void* stream) {
  using namespace u2;
  int rc = lora_check(d, "lora_dgrad");
  if (rc) return rc;
  if (!dU || !A || !dX) return set_error(U2_ERR_ARG, "lora_dgrad: null pointer");
  const LoraMask mk = lora_mask_params(d);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid((unsigned)((d->K + 63) / 64), (unsigned)((d->M + 15) / 16));
  const auto* u = reinterpret_cast<const __nv_bfloat16*>(dU);
  const auto* a = reinterpret_cast<const __nv_bfloat16*>(A);
  auto* x = reinterpret_cast<__nv_bfloat16*>(dX);
  switch (d->r) {
    case 8: lora_dgrad_kernel<8><<<grid, 256, 0, s>>>(u, d->ldu, a, x, d->ldx, d->M, d->K, d->n_adapters, d->scale, mk); break;
    case 16: lora_dgrad_kernel<16><<<grid, 256, 0, s>>>(u, d->ldu, a, x, d->ldx, d->M, d->K, d->n_adapters, d->scale, mk); break;
    case 32: lora_dgrad_kernel<32><<<grid, 256, 0, s>>>(u, d->ldu, a, x, d->ldx, d->M, d->K, d->n_adapters, d->scale, mk); break;
    default: lora_dgrad_kernel<64><<<grid, 256, 0, s>>>(u, d->ldu, a, x, d->ldx, d->M, d->K, d->n_adapters, d->scale, mk); break;
  }
  U2_CHECK_LAUNCH("lora_dgrad launch");
  return U2_OK;
}
