// Fused (flash-style) attention forward on wgmma for head_dim 64, non-causal - the ViT3D tower's attention
// (12 heads, S = 2049 tokens per frame): O = softmax(Q K^T * scale) V without materialising the S x S scores.
//
// One CTA owns a 128-row query tile of one (frame, head) and walks the keys in tiles of 128:
//   warp 0      : TMA producer  Q once, then (K_j, V_j) into a 2-deep ring
//   warps 4-7   : consumer warpgroup 0, query rows 0..63 of the tile
//   warps 8-11  : consumer warpgroup 1, query rows 64..127
// A consumer warpgroup keeps everything in registers: S_j = Q K_j^T (64 x 128, fp32 wgmma fragment), the online
// max / sum in the log2 domain (a row lives in the four lanes of a quad), P_j converted in place into the bf16 A
// fragment of the PV product (wgmma with A from registers), and the running O (64 x 64 fp32).
// Q / K / V are 4-D TMA views of the fused QKV activation ([frame, token, 3, head, d]). V is consumed AS STORED: a
// {64 d, 128 keys} box with the 128-byte swizzle is the canonical MN-major wgmma B operand (one 64-wide N chunk,
// groups of 8 key rows 1024 B apart), so the PV product needs no transposed copy of V.
//
// Replaces MONAI SABlock's einsum / softmax / einsum (reference call site src/model/multimodal_encoder/vit.py:
// 100-105,120-122), which materialises a [frames*12, 2049, 2049] fp32 score tensor per block.
#include <cuda_bf16.h>
#include <math.h>
#include <stdlib.h>

#include "host_util.h"
#include "ptx.cuh"
#include "u2b200.h"

namespace u2 {

constexpr int kFaDh = 64;
constexpr int kFaBM = 128;   // query rows per CTA (64 per consumer warpgroup)
constexpr int kFaBN = 128;   // keys per tile
constexpr int kFaThreads = 384;
constexpr int kFaQBytes = kFaBM * kFaDh * 2;          // 16 KB
constexpr int kFaKBytes = kFaBN * kFaDh * 2;          // 16 KB
constexpr int kFaVBytes = kFaBN * kFaDh * 2;          // 16 KB (128 key rows of 128 B)
constexpr int kFaSmem = kFaQBytes + 2 * kFaKBytes + 2 * kFaVBytes + 1024 + 256;

struct FaArgs {
  int Sq, Sk;              // valid query rows / keys per (batch, head)
  float scale_log2e;       // softmax scale * log2(e)
  __nv_bfloat16* out;      // [b][s][h*64 + d]
  long long out_sb, out_ss;  // element strides of batch and token
  float* lse;              // optional [b][h][Sq]: log-sum-exp of the scaled scores (the attention backward rebuilds P from it)
  int H;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(kFaThreads, 1)
fa_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                    const __grid_constant__ CUtensorMap tmap_v, const FaArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kFaQBytes;            // [2]
  uint8_t* sV = sK + 2 * kFaKBytes;        // [2]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * kFaVBytes);
  uint64_t* q_full = bars;          // 1
  uint64_t* kv_full = bars + 1;     // 2
  uint64_t* kv_empty = bars + 3;    // 2

  const int warp_idx = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = blockIdx.x * kFaBM;
  const int J = (p.Sk + kFaBN - 1) / kFaBN;

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
  }
  if (warp_idx == 1 && lane == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp_idx == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, kFaQBytes);
      tma_load_4d(sQ, &tmap_q, q_full, 0, q0, h, b);
      for (int j = 0; j < J; ++j) {
        const int buf = j & 1, n = j >> 1;
        mbar_wait(&kv_empty[buf], (n & 1) ^ 1);
        mbar_arrive_expect_tx(&kv_full[buf], kFaKBytes + kFaVBytes);
        tma_load_4d(sK + buf * kFaKBytes, &tmap_k, &kv_full[buf], 0, j * kFaBN, h, b);
        tma_load_4d(sV + buf * kFaVBytes, &tmap_v, &kv_full[buf], 0, j * kFaBN, h, b);
      }
    }
  } else if (warp_idx >= 4) {
    // ===================== consumer warpgroups =====================
    const int cg = (warp_idx - 4) >> 2;  // query rows 64 cg .. 64 cg + 63 of the tile
    const int w = (warp_idx - 4) & 3;
    const int quad = lane & 3;
    // this thread's rows (fragment rows r and r + 8 of its warp's 16) and the key / d columns it holds:
    // element 4 i + e of a fragment sits at row r + 8 (e >> 1), column 8 i + 2 quad + (e & 1)
    const int r_lo = q0 + cg * 64 + w * 16 + (lane >> 2);
    const uint64_t q_desc = gmma_desc_sw128(smem_u32(sQ + cg * (kFaQBytes / 2)));
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // l: this thread's partial row sums
    mbar_wait(q_full, 0);
    for (int j = 0; j < J; ++j) {
      const int buf = j & 1, n = j >> 1;
      const int nk = min(kFaBN, p.Sk - j * kFaBN);  // valid keys in this tile
      mbar_wait(&kv_full[buf], n & 1);
      // ---- S = Q K^T: 64 x 128 as two 64-key chunks (K rows 64..127 start 8 KB further)
      float s[64];
      const uint64_t k_desc = gmma_desc_sw128(smem_u32(sK + buf * kFaKBytes));
      float (&s0)[32] = *reinterpret_cast<float(*)[32]>(s);
      float (&s1)[32] = *reinterpret_cast<float(*)[32]>(s + 32);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kFaDh / 16; ++k) {
        wgmma_m64n64k16_ss<0, 0>(s0, q_desc + 2 * k, k_desc + 2 * k, k != 0);
        wgmma_m64n64k16_ss<0, 0>(s1, q_desc + 2 * k, k_desc + 512 + 2 * k, k != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // ---- online softmax (log2 domain); keys past Sk (zero-filled by TMA) do not take part
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = 8 * i + 2 * quad + (e & 1);
          if (key >= nk) s[4 * i + e] = -INFINITY;
          mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * i + e]);
        }
      }
      float alpha[2], mnew[2];
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 1));
        mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 2));
        mnew[hr] = fmaxf(m[hr], mx[hr] * p.scale_log2e);
        alpha[hr] = ex2_approx(m[hr] - mnew[hr]);  // m == -inf on the first tile -> 0
        m[hr] = mnew[hr];
      }
      float rs[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const float e = ex2_approx(s[i] * p.scale_log2e - mnew[(i >> 1) & 1]);  // -inf -> 0
        s[i] = e;
        rs[(i >> 1) & 1] += e;
      }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) l[hr] = l[hr] * alpha[hr] + rs[hr];
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
      // ---- O += P V: P (bf16) straight from the S fragment as the register A operand, V MN-major (16 keys per
      //      step = two 1024-byte groups of 8 key rows)
      const uint64_t v_desc = gmma_desc_sw128(smem_u32(sV + buf * kFaVBytes), kFaVBytes);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kFaBN / 16; ++kk) {
        const uint32_t a[4] = {pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                               pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
        wgmma_m64n64k16_rs<1>(o, a, v_desc + 128 * kk);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&kv_empty[buf]);
    }
    // ---- normalise, store
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      l[hr] += __shfl_xor_sync(0xffffffffu, l[hr], 1);
      l[hr] += __shfl_xor_sync(0xffffffffu, l[hr], 2);
      const int row = r_lo + 8 * hr;
      if (row < p.Sq) {
        const float inv = 1.f / l[hr];
        if (p.lse && quad == 0) p.lse[((long long)b * p.H + h) * p.Sq + row] = (m[hr] + log2f(l[hr])) * 0.6931471805599453f;
        __nv_bfloat16* dst = p.out + (long long)b * p.out_sb + (long long)row * p.out_ss + h * kFaDh + 2 * quad;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          *reinterpret_cast<__nv_bfloat162*>(dst + 8 * i) =
              __floats2bfloat162_rn(o[4 * i + 2 * hr] * inv, o[4 * i + 2 * hr + 1] * inv);
      }
    }
  }
}

}  // namespace u2

extern "C" U2_API int u2_flash_attention_d64_bf16(const void* q, const void* k, const void* v, void* out,
                                                  const u2_fa_desc* d, void* stream) {
  using namespace u2;
  if (!q || !k || !v || !out || !d) return set_error(U2_ERR_ARG, "flash_attention: null pointer");
  if (d->dh != kFaDh) return set_error(U2_ERR_UNSUPPORTED, "flash_attention: head_dim %d (this kernel: 64)", d->dh);
  if (d->B <= 0 || d->H <= 0 || d->Sq <= 0 || d->Sk <= 0) return set_error(U2_ERR_ARG, "flash_attention: bad extents");
  if (d->B > 65535 || d->H > 65535) return set_error(U2_ERR_ARG, "flash_attention: B, H must be <= 65535");
  if ((d->q_ss & 7) || (d->q_sh & 7) || (d->q_sb & 7) || (d->k_ss & 7) || (d->k_sh & 7) || (d->k_sb & 7) || (d->v_ss & 7) ||
      (d->v_sh & 7) || (d->v_sb & 7) || (d->out_ss & 7))
    return set_error(U2_ERR_ARG, "flash_attention: strides must be multiples of 8 elements");
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(fa_fwd_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFaSmem);
    if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "flash_attention: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  CUtensorMap tq, tk, tv;
  int rc = make_tmap_bf16_4d(&tq, q, kFaDh, d->Sq, d->H, d->B, d->q_ss, d->q_sh, d->q_sb, kFaDh, kFaBM);
  if (rc) return rc;
  rc = make_tmap_bf16_4d(&tk, k, kFaDh, d->Sk, d->H, d->B, d->k_ss, d->k_sh, d->k_sb, kFaDh, kFaBN);
  if (rc) return rc;
  // V as stored: dims {d, token, head, batch}, box {64 d, 128 keys} = the MN-major B operand of the PV product
  rc = make_tmap_bf16_4d(&tv, v, kFaDh, d->Sk, d->H, d->B, d->v_ss, d->v_sh, d->v_sb, kFaDh, kFaBN);
  if (rc) return rc;
  FaArgs a;
  a.Sq = d->Sq; a.Sk = d->Sk;
  a.scale_log2e = d->scale * 1.4426950408889634f;
  a.out = reinterpret_cast<__nv_bfloat16*>(out);
  a.out_sb = d->out_sb; a.out_ss = d->out_ss;
  a.lse = d->lse; a.H = d->H;
  dim3 grid((unsigned)((d->Sq + kFaBM - 1) / kFaBM), (unsigned)d->H, (unsigned)d->B);
  fa_fwd_wgmma_kernel<<<grid, kFaThreads, kFaSmem, reinterpret_cast<cudaStream_t>(stream)>>>(tq, tk, tv, a);
  U2_CHECK_LAUNCH("flash_attention");
  return U2_OK;
}
