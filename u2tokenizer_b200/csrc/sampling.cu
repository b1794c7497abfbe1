// Sampled decoding head: temperature -> top-k -> top-p (nucleus) -> multinomial draw, one CTA per sequence.
// This is what every eval script of the reference asks HF generate() for (eval/mrg.py:74-75,
// evalscipt/ourmodel_amos.py:76-78: do_sample=True, top_p, temperature; HF's default top_k = 50 applies too).
//
// No sort: the k-th largest logit and the nucleus cut are found by bisection on the logit value (each probe is one
// pass over the V logits held in L2 + a block reduction), then the draw walks the kept tokens in index order.
// HF semantics reproduced: TemperatureLogitsWarper, TopKLogitsWarper (keep the k largest), TopPLogitsWarper
// (keep the smallest set of most-probable tokens whose mass reaches top_p, at least one token).
// The random stream is a counter-based hash (seed, step, row): it cannot equal torch's Philox stream, so parity
// is statistical (tests/test_ops_gpu.py::test_sampling_distribution).
#include <cuda_bf16.h>
#include <math.h>

#include "host_util.h"
#include "u2b200.h"

namespace u2 {

constexpr int kSampThreads = 1024;

__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < kSampThreads / 32; ++w) t += red[w];
  return t;
}

__device__ __forceinline__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = -INFINITY;
  for (int w = 0; w < kSampThreads / 32; ++w) t = fmaxf(t, red[w]);
  return t;
}

__device__ __forceinline__ unsigned int mix32(unsigned int x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}

// kOut: also write the warped scores row (x * inv_temp where kept, -inf elsewhere) into the step-indexed row store
// `scores` (when not null) and the pick's log-prob under the kept distribution into logprob[b] (when not null). The
// draw is the same code in both instantiations, so the ids are bit-identical.
template <bool kOut>
__global__ void __launch_bounds__(kSampThreads)
sample_kernel(const float* __restrict__ logits, long long ld, int V, float inv_temp, int top_k, float top_p,
              unsigned long long seed, const u2_sample_params* __restrict__ pdev, const int* __restrict__ step_dev,
              int step_host, const u2_slot_state* __restrict__ slots, long long* __restrict__ out,
              const u2_row_store_params* __restrict__ scores = nullptr, float* __restrict__ logprob = nullptr) {
  __shared__ float red[kSampThreads / 32];
  __shared__ float s_scan[kSampThreads];
  if (pdev) {
    // parameters live in device memory: a captured CUDA graph keeps replaying while the host changes them
    inv_temp = 1.0f / pdev->temperature;
    top_k = pdev->top_k;
    top_p = pdev->top_p;
    seed = pdev->seed;
  }
  const int b = blockIdx.x;
  if (slots) seed = slots[b].seed;  // continuous batching: the slot's request keys its own stream
  const float* l = logits + (long long)b * ld;
  const int tid = threadIdx.x;
  // contiguous chunk per thread (index order matters for the final walk)
  const int per = (V + kSampThreads - 1) / kSampThreads;
  const int i0 = min(V, tid * per), i1 = min(V, i0 + per);

  float mx = -INFINITY;
  for (int i = i0; i < i1; ++i) mx = fmaxf(mx, l[i] * inv_temp);
  mx = block_max(mx, red);

  // ---- top-k: largest cut `ck` (in scaled-logit units) such that count(x >= ck) >= k
  float cut = -INFINITY;
  if (top_k > 0 && top_k < V) {
    float lo = mx - 60.f, hi = mx;  // anything below mx - 60 has probability < e^-60
    for (int it = 0; it < 32; ++it) {
      const float mid = 0.5f * (lo + hi);
      float c = 0.f;
      for (int i = i0; i < i1; ++i) c += (l[i] * inv_temp >= mid) ? 1.f : 0.f;
      c = block_sum(c, red);
      if (c >= (float)top_k) lo = mid; else hi = mid;
    }
    cut = lo;
  }
  // ---- softmax mass over the top-k survivors
  float z = 0.f;
  for (int i = i0; i < i1; ++i) {
    const float x = l[i] * inv_temp;
    if (x >= cut) z += __expf(x - mx);
  }
  z = block_sum(z, red);
  // ---- top-p: largest cut such that mass(x >= cut) >= top_p * z
  if (top_p < 1.f) {
    float lo = fmaxf(cut, mx - 60.f), hi = mx;
    const float want = top_p * z;
    for (int it = 0; it < 32; ++it) {
      const float mid = 0.5f * (lo + hi);
      float m = 0.f;
      for (int i = i0; i < i1; ++i) {
        const float x = l[i] * inv_temp;
        if (x >= mid) m += __expf(x - mx);
      }
      m = block_sum(m, red);
      if (m >= want) lo = mid; else hi = mid;
    }
    cut = lo;
  }
  if constexpr (kOut) {
    // the warped row, in index-strided order so that a warp's stores are coalesced (the row is L2-resident)
    const long long t = slots ? slots[b].count : step_dev ? *step_dev : step_host;
    if (scores && t >= 0 && t < scores->steps) {
      float* srow = scores->dst + t * scores->ld_step + b * scores->ld_row;
      for (int i = tid; i < V; i += kSampThreads) {
        const float x = l[i] * inv_temp;
        srow[i] = x >= cut ? x : -INFINITY;
      }
    }
  }
  // ---- draw: u * kept mass, then locate it in index order
  float mine = 0.f;
  for (int i = i0; i < i1; ++i) {
    const float x = l[i] * inv_temp;
    if (x >= cut) mine += __expf(x - mx);
  }
  s_scan[tid] = mine;
  __syncthreads();
  if (tid == 0) {
    const int step = slots ? slots[b].count : step_dev ? *step_dev : step_host;
    const int row = slots ? slots[b].row : b;
    unsigned int h = mix32((unsigned int)seed ^ mix32((unsigned int)(seed >> 32) + 0x9e3779b9u * (unsigned int)(step + 1)));
    h = mix32(h ^ (0x85ebca6bu * (unsigned int)(row + 1)));
    const float u = ((h >> 8) + 0.5f) * (1.0f / 16777216.0f);  // (0,1)
    float total = 0.f;
    for (int t = 0; t < kSampThreads; ++t) total += s_scan[t];
    float target = u * total;
    int owner = kSampThreads - 1;
    float acc = 0.f;
    for (int t = 0; t < kSampThreads; ++t) {
      if (acc + s_scan[t] >= target && s_scan[t] > 0.f) { owner = t; break; }
      acc += s_scan[t];
    }
    // walk the owner's chunk
    const int j0 = min(V, owner * per), j1 = min(V, j0 + per);
    long long pick = -1;
    long long last_kept = -1;
    for (int i = j0; i < j1; ++i) {
      const float x = l[i] * inv_temp;
      if (x >= cut) {
        last_kept = i;
        acc += __expf(x - mx);
        if (acc >= target) { pick = i; break; }
      }
    }
    if (pick < 0) pick = last_kept >= 0 ? last_kept : 0;
    out[b] = pick;
    if constexpr (kOut) {
      if (logprob) logprob[b] = (l[pick] * inv_temp - mx) - logf(total);
    }
  }
}

}  // namespace u2

extern "C" U2_API int u2_sample_f32(const float* logits, int64_t* out, int32_t B, int32_t V, int64_t ld,
                                    float temperature, int32_t top_k, float top_p, uint64_t seed,
                                    const int32_t* step_dev, int32_t step, void* stream) {
  using namespace u2;
  if (!logits || !out) return set_error(U2_ERR_ARG, "sample: null pointer");
  if (B <= 0 || V <= 0) return U2_OK;
  if (!(temperature > 0.f)) return set_error(U2_ERR_ARG, "sample: temperature must be > 0");
  if (!(top_p > 0.f) || top_p > 1.f) return set_error(U2_ERR_ARG, "sample: top_p must be in (0, 1]");
  sample_kernel<false><<<B, kSampThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, ld, V, 1.0f / temperature, top_k, top_p, seed, nullptr, step_dev, step, nullptr,
      reinterpret_cast<long long*>(out));
  U2_CHECK_LAUNCH("sample");
  return U2_OK;
}

extern "C" U2_API int u2_sample_dev_f32(const float* logits, int64_t* out, int32_t B, int32_t V, int64_t ld,
                                        const u2_sample_params* params_dev, const int32_t* step_dev, int32_t step,
                                        void* stream) {
  using namespace u2;
  if (!logits || !out || !params_dev) return set_error(U2_ERR_ARG, "sample_dev: null pointer");
  if (B <= 0 || V <= 0) return U2_OK;
  sample_kernel<false><<<B, kSampThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, ld, V, 1.0f, 0, 1.0f, 0ull, params_dev, step_dev, step, nullptr, reinterpret_cast<long long*>(out));
  U2_CHECK_LAUNCH("sample_dev");
  return U2_OK;
}

extern "C" U2_API int u2_sample_slots_f32(const float* logits, int64_t* out, int32_t B, int32_t V, int64_t ld,
                                          const u2_sample_params* params_dev, const u2_slot_state* slots, void* stream) {
  using namespace u2;
  if (!logits || !out || !params_dev || !slots) return set_error(U2_ERR_ARG, "sample_slots: null pointer");
  if (B <= 0 || V <= 0) return U2_OK;
  sample_kernel<false><<<B, kSampThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, ld, V, 1.0f, 0, 1.0f, 0ull, params_dev, nullptr, 0, slots, reinterpret_cast<long long*>(out));
  U2_CHECK_LAUNCH("sample_slots");
  return U2_OK;
}

extern "C" U2_API int u2_sample_out_f32(const float* logits, int64_t* out, int32_t B, int32_t V, int64_t ld,
                                        const u2_sample_params* params_dev, const int32_t* step_dev, int32_t step,
                                        const u2_slot_state* slots, const u2_row_store_params* scores_dev,
                                        float* logprob, void* stream) {
  using namespace u2;
  if (!logits || !out || !params_dev) return set_error(U2_ERR_ARG, "sample_out: null pointer");
  if (slots && step_dev) return set_error(U2_ERR_ARG, "sample_out: the step comes from slots or step_dev, not both");
  if (B <= 0 || V <= 0) return U2_OK;
  sample_kernel<true><<<B, kSampThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, ld, V, 1.0f, 0, 1.0f, 0ull, params_dev, step_dev, step, slots, reinterpret_cast<long long*>(out),
      scores_dev, logprob);
  U2_CHECK_LAUNCH("sample_out");
  return U2_OK;
}
