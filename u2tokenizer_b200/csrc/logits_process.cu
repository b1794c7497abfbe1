// HF generate() logits processors, applied in place to the fp32 logits of a decode step before the argmax / sampler
// (transformers generation/logits_process.py, in the order _get_logits_processor builds them):
//   RepetitionPenaltyLogitsProcessor -> NoRepeatNGramLogitsProcessor -> NoBadWordsLogitsProcessor ->
//   MinLengthLogitsProcessor / MinNewTokensLengthLogitsProcessor.
// One CTA per sequence. The history is the generated tokens only (HF starts input_ids as [B, 0] when generate() gets
// inputs_embeds), so every row has the same history length: *step_dev (or step) tokens, the last of which is the token
// fed to this step (ids[b]). The kernel appends it to hist[b] first, so a captured decode step keeps its own history.
#include <cuda_runtime.h>
#include <math.h>

#include "host_util.h"
#include "u2b200.h"

namespace u2 {

constexpr int kLpThreads = 1024;

__global__ void __launch_bounds__(kLpThreads)
logits_process_kernel(float* __restrict__ logits, long long ld, int V, const long long* __restrict__ ids,
                      int* __restrict__ hist, long long ldh, int hist_cap, const u2_logits_proc_params* __restrict__ p,
                      const int* __restrict__ step_dev, int step_host, const u2_slot_state* __restrict__ slots) {
  extern __shared__ unsigned int s_seen[];  // one bit per vocabulary entry
  const int b = blockIdx.x;
  float* l = logits + (long long)b * ld;
  int* h = hist + (long long)b * ldh;
  // history length; continuous batching: the slot's own generated count
  const int t = min(slots ? slots[b].count : step_dev ? *step_dev : step_host, hist_cap);
  const int cur = t > 0 ? (int)ids[b] : 0;
  if (threadIdx.x == 0 && t > 0) h[t - 1] = cur;
  // slot t - 1 is read from `cur`, never from memory thread 0 is writing
  auto tok = [&](int i) { return i == t - 1 ? cur : h[i]; };

  // ---- repetition penalty, once per distinct token, from its unprocessed logit (HF: gather -> where -> scatter)
  const float pen = p->penalty;
  if (pen != 1.0f && t > 0) {
    const int nw = (V + 31) >> 5;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) s_seen[i] = 0u;
    __syncthreads();
    for (int i = threadIdx.x; i < t; i += blockDim.x) {
      const int v = tok(i);
      atomicOr(&s_seen[v >> 5], 1u << (v & 31));
    }
    __syncthreads();
    // `scores / penalty` with a Python float on a CUDA tensor is computed by torch as scores * (1.0f / float(penalty))
    // (div_true_kernel_cuda, CPU-scalar branch); inv_penalty holds that fp32 reciprocal, rounded on the host
    const float inv = p->inv_penalty;
    for (int i = threadIdx.x; i < t; i += blockDim.x) {
      const int v = tok(i);
      const unsigned int m = 1u << (v & 31);
      if (atomicAnd(&s_seen[v >> 5], ~m) & m) {  // the first slot to clear the bit owns the token
        const float x = l[v];
        l[v] = x < 0.f ? x * pen : x * inv;
      }
    }
  }
  const int nb = p->n_bad;
  if (nb > 0) {
    // HF adds a bias row (0 or -inf) to every score: x + 0.0f turns -0.0 into +0.0, everything else keeps its bits
    __syncthreads();
    if ((ld & 3) == 0 && (reinterpret_cast<size_t>(logits) & 15) == 0) {
      float4* l4 = reinterpret_cast<float4*>(l);
      const int n4 = V >> 2;
#pragma unroll 4
      for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        float4 x = l4[i];
        if (__float_as_uint(x.x) == 0x80000000u || __float_as_uint(x.y) == 0x80000000u ||
            __float_as_uint(x.z) == 0x80000000u || __float_as_uint(x.w) == 0x80000000u) {
          x.x += 0.f; x.y += 0.f; x.z += 0.f; x.w += 0.f;
          l4[i] = x;
        }
      }
      for (int i = (n4 << 2) + threadIdx.x; i < V; i += blockDim.x) l[i] += 0.f;
    } else {
      for (int i = threadIdx.x; i < V; i += blockDim.x) l[i] += 0.f;
    }
  }
  __syncthreads();  // every value the penalty or the bias rewrites is final before any -inf lands

  // ---- no_repeat_ngram_size n: one thread per earlier n-gram start i; its last token is banned when its first n - 1
  // tokens equal the last n - 1 generated ones (HF _calc_banned_ngram_tokens)
  const int n = p->ngram;
  if (n > 0 && t >= n) {
    for (int i = threadIdx.x; i + n <= t; i += blockDim.x) {
      bool match = true;
      for (int j = 0; j < n - 1 && match; ++j) match = tok(i + j) == tok(t - n + 1 + j);
      if (match) l[tok(i + n - 1)] = -INFINITY;
    }
  }
  // ---- bad words: a single token always, a longer word when its prefix ends the history (SequenceBias with -inf;
  // words longer than the history are skipped, as HF skips them)
  for (int w = threadIdx.x; w < nb; w += blockDim.x) {
    const int o0 = p->bad_off[w], o1 = p->bad_off[w + 1], len = o1 - o0;
    bool hit = len == 1;
    if (len > 1 && len <= t) {
      hit = true;
      for (int j = 0; j < len - 1 && hit; ++j) hit = p->bad_tok[o0 + j] == tok(t - len + 1 + j);
    }
    if (hit) l[p->bad_tok[o1 - 1]] = -INFINITY;
  }
  // ---- min_new_tokens: every EOS id is banned while fewer than min_new tokens have been generated
  if (t < p->min_new && (int)threadIdx.x < p->n_eos) l[p->eos[threadIdx.x]] = -INFINITY;
}

}  // namespace u2

static int logits_process_launch(float* logits, int32_t B, int32_t V, int64_t ld, const int64_t* ids, int32_t* hist,
                                 int64_t ld_hist, int32_t hist_cap, const u2_logits_proc_params* params_dev,
                                 const int32_t* step_dev, int32_t step, const u2_slot_state* slots, void* stream) {
  using namespace u2;
  if (!logits || !ids || !hist || !params_dev) return set_error(U2_ERR_ARG, "logits_process: null pointer");
  if (B <= 0 || V <= 0) return U2_OK;
  if (ld < V || ld_hist < hist_cap || hist_cap < 0 || step < 0)
    return set_error(U2_ERR_ARG, "logits_process: bad strides, history capacity or step");
  const size_t smem = (size_t)((V + 31) / 32) * sizeof(unsigned int);
  if (smem > 227 * 1024) return set_error(U2_ERR_ARG, "logits_process: vocabulary too large for the presence bitmap");
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(logits_process_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_error(U2_ERR_CUDA, "logits_process: cudaFuncSetAttribute failed");
  }
  logits_process_kernel<<<B, kLpThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, ld, V, reinterpret_cast<const long long*>(ids), hist, ld_hist, hist_cap, params_dev, step_dev, step, slots);
  U2_CHECK_LAUNCH("logits_process");
  return U2_OK;
}

extern "C" U2_API int u2_logits_process_f32(float* logits, int32_t B, int32_t V, int64_t ld, const int64_t* ids,
                                            int32_t* hist, int64_t ld_hist, int32_t hist_cap,
                                            const u2_logits_proc_params* params_dev, const int32_t* step_dev,
                                            int32_t step, void* stream) {
  return logits_process_launch(logits, B, V, ld, ids, hist, ld_hist, hist_cap, params_dev, step_dev, step, nullptr,
                               stream);
}

extern "C" U2_API int u2_logits_process_slots_f32(float* logits, int32_t B, int32_t V, int64_t ld, const int64_t* ids,
                                                  int32_t* hist, int64_t ld_hist, int32_t hist_cap,
                                                  const u2_logits_proc_params* params_dev, const u2_slot_state* slots,
                                                  void* stream) {
  if (!slots) return u2::set_error(U2_ERR_ARG, "logits_process_slots: null pointer");
  return logits_process_launch(logits, B, V, ld, ids, hist, ld_hist, hist_cap, params_dev, nullptr, 0, slots, stream);
}
