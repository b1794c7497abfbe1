// Beam search inside the captured decode step: HF GenerationMixin._beam_search (transformers generation/utils.py) with
// the prompt length 0 of generate(inputs_embeds=...), so every length below counts generated tokens only.
//   u2_log_softmax_f32   log_probs = log_softmax(logits) into a separate buffer (the logits processors then run on it)
//   u2_beam_topk_f32     one CTA per row: the top C = beams_to_keep of log_prob + running_score[row] (radix select).
//                        A prompt's top C over its K * V continuations is a subset of the union of its rows' top C
//   u2_beam_step         one CTA per prompt: merge the K * C row candidates, then the bookkeeping of
//                        _get_top_k_continuations / _get_running_beams_for_next_iteration / _update_finished_beams /
//                        _check_early_stop_heuristic, and the reorder of the KV-cache indirection table and history
// Ties among equal scores go to the lower flat index (beam * V + token), as in u2_topk_rows_f32.
#include <cuda_runtime.h>
#include <math.h>

#include "host_util.h"
#include "u2b200.h"

namespace u2 {

constexpr int kBsThreads = 1024;
constexpr float kBig = -1.0e9f;  // HF's -1e9 masks (exact in fp32)

__device__ __forceinline__ unsigned int order_key(float f) {  // larger float -> larger key
  const unsigned int u = __float_as_uint(f);
  if (f != f) return 0u;  // NaN sorts last
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, w) : v + w;
  }
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < (int)(blockDim.x >> 5) ? s_red[lane] : (is_max ? -INFINITY : 0.f);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float w = __shfl_xor_sync(0xffffffffu, v, o);
      v = is_max ? fmaxf(v, w) : v + w;
    }
    if (lane == 0) s_red[32] = v;
  }
  __syncthreads();
  return s_red[32];
}

// y = x - max - log(sum exp(x - max)), as torch's log_softmax computes it on CUDA
__global__ void __launch_bounds__(kBsThreads)
log_softmax_kernel(const float* __restrict__ x, float* __restrict__ y, int V, long long ldx, long long ldy) {
  __shared__ float s_red[33];
  const float* xr = x + (long long)blockIdx.x * ldx;
  float* yr = y + (long long)blockIdx.x * ldy;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < V; i += blockDim.x) m = fmaxf(m, xr[i]);
  m = block_reduce(m, true, s_red);
  float s = 0.f;
  for (int i = threadIdx.x; i < V; i += blockDim.x) s += expf(xr[i] - m);
  s = block_reduce(s, false, s_red);
  const float ls = logf(s);
  for (int i = threadIdx.x; i < V; i += blockDim.x) yr[i] = xr[i] - m - ls;
}

// ---- per-row top C of lp[v] + running[row] by radix select on the order-preserving 32-bit key ----
__global__ void __launch_bounds__(kBsThreads)
beam_topk_kernel(const float* __restrict__ lp, long long ld, int V, const float* __restrict__ running,
                 const int* __restrict__ state_flags, const u2_beam_params* __restrict__ p, float* __restrict__ cand_val,
                 int* __restrict__ cand_tok) {
  __shared__ unsigned int s_hist[256];
  __shared__ unsigned int s_prefix, s_mask, s_remaining, s_eq, s_n;
  __shared__ unsigned int s_warp[32];
  __shared__ unsigned int s_key[U2_BEAM_MAX_KEEP];
  __shared__ int s_tok[U2_BEAM_MAX_KEEP];
  const int row = blockIdx.x;
  const int K = p->num_beams, C = p->beams_to_keep;
  if (state_flags[2 * (row / K) + 1]) return;  // the prompt is done: frozen
  const float* x = lp + (long long)row * ld;
  const float sc = running[row];
  const int tid = threadIdx.x;
  if (tid == 0) {
    s_prefix = 0u;
    s_mask = 0u;
    s_remaining = (unsigned int)C;
    s_n = 0u;
  }
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += blockDim.x) s_hist[i] = 0u;
    __syncthreads();
    const unsigned int prefix = s_prefix, mask = s_mask;
    for (int v = tid; v < V; v += blockDim.x) {
      const unsigned int k = order_key(__fadd_rn(x[v], sc));
      const bool in = (k & mask) == prefix;
      const unsigned int bin = in ? (k >> shift) & 255u : 256u + (threadIdx.x & 31);
      // aggregate equal bins within the warp: the high digits of nearby log-probs coincide
      const unsigned int peers = __match_any_sync(__activemask(), bin);
      if (in && (__ffs(peers) - 1) == (threadIdx.x & 31)) atomicAdd(&s_hist[bin], (unsigned int)__popc(peers));
    }
    __syncthreads();
    if (tid == 0) {
      unsigned int rem = s_remaining, cum = 0u;
      int bin = 255;
      for (; bin > 0; --bin) {
        if (cum + s_hist[bin] >= rem) break;
        cum += s_hist[bin];
      }
      s_remaining = rem - cum;
      s_prefix = prefix | ((unsigned int)bin << shift);
      s_mask = mask | (255u << shift);
      s_eq = s_hist[bin];
    }
    __syncthreads();
  }
  const unsigned int thr = s_prefix;
  const unsigned int need_eq = s_remaining;  // keys == thr to take, lowest token first
  const bool all_eq = s_eq <= need_eq;
  for (int v = tid; v < V; v += blockDim.x) {
    const unsigned int k = order_key(__fadd_rn(x[v], sc));
    if (k > thr || (k == thr && all_eq)) {
      const unsigned int slot = atomicAdd(&s_n, 1u);
      s_key[slot] = k;
      s_tok[slot] = v;
    }
  }
  __syncthreads();
  if (!all_eq) {  // more ties at the threshold than places: take them in token order
    unsigned int left = need_eq;
    const int lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    for (int v0 = 0; v0 < V && left > 0; v0 += blockDim.x) {
      const int v = v0 + tid;
      const bool eq = v < V && order_key(__fadd_rn(x[v], sc)) == thr;
      const unsigned int bal = __ballot_sync(0xffffffffu, eq);
      if (lane == 0) s_warp[warp] = __popc(bal);
      __syncthreads();
      unsigned int base = 0u, total = 0u;
      for (int w = 0; w < nw; ++w) {
        if (w < warp) base += s_warp[w];
        total += s_warp[w];
      }
      const unsigned int rank = base + __popc(bal & ((1u << lane) - 1u));
      if (eq && rank < left) {
        const unsigned int slot = (unsigned int)C - left + rank;
        s_key[slot] = thr;
        s_tok[slot] = v;
      }
      left = total >= left ? 0u : left - total;
      __syncthreads();
    }
  }
  __syncthreads();
  // rank sort of the C picks: score descending, token ascending
  for (int i = tid; i < C; i += blockDim.x) {
    const unsigned int ki = s_key[i];
    const int ti = s_tok[i];
    int r = 0;
    for (int j = 0; j < C; ++j) r += (s_key[j] > ki) || (s_key[j] == ki && s_tok[j] < ti);
    cand_val[(long long)row * U2_BEAM_MAX_KEEP + r] = __fadd_rn(x[ti], sc);
    cand_tok[(long long)row * U2_BEAM_MAX_KEEP + r] = ti;
  }
}

__device__ __forceinline__ bool better(float va, int ia, float vb, int ib) {
  return va > vb || (va == vb && ia < ib);
}

// fp32 `x / (n ** length_penalty)` as torch evaluates a CUDA tensor divided by a Python float: x * (1.0f / float(p))
__device__ __forceinline__ float lp_inv(double n, double length_penalty) {
  return 1.0f / (float)pow(n, length_penalty);
}

constexpr int kMergeThreads = 256;

__global__ void __launch_bounds__(kMergeThreads)
beam_step_kernel(const u2_beam_step_desc d, int step_host) {
  __shared__ float s_cv[U2_BEAM_MAX_BEAMS * U2_BEAM_MAX_KEEP];
  __shared__ int s_cf[U2_BEAM_MAX_BEAMS * U2_BEAM_MAX_KEEP];
  __shared__ float s_val[U2_BEAM_MAX_KEEP];       // the prompt's top C, sorted
  __shared__ int s_flat[U2_BEAM_MAX_KEEP];
  __shared__ float s_mv[U2_BEAM_MAX_BEAMS + U2_BEAM_MAX_KEEP];  // merged finished candidates
  __shared__ int s_minfo[U2_BEAM_MAX_BEAMS + U2_BEAM_MAX_KEEP][4];
  __shared__ int s_parent[U2_BEAM_MAX_BEAMS];
  __shared__ float s_newfin[U2_BEAM_MAX_BEAMS];
  __shared__ int s_newdone[U2_BEAM_MAX_BEAMS];
  __shared__ float s_pen[U2_BEAM_MAX_KEEP];
  __shared__ int s_hit[U2_BEAM_MAX_KEEP];
  __shared__ int s_nhit;
  const u2_beam_params* p = d.params;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int K = p->num_beams, C = p->beams_to_keep, V = d.V;
  int* flags = d.flags + 2 * b;  // [heuristic unsatisfied, done]
  if (flags[1]) return;  // frozen until the host sees it
  const int t = d.step_dev ? *d.step_dev : step_host;  // tokens generated before this one
  const int r0 = b * K;
  // ---- 1. merge the K row lists into the prompt's top C (rank by binary search in the other sorted lists)
  const int n = K * C;
  for (int i = tid; i < n; i += blockDim.x) {
    const int k = i / C, j = i - k * C;
    s_cv[i] = d.cand_val[(long long)(r0 + k) * U2_BEAM_MAX_KEEP + j];
    s_cf[i] = k * V + d.cand_tok[(long long)(r0 + k) * U2_BEAM_MAX_KEEP + j];
  }
  if (tid == 0) s_nhit = 0;
  __syncthreads();
  for (int i = tid; i < n; i += blockDim.x) {
    const int k = i / C;
    const float v = s_cv[i];
    const int f = s_cf[i];
    int r = i - k * C;
    for (int k2 = 0; k2 < K && r < C; ++k2) {
      if (k2 == k) continue;
      int lo = 0, hi = C;  // first entry of list k2 that is not better than (v, f)
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (better(s_cv[k2 * C + mid], s_cf[k2 * C + mid], v, f)) lo = mid + 1; else hi = mid;
      }
      r += lo;
    }
    if (r < C) {
      s_val[r] = v;
      s_flat[r] = f;
    }
  }
  __syncthreads();
  // ---- 2. stopping criteria, next running beams (hits get -1e9 first), finished candidates
  const int max_new = p->max_new_tokens;
  for (int i = tid; i < C; i += blockDim.x) {
    const int tok = s_flat[i] % V;
    bool hit = t + 1 >= max_new;
    for (int e = 0; e < p->n_eos; ++e) hit = hit || tok == p->eos[e];
    s_hit[i] = hit;
    s_pen[i] = __fadd_rn(s_val[i], hit ? kBig : 0.f);
    if (hit) atomicAdd(&s_nhit, 1);
  }
  __syncthreads();
  const float inv_len = lp_inv((double)(t + 1), p->length_penalty);
  bool full = p->early_stopping == 1;
  for (int k = 0; k < K; ++k) full = full && d.fin_info[4 * (r0 + k)] != 0;
  const bool unsat = flags[0] != 0;
  for (int i = tid; i < C; i += blockDim.x) {
    const int tok = s_flat[i] % V, beam = s_flat[i] / V;
    const float pen = s_pen[i];
    int r = 0;
    for (int j = 0; j < C; ++j) r += better(s_pen[j], j, pen, i);
    if (r < K) {
      s_parent[r] = beam;
      d.running[r0 + r] = pen;
      d.ids[r0 + r] = tok;
      if (t < d.rec_rows) {
        d.rec[(long long)t * d.ld_rec + 2 * (r0 + r)] = tok;
        d.rec[(long long)t * d.ld_rec + 2 * (r0 + r) + 1] = beam;
      }
    }
    const bool did = s_hit[i] && i < K;
    float s = s_val[i] * inv_len;
    s = __fadd_rn(s, full ? kBig : 0.f);
    s = __fadd_rn(s, unsat ? 0.f : kBig);
    s = __fadd_rn(s, did ? 0.f : kBig);
    s_mv[K + i] = s;
    s_minfo[K + i][0] = did;
    s_minfo[K + i][1] = t;
    s_minfo[K + i][2] = beam;
    s_minfo[K + i][3] = tok;
  }
  for (int k = tid; k < K; k += blockDim.x) {
    s_mv[k] = d.fin_score[r0 + k];
#pragma unroll
    for (int q = 0; q < 4; ++q) s_minfo[k][q] = d.fin_info[4 * (r0 + k) + q];
  }
  __syncthreads();
  // ---- 3. the best K of (old finished, new candidates), old first on ties
  const int m = K + C;
  for (int i = tid; i < m; i += blockDim.x) {
    const float v = s_mv[i];
    int r = 0;
    for (int j = 0; j < m; ++j) r += better(s_mv[j], j, v, i);
    if (r < K) {
      d.fin_score[r0 + r] = v;
      s_newfin[r] = v;
      s_newdone[r] = s_minfo[i][0];
#pragma unroll
      for (int q = 0; q < 4; ++q) d.fin_info[4 * (r0 + r) + q] = s_minfo[i][q];
    }
  }
  __syncthreads();
  // ---- 4. early-stop heuristic and the prompt's own stopping condition
  if (tid == 0) {
    const double hyp = (p->early_stopping == 2 && p->length_penalty > 0.0) ? (double)max_new : (double)(t + 1);
    const float best = d.running[r0] * lp_inv(hyp, p->length_penalty);
    float mn = s_newfin[0];
    bool all_done = true;
    for (int k = 0; k < K; ++k) {
      mn = fminf(mn, s_newfin[k]);
      all_done = all_done && s_newdone[k];
    }
    bool any = false;
    for (int k = 0; k < K; ++k) any = any || best > (s_newdone[k] ? mn : kBig);
    const bool unsat_new = unsat && any;
    flags[0] = unsat_new;
    flags[1] = !unsat_new || (p->early_stopping == 1 && all_done) || s_nhit == C;
  }
  // ---- 5. the new beams continue their parents: KV indirection table and processor history, column by column
  const int pos = d.pos_dev[r0];
  const int ncopy = t > 0 ? pos + 1 : pos;  // positions with K/V in the cache (the first pick follows the prefill)
  for (int c = tid; c <= ncopy && c < d.ld_kv_src; c += blockDim.x) {
    int old[U2_BEAM_MAX_BEAMS];
#pragma unroll
    for (int k = 0; k < U2_BEAM_MAX_BEAMS; ++k)
      if (k < K) old[k] = d.kv_src[(long long)(r0 + k) * d.ld_kv_src + c];
#pragma unroll
    for (int k = 0; k < U2_BEAM_MAX_BEAMS; ++k) {
      if (k < K) {
        int v = r0 + k;  // the next position is the row's own slot
        if (c < ncopy) {
          const int par = s_parent[k];
#pragma unroll
          for (int q = 0; q < U2_BEAM_MAX_BEAMS; ++q)
            if (q == par) v = old[q];
        }
        d.kv_src[(long long)(r0 + k) * d.ld_kv_src + c] = v;
      }
    }
  }
  if (d.hist) {
    for (int c = tid; c < t && c < d.hist_cap; c += blockDim.x) {
      int old[U2_BEAM_MAX_BEAMS];
#pragma unroll
      for (int k = 0; k < U2_BEAM_MAX_BEAMS; ++k)
        if (k < K) old[k] = d.hist[(long long)(r0 + k) * d.ld_hist + c];
#pragma unroll
      for (int k = 0; k < U2_BEAM_MAX_BEAMS; ++k) {
        if (k < K) {
          int v = 0;
          const int par = s_parent[k];
#pragma unroll
          for (int q = 0; q < U2_BEAM_MAX_BEAMS; ++q)
            if (q == par) v = old[q];
          d.hist[(long long)(r0 + k) * d.ld_hist + c] = v;
        }
      }
    }
  }
}

}  // namespace u2

#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" U2_API int u2_log_softmax_f32(const float* x, float* y, int32_t rows, int32_t V, int64_t ldx, int64_t ldy,
                                         void* stream) {
  using namespace u2;
  if (!x || !y) return set_error(U2_ERR_ARG, "log_softmax: null pointer");
  if (rows <= 0 || V <= 0) return U2_OK;
  if (ldx < V || ldy < V) return set_error(U2_ERR_ARG, "log_softmax: row stride < V");
  log_softmax_kernel<<<rows, kBsThreads, 0, ST(stream)>>>(x, y, V, ldx, ldy);
  U2_CHECK_LAUNCH("log_softmax");
  return U2_OK;
}

extern "C" U2_API int u2_beam_topk_f32(const float* logprobs, int64_t ld, int32_t rows, int32_t V,
                                       const float* running, const int32_t* flags, const u2_beam_params* params_dev,
                                       float* cand_val, int32_t* cand_tok, void* stream) {
  using namespace u2;
  if (!logprobs || !running || !flags || !params_dev || !cand_val || !cand_tok)
    return set_error(U2_ERR_ARG, "beam_topk: null pointer");
  if (rows <= 0) return U2_OK;
  if (ld < V || V < U2_BEAM_MAX_KEEP) return set_error(U2_ERR_ARG, "beam_topk: row stride < V or V < %d", U2_BEAM_MAX_KEEP);
  beam_topk_kernel<<<rows, kBsThreads, 0, ST(stream)>>>(logprobs, ld, V, running, flags, params_dev, cand_val, cand_tok);
  U2_CHECK_LAUNCH("beam_topk");
  return U2_OK;
}

extern "C" U2_API int u2_beam_step(const u2_beam_step_desc* d, int32_t step, void* stream) {
  using namespace u2;
  if (!d || !d->params || !d->cand_val || !d->cand_tok || !d->running || !d->fin_score || !d->fin_info || !d->flags ||
      !d->ids || !d->rec || !d->kv_src || !d->pos_dev)
    return set_error(U2_ERR_ARG, "beam_step: null pointer");
  if (d->prompts <= 0) return U2_OK;
  if (d->V < U2_BEAM_MAX_KEEP || d->ld_rec <= 0 || d->ld_kv_src <= 0 || (d->hist && d->ld_hist < d->hist_cap))
    return set_error(U2_ERR_ARG, "beam_step: bad strides");
  beam_step_kernel<<<d->prompts, kMergeThreads, 0, ST(stream)>>>(*d, step);
  U2_CHECK_LAUNCH("beam_step");
  return U2_OK;
}
