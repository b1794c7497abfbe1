// Slot bookkeeping of continuous batching (generate_batch), launched after the token pick inside the captured decode
// step: each decode row is a slot holding one sample of one request, with its own generated count, max_new_tokens and
// done flag (u2_slot_state). The kernel does per slot what the host does per step for a generate() call, so the host
// only has to poll the done flags to retire finished slots and admit new requests between graph replays.
#include <cuda_runtime.h>

#include "host_util.h"
#include "u2b200.h"

namespace u2 {

// kLp: also append the pick's log-prob lp_in[b] at the same count into lp_out (generate_batch(return_logprobs=True)).
template <bool kLp>
__global__ void slot_update_kernel(long long* __restrict__ ids, int B, u2_slot_state* __restrict__ slots,
                                   long long* __restrict__ out, long long ld_out, const u2_slot_params* __restrict__ p,
                                   int* __restrict__ length, int* __restrict__ length_plus1,
                                   const float* __restrict__ lp_in = nullptr, float* __restrict__ lp_out = nullptr) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  u2_slot_state s = slots[b];
  if (s.done) {
    ids[b] = p->pad;  // a finished or empty slot decodes pad at a frozen position until it is refilled
    return;
  }
  const long long tok = ids[b];
  if (s.count < ld_out) out[b * ld_out + s.count] = tok;
  if constexpr (kLp) {
    if (s.count < ld_out) lp_out[b * ld_out + s.count] = lp_in[b];
  }
  s.count += 1;
  bool fin = s.count >= s.max_new;
  for (int i = 0; i < p->n_eos; ++i) fin |= tok == (long long)p->eos[i];
  if (fin) {
    s.done = 1;
    ids[b] = p->pad;
  } else if (length) {
    length[b] += 1;
    length_plus1[b] += 1;
  }
  slots[b].count = s.count;
  slots[b].done = s.done;
}

}  // namespace u2

extern "C" U2_API int u2_slot_update(int64_t* ids, int32_t B, u2_slot_state* slots, int64_t* out, int64_t ld_out,
                                     const u2_slot_params* params_dev, int32_t* length, int32_t* length_plus1,
                                     void* stream) {
  using namespace u2;
  if (!ids || !slots || !out || !params_dev) return set_error(U2_ERR_ARG, "slot_update: null pointer");
  if (!length != !length_plus1) return set_error(U2_ERR_ARG, "slot_update: length and length_plus1 go together");
  if (ld_out < 1) return set_error(U2_ERR_ARG, "slot_update: ld_out must be >= 1");
  if (B <= 0) return U2_OK;
  slot_update_kernel<false><<<(B + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<long long*>(ids), B, slots, reinterpret_cast<long long*>(out), ld_out, params_dev, length,
      length_plus1);
  U2_CHECK_LAUNCH("slot_update");
  return U2_OK;
}

extern "C" U2_API int u2_slot_update_lp(int64_t* ids, int32_t B, u2_slot_state* slots, int64_t* out, int64_t ld_out,
                                        const float* lp_in, float* lp_out, const u2_slot_params* params_dev,
                                        int32_t* length, int32_t* length_plus1, void* stream) {
  using namespace u2;
  if (!ids || !slots || !out || !lp_in || !lp_out || !params_dev) return set_error(U2_ERR_ARG, "slot_update_lp: null pointer");
  if (!length != !length_plus1) return set_error(U2_ERR_ARG, "slot_update_lp: length and length_plus1 go together");
  if (ld_out < 1) return set_error(U2_ERR_ARG, "slot_update_lp: ld_out must be >= 1");
  if (B <= 0) return U2_OK;
  slot_update_kernel<true><<<(B + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<long long*>(ids), B, slots, reinterpret_cast<long long*>(out), ld_out, params_dev, length,
      length_plus1, lp_in, lp_out);
  U2_CHECK_LAUNCH("slot_update_lp");
  return U2_OK;
}
