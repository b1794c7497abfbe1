/*
 * u2b200_train.h - C ABI of the TRAINING side of libu2b200.so: the backward kernels, loss heads and the fused
 * sharded optimizer step behind `model(**batch).loss.backward()` and the data-parallel training step
 * (reference src/train/train_stage1.py:244-250 -> HF Trainer / DeepSpeed ZeRO-1, config/ds_config.json:27-39;
 * src/train/dpo_u2trainer.py:185-359 for the DPO step). The contractions of the backward pass (dgrad, wgrad,
 * dP = dO V^T, dQ = dS K, dK = dS^T Q, dV = P^T dO) run on u2_gemm_bf16 (u2b200.h) with its transposed-operand
 * flags; this header holds everything that is not a GEMM.
 *
 * Conventions as in u2b200.h: device pointers owned by the caller, stream-ordered, 0 / negative U2_ERR_* return.
 * Parameter gradients of VECTOR parameters (biases, norm weights, relative-bias tables) are fp32 accumulators that
 * the kernels ADD into (the caller zeroes them once per step); activations and their gradients are bf16.
 */
#ifndef U2B200_TRAIN_H_
#define U2B200_TRAIN_H_

#include "u2b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* out[b][c][r] = in[b][r][c]   (bf16; element strides ld_in / ld_out, batch strides in_bs / out_bs): layout plumbing of
 * the backward (the autograd transposes behind `.transpose(-2, -1)` in src/model/u2tokenizer/rma.py:60, tta.py:52). */
U2_API int u2_transpose_bf16(const void* in, void* out, int32_t rows, int32_t cols, int64_t ld_in, int64_t ld_out,
                             int32_t batch, int64_t in_bs, int64_t out_bs, void* stream);

/* out[c] += sum_r x[r, c]  (x bf16 [rows, cols], row stride ld, cols % 8 == 0; out fp32 [cols]): bias gradients
 * (sum over rows of dY), position-embedding / cls gradients (sum over frames): autograd's bias gradient of every nn.Linear
 * on the path (rma.py:22-33, tta.py:16-19, spatial_pooling_projector.py:24-28, MONAI blocks vit.py:90-105) and of the
 * broadcast adds in vit.py:115-118. */
U2_API int u2_colsum_bf16(const void* x, float* out, int64_t rows, int64_t cols, int64_t ld, void* stream);

/* exact (erf) GELU and its derivative, elementwise over n elements (n % 8 == 0): y = gelu(x);
 * dx = dy * gelu'(x_pre).  (nn.GELU in MONAI MLPBlock and the projector MLP, spatial_pooling_projector.py:24-28) */
U2_API int u2_gelu_bf16(const void* x, void* y, int64_t n, void* stream);
U2_API int u2_gelu_bwd_bf16(const void* x_pre, const void* dy, void* dx, int64_t n, void* stream);

/* Backward of out = silu(gate) * up on a [rows, 2I] gate|up buffer (gate = columns [0, I), up = [I, 2I)):
 * dgu[:, :I] = dact * up * silu'(gate), dgu[:, I:] = dact * silu(gate).   (autograd of the HF decoder MLP,
 * transformers models/qwen3/modeling_qwen3.py:81-83, reached through src/model/language_model/u2llama.py:76-87) */
U2_API int u2_silu_mul_bwd_bf16(const void* gate_up, const void* dact, void* dgu, int64_t rows, int32_t I,
                                int64_t ldg, int64_t ldd, void* stream);

/* LayerNorm / RMSNorm backward over rows of E (E % 8 == 0, E <= 8192): autograd of nn.LayerNorm in
 * src/model/u2tokenizer/tta.py:95,99,103, MONAI TransformerBlock norm1 / norm2 and src/model/multimodal_encoder/vit.py:123,
 * and of HF Qwen3RMSNorm (modeling_qwen3.py:50-67). x is the tensor that was normalised
 * (for `LN(x + residual)` pass the stored sum), dy the gradient of the output.
 *   dx_out = d(norm)/dx * dy  (+ dres when dres != NULL: the gradient arriving through the residual branch)
 *   dgamma += sum_rows dy * xhat,  dbeta += sum_rows dy   (fp32 accumulators, may be NULL when frozen)
 * dx_out may alias dres or dy. */
U2_API int u2_layernorm_bwd_bf16(const void* x, const float* gamma, const void* dy, const void* dres, void* dx_out,
                                 float* dgamma, float* dbeta, int64_t rows, int32_t E, int64_t ldx, int64_t ldy,
                                 int64_t ldr, int64_t ldo, float eps, void* stream);
U2_API int u2_rmsnorm_bwd_bf16(const void* x, const float* gamma, const void* dy, const void* dres, void* dx_out,
                               float* dgamma, int64_t rows, int32_t E, int64_t ldx, int64_t ldy, int64_t ldr,
                               int64_t ldo, float eps, void* stream);

/* Softmax backward (autograd of F.softmax in src/model/u2tokenizer/rma.py:72, tta.py:55-57, svr.py:108 and of the HF
 * eager attention softmax) over rows indexed (i0, i1, i2) like u2_softmax_f32_bf16:
 *   dS[j] = P[j] * (dP[j] - sum_k dP[k] P[k])      (gradient w.r.t. the softmax INPUT, before any scale)
 * P bf16 probabilities (masked entries are 0 and stay 0), dP fp32, dS bf16 (may alias P); columns
 * [n, zero_pad_to) of dS are written 0. */
typedef struct u2_softmax_bwd_desc {
  int64_t p_s0, p_s1, p_s2;
  int64_t dp_s0, dp_s1, dp_s2;
  int64_t ds_s0, ds_s1, ds_s2;
  int32_t n0, H, S, n;
  int32_t zero_pad_to;
} u2_softmax_bwd_desc;
U2_API int u2_softmax_bwd_bf16(const void* P, const float* dP, void* dS, const u2_softmax_bwd_desc* desc, void* stream);
/* drel[(j - i2 + rel_max - 1) * H + i1] += sum_{i0} dS[i0, i1, i2, j]: gradient of the RelativeMultiheadAttention
 * bias table (reference rma.py:35,64-69). dS bf16 with the strides given. */
U2_API int u2_relbias_grad_bf16(const void* dS, float* drel, int32_t n0, int32_t H, int32_t S, int32_t n, int64_t s0,
                                int64_t s1, int64_t s2, int32_t rel_max, void* stream);

/* out[b, h, s] = sum_d a[b, s, h, d] * c[b, s, h, d] (bf16 views with element strides *_sb batch, *_ss token, *_sh head;
 * out fp32 [B, H, S]): D = rowsum(dO * O), the term that turns dP into dS without the probabilities' row sums (attention
 * backward of MONAI SABlock, vit.py:100-105, with the probabilities rebuilt from the forward's log-sum-exp). */
U2_API int u2_rowdot_bf16(const void* a, const void* c, float* out, int32_t B, int32_t S, int32_t H, int32_t dh,
                          int64_t a_sb, int64_t a_ss, int64_t a_sh, int64_t c_sb, int64_t c_ss, int64_t c_sh,
                          void* stream);

/* Backward of u2_temporal_attention_bf16 (svr.py:33-36 over rma.py:60-73): recomputes the C x C probabilities of
 * every (batch, token, head) from qkv, then dqkv (same layout as qkv: [q|k|v] columns) from dout; drel (fp32
 * [2*rel_max-1, H], may be NULL) accumulates the relative-bias gradient. C <= 128. */
U2_API int u2_temporal_attention_bwd_bf16(const void* qkv, const void* dout, void* dqkv, int32_t B, int32_t C,
                                          int32_t N, int32_t H, int32_t dh, int64_t ld_qkv, int64_t ld_dout,
                                          int64_t ld_dqkv, float scale, const float* rel_bias, float* drel,
                                          int32_t rel_max, void* stream);

/* Backward of u2_rope_bf16 without cache append (autograd of src/model/u2tokenizer/rope.py:77-80 and of q_norm / k_norm +
 * apply_rotary_pos_emb in transformers models/qwen3/modeling_qwen3.py:263-268): dx (gradient w.r.t. the roped / normed heads, in place) becomes the
 * gradient w.r.t. the raw projections x_raw (needed when the per-head RMSNorm of Qwen3 is on); V heads pass
 * through. dq_norm_w / dk_norm_w: fp32 [dh] accumulators (NULL when q_norm_w / k_norm_w are). Uses the fields
 * rows, ld, dh, n_*_heads, *_norm_w, eps, inv_freq, pos0, pos_div, pos_mod of the descriptor. */
U2_API int u2_rope_bwd_bf16(void* dx, const void* x_raw, const u2_rope_desc* desc, float* dq_norm_w, float* dk_norm_w,
                            void* stream);

/* Backward of u2_spp_pool_bf16 (autograd of avg_pool3d / the sequence pooling in
 * src/model/multimodal_projector/spatial_pooling_projector.py:38-46): dx[f, in_off + token, :] = dy[f, pooled(token), :] / ps^3 (rows outside the
 * pooled grid - the cls row, the padding rows - are written 0; dx row stride ldx, frame stride in_frame_stride
 * rows, rows_per_frame rows are written per frame). */
U2_API int u2_spp_pool_bwd_bf16(const void* dy, void* dx, int64_t frames, int32_t g0, int32_t g1, int32_t g2,
                                int32_t ps, int32_t E, int64_t in_frame_stride, int64_t in_off, int64_t ldx,
                                int64_t rows_per_frame, int32_t sequence, void* stream);

/* Backward of u2_multiscale_pool_bf16 (autograd of src/model/u2tokenizer/svr.py:126-151 / 175-184). logits: the [B, 3] gate logits the forward left in its workspace.
 * dx [B, K, E] = sum_k w_k pool_k^T(dy_k) + (dynamic) the gradient through the gates; dgate_w (fp32 [E], += ),
 * ws: fp32 [B, 8] scratch (zeroed by the call). */
U2_API int u2_multiscale_pool_bwd_bf16(const void* x, const void* dy, void* dx, const float* gate_w,
                                       const float* logits, float* dgate_w, float* ws, int32_t B, int32_t K,
                                       int32_t E, int32_t dynamic, void* stream);

/* Scatter-add of row gradients (embedding / hard token selection backward):
 *   l in [1, n_vis] and dvis != NULL:  dvis[b, l - 1, :] = drows[b, l, :]        (the spliced visual tokens)
 *   else                              dtable[ids[b, l], :] += drows[b, l, :]     (bf16 atomics; skipped when
 *                                                                                  dtable == NULL)
 * (reference u2_arch.py:114,118-121 backward). ids int64 [B, L]. */
U2_API int u2_embed_scatter_add_bf16(const int64_t* ids, const void* drows, void* dtable, void* dvis, int32_t B,
                                     int32_t L, int32_t E, int32_t n_vis, int64_t vocab, void* stream);
/* out[r * ld_out + h * dh + e] = sum_{g < G} in[r * ld_in + (h * G + g) * dh + e]: sum of the G query-head
 * gradients that share one KV head (GQA dK / dV written per query head by the batched GEMMs; autograd of repeat_kv,
 * transformers models/qwen3/modeling_qwen3.py:184-194). dh % 8 == 0. */
U2_API int u2_group_sum_bf16(const void* in, void* out, int64_t rows, int32_t heads, int32_t G, int32_t dh,
                             int64_t ld_in, int64_t ld_out, void* stream);

/* Cross-entropy / log-probability head backward: fp32 logits [R, V] (row stride ld_in) -> bf16 dlogits (ld_out):
 *   dlogits[r, v] = coef[r] * (exp(logits[r, v] - lse[r]) - [v == labels[r]])
 * coef fp32 [R] (0 for rows without a label): 1 / #labelled rows for the mean-NLL loss of forward(labels=...)
 * (u2llama.py:76-87), -dLoss/dlogp[r] for the DPO loss (dpo_u2trainer.py:296 and trl's sigmoid loss). V % 8 == 0. */
U2_API int u2_ce_bwd_f32_bf16(const float* logits, void* dlogits, const float* lse, const int64_t* labels,
                              const float* coef, int64_t R, int32_t V, int64_t ld_in, int64_t ld_out, void* stream);
/* Sigmoid DPO loss head (trl DPOTrainer.dpo_loss, loss_type "sigmoid", reference_free False; beta from
 * train_stage2.py:83): per_tok fp32 [2P, L] policy log-probs (chosen rows first, then rejected), ref_sum fp32 [2P]
 * summed reference log-probs, mask [2P, L] (uint8).  loss = mean_p -logsigmoid(beta * ((pc - pr) - (rc - rr)));
 * out[0] = loss, out[1] = mean reward accuracy, out[2] = mean reward margin;
 * coef[r, l] = -dloss/dlogp[r, l] (feeds u2_ce_bwd_f32_bf16). One block, P <= 1024. */
U2_API int u2_dpo_loss_f32(const float* per_tok, const float* ref_sum, const uint8_t* mask, float* out, float* coef,
                           int32_t P, int32_t L, float beta, void* stream);

/* Fused AdamW on a (ZeRO-1) shard of the flat parameter buffer (the optimizer step DeepSpeed runs for the reference:
 * optim adamw_torch, src/train/train_stage1.py:113-131, ZeRO stage 1 config/ds_config.json:27-39): fp32 master / m / v, bf16 gradient shard (already
 * averaged over the data-parallel ranks), bf16 parameter shard written back for the all-gather.
 *   g = grad * (*grad_scale)  (grad_scale: device scalar, e.g. the clipping factor; NULL = 1)
 *   torch.optim.AdamW semantics (decoupled weight decay, bias correction with `step`).
 * u2_sumsq_bf16: out[0] += sum g^2 (fp32 atomics; gradient-norm clipping, HF Trainer max_grad_norm). */
typedef struct u2_adamw_desc {
  float lr, beta1, beta2, eps, weight_decay;
  int32_t step;               /* 1-based */
  const float* grad_scale;
  uint64_t seed;              /* stochastic rounding of bf16 moments (u2_adamw_bf16_mom16); unused with fp32 moments */
  int64_t index_offset;       /* >= 0: global index of element 0 of this call (ZeRO-1 slice / bucket offset) */
} u2_adamw_desc;
U2_API int u2_adamw_bf16(float* master, float* m, float* v, const void* grad, void* param_out, int64_t n,
                         const u2_adamw_desc* desc, void* stream);
/* same update with bf16 first / second moments (8 instead of 12 bytes of state per parameter: the mode a single GPU
 * needs to hold the whole optimizer state of the 8B model; the sharded multi-GPU step keeps fp32 moments). The new m
 * and v are computed in fp32 (and the master update uses those fp32 values), then stored with STOCHASTIC rounding to
 * bf16: round-to-nearest would freeze v whenever (1 - beta2) |g^2 - v| is below half a bf16 ulp of v (g^2 < ~3 v at
 * beta2 0.999), so v could only grow and the step size would drift away from fp32 AdamW's. The random bits of element
 * e are fmix32(fmix32(key ^ lo32(e)) ^ hi32(e)), key = fmix32(lo32(seed) ^ fmix32(hi32(seed) + step * 0x9E3779B9)),
 * e = index_offset + the element's index in this call; the low 16 bits round m, the high 16 bits round v. Same seed,
 * step and global index give the same bits, however the buffer is split into calls. */
U2_API int u2_adamw_bf16_mom16(float* master, void* m, void* v, const void* grad, void* param_out, int64_t n,
                               const u2_adamw_desc* desc, void* stream);
U2_API int u2_adamw_f32grad(float* master, float* m, float* v, const float* grad, void* param_out_bf16,
                            float* param_out_f32, int64_t n, const u2_adamw_desc* desc, void* stream);
U2_API int u2_sumsq_bf16(const void* x, float* out, int64_t n, void* stream);
U2_API int u2_sumsq_f32(const float* x, float* out, int64_t n, void* stream);
/* dst += src (bf16, n % 8 == 0): gradient accumulation where two branches meet (residual connections, the visual /
 * text tokens that feed every TTA layer, src/model/u2tokenizer/tta.py:93-107). */
U2_API int u2_add_bf16(void* dst, const void* src, int64_t n, void* stream);
/* dtype plumbing between the flat buffers: fp32 -> bf16 and bf16 -> fp32 (n elements); stands in for the bf16 autocast
 * of fp32 parameters the reference trains with (src/train/train_stage1.py:116). */
U2_API int u2_cast_f32_bf16(const float* in, void* out, int64_t n, void* stream);
U2_API int u2_cast_bf16_f32(const void* in, float* out, int64_t n, void* stream);

/* LoRA adapters of the decoder linears (PEFT LoraLayer.forward: y = W x + s * B_j A_j dropout_j(x), s = lora_alpha / r;
 * reference src/train/train_stage1.py:342-353). The 1-3 adapters of one call share the input X [M, K] (q|k|v, gate|up,
 * or o / down alone); their A matrices are stacked [n_adapters * r, K] (row stride K), U / dU are [M, n_adapters * r]
 * with adapter j in columns [j r, (j + 1) r). r in {8, 16, 32, 64}; bf16 data, fp32 accumulation.
 *
 * Dropout mask (inverted dropout, one independent mask per adapter as PEFT has one nn.Dropout per LoRA layer):
 *   fmix32(h) = h ^= h >> 16; h *= 0x85EBCA6B; h ^= h >> 13; h *= 0xC2B2AE35; h ^= h >> 16      (uint32 arithmetic)
 *   key_j     = fmix32(lo32(seed) ^ fmix32(hi32(seed) + stream[j] * 0x9E3779B9))
 *   h         = fmix32(fmix32(key_j ^ row) ^ col)                  (row of X in [0, M), column in [0, K))
 *   D_j(row, col) = 0 if h < floor(p * 2^32), else 1 / (1 - p)     (p = 0: every element kept, D = 1)
 * stream[j] names the adapter: the training engine passes layer * 8 + t with t = 0..6 for q, k, v, o, gate, up, down.
 * Phi-3 (fused HF Phi3 linears, one adapter per call) has its own streams, disjoint from those: 2^24 + layer * 4 + t
 * with t = 0..3 for qkv_proj, o_proj, gate_up_proj, down_proj.
 * The masked input D_j o X is rounded to bf16 (the dtype PEFT's dropout returns) wherever it is an operand.
 *
 *   u2_lora_down_bf16:  U[:, j] = s * (D_j o X) A_j^T
 *   u2_lora_wgrad_bf16: dA_j = s * dU_j^T (D_j o X)      written to the stacked bf16 gradient [n_adapters * r, K]
 *                       (accumulate != 0: added to what it holds)
 *   u2_lora_dgrad_bf16: dX += sum_j D_j o (s * dU_j A_j) (in place, row stride ldx)
 * ldx is the row stride of X (down, wgrad) or dX (dgrad); ldu that of U / dU. */
typedef struct u2_lora_desc {
  int32_t M, K, r, n_adapters;
  int64_t ldx, ldu;
  float scale;
  float p;
  uint64_t seed;
  int32_t stream[3];
  int32_t accumulate;
} u2_lora_desc;
U2_API int u2_lora_down_bf16(const void* X, const void* A, void* U, const u2_lora_desc* desc, void* stream);
U2_API int u2_lora_wgrad_bf16(const void* dU, const void* X, void* dA, const u2_lora_desc* desc, void* stream);
U2_API int u2_lora_dgrad_bf16(const void* dU, const void* A, void* dX, const u2_lora_desc* desc, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* U2B200_TRAIN_H_ */
