/*
 * u2b200.h - C ABI of libu2b200.so: the sm_90a kernels behind the mu2-LLM
 * "visual-tokenize-then-decode" hot path (CT volume -> 3D patch embed -> ViT3D -> spatial-pooling
 * projector -> mu2-Tokenizer -> splice -> Qwen3/Llama decoder forward / greedy decode).
 *
 * The reference (Siyou-Li/u2Tokenizer) is pure Python: it has no FFI of its own. The boundary it
 * exposes is the HuggingFace module surface (forward()/generate(), reference
 * src/model/language_model/u2llama.py:41-127); that surface is mirrored in Python by
 * u2tokenizer_b200/modeling.py and everything underneath it calls the entry points declared
 * here. Each entry point cites the reference call site whose arithmetic it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (torch allocates), no allocation inside;
 *   - `stream` is a cudaStream_t passed as void*; all work is stream-ordered, re-entrant;
 *   - return value: 0 (U2_OK) or a negative U2_ERR_* code; u2_last_error() gives the message;
 *   - bf16 = __nv_bfloat16 bits, "f32" = float; row-major unless stated otherwise.
 */
#ifndef U2B200_H_
#define U2B200_H_

#include <stdint.h>

#if defined(__GNUC__)
#define U2_API __attribute__((visibility("default")))
#else
#define U2_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define U2_OK 0
#define U2_ERR_ARG (-1)
#define U2_ERR_CUDA (-2)
#define U2_ERR_UNSUPPORTED (-3)

#define U2_DT_BF16 0
#define U2_DT_F32 1

#define U2_ACT_NONE 0
#define U2_ACT_GELU 1 /* exact erf GELU (torch.nn.GELU default) */
#define U2_ACT_SILU 2

#define U2_EPI_NONE 0
#define U2_EPI_EXP_ROW 1
#define U2_EPI_DS_ROW 2

/* Library / device info ----------------------------------------------------------------------- */
U2_API int u2_version(void);                 /* ABI version, currently 1 */
U2_API const char* u2_last_error(void);      /* message of the last failing call on this thread */
U2_API int u2_device_sm_count(void);         /* SMs of the current device (132 on H100), <0 on error */

/* GEMM --------------------------------------------------------------------------------------------
 * For every batch z = (zo, zi):
 *     C[z] (M x N) = act( alpha * A[z] (M x K) * B[z'] (N x K)^T + bias[n] ) + residual
 * A, B are bf16, K-major (row stride lda/ldb elements, multiples of 8) unless a_mn / b_mn say otherwise;
 * fp32 accumulation in registers. residual == C (same ld) accumulates into a bf16 C (gradient accumulation).
 * Batch offsets (elements): A: zi*a_stride_zi + zo*a_stride_zo; B: (zi / b_zi_div)*b_stride_zi +
 * zo*b_stride_zo (b_zi_div > 1 shares one B among consecutive inner batches: GQA);
 * C: zi*c_stride_zi + zo*c_stride_zo.
 * Output row remap (row_div > 0): out_row = (r / row_div) * row_stride + row_off + r % row_div.
 * Residual (bf16, row stride ldr): row = r % res_row_mod when res_row_mod > 0 (broadcast table,
 * e.g. the ViT position embedding) else the output row (same batch offsets as C).
 * Replaces: every nn.Linear / torch.matmul on the path (reference src/model/u2tokenizer/rma.py:52-73,
 * tta.py:42-69, svr.py:107, spatial_pooling_projector.py:48-50; MONAI blocks; HF decoder Linears).
 */
typedef struct u2_gemm_desc {
  int32_t M, N, K;
  int32_t zi, zo;     /* inner / outer batch counts (<=0 means 1) */
  int32_t b_zi_div;   /* <=0 means 1 */
  int64_t lda, a_stride_zi, a_stride_zo;
  int64_t ldb, b_stride_zi, b_stride_zo;
  int64_t ldc, c_stride_zi, c_stride_zo;
  int32_t c_dtype;    /* U2_DT_BF16 or U2_DT_F32 */
  float alpha;
  const float* bias;  /* [N] fp32 or NULL */
  int32_t act;        /* U2_ACT_* */
  const void* residual; /* bf16 or NULL */
  int64_t ldr;
  int32_t res_row_mod;
  int32_t row_div, row_stride, row_off;
  int32_t block_n;    /* 0 = auto, else 64/128/256 (256: the widest tile, 128 columns on sm_90) */
  /* transposed operands (training: dgrad = dY * W, wgrad = dY^T * X, P^T dO ...): a_mn != 0 -> A is stored
   * [K][M] (element (m, k) at A[k * lda + m]); b_mn != 0 -> B is stored [K][N]. lda / ldb are then the strides
   * between consecutive contraction indices. No transposed copy is made: the tile is loaded MN-major. */
  int32_t a_mn, b_mn;
  /* fused epilogue of the attention backward (applied after alpha, before bias / act / residual; rowvec is indexed
   * rowvec[zo * rv_stride_zo + zi * rv_stride_zi + row]):
   *   U2_EPI_EXP_ROW:  v = exp(v - rowvec[row])             P = exp(scale * q.k - lse) straight out of the score GEMM
   *   U2_EPI_DS_ROW:   v = mul[row, col] * (v - rowvec[row]) dS = P * (dO.V^T - rowsum(dO * O)); mul (bf16) has C's
   *                                                          layout (ldc, c_stride_*) and may BE C (in place) */
  int32_t epi_op;
  const float* rowvec;
  int64_t rv_stride_zi, rv_stride_zo;
  const void* mul;
} u2_gemm_desc;

U2_API int u2_gemm_bf16(const void* A, const void* B, void* C, const u2_gemm_desc* desc, void* stream);

/* Row-wise normalisation ----------------------------------------------------------------------------
 * y = LayerNorm(x [+ residual]) * gamma + beta   (fp32 statistics, eps inside the sqrt)
 * y = RMSNorm (x [+ residual]) * gamma
 * x, residual, y, sum_out: bf16 rows of E elements (row strides ldx/ldr/ldy, multiples of 8);
 * gamma/beta fp32 [E]. When residual and sum_out are given, sum_out receives x + residual (the new
 * residual stream, row stride ldy). Replaces nn.LayerNorm (MONAI TransformerBlock norm1/norm2, ViT
 * final norm vit.py:123; tta.py:95,99,103) and HF Qwen3RMSNorm / LlamaRMSNorm.
 */
U2_API int u2_layernorm_bf16(const void* x, const void* residual, const float* gamma, const float* beta,
                             void* y, void* sum_out, int64_t rows, int32_t E, int64_t ldx, int64_t ldr,
                             int64_t ldy, float eps, void* stream);
U2_API int u2_rmsnorm_bf16(const void* x, const void* residual, const float* gamma, void* y, void* sum_out,
                           int64_t rows, int32_t E, int64_t ldx, int64_t ldr, int64_t ldy, float eps,
                           void* stream);

/* Softmax over fp32 score rows -> bf16 probabilities ---------------------------------------------------
 * Rows are indexed (i0 batch, i1 head in [0,H), i2 query in [0,S)); element strides given for input
 * and output. p[j] = softmax_j(in[j] * scale + rel_bias[(j - i2 + rel_max - 1) * H + i1]) over the
 * visible keys j < n (and j <= i2 + causal_off when causal). Columns [n, zero_pad_to) are written 0.
 * window > 0 (needs causal): key j is also hidden unless j > i2 + causal_off - window, the sliding-window mask of HF
 * Phi-3 (transformers masking_utils.py:90-97 sliding_window_overlay `kv_idx > q_idx - sliding_window`, applied through
 * models/phi3/modeling_phi3.py:265,403); 0 = no window.
 * Replaces F.softmax in rma.py:60-73 (relative bias gather included), tta.py:55-57, the MONAI
 * SABlock softmax and the HF eager attention softmax + causal (+ sliding-window) mask.
 */
typedef struct u2_softmax_desc {
  int64_t in_s0, in_s1, in_s2;
  int64_t out_s0, out_s1, out_s2;
  int32_t n0, H, S, n;
  float scale;
  const float* rel_bias;
  int32_t rel_max;
  int32_t causal, causal_off;
  int32_t zero_pad_to;
  int32_t window;
} u2_softmax_desc;
U2_API int u2_softmax_f32_bf16(const float* in, void* out, const u2_softmax_desc* desc, void* stream);

/* out[r, i] = silu(g) * u with (g, u) = gate_up[r, i], gate_up[r, I + i]  (interleaved == 0) or
 * gate_up[r, 2i], gate_up[r, 2i + 1] (interleaved != 0). Replaces `act_fn(gate_proj(x)) * up_proj(x)` of the HF decoder MLP
 * (transformers models/qwen3/modeling_qwen3.py:81-83, reached from the reference through super().forward,
 * src/model/language_model/u2llama.py:76-87). */
U2_API int u2_silu_mul_bf16(const void* gate_up, void* out, int64_t rows, int32_t I, int64_t ldg,
                            int64_t ldo, int32_t interleaved, void* stream);

/* Vision-front data movement ----------------------------------------------------------------------------
 * patchify: fp32 volume [frames, d0, d1, d2] -> bf16 patch rows [frames * n_patches, p0*p1*p2] in the
 * MONAI "perceptron" order "b c (h p1) (w p2) (d p3) -> b (h w d) (p1 p2 p3 c)", c == 1
 * (reference vit.py:90-99 -> MONAI PatchEmbeddingBlock).
 */
U2_API int u2_patchify_f32_bf16(const float* vol, void* rows, int64_t frames, int32_t d0, int32_t d1,
                                int32_t d2, int32_t p0, int32_t p1, int32_t p2, void* stream);
/* Fused 3-D patch embedding: out[f, 1 + t, :] = bf16(patch(f, t) . W^T + bias + pos[t]) for the fp32 volume
 * vol [frames, d0, d1, d2] (single channel), W [N, p0*p1*p2] bf16 in MONAI's (p1 p2 p3 c) feature order, bias fp32 [N],
 * pos bf16 [tokens, N], out bf16 [frames, out_frame_rows, N] (row 0 = cls and the rows behind the tokens are left to
 * u2_vit_frame_rows_bf16). 5-D TMA slabs of the volume are converted to the swizzled bf16 A operand in shared memory: the
 * einops gather of MONAI PatchEmbeddingBlock + Linear + position add (reference vit.py:90-99,115) in one kernel, the volume
 * is read once. Covers patch (p0, 4k, 16) on a (g0, 8m, 16) token grid (the canonical 4 x 16 x 16 patches of
 * 32 x 256 x 256 frames); other geometries return U2_ERR_UNSUPPORTED (use u2_patchify_f32_bf16 + u2_gemm_bf16). */
U2_API int u2_patch_embed_f32_bf16(const float* vol, const void* W, const float* bias, const void* pos, void* out,
                                   int64_t frames, int32_t d0, int32_t d1, int32_t d2, int32_t p0, int32_t p1, int32_t p2,
                                   int32_t N, int64_t out_frame_rows, void* stream);
/* dst[(r * row_stride + row_off), :] = vec for r in [0, n_rows)   (cls token rows, vit.py:116-118) */
U2_API int u2_set_rows_bf16(void* dst, const void* vec, int64_t n_rows, int64_t row_stride, int64_t row_off,
                            int32_t E, void* stream);
/* ViT sequence buffer dst [frames][Sp][E]: row 0 of every frame = cls, rows [S, Sp) = 0 (the padding that keeps the
 * frame stride a multiple of 16 bytes); rows 1..S-1 come from the patch-embed GEMM (vit.py:116-118 cls concat). */
U2_API int u2_vit_frame_rows_bf16(void* dst, const void* cls, int64_t frames, int32_t Sp, int32_t S, int32_t E,
                                  void* stream);
/* in[b][s][h][d] (element strides in_sb, in_ss, in_sh; d contiguous) -> out[b][h][d][s] with the s axis
 * padded to ld_out (zeros): a K-major V^T / X^T operand. Replaces the `split_heads` + `transpose(-2, -1)` copies of
 * src/model/u2tokenizer/rma.py:41-44,60 and tta.py:24-26,52. The path itself no longer calls it: V and the DiffTS token
 * matrix are consumed in place as MN-major operands (u2_gemm_desc.b_mn, u2_flash_attention_d64_bf16). */
U2_API int u2_transpose_heads_bf16(const void* in, void* out, int32_t B, int32_t S, int32_t H, int32_t Dh,
                                   int64_t in_sb, int64_t in_ss, int64_t in_sh, int64_t out_sb,
                                   int64_t out_sh, int64_t ld_out, void* stream);
/* SpatialPoolingProjector pooling (spatial_pooling_projector.py:38-46): token (a0,a1,a2) of frame f lives
 * at row f*in_frame_stride + in_off + (a0*g1+a1)*g2+a2 (row stride ldx); out [frames, n_out, E] dense.
 * sequence != 0 selects the avg_pool1d(ps^3) variant. */
U2_API int u2_spp_pool_bf16(const void* x, void* out, int64_t frames, int32_t g0, int32_t g1, int32_t g2,
                            int32_t ps, int32_t E, int64_t in_frame_stride, int64_t in_off, int64_t ldx,
                            int32_t sequence, void* stream);
/* Multi-scale token pooling, scales (1,2,4) over the token dim of x [B, K, E] -> out [B, K+K/2+K/4, E];
 * dynamic != 0: DynamicMultiScalePooling gate (svr.py:126-151) with gate_w [E] fp32, gate_bias scalar and an fp32
 * workspace of u2_multiscale_pool_ws_elems(B, K) floats whose first B*3 hold the gate logits [B,3] on return (the
 * rest: per-block partial sums, added in a fixed order); dynamic == 0: the plain concat (svr.py:175-184). */
U2_API int u2_multiscale_pool_bf16(const void* x, void* out, const float* gate_w, float gate_bias,
                                   float* logits_ws, int32_t B, int32_t K, int32_t E, int32_t dynamic,
                                   void* stream);
U2_API int64_t u2_multiscale_pool_ws_elems(int32_t B, int32_t K);
/* out[b][l] = vis[b][l-1] for 1 <= l <= n_vis (when vis != NULL) else table[ids[b][l]]
 * (u2_arch.py:118-121: embed_tokens gather + cat splice). ids int64. */
U2_API int u2_embed_splice_bf16(const int64_t* ids, const void* table, const void* vis, void* out, int32_t B,
                                int32_t L, int32_t E, int32_t n_vis, int64_t vocab, void* stream);

/* Small attention pieces ----------------------------------------------------------------------------------
 * temporal attention of the SVR layer (svr.py:33-36 with rma.py:60-73): qkv rows ordered (b, c, n),
 * columns [q|k|v] (E each); attends across the C <= 32 frames of each (b, n, head). rel_bias as above. */
U2_API int u2_temporal_attention_bf16(const void* qkv, void* out, int32_t B, int32_t C, int32_t N, int32_t H,
                                      int32_t dh, int64_t ld_qkv, int64_t ld_out, float scale,
                                      const float* rel_bias, int32_t rel_max, void* stream);

/* In-place rotate-half RoPE on the first n_q_heads + n_k_heads heads of every row (optionally preceded by
 * the per-head RMSNorm of Qwen3, HF modeling_qwen3.py:263-268), and optional KV-cache append
 * (caches [B, n_k_heads, Tmax, dh]). position(row) = pos0 + (row / pos_div) % pos_mod; pos0 may be read
 * from the device (pos0_dev). Also used for attn_type == "rope" of the tokenizer (rope.py:77-80). */
typedef struct u2_rope_desc {
  int64_t rows, ld;
  int32_t dh, n_q_heads, n_k_heads, n_v_heads;
  const float* q_norm_w;
  const float* k_norm_w;
  float eps;
  const float* inv_freq; /* [dh/2] fp32 */
  int32_t pos0, pos_div, pos_mod;
  const int32_t* pos0_dev;
  void* k_cache;
  void* v_cache;
  int32_t Tmax, rows_per_batch;
  int32_t pos0_per_batch; /* != 0: pos0 = pos0_dev[row / rows_per_batch] (one position per sequence of a batch whose
                             prompts have different lengths); 0: pos0_dev[0] (or pos0) for every row */
} u2_rope_desc;
U2_API int u2_rope_bf16(void* x, const u2_rope_desc* desc, void* stream);

/* One query token per sequence against the KV cache (GQA). q [B, Hq*dh] (row stride ldq), caches
 * [B, Hkv, Tmax, dh]; T valid keys (or *T_dev when T_dev != NULL; T_dev[b] for sequence b when T_per_seq != 0,
 * which needs T_dev). Replaces the HF eager attention at q_len == 1
 * (transformers models/qwen3/modeling_qwen3.py:252-291) inside generate() (src/model/language_model/u2llama.py:123-126);
 * unfused variant used by the CUDA-core decode path. kv_src (int32 [B, ld_kv_src] or NULL): the beam-indirect cache of
 * u2_fused_decode_desc, key t < T - 1 of sequence b from cache row kv_src[b * ld_kv_src + t]. */
U2_API int u2_decode_attention_bf16(const void* q, const void* k_cache, const void* v_cache, void* out,
                                    int32_t B, int32_t Hq, int32_t Hkv, int32_t dh, int32_t Tmax, int32_t T,
                                    const int32_t* T_dev, int64_t ldq, int64_t ldo, float scale, int32_t T_per_seq,
                                    const int32_t* kv_src, int64_t ld_kv_src, void* stream);
/* u2_decode_attention_bf16 with a sliding window: sequence b attends keys [max(0, T_b - window), T_b) only and reads
 * nothing below them (window 0 = no window). The Phi-3 decode step (HF masking_utils.py:90-97, modeling_phi3.py:403).
 * head_dim 32, 64, 96 or 128 (as u2_decode_attention_bf16). */
U2_API int u2_decode_attention_window_bf16(const void* q, const void* k_cache, const void* v_cache, void* out,
                                           int32_t B, int32_t Hq, int32_t Hkv, int32_t dh, int32_t Tmax, int32_t T,
                                           const int32_t* T_dev, int64_t ldq, int64_t ldo, float scale,
                                           int32_t T_per_seq, const int32_t* kv_src, int64_t ld_kv_src,
                                           int32_t window, void* stream);

/* Decode-step linear (weight streaming, HBM-bound): y[b, n] = sum_k norm(x)[b, k] * w[n, k] (+ residual).
 * CUDA-core variant of the HF decoder Linears (+ Qwen3RMSNorm, modeling_qwen3.py:50-67) at q_len == 1 inside generate()
 * (src/model/language_model/u2llama.py:123-126) for shapes the wgmma path does not take (K % 64 != 0).
 * B <= 8. norm_gamma != NULL fuses the input RMSNorm; silu_pair != 0 treats rows (2j, 2j+1) of w as
 * (gate_j, up_j) and writes silu(gate) * up (N/2 outputs). */
typedef struct u2_gemv_desc {
  int32_t B, N, K;
  int64_t ldx, ldw, ldy, ldr;
  int32_t y_dtype;
  const void* residual;
  const float* norm_gamma;
  float norm_eps;
  int32_t silu_pair;
} u2_gemv_desc;
U2_API int u2_gemv_bf16(const void* x, const void* w, void* y, const u2_gemv_desc* desc, void* stream);
/* ids[b] = argmax_v logits[b, v] (first index on ties). scratch: uint64 [B], zero on entry and zero again on exit.
 * Replaces `torch.argmax(next_token_scores, dim=-1)` of HF GenerationMixin._sample with do_sample=False
 * (transformers generation/utils.py:2793; reference call src/model/language_model/u2llama.py:123-126). */
U2_API int u2_argmax_f32(const float* logits, int64_t* out, uint64_t* scratch, int32_t B, int32_t V, int64_t ld,
                         void* stream);

/* Decode-step linear on the tensor cores (swap-AB, stream-K over all SMs, TMA weight stream; HBM-bound):
 *   acc[b, n] = sum_k x[b, k] * w[n, k]                       B <= 16, K % 64 == 0
 *   v = acc * rsqrt(ssq_in[b] / K + eps)   (when ssq_in != NULL: fused RMSNorm, x must already carry gamma)
 *   silu_pair: rows (2j, 2j+1) of w are (gate_j, up_j):  y[b, j] = silu(v_2j) * v_2j+1
 *   else:      y[b, n] = v + residual[b, n];  optionally xg[b, n] = bf16(y * gamma_next[n]) and
 *              ssq_out[b] += sum_n y^2 (prepares the next fused norm); ssq_zero[0..15] is reset to 0.
 * ws: fp32 partial-sum slots (ws_elems floats; u2_dlinear_ws_elems(N, K) gives the size needed by the stream-K
 * schedule and the per-tile sums of squares behind the slots): every 32-bit word must hold 0xffffffff ("empty") on
 * entry and does so again on exit;
 * counters: int32 [ceil(N/64)] (+1 when ssq_out != NULL: the op's tile ticket), zero on entry and on exit.
 * ssq_out is added in a fixed order, so repeated launches on the same inputs give identical results.
 * Replaces the HF decoder Linears at q_len == 1 (reference u2llama.py:123-126 -> GenerationMixin._sample). */
#define U2_DLIN_STREAMK128 0
#define U2_DLIN_TILES64 1
#define U2_DLIN_W_BF16 0     /* w: bf16 [N, K], row stride ldw */
#define U2_DLIN_W_PACKED13 1 /* w: the units u2_dlinear_pack_bf16 wrote (stream-K schedule only; ldw unused) */
typedef struct u2_dlinear_desc {
  int32_t B, N, K;
  int64_t ldx, ldw, ldy, ldr, ldxg;
  int32_t y_dtype;
  float* ws;
  int32_t* counters;
  const float* ssq_in;
  float eps;
  const void* residual;
  int32_t silu_pair;
  const float* gamma_next;
  void* xg;
  float* ssq_out;
  float* ssq_zero;
  int32_t pdl; /* != 0: launch with programmatic stream serialization (weight prefetch overlaps the previous kernel) */
  void* dbg;   /* optional uint64 [grid][4][8] globaltimer stamps (tuning aid), normally NULL */
  int64_t ws_elems; /* capacity of ws in floats */
  /* multi-op launches only - fine-grained dataflow instead of a grid-wide wait before the first MMA of an op:
   * out_flags: int32 [ceil(N/128)] set to the step counter when a tile of THIS op is final;
   * dep_flags/dep_shift: flags of the op producing our x; k-block kb needs producer tile kb >> dep_shift
   * (1: 128 producer rows = 2 k-blocks; 0: a silu_pair producer, 128 rows = 64 activations = 1 k-block).
   * Ops linked this way must use disjoint ws / counters / x buffers (see engine.py). */
  const int32_t* dep_flags;
  int32_t dep_shift;
  int32_t* out_flags;
  int32_t sched; /* U2_DLIN_STREAMK128 (128-row tiles, stream-K + workspace reduction) or
                    U2_DLIN_TILES64 (whole 64-row tiles per CTA, no inter-CTA reduction) */
  int32_t w_format; /* U2_DLIN_W_BF16 or U2_DLIN_W_PACKED13; all ops of one multi-op launch share it */
} u2_dlinear_desc;
U2_API int u2_dlinear_bf16(const void* x, const void* w, void* y, const u2_dlinear_desc* desc, void* stream);
U2_API int64_t u2_dlinear_ws_elems(int32_t N, int32_t K); /* fp32 elements of workspace for an N x K linear */
/* Up to four DEPENDENT decode linears in one launch (o_proj -> gate|up -> down -> next qkv; the Linears of
 * Qwen3DecoderLayer.forward, transformers models/qwen3/modeling_qwen3.py:305-336, at q_len == 1): software grid
 * barriers between them (gridbar: uint32[4], monotonically increasing; target = *step_dev * #SMs, step_dev is
 * the per-step counter u2_decode_embed_bf16 bumps), the weight stream of op i+1 is prefetched while op i
 * drains. x[i], w[i], y[i], descs[i] as for u2_dlinear_bf16. */
/* Optional L2 look-ahead for u2_dlinear_multi_bf16: lookahead_units = per-CTA number of 16 KB weight tiles
 * prefetched into L2 beyond the shared-memory ring while an in-launch dependency is pending; w[j] (N[j] x K[j],
 * row stride ldw[j]) = weights the NEXT launch streams first, units[j] leading tiles per CTA are prefetched when
 * this launch has issued all of its own loads (covers the launch gap / the attention kernel in between). */
typedef struct u2_dlinear_next {
  int32_t pre_stages;   /* ring stages of the next op's weights requested before its dependency resolves (0 = all) */
  int32_t lookahead_units;
  int32_t n;            /* 0..2 */
  const void* w[2];
  int32_t N[2], K[2];
  int64_t ldw[2];
  int32_t units[2];
  int32_t w_format[2];  /* U2_DLIN_W_BF16 or U2_DLIN_W_PACKED13 (w[j] then holds packed units; N, K as unpacked) */
} u2_dlinear_next;
U2_API int u2_dlinear_multi_bf16(const void* const* x, const void* const* w, void* const* y,
                                 const u2_dlinear_desc* descs, int32_t n_ops, uint32_t* gridbar,
                                 const int32_t* step_dev, int32_t pdl, const u2_dlinear_next* next, void* stream);
/* Lossless 13-bit packing of a decode-linear weight w (bf16 [N, K], row stride ldw, K % 64 == 0) for the stream-K
 * schedule: every 128 x 64 unit becomes 13 328 B (out: ceil(N / 128) * K / 64 units, 16-byte aligned). Per unit,
 * base = max(emax - 31, 0) over the unit's exponent fields; an exponent e is stored as 0 when e == 0 and as e - base
 * otherwise, sign and mantissa as they are, every plane in wgmma A-fragment order (layout: csrc/dlinear_wgmma.cu).
 * Rows >= N are packed as +0. *bad (device int32) is incremented once per unit with a nonzero exponent <= base: a
 * matrix with any such unit must stay in bf16. Unpacking reproduces every bf16 bit. */
U2_API int u2_dlinear_pack_bf16(const void* w, int32_t N, int32_t K, int64_t ldw, void* out, int32_t* bad, void* stream);
/* x[b] = table[ids[b]]; xg[b] = bf16(x * gamma); ssq[b] = sum x^2; ssq_zero[b] = 0; *step_counter += 1
 * (start of a decode step; step_counter may be NULL). Replaces `embed_tokens(input_ids)` of the cached decode step
 * (transformers models/qwen3/modeling_qwen3.py:392) + the first half of the first layer's input RMSNorm. */
U2_API int u2_decode_embed_bf16(const int64_t* ids, const void* table, const float* gamma, void* x, void* xg,
                                float* ssq, float* ssq_zero, int32_t* step_counter, int32_t B, int32_t E,
                                int64_t vocab, void* stream);

/* Fused decode-step attention (one launch per layer): per-head RMSNorm (optional) + RoPE of the new q/k,
 * KV-cache append at position pos (or *pos_dev) and GQA attention over the pos + 1 cached keys.
 * qkv [B, (Hq + 2 Hkv) * dh] raw projections; caches [B, Hkv, Tmax, dh]; out [B, Hq * dh]. dh 32, 64, 96 or 128
 * (96: Phi-3-mini; the PV phase runs 24 lanes x 4 elements).
 * Replaces HF modeling_qwen3.py:263-288 at q_len == 1. */
typedef struct u2_fused_decode_desc {
  int32_t B, Hq, Hkv, dh, Tmax, pos;
  const int32_t* pos_dev;
  int64_t ldq, ldo;
  const float* q_norm_w;
  const float* k_norm_w;
  float eps;
  const float* inv_freq;
  float scale;
  int32_t kv_splits;   /* 0/1: one CTA per (sequence, KV head); 2/4/8: a cluster of that many CTAs splits the cached
                          keys and merges over distributed shared memory (fills the SMs when B * Hkv is small) */
  int32_t pdl;         /* != 0 (split-KV variant only): launch with programmatic stream serialisation - position read
                          and K/V prefetch overlap the tail of the preceding kernel, which must not write the cache */
  int32_t pos_per_seq; /* != 0: sequence b appends at pos_dev[b] and attends over pos_dev[b] + 1 keys (a batch of
                          prompts of different lengths; needs pos_dev); 0: pos_dev[0] (or pos) for every sequence */
  const int32_t* kv_src; /* beam-indirect cache: int32 [B, ld_kv_src]; sequence b reads the key / value of position
                            t < pos from cache row kv_src[b * ld_kv_src + t] (its new token is always appended to and
                            read from its own row). NULL: every sequence reads its own row (compiled without lookups) */
  int64_t ld_kv_src;     /* >= Tmax when kv_src != NULL */
  int32_t window;        /* sliding window (Phi-3): attend keys [max(0, pos - window + 1), pos] only, i.e. HF's
                            `kv_idx > q_idx - sliding_window` (transformers masking_utils.py:90-97, modeling_phi3.py:403);
                            the split-KV variant deals only the window's 32-key groups to its cluster. 0: no window
                            (compiled without it). The cache stays full-length: positions index it as before */
} u2_fused_decode_desc;
U2_API int u2_decode_attention_fused_bf16(const void* qkv, void* k_cache, void* v_cache, void* out,
                                          const u2_fused_decode_desc* desc, void* stream);

/* Row-wise top-k of fp32 scores, sorted descending (ties: lower index first), as torch.topk in the hard
 * TokenSelection (reference svr.py:75-91). out_idx[r, i] = index + r * idx_offset_per_row (int64). T <= 16384. */
U2_API int u2_topk_rows_f32(const float* scores, int64_t* out_idx, int32_t rows, int32_t T, int32_t K, int64_t ld,
                            int64_t idx_offset_per_row, void* stream);

/* Fused attention forward, head_dim 64, non-causal (ViT3D): out = softmax(q k^T * scale) v, scores never leave
 * the SM (wgmma: S, P and the running O stay in registers).
 * q [B, Sq, H, 64], k [B, Sk, H, 64], v [B, Sk, H, 64] as strided views (element strides *_sb batch, *_ss token,
 * *_sh head; d contiguous) - typically the three slices of one fused QKV activation; v is consumed as stored (MN-major
 * B operand of the PV product, no transposed copy); out [B, Sq, H*64] (strides out_sb, out_ss). All strides multiples
 * of 8 elements.
 * Replaces MONAI SABlock einsum/softmax/einsum (reference vit.py:100-105,120-122). */
typedef struct u2_fa_desc {
  int32_t B, H, Sq, Sk, dh;
  float scale;
  int64_t q_sb, q_ss, q_sh;
  int64_t k_sb, k_ss, k_sh;
  int64_t v_sb, v_ss, v_sh;
  int64_t out_sb, out_ss;
  float* lse; /* optional fp32 [B, H, Sq]: log-sum-exp of the scaled score rows (training: the backward rebuilds the
                 probabilities as exp(scale * q.k - lse) in the score GEMM's epilogue); NULL at inference */
} u2_fa_desc;
U2_API int u2_flash_attention_d64_bf16(const void* q, const void* k, const void* v, void* out, const u2_fa_desc* desc,
                                       void* stream);

/* Sampled decoding head: ids[b] ~ multinomial(top_p(top_k(softmax(logits[b] / temperature)))) - the HF warper chain
 * behind generate(do_sample=True, temperature, top_k, top_p) used by the reference's eval scripts
 * (eval/mrg.py:74-75). top_k <= 0 disables top-k, top_p = 1 disables nucleus filtering. Counter-based RNG
 * keyed by (seed, step or *step_dev, row). */
U2_API int u2_sample_f32(const float* logits, int64_t* out, int32_t B, int32_t V, int64_t ld, float temperature,
                         int32_t top_k, float top_p, uint64_t seed, const int32_t* step_dev, int32_t step,
                         void* stream);

/* Same head (HF _sample with do_sample=True, generation/utils.py:2791; reference eval/mrg.py:74-75,
 * src/train/dpo_u2trainer.py:71-79) with its parameters in DEVICE memory (24 bytes): a captured decode step reads them at
 * replay time, so a new seed / temperature / top-k / top-p per request (HF generate kwargs) needs one small
 * host-to-device copy, not a new capture. The caller validates temperature > 0 and 0 < top_p <= 1. */
typedef struct u2_sample_params {
  float temperature;
  int32_t top_k;
  float top_p;
  int32_t reserved;
  uint64_t seed;
} u2_sample_params;
U2_API int u2_sample_dev_f32(const float* logits, int64_t* out, int32_t B, int32_t V, int64_t ld,
                             const u2_sample_params* params_dev, const int32_t* step_dev, int32_t step, void* stream);

/* Logits processors of HF generate(repetition_penalty, no_repeat_ngram_size, bad_words_ids, min_new_tokens /
 * min_length), in place on logits [B, V] (row stride ld) before u2_argmax_f32 / u2_sample_dev_f32. Replaces, in this
 * order, RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor, NoBadWordsLogitsProcessor and
 * MinLengthLogitsProcessor / MinNewTokensLengthLogitsProcessor (transformers generation/logits_process.py, built by
 * GenerationMixin._get_logits_processor; reference call src/model/language_model/u2llama.py:123-126).
 * History: t = *step_dev (or step when step_dev is NULL) generated tokens, t <= hist_cap. When t > 0 the token fed to
 * this step, ids[b], is first stored at hist[b * ld_hist + t - 1]; the processors then read hist[b, 0..t-1]. A decode
 * step that bumps *step_dev before this launch can therefore be captured in a CUDA graph.
 *   penalty != 1: every distinct history token v gets x < 0 ? x * penalty : x * inv_penalty, from its unprocessed x
 *                 (inv_penalty = fp32(1 / fp32(penalty)), which is how torch evaluates `scores / penalty` on CUDA);
 *   ngram = n > 0: hist[i + n - 1] -> -inf for every i with hist[i .. i+n-2] == hist[t-n+1 .. t-1];
 *   bad words:    word w is bad_tok[bad_off[w] .. bad_off[w+1]); a one-token word is always -inf, a longer word bans its
 *                 last token when its length is <= t and its prefix equals the end of the history; -0.0 becomes +0.0
 *                 in every row (HF adds a 0 / -inf bias row);
 *   min_new:      eos[0 .. n_eos) -> -inf while t < min_new.
 * The parameters live in DEVICE memory (like u2_sample_params): a captured step picks up a new request's values from
 * one host-to-device copy. The caller validates them: penalty > 0, ngram >= 0, every token id in [0, V), n_bad words
 * of at least one token within the capacities below. Dynamic shared memory: one bit per vocabulary entry. */
#define U2_LP_MAX_EOS 8
#define U2_LP_MAX_BAD_WORDS 256
#define U2_LP_MAX_BAD_TOKENS 2048
typedef struct u2_logits_proc_params {
  float penalty;     /* 1.0: off */
  float inv_penalty;
  int32_t ngram;     /* 0: off */
  int32_t min_new;   /* 0: off */
  int32_t n_eos;
  int32_t n_bad;     /* 0: off */
  int32_t eos[U2_LP_MAX_EOS];
  int32_t bad_off[U2_LP_MAX_BAD_WORDS + 1];
  int32_t bad_tok[U2_LP_MAX_BAD_TOKENS];
} u2_logits_proc_params;
U2_API int u2_logits_process_f32(float* logits, int32_t B, int32_t V, int64_t ld, const int64_t* ids, int32_t* hist,
                                 int64_t ld_hist, int32_t hist_cap, const u2_logits_proc_params* params_dev,
                                 const int32_t* step_dev, int32_t step, void* stream);

/* Continuous batching (generate_batch): every row of the decode batch is a slot that holds one sample of one request,
 * admitted and retired independently of the other rows. The per-slot state lives in DEVICE memory, one record per row,
 * so one captured decode step serves every request that passes through the slots:
 *   seed     the request's sampling seed;
 *   row      the RNG row: j for the request's j-th sample (num_return_sequences);
 *   count    tokens generated so far = the request's own step (what *step_dev is for a request decoded alone);
 *   max_new  the request's max_new_tokens;
 *   done     0: decoding; 1: finished or never admitted (the slot feeds pad and keeps its cache length).
 * u2_sample_slots_f32 and u2_logits_process_slots_f32 are u2_sample_dev_f32 / u2_logits_process_f32 with the seed,
 * the RNG row and the step (history length) of row b read from slots[b]: a slot draws and processes exactly what its
 * request would draw and process alone. u2_slot_update runs after the pick: for every slot with done == 0 it stores
 * ids[b] at out[b * ld_out + count] (when count < ld_out), increments count, and sets done on an EOS id of
 * params_dev->eos or on count == max_new; a slot that goes on advances length[b] and length_plus1[b] (both optional).
 * Every done slot gets ids[b] = params_dev->pad. */
typedef struct u2_slot_state {
  uint64_t seed;
  int32_t row;
  int32_t count;
  int32_t max_new;
  int32_t done;
} u2_slot_state;
typedef struct u2_slot_params {
  int64_t pad;
  int32_t n_eos;     /* <= U2_LP_MAX_EOS */
  int32_t eos[U2_LP_MAX_EOS];
  int32_t reserved;
} u2_slot_params;
U2_API int u2_sample_slots_f32(const float* logits, int64_t* out, int32_t B, int32_t V, int64_t ld,
                               const u2_sample_params* params_dev, const u2_slot_state* slots, void* stream);
U2_API int u2_logits_process_slots_f32(float* logits, int32_t B, int32_t V, int64_t ld, const int64_t* ids,
                                       int32_t* hist, int64_t ld_hist, int32_t hist_cap,
                                       const u2_logits_proc_params* params_dev, const u2_slot_state* slots,
                                       void* stream);
U2_API int u2_slot_update(int64_t* ids, int32_t B, u2_slot_state* slots, int64_t* out, int64_t ld_out,
                          const u2_slot_params* params_dev, int32_t* length, int32_t* length_plus1, void* stream);

/* Generation scores (HF generate(return_dict_in_generate, output_scores, output_logits) and continuous batching's
 * return_logprobs), written inside the captured decode step. A feature that is off launches none of these.
 * u2_row_store_params: the destination of a step-indexed row store, in DEVICE memory so that one captured step serves
 * every call and chunk (the host rewrites the block before the first, eager, step of each chunk). Row r of step t is
 * stored at dst + t * ld_step + r * ld_row; a step outside [0, steps) is not stored.
 *   u2_store_rows_f32    copies src [rows, V] (row stride ld_src) to the rows of step t = *step_dev (or step when
 *                        step_dev is NULL): the raw logits, greedy scores and beam scores of that step.
 *   u2_sample_out_f32    u2_sample_dev_f32 (step from step_dev / step) or u2_sample_slots_f32 (slots not NULL; then
 *                        step_dev must be NULL) with the same draw, bit for bit, that also writes, when not NULL,
 *                        scores_dev's row: x * (1 / temperature) where the top-k / top-p cut keeps it, -inf elsewhere
 *                        (what HF's warpers hand the multinomial), and logprob[b] = log softmax of that row at the pick.
 *   u2_pick_logprob_f32  logprob[b] = logits[b, ids[b]] - logsumexp(logits[b]) (the greedy pick's log-prob).
 *   u2_slot_update_lp    u2_slot_update that also stores lp_in[b] at lp_out[b * ld_out + count] for every live slot. */
typedef struct u2_row_store_params {
  float* dst;
  int64_t ld_step;
  int64_t ld_row;
  int32_t steps;
  int32_t reserved;
} u2_row_store_params;
U2_API int u2_store_rows_f32(const float* src, int32_t rows, int32_t V, int64_t ld_src,
                             const u2_row_store_params* params_dev, const int32_t* step_dev, int32_t step, void* stream);
U2_API int u2_sample_out_f32(const float* logits, int64_t* out, int32_t B, int32_t V, int64_t ld,
                             const u2_sample_params* params_dev, const int32_t* step_dev, int32_t step,
                             const u2_slot_state* slots, const u2_row_store_params* scores_dev, float* logprob,
                             void* stream);
U2_API int u2_pick_logprob_f32(const float* logits, int32_t B, int32_t V, int64_t ld, const int64_t* ids,
                               float* logprob, void* stream);
U2_API int u2_slot_update_lp(int64_t* ids, int32_t B, u2_slot_state* slots, int64_t* out, int64_t ld_out,
                             const float* lp_in, float* lp_out, const u2_slot_params* params_dev, int32_t* length,
                             int32_t* length_plus1, void* stream);

/* Beam search (HF generate(num_beams=K, length_penalty, early_stopping): GenerationMixin._beam_search, transformers
 * generation/utils.py, with the prompt length 0 of generate(inputs_embeds=...)) inside the captured decode step.
 * Prompt b owns rows b*K .. b*K+K-1 of the decode batch; row b*K+k is HF's running beam k. One step:
 *   u2_log_softmax_f32: lp = log_softmax(logits) (fp32, separate buffer; u2_logits_process_f32 may then run on lp);
 *   u2_beam_topk_f32:   per row, the top C = beams_to_keep of lp[v] + running[row], sorted (score descending, token
 *                       ascending on ties) into cand_val / cand_tok [rows, U2_BEAM_MAX_KEEP];
 *   u2_beam_step:       per prompt, the top C of its K*C row candidates (ties: lower beam * V + token), the stopping
 *                       criteria (token in eos, or t + 1 == max_new_tokens), the next running beams, the finished
 *                       hypotheses (score logprob_sum / (t+1)^length_penalty, -1e9 masks as HF adds them), the early-stop
 *                       heuristic and the prompt's done flag. A done prompt is frozen: later steps change nothing of it.
 * t = *step_dev (or step) = tokens generated before this step's. State (device memory, set up by the caller):
 *   running [rows]          running beam scores, {0, -1e9, ...} per prompt at t = 0
 *   fin_score [rows]        finished hypotheses per prompt, best first, -1e9 at t = 0
 *   fin_info [rows][4]      (is finished, step t of its last token or -1, parent beam, last token), (0, -1, 0, 0) at t = 0
 *   flags [prompts][2]      (early-stop heuristic unsatisfied, done), (1, 0) at t = 0
 *   ids [rows] int64        the next token of every row (the decode step's input)
 *   rec [rec_rows][rows][2] (token, parent beam) of every running row after step t: the output is backtracked from it
 *   kv_src [rows, ld_kv_src] the cache indirection of u2_fused_decode_desc: row k of prompt b takes row parent_k's
 *                           entries at the positions that hold K/V (pos_dev[b*K] + 1 of them after a decode step, pos_dev[b*K]
 *                           at t = 0) and its own row at the next position
 *   hist [rows, ld_hist]    optional: the u2_logits_process_f32 history, first t columns reordered like kv_src.
 * Parameters in DEVICE memory, so a captured step picks up a new request's values; the caller validates them. */
#define U2_BEAM_MAX_BEAMS 16
#define U2_BEAM_MAX_EOS 8
#define U2_BEAM_MAX_KEEP 144 /* max(2, 1 + n_eos) * num_beams */
typedef struct u2_beam_params {
  double length_penalty;
  int32_t num_beams;       /* K, 2..U2_BEAM_MAX_BEAMS */
  int32_t beams_to_keep;   /* max(2, 1 + n_eos) * K */
  int32_t early_stopping;  /* 0: False (heuristic), 1: True, 2: "never" */
  int32_t max_new_tokens;
  int32_t n_eos;
  int32_t reserved;
  int32_t eos[U2_BEAM_MAX_EOS];
} u2_beam_params;
typedef struct u2_beam_step_desc {
  const u2_beam_params* params;
  int32_t prompts, V;
  const float* cand_val;
  const int32_t* cand_tok;
  float* running;
  float* fin_score;
  int32_t* fin_info;
  int32_t* flags;
  int64_t* ids;
  int32_t* rec;
  int64_t ld_rec;
  int32_t rec_rows;
  int32_t* kv_src;
  int64_t ld_kv_src;
  const int32_t* pos_dev;
  int32_t* hist;
  int64_t ld_hist;
  int32_t hist_cap;
  const int32_t* step_dev;
} u2_beam_step_desc;
U2_API int u2_log_softmax_f32(const float* x, float* y, int32_t rows, int32_t V, int64_t ldx, int64_t ldy, void* stream);
U2_API int u2_beam_topk_f32(const float* logprobs, int64_t ld, int32_t rows, int32_t V, const float* running,
                            const int32_t* flags, const u2_beam_params* params_dev, float* cand_val, int32_t* cand_tok,
                            void* stream);
U2_API int u2_beam_step(const u2_beam_step_desc* desc, int32_t step, void* stream);

/* Fused lm_head + selective log-softmax (the DPO / SFT log-probability head) -----------------------------------
 * logp[r] = log_softmax(hidden[r] . W^T)[labels[r]]  (0 where labels[r] < 0) without materialising the [R, V] logits:
 * the GEMM's epilogue reduces every 128-column half tile to (max, sum exp, sum) per row, a second small kernel merges
 * them. Replaces lm_head + `selective_log_softmax(logits, labels)` in u2DPOTrainer.concatenated_forward
 * (src/train/dpo_u2trainer.py:267-300; [2B, 1024, 151936] logits = 622 MB per pair in bf16) and HF's
 * ForCausalLMLoss in forward(labels=...) (src/model/language_model/u2llama.py:76-87).
 * hidden [R, E] bf16 (row stride ldh), W [V, E] bf16 (row stride ldw), labels int64 [R]; optional outputs: lse [R]
 * (log-sum-exp), logit_sum [R] (sum of the row's V logits: the trainer's mean_*_logits statistics,
 * dpo_u2trainer.py:343-350), nll_acc [2] (+= sum of -logp and the number of labelled rows; the caller zeroes it).
 * ws: workspace of u2_logprob_ws_bytes(R, V) bytes, 16-byte aligned. */
typedef struct u2_logprob_desc {
  int32_t R, V, E;
  int64_t ldh, ldw;
  const int64_t* labels;
  void* ws;
  int64_t ws_bytes;
  float* lse;
  float* logit_sum;
  float* nll_acc;
} u2_logprob_desc;
U2_API int64_t u2_logprob_ws_bytes(int32_t R, int32_t V);
U2_API int u2_lmhead_logprob_bf16(const void* hidden, const void* W, float* logp, const u2_logprob_desc* desc,
                                  void* stream);

/* Volume preprocessing in front of the path (SURVEY.md section 8f-1) ------------------------------------------------
 * The reference's u2Transform.adaptive_resize (src/utils/u2Transform.py:62-122, validation pipeline :47-56) on a volume
 * that is already on the device: ScaleIntensityRangePercentiles(lower, upper -> [0, 1], clip) -> CropForeground (> 0) ->
 * anti-aliased trilinear resize (align_corners) so that the larger in-plane side becomes `target` (depth kept when it is
 * <= pad_depth, resized to pad_depth otherwise) -> zero pad to [pad_depth, target, target].
 * vol: fp32 [D, H, W] (the reference's data[0] after get_fdata().transpose(2, 0, 1)); out: fp32 [pad_depth, target,
 * target] (viewed as [pad_depth / 32, 32, target, target] it is the `images` tensor of one study). info (device memory)
 * receives the data-dependent quantities; nothing is synchronised with the host. status != 0 flags the inputs on which
 * the reference itself fails or degenerates (the output is then all zeros, except U2_PP_FLAT_INTENSITY). */
#define U2_PP_OK 0
#define U2_PP_EMPTY_FOREGROUND 1  /* no voxel above the lower percentile */
#define U2_PP_DEGENERATE_SHAPE 2  /* a resized extent of 0, or an anti-aliasing kernel wider than 129 taps */
#define U2_PP_FLAT_INTENSITY 3    /* a_min == a_max: MONAI returns img - a_min unscaled */
typedef struct u2_preprocess_info {
  double a_min, a_max;      /* the two percentiles (np.percentile, linear interpolation, float64) */
  int32_t lo[3], hi[3];     /* foreground box [lo, hi) on (D, H, W) */
  int32_t out[3];           /* resized extents on (D, H, W) before padding */
  float sigma[3];           /* anti-aliasing sigma per axis (0: none) */
  int32_t tail[3];          /* Gaussian half width in taps */
  int32_t status;           /* U2_PP_* */
} u2_preprocess_info;
typedef struct u2_preprocess_desc {
  int32_t D, H, W;
  int32_t target, pad_depth;
  double lower_pct, upper_pct;
  void* ws;                 /* u2_preprocess_ws_bytes(D, H, W) bytes, 256-byte aligned */
  int64_t ws_bytes;
} u2_preprocess_desc;
U2_API int64_t u2_preprocess_ws_bytes(int32_t D, int32_t H, int32_t W);
U2_API int u2_preprocess_volume_f32(const float* vol, float* out, u2_preprocess_info* info,
                                    const u2_preprocess_desc* desc, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* U2B200_H_ */
