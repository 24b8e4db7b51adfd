/*
 * jlama_b200.h -- C ABI of libjlama_b200.so, the Hopper (sm_90a) back-end for
 * tjake/Jlama's quantized forward pass.
 *
 * This is the drop-in boundary: plain C types only (pointers, ints, sizes), the
 * conventions jextract/Panama-FFI binds (the reference's existing natives:
 * jlama-native/src/main/c/simd/vector_simd.h:22-39 and
 * jlama-native/src/main/c/gpu/vector_gpu.h:7-19).  Each entry point cites the
 * reference interface it replaces.  Reference paths are relative to
 * /root/reference; "core/" = jlama-core/src/main/java/com/github/tjake/jlama/,
 * "native/java/" = jlama-native/src/main/java/com/github/tjake/jlama/tensor/operations/.
 *
 * Conventions
 *  - every function returns int status (JL_OK or a negative JL_ERR_*) or an
 *    int64 handle with -1 = failure (vector_gpu.h:10-15 convention).  Nothing
 *    aborts the process (the reference GPU natives call exit(),
 *    vector_gpu.c:96,116 -- deliberately not reproduced).
 *  - there is no CPU fallback: with no usable sm_90 device jl_init fails.
 *  - thread-safe: calls on one jl_ctx are serialised internally; the entry points
 *    of one jl_model serialise on the model's own lock and run on its own stream
 *    (request threads may call jl_model_generate concurrently, one session each).
 *  - dtype codes: Jlama DType (core/safetensors/DType.java) subset.
 */
#ifndef JLAMA_B200_H
#define JLAMA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define JL_OK 0
#define JL_ERR_INVALID (-1)     /* IllegalArgumentException analogue (Guava Preconditions in the reference) */
#define JL_ERR_CUDA (-2)        /* CUDA runtime error; see jl_last_error */
#define JL_ERR_OOM (-3)         /* device memory exhausted (NativeGPUTensorOperations.java:145-150 "limitReached") */
#define JL_ERR_UNSUPPORTED (-4) /* UnsupportedOperationException analogue (TestOperations.java:140 relies on it) */
#define JL_ERR_NCCL (-5)

/* most sessions one jl_model_decode / jl_model_decode_sample call accepts (also bounded by the model's max_sessions) */
#define JL_MAX_DECODE_ROWS 64
/* most top alternatives a logprob call returns per token (OpenAI's top_logprobs limit) */
#define JL_MAX_LOGPROBS 20

/* dtypes */
#define JL_F32 0
#define JL_BF16 1
#define JL_Q4 2 /* core/tensor/Q4ByteBufferTensor.java:34-259: 32-element blocks, byte j = q[j] | q[j+16]<<4, separate f32 scales [rows, cols/32] */
#define JL_I8 3 /* core/tensor/Q8ByteBufferTensor.java:37-223: int8 + f32 scale per 32 */

typedef struct jl_ctx jl_ctx;
typedef struct jl_model jl_model;

/* ---- lifecycle: replaces init_gpu (vector_gpu.h:7, vector_gpu.c:227-239) -------------- */
/* info[0]=free bytes, [1]=total bytes, [2]=SM count, [3]=compute capability*10 (90 for H100). */
int jl_init(int device, jl_ctx **out, int64_t *info /* nullable, int64[4] */);
int jl_shutdown(jl_ctx *ctx);
/* never NULL.  errno style: the text of the calling thread's most recent failing call (any entry point of this library), or, if this
 * thread has not failed yet, the most recent failure of any thread on `ctx`.  Valid until the calling thread's next failing call. */
const char *jl_last_error(jl_ctx *ctx);
const char *jl_version(void);
int jl_sync(jl_ctx *ctx);
/* number of kernels this library launched since jl_init (bench.py's gpu_launches claim) */
int64_t jl_kernel_launches(jl_ctx *ctx);

/* kernel timeline: every GEMV / decode-attention launch made while tracing is on gets a slot of 16 words
 * {first CTA start ns, last CTA end ns, CTA 0 after its prologue ns, tag, CTA 0 start ns, 11 stage stamps}; tools/ktrace.py */
int jl_debug_ktrace(jl_ctx *ctx, int capacity);
int jl_debug_ktrace_clear(jl_ctx *ctx);
int jl_debug_ktrace_read(jl_ctx *ctx, uint64_t *out, int max_slots);
/* diagnostic: time the quantised GEMV kernel on device-resident operands.  `b_id` is a registered weight
 * [rows, k]; each of `iters` launches handles `n` consecutive rows starting at a rotating offset so that the
 * stream of weights is larger than L2; activations [m, k] f32 live in HBM.  mode: 0 = Q8-quantising prologue +
 * store, 1 = RMSNorm + Q8 prologue + store, 2 = f32 activations + store, 3 = Q8 prologue + residual epilogue.
 * Returns the average microseconds per launch measured with CUDA events around the whole sequence. */
int jl_debug_gemv_bench(jl_ctx *ctx, int64_t b_id, int n, int m, int mode, int iters, double *avg_us);

/* diagnostic: average microseconds of one wgmma prefill GEMM launch C[t, rows] = A_bf16[t, k] * W^T on
 * device-resident operands (W = registered Q4 tensor [rows, k]). */
int jl_debug_gemm_tc_bench(jl_ctx *ctx, int64_t b_id, int t, int iters, double *avg_us);

/* ---- TensorOperations.registerModelTensor (core/tensor/operations/TensorOperations.java:39;
 *      NativeGPUTensorOperations.java:104-151 -> register_tensor, vector_gpu.h:10) ------------
 * Copies a weight (and its Q4/I8 block scales) to HBM once; returns a tensor id, -1 on failure.
 * `rows` x `cols` is the logical shape; Q4 data is rows*cols/2 bytes, scales rows*cols/32 floats.
 * Unlike the reference (int size => < 2 GiB) sizes are 64-bit. */
int64_t jl_register_tensor(jl_ctx *ctx, int dtype, int64_t rows, int64_t cols, const void *data, const float *scales);
int jl_unregister_tensor(jl_ctx *ctx, int64_t id);

/* ---- TensorOperations.batchDotProduct (TensorOperations.java:62-72) with a registered B ----
 * Drop-in for gpu_gemm (vector_gpu.h:17) / gemm_q8_q4, gemm_f32_q4, gemm_f32, gemm_f32_bf16
 * (vector_simd.h:22-39).  A and R are HOST buffers (the Java MemorySegments):
 *   r[ldc*i + j - roffset] = sum_{t<k} A[i, a_col_off+t] * B[j, b_col_off+t],  i in [0,m), j in [n0,n0+n)
 * a_dtype in {JL_F32, JL_BF16, JL_I8}; for JL_I8 `a_scales` are the Q8 block scales [m, lda/32]
 * (produced by jl_quantize_q8 or by Jlama itself).  lda/ldc in elements.
 * Offsets follow NativeSimdTensorOperations.java:96-107 (roffset is subtracted from the output index,
 * vector_simd.c:344). */
int jl_gemm(jl_ctx *ctx, int a_dtype, const void *a, const float *a_scales, int a_col_off, int lda, int64_t b_id,
            int b_col_off, float *r, int roffset, int m, int n0, int n, int k, int ldc);
/* dotProductBatchChunk (TensorOperations.java:86-99; gemm_*_batch, vector_simd.h:24-39): one A, several B/R. */
int jl_gemm_batch(jl_ctx *ctx, int batch_num, int a_dtype, const void *a, const float *a_scales, int a_col_off, int lda,
                  const int64_t *b_ids, int b_col_off, float *const *r, int roffset, int m, int n0, int n, int k,
                  int ldc);
/* batchDotProduct on the wgmma tensor cores for m >= 16 rows of F32/BF16 activations against a registered Q4 or Q8_0 (JL_I8)
 * weight (prefill shape).  Same index semantics as jl_gemm; operands are rounded to BF16 (accumulation in F32), so
 * the result matches the reference's F32 x Q4 GEMM (PanamaTensorOperations.java:289-548) to ~1e-3 of max|C|, not bit-wise.
 * Requires k %% 64 == 0, n %% 128 == 0, n0 %% 128 == 0, b_col_off %% 64 == 0 (JL_ERR_UNSUPPORTED otherwise). */
int jl_gemm_tc(jl_ctx *ctx, int a_dtype, const void *a, int a_col_off, int lda, int64_t b_id, int b_col_off, float *r,
               int roffset, int m, int n0, int n, int k, int ldc);
/* batchDotProduct where B is a HOST tensor too (attention scores against a KV page held by Java,
 * CausalSelfAttention.java:324-330).  b_dtype in {JL_F32, JL_BF16}. */
int jl_gemm_host(jl_ctx *ctx, int a_dtype, const void *a, int a_col_off, int lda, int b_dtype, const void *b,
                 int b_col_off, int ldb, float *r, int roffset, int m, int n0, int n, int k, int ldc);

/* ---- remaining TensorOperations methods on HOST f32 buffers (TensorOperations.java:101-149) ----
 * All run as CUDA kernels (upload, kernel, read back); there is no CPU path. */
/* a[r, off:off+len] += b[(r or 0), off:off+len]; b_dtype in {JL_F32, JL_BF16, JL_Q4 (+b_scales)}
 * (PanamaTensorOperations.java:2151-2325) */
int jl_accumulate(jl_ctx *ctx, float *a, int a_rows, int lda, int b_dtype, const void *b, const float *b_scales,
                  int b_rows, int ldb, int offset, int length);
/* a *= b (PanamaTensorOperations.java:2062-2097) */
int jl_maccumulate(jl_ctx *ctx, float *a, int a_rows, int lda, const float *b, int b_rows, int ldb, int offset,
                   int length);
/* x[r, off:off+len] *= factor (PanamaTensorOperations.java:2474-2514) */
int jl_scale(jl_ctx *ctx, float factor, float *x, int rows, int ldx, int offset, int length);
/* y[yoff+i] += alpha * x[xoff+i] (PanamaTensorOperations.java:2567-2611) */
int jl_saxpy(jl_ctx *ctx, float alpha, const float *x, float *y, int xoffset, int yoffset, int limit);
/* y[0, yoff+i] += sum_r alpha[aoff+r] * x[xrow+r, xoff+i]  (TensorOperations.java:122-137,
 * PanamaTensorOperations.java:2614-2698) */
int jl_saxpy_batch(jl_ctx *ctx, const float *alpha, const float *x, int ldx, float *y, int xoffset, int yoffset,
                   int limit, int a_offset, int x_row_offset, int batch);
/* quantize(t, I8, offset, length) (TensorOperations.java:145-149; PanamaTensorOperations.java:1684-1774):
 * d = max/127, q = (byte)(x*(127/max) + 0.5f) truncating; writes q[rows, ldx] (only [offset, offset+length))
 * and scales[rows, ldx/32]. */
int jl_quantize_q8(jl_ctx *ctx, const float *x, int rows, int ldx, int offset, int length, int8_t *q, float *scales);
/* quantize(t, BF16, ...) : FloatConversions.float32ToBFloat16 RNE (core/math/FloatConversions.java:35-61) */
int jl_quantize_bf16(jl_ctx *ctx, const float *x, int rows, int ldx, int offset, int length, uint16_t *out);
/* AbstractTensor.quantize(Q4) weight quantiser on the GPU (Q4ByteBufferTensor.java:66-120);
 * byte-identical to the reference's files (SURVEY 8f.1). */
int jl_quantize_q4_weights(jl_ctx *ctx, const float *x, int64_t rows, int64_t cols, uint8_t *q, float *scales);
/* AbstractTensor.quantize(I8) weight quantiser on the GPU (Q8ByteBufferTensor.java:47-90): iscale = 127/max,
 * q = (byte)Math.round(x * iscale) -- round half up, unlike the truncating activation quantiser above. */
int jl_quantize_q8_weights(jl_ctx *ctx, const float *x, int64_t rows, int64_t cols, int8_t *q, float *scales);

/* ---- layer-level fused entry points on HOST buffers --------------------------------------
 * The reference does these as scalar Java loops outside TensorOperations (SURVEY 7 "hard parts");
 * a device-resident layer subclass calls them instead. */
/* RMSNorm.forward (core/model/RMSNorm.java:34-56) */
int jl_rmsnorm(jl_ctx *ctx, const float *x, int rows, int ldx, int w_dtype, const void *w, float weight_adjustment,
               float eps, int embedding_length, int offset, int length, float *out);
/* LayerNorm.forward (core/model/LayerNorm.java:41-67; GPT-2 family): statistics over [offset, offset+length) divided by
 * embedding_length, out = (x - mean) * invStddev * w + bias.  Weights / bias F32 or BF16. */
int jl_layernorm(jl_ctx *ctx, const float *x, int rows, int ldx, int w_dtype, const void *w, int b_dtype, const void *bias, float eps,
                 int embedding_length, int offset, int length, float *out);
/* ActivationFunction.eval in place (core/math/ActivationFunction.java:29-37): type 0 SILU, 1 GELU (tanh form, also
 * GELU_PYTORCH_TANH), 2 TANH; double-precision math cast to float like the reference. */
#define JL_ACT_SILU 0
#define JL_ACT_GELU 1
#define JL_ACT_TANH 2
int jl_activation(jl_ctx *ctx, int type, float *x, int rows, int ld, int offset, int length);
/* VectorMath.softMax (core/math/VectorMath.java:69-90) */
int jl_softmax(jl_ctx *ctx, float *x, int offset, int length);
/* MLPBlock activation loop + maccumulate (core/model/MLPBlock.java:132-141): gate = silu(gate) * up */
int jl_silu_mul(jl_ctx *ctx, float *gate, const float *up, int rows, int ld, int offset, int length);
/* VectorMath.precomputeFreqsCis (core/math/VectorMath.java:148-165): out[end*dim/2][2] (cos,sin).
 * Host-side double libm, identical recipe to the reference. */
int jl_precompute_freqs_cis(int dim, int end, double theta, double scaling_factor, float *out);

/* ---- DistributedContext / KvBufferCache host logic (pure functions) -----------------------
 * core/model/DistributedContext.java:60-98 */
typedef struct {
    int embeddingSegmentStart, embeddingSegmentLength;
    int attentionSegmentStart, attentionSegmentLength;
    int hiddenSegmentStart, hiddenSegmentLength;
    int kvSegmentStart, kvSegmentLength;
    int headStart, headEnd, groupHeadStart, groupHeadEnd;
    int numberOfLayers, layerStart, layerEnd;
} jl_dctx;
int jl_dctx_build(int embedding_length, int attention_length, int hidden_length, int head_size, int head_group_size,
                  int num_layers, int model_shard, int num_model_shards, int layer_shard, int num_layer_shards,
                  jl_dctx *out);
/* KvBufferCache.computePageSize (core/tensor/KvBufferCache.java:224-280) */
int jl_kv_page_geometry(int num_layers, int context_length, int kv_segment_length, int dtype_size,
                        int64_t max_page_bytes, int *layers_per_page, int *ctx_per_page);

/* ---- device-resident model: AbstractModel / LlamaModel mirror -----------------------------
 * core/model/AbstractModel.java:100-183,295-329,443-491,516-646; core/model/llama/LlamaModel.java:68-184.
 * The host driver (C++) replays generate()'s exact call sequence with every layer op as a CUDA
 * kernel on device-resident activations, paged KV in HBM, CUDA-graphed decode. */
typedef struct {
    int context_length, embedding_length, hidden_length;
    int num_heads, num_kv_heads, num_layers, vocab_size, head_size;
    float layer_norm_eps;
    double rope_theta;   /* LlamaConfig.java:27-57 */
    double rope_scaling; /* only rope_type "linear" is honoured by the reference (:55-56) */
    int working_qtype;   /* JL_I8 (default, Q8 activations), JL_F32, JL_BF16 (AbstractModel.java:119-176) */
    int kv_dtype;        /* JL_F32 (reference default workingDType), JL_BF16, or JL_I8: Q8_0 pages whose rows are kv_len int8
                          * values then kv_len / 32 f32 scales, one per 32-element block (9/8 byte per element; head_size % 32 == 0,
                          * tp_size 1).  An I8 model decodes one session on the per-op graph, not the persistent kernel. */
    int max_batch;       /* jlama.max_batch_size, 256 (AbstractModel.java:57,304) */
    int max_sessions;    /* concurrent KvBuffers (KvBufferCache.java:58-60) */
    int max_context;     /* positions to reserve pages for (<= context_length); 0 = context_length */
    int tp_rank, tp_size; /* jlama-net model shard (DistributedContext modelShard/numModelShards) */
    int prefill_tensor_core; /* 1: prompt chunks of >= 16 rows use the wgmma BF16 GEMM path; 0: exact-integer SIMT path */
    int flags;           /* JL_MODEL_* */
    int num_experts;       /* 0 = dense MLP; > 0: Mixtral-style mixture of experts (core/model/MoEBlock.java) */
    int experts_per_token; /* top-k (MixtralConfig numberOfExpertsPerToken) */
    int arch;              /* JL_ARCH_LLAMA (Llama / Mixtral blocks) or JL_ARCH_GPT2 (core/model/gpt2/GPT2Model.java) */
} jl_model_config;

#define JL_ARCH_LLAMA 0
/* GPT-2 blocks: learned position embeddings (wte + wpe, GPT2Model.java:54-69), LayerNorm with bias (LayerNorm.java:41-67), biased
 * q/k/v/o and MLP projections (CausalSelfAttention.java:184-192,380; MLPBlock.java:126-128,160), GELU, no RoPE, lm_head tied to wte.
 * Slots: JL_T_EMBED = wte, JL_T_OUT_NORM = ln_f.weight; JL_L_ATTN_NORM / JL_L_FFN_NORM = ln_1 / ln_2 weights, JL_L_Q/K/V = the three
 * row blocks of c_attn.weight^T, JL_L_O = attn c_proj^T, JL_L_GATE = c_fc^T, JL_L_DOWN = mlp c_proj^T (JL_L_UP stays empty);
 * biases and wpe through jl_model_set_aux_tensor.  Single rank, dense (non-MoE). */
#define JL_ARCH_GPT2 1
/* jl_model_set_aux_tensor `which`: layer < 0 */
#define JL_AUX_POS_EMBED 0     /* wpe.weight [context_length, E] */
#define JL_AUX_OUT_NORM_BIAS 1 /* ln_f.bias [1, E] */
/* layer >= 0 */
#define JL_AUX_ATTN_NORM_BIAS 0 /* ln_1.bias */
#define JL_AUX_Q_BIAS 1         /* c_attn.bias split in three (GPT2Model.java:79) */
#define JL_AUX_K_BIAS 2
#define JL_AUX_V_BIAS 3
#define JL_AUX_O_BIAS 4         /* attn.c_proj.bias */
#define JL_AUX_FFN_NORM_BIAS 5  /* ln_2.bias */
#define JL_AUX_FC_BIAS 6        /* mlp.c_fc.bias [1, H] */
#define JL_AUX_PROJ_BIAS 7      /* mlp.c_proj.bias */

#define JL_MODEL_NO_GRAPH 1 /* launch decode kernels eagerly instead of through a CUDA graph */
#define JL_MODEL_NO_PERSISTENT 4 /* decode through the CUDA graph of per-op kernels instead of the persistent decode kernel */
/* bits 2 and 16 are retired (callers built against older headers may still set them; they are ignored): do not reuse them */

/* tensor slots */
#define JL_T_EMBED 0
#define JL_T_OUT_NORM 1
#define JL_T_LM_HEAD 2
#define JL_L_ATTN_NORM 0
#define JL_L_Q 1
#define JL_L_K 2
#define JL_L_V 3
#define JL_L_O 4
#define JL_L_FFN_NORM 5
#define JL_L_GATE 6
#define JL_L_DOWN 7
#define JL_L_UP 8

/* sizeof(jl_model_config) of this build: bindings that mirror the struct by hand (ctypes, FFM StructLayout) compare it with theirs */
int jl_model_config_size(void);
int jl_model_create(jl_ctx *ctx, const jl_model_config *cfg, jl_model **out);
/* layer < 0: global slot (JL_T_*); else per-layer slot (JL_L_*).  The tensor must already hold this
 * rank's shard (rows for q/k/v/gate/up, columns for o/down: LlamaModel.java:120-133,
 * Weights.getLoadOffsets core/safetensors/Weights.java:99-117).  The model holds a reference on every bound tensor until it is
 * freed; binding a slot again (here or in the two calls below) drops the reference on the tensor the slot held. */
int jl_model_set_tensor(jl_model *m, int layer, int slot, int64_t tensor_id);
/* Mixture-of-experts layers (core/model/mixtral/MixtralModel.java:88-105): expert = -1 binds the router
 * ("block_sparse_moe.gate.weight" [num_experts, E]); otherwise which = 0 w1 (gate_proj [H, E]), 1 w2 (down_proj [E, H]),
 * 2 w3 (up_proj [H, E]) of that expert.  The dense JL_L_GATE / JL_L_UP / JL_L_DOWN slots stay empty for MoE models. */
int jl_model_set_expert_tensor(jl_model *m, int layer, int expert, int which, int64_t tensor_id);
/* GPT-2 family: bias vectors ([1, n] F32/BF16) and the position-embedding table, see JL_AUX_* */
int jl_model_set_aux_tensor(jl_model *m, int layer, int which, int64_t tensor_id);
/* allocate scratch + KV page pool, build RoPE table, capture graphs.  JL_ERR_UNSUPPORTED for weights no kernel runs: F32 / BF16
 * gate/up of a Llama model or F32 / BF16 experts (their SiLU * up epilogue is implemented for Q4 / I8 weights only). */
int jl_model_finalize(jl_model *m);
int jl_model_free(jl_model *m);
/* KvBuffer lifecycle (KvBufferCache.getKvBuffer / close) */
int jl_model_reset_session(jl_model *m, int session);
/* AbstractModel.batchForward (:295-312): prompt tokens (HOST int32) in chunks of max_batch.  The one-segment case of
 * jl_model_batch_forward_multi. */
int jl_model_batch_forward(jl_model *m, int session, const int32_t *tokens, int n, int start_pos);
/* AbstractModel.sample (:443-491) on the last forwarded row of `session`: final norm, lm_head, argmax
 * (temperature 0) or softmax sampling with `uniform`.  logits_out (HOST, [vocab]) may be NULL. */
int jl_model_sample(jl_model *m, int session, float temperature, float uniform, int32_t *token_out, float *logits_out);
/* AbstractModel.batchForward for several sessions at once.  Segment i forwards lengths[i] tokens of sessions[i] starting at
 * start_pos[i]; tokens (HOST) holds the segments back to back.  Sessions distinct, 1 <= n_seg <= max_sessions.
 * Each segment is cut into max_batch-row chunks, and each chunk takes the tensor cores (prefill_tensor_core, >= 16 rows) or the exact
 * path; round r forwards the r-th chunk of every segment, the chunks of a round sharing forward passes of up to max(max_batch, max_sessions)
 * rows, so the weights are read once per pass instead of once per session.  Tensor-core chunks are bit-identical to the same segment
 * forwarded alone (jl_model_batch_forward); exact-path chunks agree with it to rounding (their GEMM row grouping depends on the pass).
 * Every argument is checked before any device work: a refused call (JL_ERR_INVALID) leaves all KV untouched. */
int jl_model_batch_forward_multi(jl_model *m, int n_seg, const int32_t *sessions, const int32_t *start_pos, const int32_t *lengths,
                                 const int32_t *tokens);
/* AbstractModel.sample on the last forwarded row of n distinct sessions, in one lm_head pass.  temperatures NULL = all arg-max;
 * rows at temperature != 0 use AbstractModel.sample's rule with uniforms[i] (as jl_model_decode_sample).
 * 1 <= n <= min(max_sessions, JL_MAX_DECODE_ROWS); sessions / temperatures / uniforms / tokens_out HOST [n]; logits_out HOST [n, vocab]
 * (raw logits) or NULL. */
int jl_model_sample_multi(jl_model *m, int n, const int32_t *sessions, const float *temperatures, const float *uniforms,
                          int32_t *tokens_out, float *logits_out);
/* One decode step for `n` sessions at once (the reference's "batch" = concurrent sessions):
 * forward(token_i, position_i) + sample at temperature 0, one CUDA-graph launch.
 * 1 <= n <= min(max_sessions, JL_MAX_DECODE_ROWS), sessions distinct; with Q4 / Q8_0 weights and Q8 activations every layer
 * GEMM streams its weights once for all n rows.
 * tokens/positions/next_tokens are HOST int32[n]; logits_out HOST [n, vocab] or NULL. */
int jl_model_decode(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                    int32_t *next_tokens, float *logits_out);
/* jl_model_decode with per-row sampling: a row whose temperature is not 0 draws its token with AbstractModel.sample's rule (:475-489:
 * exp((l - max) / T) in double, float running sum against `uniform`) from its logits row; rows at temperature 0 keep the arg-max.
 * temperatures / uniforms: HOST float[n].  logits_out receives the raw logits.  n is bounded as for jl_model_decode. */
int jl_model_decode_sample(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                           const float *temperatures, const float *uniforms, int32_t *next_tokens, float *logits_out);
/* generate() with a temperature: uniforms[i] (HOST float[n_new]) stands for the i-th ThreadLocalRandom.nextFloat() of the loop */
int jl_model_generate_sample(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, float temperature,
                             const float *uniforms, int32_t *out_tokens, double *timings_ms);
/* ---- top-k / top-p (nucleus) sampling: this project's rule (DESIGN §3.12), not the reference's -------------------------------
 * A row is FILTERED when temperature > 0 and (1 <= top_k < vocab or top_p < 1).  Filtered rows draw with integer weights
 * w_i = (uint64)(exp((l_i - max) / T) * 2^40): top-k keeps the weights >= the k-th largest (ties stay in), top-p then keeps the tokens
 * whose strictly-heavier kept mass is < top_p * (kept mass), and the token is the first kept one, in vocabulary order, whose prefix
 * sum of kept weights exceeds min(W - 1, floor(u * W)).  Every filtered row of a call is sampled in one kernel launch.  Unfiltered rows
 * keep the reference's rule (jl_model_decode_sample) bit for bit; rows at temperature 0 take the arg-max.
 * top_k (int32) and top_p (float) are nullable HOST [n] arrays (NULL = unfiltered).  Refused before any device work (JL_ERR_INVALID):
 * a temperature < 0 or NaN, top_k < 0, top_p outside (0, 1], a filtered row without uniforms or with a uniform outside [0, 1], or a
 * filtered row with a vocabulary above 2^23.  logits_out (nullable) always receives the raw logits. */
/* jl_model_decode_sample with per-row top_k / top_p; limits and session checks as jl_model_decode_sample */
int jl_model_decode_sample_topkp(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                                 const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms,
                                 int32_t *next_tokens, float *logits_out);
/* jl_model_sample_multi with per-row top_k / top_p; limits and session checks as jl_model_sample_multi */
int jl_model_sample_multi_topkp(jl_model *m, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                const float *top_p, const float *uniforms, int32_t *tokens_out, float *logits_out);
/* jl_model_generate_sample with one top_k / top_p for every token (top_k 0 and top_p 1: the reference's rule) */
int jl_model_generate_sample_topkp(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, float temperature,
                                   int top_k, float top_p, const float *uniforms, int32_t *out_tokens, double *timings_ms);
/* The sampling kernel on HOST buffers, for crafted rows: n rows of `vocab` logits at stride ld.  Every row at temperature > 0 is drawn
 * by the integer rule above (a row without a filter draws from the whole vocabulary), so uniforms[i] must lie in [0, 1] for those rows;
 * rows at temperature 0 take the arg-max (first index on ties).  1 <= vocab <= 2^23. */
int jl_sample_topkp(jl_ctx *ctx, int n, int vocab, const float *logits, int64_t ld, const float *temperatures, const int32_t *top_k,
                    const float *top_p, const float *uniforms, int32_t *out);
/* ---- token log-probabilities: this project's rule (DESIGN §3.13) ----------------------------------------------------------------
 * For a raw logits row l (what logits_out returns), m = max l and Z = sum_i exp(l_i - m) in double, lp_i = (float)((l_i - m) - log Z):
 * the model's distribution at temperature 1, before temperature and top-k / top-p, so a value does not depend on the sampling
 * parameters.  top_n (HOST int32 [n]) per row: -1 = no logprobs, 0 = the chosen token's only, up to JL_MAX_LOGPROBS alternatives: the
 * top_n tokens of largest logit (ties: lower id first).  Outputs, each HOST and nullable: lp_out [n] (the chosen token's logprob),
 * top_ids_out [n][JL_MAX_LOGPROBS] and top_lp_out [n][JL_MAX_LOGPROBS]; rows at -1 get NaN, slots past top_n get id -1 and NaN.
 * The bits depend on the row alone.  Refused before any device work: top_n outside -1..20 (JL_ERR_INVALID); tp_size > 1
 * (JL_ERR_UNSUPPORTED).  Tokens, logits_out and KV are those of the matching _topkp call with the same arguments. */
int jl_model_decode_logprobs(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                             const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms,
                             const int32_t *top_n, int32_t *next_tokens, float *lp_out, int32_t *top_ids_out, float *top_lp_out,
                             float *logits_out);
int jl_model_sample_multi_logprobs(jl_model *m, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                   const float *top_p, const float *uniforms, const int32_t *top_n, int32_t *tokens_out, float *lp_out,
                                   int32_t *top_ids_out, float *top_lp_out, float *logits_out);
/* jl_model_generate_sample_topkp with one top_n for every token; outputs [n_new] / [n_new][JL_MAX_LOGPROBS] */
int jl_model_generate_logprobs(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, float temperature, int top_k,
                               float top_p, const float *uniforms, int top_n, int32_t *out_tokens, float *lp_out, int32_t *top_ids_out,
                               float *top_lp_out, double *timings_ms);
/* Prompt scoring: jl_model_batch_forward_multi (same arguments, checks, KV and last-row effects, bit for bit) that also returns, for
 * entry k of each segment (laid out back to back like tokens), the logprob of token k given everything before it in the session and
 * the top_n (0..JL_MAX_LOGPROBS) alternatives at that position.  Entry 0 of every segment is NaN with id -1, also when the segment
 * continues a session (score context + continuation in one call to get the continuation's first token).  lp_out HOST [sum lengths];
 * top_ids_out / top_lp_out HOST [sum lengths][JL_MAX_LOGPROBS], nullable.  The first call allocates the scoring buffers (a 64-row logits
 * buffer when max_sessions is smaller); they live until jl_model_free. */
int jl_model_score_multi(jl_model *m, int n_seg, const int32_t *sessions, const int32_t *start_pos, const int32_t *lengths,
                         const int32_t *tokens, int top_n, float *lp_out, int32_t *top_ids_out, float *top_lp_out);
int jl_model_score(jl_model *m, int session, const int32_t *tokens, int n, int start_pos, int top_n, float *lp_out, int32_t *top_ids_out,
                   float *top_lp_out);
/* The logprob kernel on HOST buffers, for crafted rows: n rows of `vocab` logits at stride ld; targets (nullable) [n] in [-1, vocab), -1 =
 * none.  lp_out is required.  Refused (JL_ERR_INVALID) before any device work: n < 1, top_n outside -1..20, a target outside [-1, vocab),
 * a row with NaN or +inf or without a finite logit, a vocabulary above 2^20. */
int jl_logprobs(jl_ctx *ctx, int n, int vocab, const float *logits, int64_t ld, const int32_t *targets, const int32_t *top_n,
                float *lp_out, int32_t *top_ids_out, float *top_lp_out);
/* ---- frequency, presence and repetition penalties and logit bias: this project's rule (DESIGN §3.14) ------------------------------
 * Per row i (every array HOST):  history ids hist_ids[hist_off[i] .. hist_off[i+1]), of which the first hist_prompt[i] are prompt tokens
 * and the rest generated tokens in order (in a decode call including the token fed in that step); bias entries
 * (bias_ids[j], bias_vals[j]) for j in [bias_off[i], bias_off[i+1]).  With c = the count of a token among the generated tokens and s =
 * whether it occurs anywhere in the history, the processed logit of token t is, in float32 with one rounding per operation:
 *   b = l + bias_t (0 when t is not listed);  if s: b = b < 0 ? b * repetition : b / repetition;  b = b - (float)c * frequency;
 *   if c > 0: b = b - presence.
 * b replaces the raw logits as the input of the row's selection (arg-max, reference rule or top-k / top-p).  Logprobs, logits_out and
 * the KV stay those of the raw logits.  A NULL presence / frequency / repetition array is 0 / 0 / 1 for every row; a NULL hist_off or
 * bias_off is an empty list for every row; a NULL hist_prompt counts every history token as generated.  A row with presence = frequency
 * = 0, repetition = 1 and no bias entry is unpenalised: its processed row is its raw row. */
typedef struct {
    const float *presence, *frequency, *repetition;                   /* [n] each, nullable */
    const int32_t *hist_off /*[n+1]*/, *hist_prompt /*[n]*/, *hist_ids;
    const int32_t *bias_off /*[n+1]*/, *bias_ids;
    const float *bias_vals;
} jl_penalties;
/* The _logprobs calls with penalties (pen nullable: exactly the _logprobs call).  Refused before any device work, leaving the KV as it
 * was: presence or frequency outside [-2, 2], repetition outside (0, 100], a value that is not finite, a history or bias id outside
 * [0, vocab), hist_prompt outside [0, history length], a bias id twice in one row, a bias value outside [-100, 100], offsets that are
 * negative or decreasing (JL_ERR_INVALID); tp_size > 1 (JL_ERR_UNSUPPORTED).  The first call with a penalised row allocates the penalty
 * buffers (three min(max_sessions, 64) x vocab arrays); they live until jl_model_free. */
int jl_model_decode_penalized(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                              const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms,
                              const int32_t *top_n, const jl_penalties *pen, int32_t *next_tokens, float *lp_out, int32_t *top_ids_out,
                              float *top_lp_out, float *logits_out);
int jl_model_sample_multi_penalized(jl_model *m, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                    const float *top_p, const float *uniforms, const int32_t *top_n, const jl_penalties *pen,
                                    int32_t *tokens_out, float *lp_out, int32_t *top_ids_out, float *top_lp_out, float *logits_out);
/* jl_model_generate_logprobs with one presence / frequency / repetition and one bias list (n_bias entries) for every token; the history
 * of token k is the prompt followed by the k tokens generated before it. */
int jl_model_generate_penalized(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, float temperature, int top_k,
                                float top_p, const float *uniforms, int top_n, float presence, float frequency, float repetition,
                                int n_bias, const int32_t *bias_ids, const float *bias_vals, int32_t *out_tokens, float *lp_out,
                                int32_t *top_ids_out, float *top_lp_out, double *timings_ms);
/* The penalty kernel on HOST buffers, for crafted rows: n rows of `vocab` logits at stride ld -> out [n][vocab], the processed rows.
 * pen nullable.  Refused (JL_ERR_INVALID) before any device work as the model calls, and for n < 1. */
int jl_apply_penalties(jl_ctx *ctx, int n, int vocab, const float *logits, int64_t ld, const jl_penalties *pen, float *out);
/* ---- constrained decoding: per-row allowed-token masks, this project's rule (DESIGN §3.18) ----------------------------------------
 * A grammar engine above the model (JSON mode, JSON schema, regex, choices) turns its state into the set A of tokens allowed at the next
 * position; the calls below apply it.  A is a bitmask of words = (vocab + 31) / 32 uint32 words: token t is allowed when bit t % 32 of
 * word t / 32 is set; bits at or above vocab are ignored.  allow (HOST [n_allow][words]) holds the call's mask rows and allow_row (HOST
 * [n], -1 = unconstrained; NULL = no constrained row) gives each row its mask row; rows may share one.  For a constrained row:
 *   p_t = t in A ? b_t : -inf, b the processed row of the penalties (the raw row without them), so a penalty never brings a banned
 *   token back;  temperature 0: the arg-max of p, first index on ties;  temperature > 0: the top-k / top-p rule (DESIGN §3.12) on p
 *   with the row's top_k / top_p (0 / 1 = none), never the reference's prefix-sum rule, which can return a banned token.
 * Logprobs, logits_out and the KV stay those of the raw logits.  Unconstrained rows get exactly what the _penalized call gives them.
 * Refused before any device work, leaving the KV as it was: allow_row[i] outside [-1, n_allow), n_allow > 0 with a NULL allow, a
 * constrained row whose mask allows no token below vocab, everything the _penalized calls refuse (JL_ERR_INVALID); tp_size > 1
 * (JL_ERR_UNSUPPORTED).  allow_row NULL is the _penalized call, kernel launches included.  The first call with a constrained row
 * allocates the mask buffers (min(max_sessions, 64) x words uint32, on the device and pinned) and the penalty buffers; they live until
 * jl_model_free. */
int jl_model_decode_constrained(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                                const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms,
                                const int32_t *top_n, const jl_penalties *pen, int n_allow, const uint32_t *allow, const int32_t *allow_row,
                                int32_t *next_tokens, float *lp_out, int32_t *top_ids_out, float *top_lp_out, float *logits_out);
int jl_model_sample_multi_constrained(jl_model *m, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                      const float *top_p, const float *uniforms, const int32_t *top_n, const jl_penalties *pen, int n_allow,
                                      const uint32_t *allow, const int32_t *allow_row, int32_t *tokens_out, float *lp_out,
                                      int32_t *top_ids_out, float *top_lp_out, float *logits_out);
/* The selection of the calls above on HOST buffers, for crafted rows: n rows of `vocab` logits at stride ld -> out [n], the tokens.
 * Unconstrained sampled rows without a filter take the reference's rule, as in the model calls.  Refused (JL_ERR_INVALID) before any
 * device work as the model calls, and for n < 1 or a vocabulary above 2^23. */
int jl_select_constrained(jl_ctx *ctx, int n, int vocab, const float *logits, int64_t ld, const float *temperatures, const int32_t *top_k,
                          const float *top_p, const float *uniforms, const jl_penalties *pen, int n_allow, const uint32_t *allow,
                          const int32_t *allow_row, int32_t *out);
/* The mixture-of-experts router kernel on HOST buffers, for crafted rows: n rows of n_experts logits (contiguous) -> probs_out [n][n_experts]
 * (the reference's float softmax: (float)exp((double)(x - max)), a float sum in index order, a divide) and sel_out [n][k], the experts
 * of the replace-the-minimum top-k scan (MoEBlock.java:151-168) in the scan's order.  Refused (JL_ERR_INVALID) before any device work:
 * n < 1, n_experts outside 1..64, k outside 1..n_experts, a NULL pointer. */
int jl_moe_route(jl_ctx *ctx, int n, int n_experts, int k, const float *logits, float *probs_out, int32_t *sel_out);
/* The mixture-of-experts grouping kernel on HOST buffers, for crafted selections: sel [n][k] (experts in 0..n_experts-1) -> the
 * pairs p = row * k + slot sorted by expert, a stable counting sort (ascending p within an expert): counts_out / offsets_out
 * [n_experts] (the first place of each expert in pairs_out), pairs_out [n * k]; tiles_out [bound][4] {expert, first place, pairs, 0}
 * cut each expert's list into runs of at most R pairs, expert by expert, *ntiles_out of them, with
 * bound = (n * k + n_experts * (R - 1)) / R.  Refused (JL_ERR_INVALID) before any device work: n < 1, n_experts outside 1..64,
 * k outside 1..min(8, n_experts), R outside 1..64, a selection out of range, a NULL pointer. */
int jl_moe_group(jl_ctx *ctx, int n, int n_experts, int k, int R, const int32_t *sel, int32_t *counts_out, int32_t *offsets_out,
                 int32_t *pairs_out, int32_t *tiles_out, int32_t *ntiles_out);
/* AbstractModel.generate (:516-646) at temperature 0 over token ids: returns n_new tokens (the first is
 * sampled from the prompt's last row).  timings_ms (nullable double[2]) = {prompt, generate} wall ms like
 * Generator.Response.  logits_out HOST [n_new, vocab] or NULL. */
int jl_model_generate(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, int32_t *out_tokens,
                      float *logits_out, double *timings_ms);
/* device-side decode loop without per-token host round trips: feeds each step's argmax into the next
 * step on the GPU (tokens stay in HBM); copies the n_new tokens back at the end.  Used for `value`
 * in bench.py (inputs resident in HBM). */
int jl_model_decode_resident(jl_model *m, int session, int32_t first_token, int start_pos, int n_new,
                             int32_t *out_tokens);
/* test hooks: copy a K/V row (f32) or the hidden rows of the last batch_forward chunk to HOST */
int jl_model_read_kv(jl_model *m, int session, int layer, int position, int which /*0=K,1=V*/, float *out);
/* KvBufferCache.KvBufferPage persistence (core/tensor/KvBufferCache.java:121-176): write / read the allocated KV pages of a session
 * as  <dir>/<session_name>-L<layerPage>C<contextPage>.page  (raw little-endian page bytes, the reference's file naming and layout).
 * Return the number of pages written / read (>= 0) or a JL_ERR_*.  After a load the caller continues at the position it saved. */
int jl_model_kv_save(jl_model *m, int session, const char *dir, const char *session_name);
int jl_model_kv_load(jl_model *m, int session, const char *dir, const char *session_name);
/* Host spill of an idle session (SURVEY 8f.3 "device page pool, host spill/restore"): offload copies the allocated KV pages of `session`
 * to host memory, frees their HBM and leaves the slot empty; returns a handle (> 0) or a negative JL_ERR_*.  restore zeroes `session`
 * (any slot), brings the pages of `handle` back and forgets the handle; the caller continues at the position it stopped at.  discard
 * drops a handle that will not be restored.  kv_pages = the page-table entries a session references (a page it shares counts too).
 * A spill undoes sharing: offload copies shared pages to the host like the session's own and detaches them (the other sessions keep
 * them), and restore brings every page back as the session's own. */
int64_t jl_model_kv_offload(jl_model *m, int session);
int jl_model_kv_restore(jl_model *m, int session, int64_t handle);
int jl_model_kv_discard(jl_model *m, int64_t handle);
int jl_model_kv_pages(jl_model *m, int session);
/* ---- shared copy-on-write KV pages (DESIGN §3.15) --------------------------------------------------------------------------------
 * Fork: each dst[i] (HOST [n]) becomes what `src` holds for positions [0, positions).  Every context page wholly below `positions` is
 * shared: dst's entry points at src's page, no bytes move.  When positions % ctx_per_page != 0 the page holding positions - 1 gets a
 * private copy per destination (rows below positions, zeros above: the page an unforked session would hold), all in one kernel launch.
 * dst's other pages are released as by jl_model_reset_session, and dst's last row becomes src's, so jl_model_sample* on dst draws from
 * the prompt's last row.  A call that writes into a shared page (a forward rewound below the fork point, kv_load) first gives the writing
 * session a private copy holding the rows below the lowest position it writes there; the others keep the original.  reset_session
 * detaches shared pages, and jl_model_free frees each page once.  Refused before any device work, every session left as it was: n < 1,
 * a dst out of range, repeated or equal to src, positions outside [1, max_context], src without a page below positions
 * (JL_ERR_INVALID); tp_size > 1 (JL_ERR_UNSUPPORTED). */
int jl_model_kv_fork(jl_model *m, int src, int positions, int n, const int32_t *dst);
/* KV memory in use: pages_allocated counts a page shared by k sessions once, page_entries k times (the sum of kv_pages); each nullable.
 * pages_allocated includes the pages only retained prefixes hold. */
int jl_model_kv_page_stats(jl_model *m, int64_t *pages_allocated, int64_t *page_entries);
/* ---- retained prefixes (DESIGN §3.17): KV pages that outlive their session, for the scheduler's prefix cache ----------------------
 * A retained prefix is a handle holding a reference to each of a session's pages wholly below some position; it owns no page-table row.
 * Its references count like page-table entries: a session writing into a retained page copies it first, and reset_session, kv_offload
 * and jl_model_free treat retained pages as shared ones.  Refused before any device work, nothing changed: an unknown or released handle,
 * positions not a positive multiple of ctx_per_page or above the reserved context or the retained length, a session out of range or
 * without a page below positions (JL_ERR_INVALID); tp_size > 1 (JL_ERR_UNSUPPORTED). */
/* hold every page of `session` wholly below `positions` (a multiple of ctx_per_page, >= ctx_per_page); returns a handle > 0.  The
 * session is unchanged and keeps writing its later positions: they lie in pages the handle does not hold. */
int64_t jl_model_kv_retain(jl_model *m, int session, int positions);
/* `session` becomes what `handle` holds for [0, positions) (a multiple of ctx_per_page, <= the retained positions): entries below point
 * at the retained pages, no bytes move; its other pages are released or zeroed as by jl_model_reset_session.  last_hidden is not set:
 * forward at least one token before sampling. */
int jl_model_kv_attach(jl_model *m, int64_t handle, int positions, int session);
/* drop the handle's references; a page nothing else holds is freed */
int jl_model_kv_release(jl_model *m, int64_t handle);
/* handles alive, and pages held by handles and by no page-table entry (what releasing every handle would free); each nullable */
int jl_model_kv_retained(jl_model *m, int64_t *handles, int64_t *pages_retained_only);
int jl_model_read_hidden(jl_model *m, int session, float *out /* [embedding_length] last row */);
/* test hook: copy `n` floats of an internal activation buffer of the LAST forward/decode call to HOST (row 0 first).
 * which: 0 = x (hidden after the last layer), 1 = xb (after attention + residual), 2 = q, 3 = k, 4 = v (raw projections),
 * 5 = att (attention output), 6 = h (silu(gate) * up; in a mixture-of-experts model [max_batch][experts_per_token][H], expert i of row b
 * at row b * experts_per_token + i), 7 = logits, and for mixture-of-experts models only (JL_ERR_INVALID otherwise) 8 = the router
 * probabilities [max_batch][num_experts] and 9 = the selected experts [max_batch][experts_per_token] as int32 bit patterns;
 * for tensor-core prefill models only 10 = the up projection [max_batch][H] and 11 = the BF16 operand buffer (two BF16 per float
 * word); for GPT-2 models only 12 = the LayerNorm output [max_batch][E]: ln_2 of the last layer (the c_fc input) after a prompt
 * forward, ln_f of the sampled rows (the lm_head input) after a decode step or a sampling call. */
int jl_model_debug_read(jl_model *m, int which, float *out, int64_t n);
/* diagnostic: CTA 0's phase stamps (globaltimer ns) of the last persistent decode launch (tools/ptrace.py); phase tracing
 * is enabled with JL_PD_TRACE=1 in the environment when the model is created.  Returns the number of words written. */
int jl_model_debug_trace(jl_model *m, uint64_t *out, int64_t out_words);
/* how jl_model_decode executes for n sessions: 3 = persistent decode kernel (one cooperative launch per token, n == 1),
 * 1 = CUDA graph of per-op kernels, 0 = eager */
int jl_model_decode_mode(jl_model *m, int n);
/* per-token algorithmic bytes of the decode weight stream on this rank (roofline numerator) */
int64_t jl_model_weight_bytes(jl_model *m);
/* event-timed duration (ms) of the last jl_model_decode / decode_resident GPU work, measured with CUDA events on the model
 * stream.  gemv_ms (nullable) is always set to 0. */
int jl_model_last_timing(jl_model *m, double *total_ms, double *gemv_ms);

/* ---- JQ4 / JQ8 checkpoints: safetensors with Jlama's dtype strings "Q4" / "I8" + "<name>.qb" f32 block scales ------------
 * core/safetensors/SafeTensorSupport.java:54-102,215-332; Weights.java:49-66,99-179; SafeTensorIndex.java:59-236.
 * Files are mapped whole (64-bit), so the reference's <= 2 GiB mmap splits (SafeTensorIndex.java:121-236) are not needed. */
typedef struct jl_st jl_st;
#define JL_ST_F16 4 /* dtype code reported for F16 tensors (read-only; bound to a model as F32, Weights.java:137-152) */
/* path: a .safetensors file, or a directory with model.safetensors or model.safetensors.index.json + shards */
int jl_st_open(const char *path, jl_st **out);
int jl_st_close(jl_st *st);
const char *jl_st_last_error(void);
int jl_st_count(jl_st *st);
int jl_st_find(jl_st *st, const char *name); /* index or -1 */
/* tensors are ordered by data offset (TensorInfo.compareTo); dtype -1 = a dtype string this library does not know */
int jl_st_info(jl_st *st, int i, const char **name, int *dtype, int *ndim, int64_t *shape4, int64_t *nbytes);
const void *jl_st_data(jl_st *st, int i); /* pointer into the read-only mapping */
const char *jl_st_metadata(jl_st *st, const char *key); /* "__metadata__" entry or NULL */
int jl_st_majority_dtype(jl_st *st); /* Weights.findDType: ".qb" tensors not counted, F16 counts as F32 */
/* one file: 8-byte LE header length, JSON header (data_offsets relative to the data section), raw bytes in the given order */
int jl_st_write(const char *path, int n, const char *const *names, const int *dtypes, const int *ndims, const int64_t *shapes4,
                const void *const *data, const int64_t *nbytes, int n_meta, const char *const *meta_kv);
/* SafeTensorSupport.quantizeModel with the block quantisers on the GPU (byte-identical files): 2-D tensors whose name contains
 * none of the comma-separated `skip_csv` substrings (NULL = "norm", QuantizeCommand.java:36-38) and whose first dim is not 1
 * (AbstractTensor.java:284) become qtype (JL_Q4 / JL_I8) + "<name>.qb"; names starting with a `drop_csv` prefix are omitted. */
int jl_quantize_model(jl_ctx *ctx, const char *src_dir, const char *dst_dir, int qtype, const char *skip_csv, const char *drop_csv);
/* config.json -> jl_model_config (safetensors/Config.java:253-287, llama/LlamaConfig.java:27-57); working_qtype I8, F32 KV, tp 1 */
int jl_config_from_json(const char *config_json_path, jl_model_config *cfg);
/* LlamaModel.loadInputWeights / loadTransformerBlockWeights / loadOutputWeights (llama/LlamaModel.java:68-156): registers this
 * rank's shard of every tensor of the checkpoint (rows per Weights.getLoadOffsets :99-117, columns per AbstractTensor.sparsify)
 * and binds it; call jl_model_finalize afterwards.  ids_out receives the registered tensor ids (for jl_unregister_tensor). */
int jl_model_load_safetensors(jl_model *m, jl_ctx *ctx, jl_st *st, int64_t *ids_out, int ids_cap, int *n_ids);
/* this model's DistributedContext and shard count */
int jl_model_tp_layout(jl_model *m, jl_dctx *out, int *tp_size);

/* ---- concurrent sessions: request queue + iteration-level batching (csrc/jl_sched.cu) ------------------------------------
 * The reference runs one thread per request, each calling AbstractModel.generate (core/model/AbstractModel.java:516-646) on its own
 * KvBuffer (core/tensor/KvBufferCache.java:58-60; jlama-net/.../openai/OpenAIChatService.java:64-74,107-160).  Here requests queue in
 * front of the batched decode step: every jl_sched_step admits queued requests into free session slots (FIFO), forwards prompt chunks,
 * runs ONE decode step for all generating requests (rows of different lengths side by side, at most the model's rows-per-call per
 * backend call, each row greedy or sampled at its own temperature) and retires finished requests so that their slots are reused by the
 * next step.  When no slot is free, the least
 * recently finished kept session is spilled to host memory (KvBufferCache's pages are file-backed in the reference, :121-176; here the
 * idle session's pages leave HBM) and restored into any free slot when its follow-up arrives.  Under tensor parallelism every rank runs the same scheduler on the same request stream (it is deterministic).
 * Free the scheduler before its model. */
typedef struct jl_sched jl_sched;
/* request states */
#define JL_SCHED_QUEUED 0
#define JL_SCHED_PREFILL 1
#define JL_SCHED_DECODING 2
#define JL_SCHED_FINISHED 3
#define JL_SCHED_FAILED 4
/* Generator.FinishReason (core/model/functions/Generator.java) + the scheduler's own exits */
#define JL_FINISH_NONE 0
#define JL_FINISH_MAX_TOKENS 1 /* max_new tokens produced, or the reserved context is full (generate :538,:590) */
#define JL_FINISH_STOP_TOKEN 2 /* c.eosTokens.contains(next) (:604-608) */
#define JL_FINISH_CANCELLED 3
#define JL_FINISH_ERROR 4      /* a backend call failed for this request; jl_sched_last_error */
/* submit flags */
#define JL_SCHED_KEEP_SESSION 1 /* keep the session slot and its KV after the request finishes, for a continuation (the reference's
                                   session header: the next generate() on that UUID starts at kvmem.getCurrentContextPosition(), :533) */
#define JL_SCHED_CONSTRAINED 2  /* select every token of the request under the allowed-token mask its mask provider gives for it (DESIGN
                                   §3.18); needs jl_sched_set_mask_provider and a constraint backend */
/* the four model calls the policy is written against; all return JL_OK or a JL_ERR_* */
typedef struct {
    int (*reset_session)(void *user, int session);                                                   /* jl_model_reset_session */
    int (*batch_forward)(void *user, int session, const int32_t *tokens, int n, int start_pos);       /* jl_model_batch_forward */
    int (*sample)(void *user, int session, float temperature, float uniform, int32_t *token_out);     /* jl_model_sample */
    int (*decode)(void *user, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                  const float *temperatures, const float *uniforms, int32_t *next_tokens);            /* jl_model_decode_sample */
    /* optional, all three or none: host spill of kept sessions (jl_model_kv_offload / kv_restore / kv_discard) */
    int (*offload)(void *user, int session, int64_t *handle_out);
    int (*restore)(void *user, int session, int64_t handle);
    int (*discard)(void *user, int64_t handle);
} jl_sched_backend;
/* optional batched prompt calls (jl_model_batch_forward_multi / jl_model_sample_multi without logits), installed with
 * jl_sched_set_batch_backend.  With them a step runs: the slot preparation of every admitted request (offload / restore / reset), then
 * ONE forward_multi over every prompt chunk whose preparation succeeded, then one sample_multi per max_rows prompts that completed.
 * If forward_multi or sample_multi fails, every request in that call fails with JL_FINISH_ERROR; the others go on. */
typedef struct {
    int (*forward_multi)(void *user, int n_seg, const int32_t *sessions, const int32_t *start_pos, const int32_t *lengths,
                         const int32_t *tokens);
    int (*sample_multi)(void *user, int n, const int32_t *sessions, const float *temperatures, const float *uniforms,
                        int32_t *tokens_out);
} jl_sched_batch_backend;
/* optional top-k / top-p calls (jl_model_decode_sample_topkp / jl_model_sample_multi_topkp without logits), installed with
 * jl_sched_set_topkp_backend.  A decode or first-token call that holds at least one filtered request (temperature > 0 and top_k > 0 or
 * top_p < 1) goes through these for all of its rows; a call without one is exactly the jl_sched_backend / jl_sched_batch_backend call.
 * The first token of a filtered request goes through sample_multi_topkp also when no batch backend is installed (one row per call). */
typedef struct {
    int (*decode_topkp)(void *user, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                        const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms, int32_t *next_tokens);
    int (*sample_multi_topkp)(void *user, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                              const float *top_p, const float *uniforms, int32_t *tokens_out);
} jl_sched_topkp_backend;
/* optional logprob calls (jl_model_decode_logprobs / jl_model_sample_multi_logprobs without logits), installed with
 * jl_sched_set_logprob_backend.  A decode or first-token call that holds at least one request submitted with logprobs >= 0 goes through
 * these for all of its rows (top_n[i] = that request's logprobs, -1 for the others, top-k / top-p as in the top-k / top-p calls); a call
 * without one is exactly the call it would be without this backend.  The first token of such a request goes through
 * sample_multi_logprobs also when no batch backend is installed (one row per call). */
typedef struct {
    int (*decode_logprobs)(void *user, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                           const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms, const int32_t *top_n,
                           int32_t *next_tokens, float *lp_out, int32_t *top_ids_out, float *top_lp_out);
    int (*sample_multi_logprobs)(void *user, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                 const float *top_p, const float *uniforms, const int32_t *top_n, int32_t *tokens_out, float *lp_out,
                                 int32_t *top_ids_out, float *top_lp_out);
} jl_sched_logprob_backend;
/* optional penalty calls (jl_model_decode_penalized / jl_model_sample_multi_penalized without logits), installed with
 * jl_sched_set_penalty_backend.  A decode or first-token call that holds at least one request submitted with a penalty goes through these
 * for all of its rows (the other rows unpenalised, with empty histories; top_n and top-k / top-p as in the logprob calls); a call without
 * one is exactly the call it would be without this backend.  A penalised request's history is its own prompt followed by its generated
 * tokens: for a continuation of a kept session that is the continuation's prompt, not the earlier turns. */
typedef struct {
    int (*decode_penalized)(void *user, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                            const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms, const int32_t *top_n,
                            const jl_penalties *pen, int32_t *next_tokens, float *lp_out, int32_t *top_ids_out, float *top_lp_out);
    int (*sample_multi_penalized)(void *user, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                  const float *top_p, const float *uniforms, const int32_t *top_n, const jl_penalties *pen, int32_t *tokens_out,
                                  float *lp_out, int32_t *top_ids_out, float *top_lp_out);
} jl_sched_penalty_backend;
/* optional constrained calls (jl_model_decode_constrained / jl_model_sample_multi_constrained without logits) and the vocabulary they
 * select from, installed with jl_sched_set_constraint_backend.  A decode or first-token call that holds at least one JL_SCHED_CONSTRAINED
 * request goes through these for all of its rows (the others with allow_row -1; penalties, top_n and top-k / top-p as in the penalty
 * calls); a call without one is exactly the call it would be without this backend. */
typedef struct {
    int (*decode_constrained)(void *user, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                              const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms, const int32_t *top_n,
                              const jl_penalties *pen, int n_allow, const uint32_t *allow, const int32_t *allow_row, int32_t *next_tokens,
                              float *lp_out, int32_t *top_ids_out, float *top_lp_out);
    int (*sample_multi_constrained)(void *user, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                    const float *top_p, const float *uniforms, const int32_t *top_n, const jl_penalties *pen, int n_allow,
                                    const uint32_t *allow, const int32_t *allow_row, int32_t *tokens_out, float *lp_out, int32_t *top_ids_out,
                                    float *top_lp_out);
    int vocab; /* the mask width: (vocab + 31) / 32 words */
} jl_sched_constraint_backend;
/* The mask provider of JL_SCHED_CONSTRAINED requests: the caller's grammar engine.  Called once before every selection of such a
 * request -- its first token with n_generated 0, then each decode step with every token the request has generated so far, the one fed
 * in that step included (for a continuation: this request's tokens only).  It writes the allowed set of the next token into
 * allow_out [(vocab + 31) / 32] (zeroed before the call) and returns 0.  It runs on the stepping thread without the scheduler's lock
 * and gets a copy of the tokens: it may call jl_sched_result, jl_sched_cancel and the other request calls, but must not step.  A
 * non-zero return or a mask that allows no token below vocab fails that request alone (JL_FINISH_ERROR, jl_sched_last_error says
 * why); the other rows of its call go on.  When the grammar is complete the provider allows only stop tokens, and the request ends
 * with JL_FINISH_STOP_TOKEN (its first token is not stop-checked, as everywhere). */
typedef int(jl_sched_mask_fn)(void *user, int64_t request, const int32_t *generated, int n_generated, uint32_t *allow_out); /* a function
                                                                                                                     type: take it by pointer */
typedef struct {
    int admitted, prefill_tokens, decode_rows, decode_calls, finished; /* what this step (or run) did */
    int active, queued;                                                 /* afterwards */
    int spilled;                                                        /* kept sessions moved to host memory to free their slot */
} jl_sched_stats;
typedef struct {
    int state, finish_reason, session /* -1: none, or spilled */, start_pos, n_prompt, n_prefilled, n_generated, next_position;
    int spilled; /* 1: this finished request's kept KV lives in host memory; its continuation restores it into a free slot */
    int64_t submit_step, first_token_step, finish_step; /* scheduler step counters: queueing delay and time to first token in steps */
    /* host-clock milliseconds: waiting for a slot; admission -> first token (Generator.Response promptTimeMs, AbstractModel.java:561-568);
     * first token -> finish (generateTimeMs, :589,:623).  A phase still running is measured up to the call. */
    double queue_ms, prompt_ms, generate_ms;
} jl_sched_request_info_t;
/* max_active: session slots to use (<= the model's max_sessions; 0 = all).  prefill_tokens_per_step: prompt tokens forwarded per step over
 * all admitted requests (chunked prefill, bounds the latency a long prompt adds to the running requests' decode steps); 0 = no bound.
 * Each step forwards the prompt chunks of all admitted requests in one jl_model_batch_forward_multi call, samples their first tokens in
 * jl_model_sample_multi calls, and decodes every generating request in one jl_model_decode_sample call of up to
 * min(max_sessions, JL_MAX_DECODE_ROWS) rows. */
int jl_sched_create(jl_model *m, int max_active, int prefill_tokens_per_step, jl_sched **out);
/* the same policy over caller-supplied model calls (CPU tests drive it with the oracle; a host with its own model object plugs in here) */
int jl_sched_create_backend(const jl_sched_backend *be, void *user, int n_sessions, int max_rows_per_decode, int max_context,
                            int prefill_tokens_per_step, jl_sched **out);
/* install (both calls set) or remove (bb NULL) the batched prompt calls; before the first jl_sched_step only.  jl_sched_create installs
 * the model's jl_model_batch_forward_multi / jl_model_sample_multi; without them every prompt chunk is its own batch_forward + sample. */
int jl_sched_set_batch_backend(jl_sched *s, const jl_sched_batch_backend *bb);
/* install the top-k / top-p calls (both set); before the first jl_sched_step only.  jl_sched_create installs the model's
 * jl_model_decode_sample_topkp / jl_model_sample_multi_topkp. */
int jl_sched_set_topkp_backend(jl_sched *s, const jl_sched_topkp_backend *tb);
/* install the logprob calls (both set); before the first jl_sched_step only.  jl_sched_create installs the model's
 * jl_model_decode_logprobs / jl_model_sample_multi_logprobs. */
int jl_sched_set_logprob_backend(jl_sched *s, const jl_sched_logprob_backend *lb);
/* install the penalty calls (both set); before the first jl_sched_step only.  jl_sched_create installs the model's
 * jl_model_decode_penalized / jl_model_sample_multi_penalized. */
int jl_sched_set_penalty_backend(jl_sched *s, const jl_sched_penalty_backend *pb);
/* install the constrained calls (both set, vocab >= 1); before the first jl_sched_step only.  jl_sched_create installs the model's
 * jl_model_decode_constrained / jl_model_sample_multi_constrained and its vocab_size. */
int jl_sched_set_constraint_backend(jl_sched *s, const jl_sched_constraint_backend *cb);
/* install (fn NULL: remove) the mask provider of JL_SCHED_CONSTRAINED requests, called with `user`; before the first jl_sched_step only */
int jl_sched_set_mask_provider(jl_sched *s, jl_sched_mask_fn *fn, void *user);
/* optional fork call (jl_model_kv_fork), installed with jl_sched_set_fork_backend: n completions of one prompt (jl_sched_submit_n).  In the
 * step that forwards the prompt's last chunk, after the forward, one fork(leader session, positions after the prompt, n - 1, sibling
 * sessions) call gives the siblings the prompt's KV and last row; their first tokens then come from the same first-token calls as every
 * other completed prompt. */
typedef struct {
    int (*fork)(void *user, int src, int positions, int n, const int32_t *dst);
} jl_sched_fork_backend;
/* install the fork call; before the first jl_sched_step only.  jl_sched_create installs the model's jl_model_kv_fork. */
int jl_sched_set_fork_backend(jl_sched *s, const jl_sched_fork_backend *fb);
/* prefix cache calls (jl_model_kv_retain / kv_attach / kv_release / kv_retained) and the model's ctx_per_page, installed with
 * jl_sched_set_prefix_cache (DESIGN §3.17).  A fresh request (one that does not continue a kept session) retains its prompt's whole pages
 * in the step that forwards its last chunk, and the whole pages of every position it wrote when it finishes (stop, max tokens, cancelled
 * after admission).  At admission it attaches the longest cached page-aligned prefix of its prompt below its last token and forwards the
 * rest.  Entries are evicted least recently used beyond max_pages pages held only by the cache, and when a forward, decode, fork or attach
 * runs out of memory. */
typedef struct {
    int (*retain)(void *user, int session, int positions, int64_t *handle_out);
    int (*attach)(void *user, int64_t handle, int positions, int session);
    int (*release)(void *user, int64_t handle);
    int (*retained)(void *user, int64_t *handles, int64_t *pages_retained_only);
    int ctx_per_page;
} jl_sched_prefix_backend;
/* turn the prefix cache on (max_pages > 0) or off (0, the default); before the first jl_sched_step only.  pb NULL: the model's calls, for
 * a jl_sched_create scheduler (JL_ERR_INVALID for jl_sched_create_backend).  JL_ERR_UNSUPPORTED when the backend's retained call says so
 * (a model with tp_size > 1). */
int jl_sched_set_prefix_cache(jl_sched *s, const jl_sched_prefix_backend *pb, int max_pages);
typedef struct {
    int64_t entries, lookups, hits; /* cached prefixes now; fresh requests admitted with the cache on, and those that attached a prefix */
    int64_t cached_tokens;          /* prompt tokens served from the cache instead of forwarded */
    int64_t evictions;              /* entries released for the page budget or to free memory */
    int64_t pages_retained_only;    /* pages held by the cache and by no session, as of the last step */
} jl_sched_prefix_stats_t;
int jl_sched_prefix_stats(jl_sched *s, jl_sched_prefix_stats_t *out);
/* the prompt tokens `request` took from the prefix cache (>= 0), or JL_ERR_INVALID for an unknown request */
int jl_sched_request_cached(jl_sched *s, int64_t request);
int jl_sched_free(jl_sched *s);
const char *jl_sched_last_error(jl_sched *s);
/* Queue a request: prompt token ids, at most max_new generated tokens (the first is sampled from the prompt's last row and, like the
 * reference's, not stop-checked), optional stop tokens.  flags: JL_SCHED_KEEP_SESSION, JL_SCHED_CONSTRAINED (refused, -1, without a
 * mask provider and a constraint backend); every submit call takes them.  continue_request >= 0: a finished JL_SCHED_KEEP_SESSION request whose session
 * this request appends to.  temperature 0 = arg-max; otherwise every token is drawn with the reference's rule (AbstractModel.java:475-489)
 * from a per-request uniform stream seeded with `seed` (the reference draws ThreadLocalRandom.nextFloat(), :576,:594): the k-th token of
 * a request uses its k-th draw however the steps were batched, so (seed, prompt) reproduces.  Returns the request id (> 0) or -1.
 * Callable from any thread, also while a step runs. */
int64_t jl_sched_submit(jl_sched *s, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens, int n_stop, int flags,
                        int64_t continue_request, float temperature, uint64_t seed);
/* jl_sched_submit with a token filter: top_k >= 0 (0 = none), top_p in (0, 1] (1 = none).  With temperature > 0 and a filter every
 * token is drawn by the top-k / top-p rule (jl_model_decode_sample_topkp) from the same per-request uniform stream; such a request is
 * refused (-1) when no top-k / top-p backend is installed.  top_k 0 and top_p 1 is jl_sched_submit. */
int64_t jl_sched_submit_topkp(jl_sched *s, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens, int n_stop,
                              int flags, int64_t continue_request, float temperature, int top_k, float top_p, uint64_t seed);
/* jl_sched_submit_topkp with log-probabilities (DESIGN §3.13): logprobs -1 = none (jl_sched_submit_topkp), 0 = each generated token's
 * own, 1..JL_MAX_LOGPROBS = also that many top alternatives per token.  Tokens are those of the same request without logprobs.  Refused
 * (-1) with logprobs >= 0 when no logprob backend is installed. */
int64_t jl_sched_submit_logprobs(jl_sched *s, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens, int n_stop,
                                 int flags, int64_t continue_request, float temperature, int top_k, float top_p, uint64_t seed, int logprobs);
/* jl_sched_submit_logprobs with penalties (DESIGN §3.14): presence / frequency in [-2, 2], repetition in (0, 100], and n_bias distinct
 * (bias_ids[j] >= 0, bias_vals[j] in [-100, 100]) entries; 0 / 0 / 1 and no entry is jl_sched_submit_logprobs.  Refused (-1) with a bad
 * value, or with a penalty when no penalty backend is installed.  A bias id at or above the vocabulary fails the request at its first
 * call. */
int64_t jl_sched_submit_penalized(jl_sched *s, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens, int n_stop,
                                  int flags, int64_t continue_request, float temperature, int top_k, float top_p, uint64_t seed, int logprobs,
                                  float presence, float frequency, float repetition, int n_bias, const int32_t *bias_ids,
                                  const float *bias_vals);
/* n completions of one prompt (OpenAI's `n`): n requests with ids ids_out[0..n) (HOST [n]), each an ordinary request with the other
 * arguments of jl_sched_submit_penalized (its own stop tokens, max_new, logprobs, penalty history, keep flag, result, cancel and release),
 * member j drawing from the uniform stream seeded with seed + j.  The group is admitted whole, FIFO, into n session slots (spilling kept
 * sessions as any admission does); member 0 forwards the prompt under the prefill budget while the others hold their slots in
 * JL_SCHED_PREFILL; after the prompt's last chunk its session is forked into theirs (shared KV pages, DESIGN §3.15) and from the first
 * token on the members decode independently.  With continue_request, member 0 continues the kept session and the others fork the whole
 * conversation.  A leader cancelled before the fork still forwards the prompt for the others, then ends; a failed prompt forward fails
 * the group, a failed fork the members other than 0.  n == 1 is jl_sched_submit_penalized.  Returns JL_OK, or JL_ERR_INVALID with
 * nothing queued: a bad argument, n < 1, n above the scheduler's session slots, or n > 1 without a fork backend. */
int jl_sched_submit_n(jl_sched *s, int n, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens, int n_stop, int flags,
                      int64_t continue_request, float temperature, int top_k, float top_p, uint64_t seed, int logprobs, float presence,
                      float frequency, float repetition, int n_bias, const int32_t *bias_ids, const float *bias_vals, int64_t *ids_out);
int jl_sched_cancel(jl_sched *s, int64_t request); /* takes effect at the next step boundary */
/* one scheduling iteration; returns the first backend error of the step (the affected requests are JL_SCHED_FAILED, the others go on) */
int jl_sched_step(jl_sched *s, jl_sched_stats *stats /* nullable */);
/* step until nothing is queued or running (max_steps <= 0: no limit); totals are summed over the steps */
int jl_sched_run(jl_sched *s, int max_steps, jl_sched_stats *totals /* nullable */);
/* tokens generated so far (streaming read), state and finish reason; copies min(cap, n) tokens, *n_tokens = n */
int jl_sched_result(jl_sched *s, int64_t request, int32_t *tokens, int cap, int *n_tokens, int *state, int *finish_reason);
int jl_sched_request_info(jl_sched *s, int64_t request, jl_sched_request_info_t *info);
/* streaming read of a logprob request's entries [first, first + count): entry k belongs to its k-th generated token, however the steps
 * were batched.  lp [count], top_ids / top_lp [count][JL_MAX_LOGPROBS] (each nullable; slots past the request's logprobs hold id -1 and
 * NaN); entries past the available ones are left untouched.  *n_available (nullable) = entries so far.  A request submitted without
 * logprobs is refused (JL_ERR_INVALID). */
int jl_sched_result_logprobs(jl_sched *s, int64_t request, int first, int count, float *lp, int32_t *top_ids, float *top_lp,
                             int *n_available);
/* forget a finished / failed request; frees the session slot it kept */
int jl_sched_release(jl_sched *s, int64_t request);
int jl_sched_counts(jl_sched *s, int *queued, int *active, int *free_slots);

/* ---- jlama-net replacement: NCCL over NVLink instead of gRPC -------------------------------
 * JlamaService.combine (jlama-net/src/main/java/com/github/tjake/jlama/net/grpc/JlamaService.java:300-359)
 * == all-reduce SUM of [M,E] f32.  One process per GPU; rank 0 creates the id, the launcher
 * (torch.distributed / any store) broadcasts it. */
int jl_comm_unique_id(jl_ctx *ctx, uint8_t *id128 /* 128 bytes */);
int jl_comm_init(jl_ctx *ctx, const uint8_t *id128, int rank, int world);
/* HOST-buffer all-reduce for tests of the collective itself */
int jl_comm_allreduce_f32(jl_ctx *ctx, float *host_buf, int64_t count);
int jl_comm_destroy(jl_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* JLAMA_B200_H */
