// Internal declarations shared by the translation units of libjlama_b200.so.
// sm_90a only.  No torch types anywhere in this library.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <mutex>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "../../include/jlama_b200.h"

#define QBLOCK 32

struct DevTensor {
    int dtype = 0;
    int64_t rows = 0, cols = 0;
    void *data = nullptr;    // f32 / bf16 / packed nibbles / int8
    float *scales = nullptr; // [rows, cols/32] for Q4 / I8
    size_t bytes = 0;
    int64_t id = 0;          // registry id (0 for views / temporaries)
    int refs = 0;            // models this tensor is bound to (jl_model_set_tensor); unregister refuses while > 0
};

struct jl_ctx {
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr; // op-level API stream
    std::mutex mu;
    std::mutex err_mu;      // guards last_error only: model entry points report errors without holding `mu`
    std::string last_error; // the most recent error of any thread; jl_last_error prefers the calling thread's own (jl_runtime.cu)
    std::unordered_map<int64_t, DevTensor> tensors;
    std::vector<struct jl_model *> models; // live models (freed by jl_shutdown before the tensors they point at)
    int64_t next_id = 1;
    long long launches = 0;
    // op-level scratch (grown on demand)
    void *scratch[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t scratch_bytes[4] = {0, 0, 0, 0};
    // kernel timeline diagnostics (jl_debug_ktrace): device [cap][4] globaltimer stamps, one slot per traced launch
    unsigned long long *ktrace = nullptr;
    int ktrace_cap = 0, ktrace_n = 0;
    // comm
    void *nccl_comm = nullptr;
    int rank = 0, world = 1;
};

int jl_set_error(jl_ctx *ctx, int code, const char *fmt, ...);
#define JL_CUDA_CHECK(ctx, expr)                                                                      \
    do {                                                                                              \
        cudaError_t _e = (expr);                                                                      \
        if (_e != cudaSuccess)                                                                        \
            return jl_set_error(ctx, _e == cudaErrorMemoryAllocation ? JL_ERR_OOM : JL_ERR_CUDA,      \
                                "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

void *jl_scratch(jl_ctx *ctx, int slot, size_t bytes); // nullptr on OOM
// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute: remember what was set per (device, kernel)
// so that a second context on another GPU of the same process configures its own copy.
#define JL_MAX_DEVICES 64
template <typename K>
static inline cudaError_t jl_ensure_dyn_smem(K kernel, int device, size_t bytes, size_t (&configured)[JL_MAX_DEVICES]) {
    if (bytes <= 40 * 1024) return cudaSuccess; // static shared memory counts against the 48 KB default too
    const int d = device >= 0 && device < JL_MAX_DEVICES ? device : 0;
    if (bytes <= configured[d]) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) configured[d] = bytes;
    return e;
}
// called when the timeline buffer is replaced: captured graphs hold the old slot pointers
void jl_models_invalidate_graphs(jl_ctx *ctx);

// ---------------------------------------------------------------------------------------------
// Quantised GEMV / small-M GEMM (jl_gemv.cu)
// ---------------------------------------------------------------------------------------------
enum GemvPrologue {
    PRO_Q8_GLOBAL = 0,  // activations already int8 + scales in global memory
    PRO_F32_QUANT,      // f32 activations -> Q8 (PanamaTensorOperations.quantizeQ8 semantics) in the prologue
    PRO_RMSNORM_QUANT,  // f32 hidden row -> RMSNorm (RMSNorm.java:34-56) -> Q8
    PRO_F32,            // f32 activations used as-is (F32 x W path)
    PRO_RMSNORM_F32,    // RMSNorm then f32 activations
    PRO_BF16_GLOBAL,    // bf16 activations in global -> f32
};
enum GemvEpilogue {
    EPI_STORE = 0,    // out[m, out_off + row] = acc
    EPI_ADD_RESIDUAL, // out[m, row] = acc + residual[m, row]
    EPI_SILU_MUL,     // seg0 = gate, seg1 = up: out[m,row] = silu(g) * u   (MLPBlock.java:132-141)
};

struct GemvSeg {
    const void *w;       // weight rows, leading dim = ldw elements
    const float *ws;     // block scales (Q4/I8) with leading dim ldw/32
    float *out;          // f32 output [M, out_ld]
    int rows;            // rows in this segment
    int out_ld;
    int out_off;         // added to the row index on store (already includes -roffset)
};

struct GemvParams {
    GemvSeg seg[3];
    int nseg;
    int w_dtype;             // JL_Q4 / JL_I8 / JL_BF16 / JL_F32
    int ldw;                 // weight leading dimension in elements
    int w_col_off;           // first weight column (elements, multiple of 32 for quantised)
    int K;                   // reduction length
    int M;                   // activation rows (1..GEMV_MAX_M; up to JL_MAX_DECODE_ROWS where jl_gemm64_supported)
    // activations
    const void *a;           // f32 / int8 / bf16 [M, lda]
    const float *a_scales;   // for PRO_Q8_GLOBAL: [M, lda/32]
    int lda;
    int a_col_off;
    // norm prologue
    const void *norm_w;      // f32 or bf16 [E]
    int norm_w_dtype;
    float norm_adj, norm_eps;
    int norm_E;
    double norm_inv_E;       // filled by jl_launch_gemv
    // epilogue
    const float *residual;   // [M, res_ld]
    int res_ld;
    int row0;                // first global row handled by this launch (n0)
    int total_rows;          // rows handled by this launch
    unsigned long long *trace; // diagnostics slot (jl_debug_ktrace) or nullptr
    // mixture-of-experts indirection (MoEBlock.java:98-137): when sel != nullptr the weights of segment i are
    // w_tab[i][*sel] / ws_tab[i][*sel] -- the expert index is only known on the device (router top-k of this row)
    const int *sel;
    const void *const *w_tab[2];
    const float *const *ws_tab[2];
    // many-row decode GEMM (jl_gemm64.cu), caller-owned device workspaces: quantised activations (jl_gemm64_act_bytes), split-K
    // partial tiles (jl_gemm64_part_floats) and one zero-initialised arrival counter per SM
    void *wide_act;
    float *wide_part;
    unsigned *wide_cnt;
    // grouped expert GEMM (jl_launch_gemm64_grouped): the tile table and pair list of jl_launch_moe_group; tile row r reads
    // quantised row pair / g_div of wide_act (g_div = k: the token row of gate/up, 1: the pair's own h row for down_proj) and
    // writes output row `pair`; the weights of segment i are w_tab[i][tile expert]
    const int4 *g_tiles;
    const int *g_ntiles;
    const int *g_pairs;
    int g_div;
};
__device__ __forceinline__ void gemv_seg_base(const GemvParams &p, int seg, const void *&w, const float *&ws) {
    if (p.sel) {
        const int e = __ldg(p.sel);
        w = p.w_tab[seg][e], ws = p.ws_tab[seg][e];
    } else {
        w = p.seg[seg].w, ws = p.seg[seg].ws;
    }
}

#define GEMV_MAX_M 8

// Launch on `stream`.
int jl_launch_gemv(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int epilogue);
int jl_gemv_max_m(int w_dtype, int prologue, int K);
// batched decode (2..8 rows): integer block products on the tensor cores (jl_gemm8.cu)
bool jl_gemm8_supported(const GemvParams &p, int prologue, int epilogue);
int jl_launch_gemm8(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int epilogue); // largest M chunk (1/2/4/8) that fits shared memory, 0 if none
// many-row decode (9..JL_MAX_DECODE_ROWS rows) in one weight pass (jl_gemm64.cu); two launches: activation prologue + GEMM
bool jl_gemm64_supported(const GemvParams &p, int prologue, int epilogue);
int jl_launch_gemm64(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int epilogue);
size_t jl_gemm64_act_bytes(int K);            // wide_act bytes for reduction length K
size_t jl_gemm64_part_floats(int sm_count);   // wide_part floats
// grouped expert GEMM: p.M activation rows quantised in a prologue launch, then one CTA per (tile, 128 weight rows) of the
// first `tiles` entries of p.g_tiles (CTAs past *p.g_ntiles exit); tiles of at most jl_gemm64_group_rows(rows per expert) rows
int jl_gemm64_group_rows(int max_rows_per_expert);
bool jl_gemm64_grouped_supported(const GemvParams &p, int prologue, int epilogue, int R);
int jl_launch_gemm64_grouped(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int epilogue, int R, int tiles);
size_t jl_gemm64_q8_bytes(int rows, int K);   // quantised rows + block scales of the prologue

// ---------------------------------------------------------------------------------------------
// Element-wise / normalisation / sampling kernels (jl_elementwise.cu)
// ---------------------------------------------------------------------------------------------
int jl_launch_accumulate(jl_ctx *ctx, cudaStream_t s, float *a, int a_rows, int lda, int b_dtype, const void *b,
                         const float *b_scales, int b_rows, int ldb, int offset, int length);
int jl_launch_maccumulate(jl_ctx *ctx, cudaStream_t s, float *a, int a_rows, int lda, const float *b, int b_rows, int ldb,
                          int offset, int length);
int jl_launch_scale(jl_ctx *ctx, cudaStream_t s, float f, float *x, int rows, int ldx, int offset, int length);
int jl_launch_saxpy_batch(jl_ctx *ctx, cudaStream_t s, const float *alpha, const float *x, int ldx, float *y, int xoffset,
                          int yoffset, int limit, int a_offset, int x_row_offset, int batch);
int jl_launch_quantize_q8(jl_ctx *ctx, cudaStream_t s, const float *x, int rows, int ldx, int offset, int length,
                          int8_t *q, float *scales);
int jl_launch_quantize_bf16(jl_ctx *ctx, cudaStream_t s, const float *x, int rows, int ldx, int offset, int length,
                            uint16_t *out);
int jl_launch_quantize_q4w(jl_ctx *ctx, cudaStream_t s, const float *x, int64_t rows, int64_t cols, uint8_t *q,
                           float *scales);
int jl_launch_quantize_q8w(jl_ctx *ctx, cudaStream_t s, const float *x, int64_t rows, int64_t cols, int8_t *q, float *scales);
int jl_launch_rmsnorm(jl_ctx *ctx, cudaStream_t s, const float *x, int rows, int ldx, int w_dtype, const void *w, float adj,
                      float eps, int E, int offset, int length, float *out);
int jl_launch_layernorm(jl_ctx *ctx, cudaStream_t s, const float *x, int rows, int ldx, int w_dtype, const void *w, int b_dtype,
                        const void *bias, float eps, int E, int offset, int length, float *out);
int jl_launch_activation(jl_ctx *ctx, cudaStream_t s, int type, float *x, int rows, int ld, int offset, int length);
// MoE router: softmax over the expert logits of each row (VectorMath.softMax) + top-k by the reference's replace-the-minimum
// scan (MoEBlock.java:151-168); sel[row * k + i] = i-th selected expert
int jl_launch_moe_route(jl_ctx *ctx, cudaStream_t s, float *logits, int rows, int n_experts, int k, int32_t *sel);
// MoE grouping of a step's rows by expert (one CTA): the pairs p = row * k + slot of sel [rows][k] by expert, a stable counting
// sort (ascending p within an expert); counts / offsets [n_experts]; tiles {expert, first pair, pairs, 0} cut each expert's list
// into runs of at most R, expert by expert; *ntiles = their number, at most jl_moe_tile_bound(rows * k, n_experts, R)
struct MoeGroups {
    int32_t *counts, *offsets, *pairs, *ntiles;
    int4 *tiles;
};
static inline int jl_moe_tile_bound(int pairs, int n_experts, int R) { return (pairs + n_experts * (R - 1)) / R; }
int jl_launch_moe_group(jl_ctx *ctx, cudaStream_t s, const int32_t *sel, int rows, int n_experts, int k, int R, const MoeGroups &g);
// x[b] = (d[b k + k - 1] + ... + (d[b k + 1] + d[b k])) + xb[b], floats in slot order; d [rows * k][E]
int jl_launch_moe_combine(jl_ctx *ctx, cudaStream_t s, const float *d, int rows, int k, int E, const float *xb, float *x);
int jl_launch_softmax(jl_ctx *ctx, cudaStream_t s, float *x, int offset, int length);
int jl_launch_silu_mul(jl_ctx *ctx, cudaStream_t s, float *gate, const float *up, int rows, int ld, int offset, int length);
// fused producers of the BF16 operand of the tensor-core prefill GEMMs
int jl_launch_rmsnorm_bf16(jl_ctx *ctx, cudaStream_t s, const float *x, int rows, int ldx, int w_dtype, const void *w, float adj, float eps,
                           int E, uint16_t *out, int ldo);
int jl_launch_silu_mul_bf16(jl_ctx *ctx, cudaStream_t s, const float *gate, const float *up, int rows, int ld, int length, uint16_t *out, int ldo);
// embedding rows -> f32 hidden (LlamaModel.java:68-100); tokens on device
int jl_launch_embed(jl_ctx *ctx, cudaStream_t s, const DevTensor &wte, const int32_t *tokens, int n, float *out, int E);
int jl_launch_pos_embed_add(jl_ctx *ctx, cudaStream_t s, float *x, int rows, int E, const DevTensor &wpe, const int32_t *positions);
// argmax with strict '>' (lowest index wins; AbstractModel.java:455-469): two-stage
int jl_launch_argmax(jl_ctx *ctx, cudaStream_t s, const float *logits, int rows, int vocab, int ld, int32_t *out_tokens,
                     void *scratch);
size_t jl_argmax_scratch_bytes(int rows);
// top-k / top-p sampling (jl_sample.cu; the rule is DESIGN §3.12): one CTA per entry of `rows` (DEVICE [n]) samples logits row
// rows[i].row (read-only, stride ld) into out[rows[i].row].  ex: DEVICE scratch of n * vocab floats.
struct TopkpRow {
    int32_t row;
    float temperature;
    int32_t top_k;
    float top_p;
    float uniform;
};
#define JL_TOPKP_MAX_VOCAB (1 << 23) // keeps every uint64 weight sum below 2^63
int jl_launch_sample_topkp(jl_ctx *ctx, cudaStream_t s, const float *logits, int64_t ld, int vocab, const TopkpRow *rows, int n, float *ex,
                           int32_t *out);
// Argument checks of the top-k / top-p calls, before any device work.  temperatures / top_k / top_p / uniforms: HOST [n], each nullable
// (top_k / top_p NULL = unfiltered).  filtered (HOST [n], nullable) receives 1 for the rows the top-k / top-p kernel samples: temperature
// > 0 and (1 <= top_k < vocab or top_p < 1).  Returns JL_OK or JL_ERR_INVALID with the error set; *n_filtered = count of filtered rows.
int jl_topkp_check(jl_ctx *ctx, const char *who, int n, int vocab, const float *temperatures, const int32_t *top_k, const float *top_p,
                   const float *uniforms, char *filtered, int *n_filtered);
// token log-probabilities (jl_logprobs.cu; the rule is DESIGN §3.13): one launch for the n entries of `rows` (DEVICE [n]); entry i reads
// logits row rows[i].row (read-only, stride ld) and its target targets[rows[i].row] (DEVICE, nullable; -1 = none) and writes
// out[rows[i].row] with its top rows[i].top_n (0..JL_MAX_LOGPROBS) tokens.  ws: DEVICE jl_logprobs_ws_bytes(vocab, n); cnt: DEVICE [n]
// counters, zero before the first launch (each launch leaves them zero).
struct LogprobRow {
    int32_t row;
    int32_t top_n;
};
struct LogprobOut {
    float lp;                     // the target's logprob (NaN without a target)
    int32_t ids[JL_MAX_LOGPROBS]; // top tokens, best first (-1 past top_n or the vocabulary)
    float lps[JL_MAX_LOGPROBS];   // their logprobs (NaN where ids is -1)
};
#define JL_LOGPROBS_MAX_VOCAB (1 << 20) // 128 slices: the merge of every slice's candidates fits the kernel's shared buffer
int jl_logprobs_slices(int vocab);
size_t jl_logprobs_ws_bytes(int vocab, int rows);
int jl_launch_logprobs(jl_ctx *ctx, cudaStream_t s, const float *logits, int64_t ld, int vocab, const LogprobRow *rows, int n,
                       const int32_t *targets, void *ws, unsigned *cnt, LogprobOut *out);
// top_n (HOST [n], nullable = all -1) in -1..JL_MAX_LOGPROBS, and a vocabulary the kernel takes when a row asks; *n_on = rows with top_n >= 0
int jl_logprobs_check(jl_ctx *ctx, const char *who, int n, int vocab, const int32_t *top_n, int *n_on);
// o[i] -> the HOST outputs of row i (each nullable): rows with top_n -1 get NaN, slots past top_n get id -1 and NaN
void jl_logprobs_unpack(const LogprobOut *o, const int32_t *top_n, int n, float *lp_out, int32_t *top_ids_out, float *top_lp_out);
// frequency / presence / repetition penalties and logit bias (jl_penalty.cu; the rule is DESIGN §3.14).  The penalties of n rows travel
// as one table: PenaltyRow [n], then the history ids [n_hist], the bias ids [n_bias] and the bias values [n_bias] (offsets index those).
struct PenaltyRow {
    float presence, frequency, repetition;
    int32_t on;                    // 0: the row is copied unchanged
    int32_t hist0, prompt1, hist1; // history [hist0, hist1), of which [hist0, prompt1) are prompt tokens
    int32_t bias0, bias1;          // bias entries [bias0, bias1)
    int32_t mask;                  // allowed-token mask row of the call (DESIGN §3.18), -1 = unconstrained
};
struct PenaltyPlan {
    int n_on = 0;        // penalised rows
    int n_hist = 0, n_bias = 0;
    size_t bytes = 0;    // the table's size
};
// Checks a jl_penalties (HOST, nullable) of n rows before any device work (JL_ERR_INVALID with the error set), and sizes its table.
int jl_penalty_check(jl_ctx *ctx, const char *who, int n, int vocab, const jl_penalties *pen, PenaltyPlan *plan);
// the table of a checked jl_penalties -> tab (HOST, plan.bytes)
void jl_penalty_pack(const jl_penalties *pen, int n, const PenaltyPlan &plan, void *tab);
// Two launches for all n rows: the histories and bias lists of the penalised rows are marked in cnt / bias (DEVICE [n][vocab] each; cnt
// zero before the first launch, and each launch leaves it zero), then every row of logits (read-only, stride ld) -> out [n][vocab].
// mask (DEVICE [rows][(vocab + 31) / 32], nullable): the allowed-token mask rows the table's PenaltyRow::mask index; a row's banned
// tokens become -inf after its penalties.  With a mask and no penalised row the mark launch is skipped.
int jl_launch_penalties(jl_ctx *ctx, cudaStream_t s, const float *logits, int64_t ld, int vocab, int n, const void *tab,
                        const PenaltyPlan &plan, unsigned *cnt, float *bias, const uint32_t *mask, float *out);
// Allowed-token masks of the *_constrained calls (DESIGN §3.18): allow (HOST [n_allow][(vocab + 31) / 32]) and allow_row (HOST [n],
// nullable = no constrained row; -1 = unconstrained).  Refused (JL_ERR_INVALID with the error set) before any device work: n_allow < 0,
// n_allow > 0 with a NULL allow, allow_row[i] outside [-1, n_allow), a constrained row whose mask allows no token below vocab.
// *n_on = the constrained rows.
int jl_constraint_check(jl_ctx *ctx, const char *who, int n, int vocab, int n_allow, const uint32_t *allow, const int32_t *allow_row,
                        int *n_on);
// the mask rows the constrained rows of a checked call use -> dst (HOST, at most n rows of (vocab + 31) / 32 words, each used row
// once), and PenaltyRow::mask of the packed table `tab` pointed at them.  Returns the rows written.
int jl_constraint_pack(int n, int vocab, int n_allow, const uint32_t *allow, const int32_t *allow_row, void *tab, uint32_t *dst);
// KV page copies (jl_kv_copy.cu; DESIGN §3.15): entry e makes page dst a copy of page src in positions [0, rows) of every layer's K and V
// block, zeros in the others.  One launch for the n entries of tab (DEVICE); pages are [layers][2][ctx_per_page rows of row_bytes].
struct KvCopy {
    void *dst;
    const void *src;
    int32_t rows, pad;
};
int jl_launch_kv_copy(jl_ctx *ctx, cudaStream_t s, const KvCopy *tab, int n, size_t page_bytes, int ctx_per_page, int row_bytes);

// ---------------------------------------------------------------------------------------------
// Attention over the paged KV cache (jl_attention.cu)
// ---------------------------------------------------------------------------------------------
struct KvLayout {
    // Page = [layers_per_page, 2, ctx_per_page, kv_len] (KvBufferCache.java:102); page table per session.
    int layers_per_page, ctx_per_page, kv_len; // kv_len = this rank's kvSegmentLength
    int n_ctx_pages;                            // page-table stride per (session, layer_page)
    int n_layer_pages;
    int kv_dtype;                               // JL_F32, JL_BF16 or JL_I8 (kv_row_bytes)
    void *const *page_table;                    // device: [sessions][n_layer_pages][n_ctx_pages] -> page base
};

// ---- KV page rows (DESIGN §3.16) ----
// A page row holds the kv_len elements of one (layer, K or V, position).  F32 and BF16 rows are the elements.  An I8 (Q8_0) row is
// kv_len int8 values followed by kv_len / 32 f32 scales: block b covers elements [32b, 32b + 32), its scale is at byte kv_len + 4b and
// value i of the block reads as __fmul_rn((float)q, scale).  head_size is a multiple of 32, so KV head h owns whole blocks: its int8
// values start at byte h * head_size and its scales at kv_q8_scale_off(kv_len, h * head_size).
// kv_rows_bytes: the bytes of `rows` consecutive rows, i.e. the offset of row `rows` of a page.  KVDT: the dtype when a kernel fixes
// it at compile time; -1 = `dt` at run time, F32 or BF16 only: a -1 instantiation addresses I8 pages as 2 bytes per element.  So a
// host launcher picks KVDT with kv_dispatch, which sends I8 layouts to JL_I8 instantiations only; the persistent decode kernel
// (attention_flat<HS, PD_NT>, -1) is kept off I8 models by pd_ok in jl_model_finalize.  F32 / BF16 offsets keep the element-count
// form rows * kv_len * bytes, which is what their instantiations are register-allocated with (DESIGN §3.16).
template <int KVDT = -1>
__host__ __device__ __forceinline__ size_t kv_rows_bytes(int dt, size_t kv_len, size_t rows) {
    if constexpr (KVDT == JL_I8) return rows * (kv_len + kv_len / 8);
    else return rows * kv_len * (dt == JL_F32 ? 4 : 2);
}
// one row, any dtype at run time
__host__ __device__ __forceinline__ size_t kv_row_bytes(int dt, size_t kv_len) {
    return dt == JL_I8 ? kv_rows_bytes<JL_I8>(dt, kv_len, 1) : kv_rows_bytes(dt, kv_len, 1);
}
// byte offset, inside an I8 row, of the scale of the block that holds element e
__host__ __device__ __forceinline__ size_t kv_q8_scale_off(size_t kv_len, size_t e) { return kv_len + e / 32 * 4; }
// four int8 values (little-endian in w) of one block with scale s, as stored values
__device__ __forceinline__ float4 kv_q8x4(uint32_t w, float s) {
    return make_float4(__fmul_rn((float)((int)(w << 24) >> 24), s), __fmul_rn((float)((int)(w << 16) >> 24), s),
                       __fmul_rn((float)((int)(w << 8) >> 24), s), __fmul_rn((float)((int)w >> 24), s));
}

// f(std::integral_constant<int, KVDT>) with the instantiation that reads pages of dtype dt: JL_I8 for I8 pages.  F32 and BF16 pages
// get their own JL_F32 / JL_BF16 instantiations where the kernel has them (CONCRETE), and share the run-time -1 one otherwise.
template <bool CONCRETE, typename F>
static inline auto kv_dispatch(int dt, F &&f) -> decltype(f(std::integral_constant<int, JL_I8>())) {
    if (dt == JL_I8) return f(std::integral_constant<int, JL_I8>());
    if constexpr (CONCRETE) {
        if (dt == JL_F32) return f(std::integral_constant<int, JL_F32>());
        return f(std::integral_constant<int, JL_BF16>());
    } else {
        return f(std::integral_constant<int, -1>());
    }
}

struct AttnParams {
    KvLayout kv;
    int layer;
    int heads, kv_heads, head_size; // this rank's heads
    int head0_global;               // first global head on this rank (for the RoPE table quirk)
    int kv_head0_global;
    const float *q;  // [rows, q_ld]  raw projections (pre-RoPE)
    const float *k;  // [rows, kv_ld]
    const float *v;  // [rows, kv_ld]
    int q_ld, kv_ld;
    float *out;      // [rows, q_ld] attention output (this rank's heads)
    const float *rope; // [(positions) * hs/2][2]
    int rows;                  // query rows in this launch
    const int32_t *sessions;   // device [rows] session of each row
    const int32_t *positions;  // device [rows] absolute position of each row
    float scale;
    // split-K workspace
    float *ws;       // [rows, heads, splits, hs + 2]
    int splits;
};

// Writes rotated K and V of every row into the pages and rotates q in place (CausalSelfAttention.java:199-311).
int jl_launch_rope_kv_append(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, float *q_inplace);
// Causal attention of each row against positions [0, pos] of its session (CausalSelfAttention.java:314-356).
int jl_launch_paged_attention(jl_ctx *ctx, cudaStream_t s, const AttnParams &p);
// tiled prefill attention for one session's chunk of consecutive positions (jl_attn_prefill.cu)
bool jl_prefill_attention_supported(const AttnParams &p);
int jl_launch_prefill_attention(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, int session, int pos0);
// the same for a pass whose rows hold chunks of several sessions: segs[i] = {session, pos0, first row, rows} (HOST) -> CTA block table
// (HOST, at most p.rows / 16 + nseg entries; returns the count), then one launch over the table once it is on the device
int jl_prefill_attention_table(jl_ctx *ctx, const AttnParams &p, const int4 *segs, int nseg, int4 *out);
int jl_launch_prefill_attention_table(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, const int4 *tab, int ntab);
// Decode steps (every row a different session): RoPE + KV append + attention fused in one kernel; q/k/v are the raw
// projections.  done_cnt: [rows * kv_heads] zero-initialised split-arrival counters (self-resetting).
// max_pos >= 0: the largest position among the rows (lets batched decode take the flat task); -1: tiled task only
int jl_launch_fused_decode_attention(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, unsigned *done_cnt, int max_pos = -1);

// ---------------------------------------------------------------------------------------------
// Larger-M GEMM paths for prefill (jl_gemm.cu)
// ---------------------------------------------------------------------------------------------
// wgmma tensor-core GEMM (jl_gemm_tc.cu): C[T, out_col_off+n] (+residual) = A_bf16[T,K] * dequant(W[n, w_col_off+k])^T
int jl_launch_gemm_tc(jl_ctx *ctx, cudaStream_t stream, const uint16_t *a_bf16, int lda, int T, const DevTensor &W, int n_rows,
                      int w_col_off, int K, float *out, int ldc, int out_col_off, const float *residual, int res_ld);

// ---------------------------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ uint4 ldg_nc_u4(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ float ldg_nc_f32(const float *p) {
    float r;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}
// Loads that should stay in L2 across decode steps (norm weights: 16 KB per layer, re-read every token but otherwise
// flushed by the 4.7 GB weight stream in between): L2 evict_last policy.
__device__ __forceinline__ unsigned long long l2_evict_last_policy() {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint4 ldg_keep_u4(const void *p, unsigned long long pol) {
    uint4 r;
    asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p), "l"(pol));
    return r;
}
// The decode weight stream (4.7 GB per token through a 50 MB L2) is tagged evict_first, so that it recycles its own
// lines instead of flushing what the step re-reads: activations, KV pages, RoPE and norm tables -- and kernel code.
__device__ __forceinline__ unsigned long long l2_evict_first_policy() {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint4 ldg_stream_u4(const void *p, unsigned long long pol) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ float ldg_stream_f32(const float *p, unsigned long long pol) {
    float r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(r) : "l"(p), "l"(pol));
    return r;
}

// ---- tensor-core MMAs and cp.async (decode GEMMs, prefill attention) ----
// c += a (16x32, row) * b (32x8, col): u8 x s8 (Q4 nibbles) and s8 x s8 (Q8_0) -> s32
__device__ __forceinline__ void mma_u8s8(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_s8s8(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// d += a (16x16, row) * b (16x8, col): bf16 x bf16 -> f32
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// 16-byte global -> shared copy, with an L2 cache policy or the default one
__device__ __forceinline__ void cp16(uint32_t dst, const void *src, unsigned long long pol) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp16(uint32_t dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// wait until at most `pending` of this thread's copy groups are still in flight
__device__ __forceinline__ void cp_wait(int pending) {
    switch (pending) {
        case 0: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
        case 1: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
        case 2: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
        case 3: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
        default: asm volatile("cp.async.wait_group 4;" ::: "memory"); break;
    }
}

// One pipeline stage of a 16-row weight strip (jl_gemm8.cu, jl_gemm64.cu): a 128-byte chunk of each of the 16 rows, then the
// rows' block scales.  The row stride 128 + 16 makes the fragment loads conflict free (lane (g, t) reads word g*36 + 4u + t:
// 32 distinct banks).  ROWB and SC_OFF are the same for both weight types, and so is the stage size.
#define STRIP_STAGE 3072 // bytes of one strip stage: 16 rows x 144 B of weights + 16 rows x <= 48 B of block scales
template <int WDT>
struct Strip {
    static constexpr int BPC = WDT == JL_Q4 ? 8 : 4;  // blocks per 128-byte row chunk
    static constexpr int BB = WDT == JL_Q4 ? 16 : 32; // weight bytes per block
    static constexpr int SCS = BPC * 4 + 16;          // staged scale row stride (bytes)
    static constexpr int ROWB = 144;                  // staged weight row stride (bytes)
    static constexpr int SC_OFF = 16 * ROWB;          // scales behind the 16 weight rows
};

// One warp issues stage `st` of a strip: the 128-byte chunk at block column cb of weight rows p.row0 + local0 + 0..15 of tensor
// (wb, wsb) (8 lanes per row, 4 copies per lane) and their scales.  Rows at or past rows_left do not exist and copy the strip's
// first row instead (their results are never stored).
template <int WDT>
__device__ __forceinline__ void strip_stage(uint32_t st, const GemvParams &p, const void *wb, const float *wsb, int local0, int rows_left,
                                            size_t ldb, size_t cb, int lane, unsigned long long pol) {
    using S = Strip<WDT>;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int r = (lane >> 3) + 4 * i, rl = r < rows_left ? r : 0;
        const size_t blk0 = (size_t)(p.row0 + local0 + rl) * ldb + cb;
        cp16(st + r * S::ROWB + (lane & 7) * 16, (const uint8_t *)wb + blk0 * S::BB + (lane & 7) * 16, pol);
    }
    if (WDT == JL_Q4) { // 16 rows x 32 B of scales: two lanes per row
        const int r = lane >> 1, rl = r < rows_left ? r : 0;
        const size_t blk0 = (size_t)(p.row0 + local0 + rl) * ldb + cb;
        cp16(st + S::SC_OFF + r * S::SCS + (lane & 1) * 16, wsb + blk0 + (lane & 1) * 4, pol);
    } else if (lane < 16) { // 16 rows x 16 B
        const int r = lane, rl = r < rows_left ? r : 0;
        const size_t blk0 = (size_t)(p.row0 + local0 + rl) * ldb + cb;
        cp16(st + S::SC_OFF + r * S::SCS, wsb + blk0, pol);
    }
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define KTRACE_WORDS 16 // per slot: first CTA start, last CTA end, CTA 0 after prologue, tag, CTA 0 start, 11 free stamps
__device__ __forceinline__ void ktrace_begin(unsigned long long *t, unsigned long long tag) {
    if (t && threadIdx.x == 0) {
        const unsigned long long now = globaltimer_ns();
        atomicMin(&t[0], now);
        if (blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) t[3] = tag, t[4] = now;
    }
}
// extra stamp `idx` (5..15) by thread 0 of CTA 0, ordered after `dep` has been computed
__device__ __forceinline__ void ktrace_stamp(unsigned long long *t, int idx, float dep) {
    if (t && threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
        unsigned long long now;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now) : "f"(dep) : "memory");
        t[idx] = now;
    }
}
__device__ __forceinline__ void ktrace_mid(unsigned long long *t) {
    if (t && threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) t[2] = globaltimer_ns();
}
__device__ __forceinline__ void ktrace_end(unsigned long long *t) {
    if (t && threadIdx.x == 0) atomicMax(&t[1], globaltimer_ns());
}
inline unsigned long long *jl_ktrace_slot(jl_ctx *ctx) {
    if (!ctx->ktrace || ctx->ktrace_n >= ctx->ktrace_cap) return nullptr;
    return ctx->ktrace + (size_t)KTRACE_WORDS * ctx->ktrace_n++;
}

__device__ __forceinline__ float bf16_bits_to_f32(uint16_t b) { return __uint_as_float(((uint32_t)b) << 16); }
// f32 -> bf16 round to nearest even, NaN preserving (FloatConversions.java:35-61)
__device__ __forceinline__ uint16_t f32_to_bf16_rne(float n) {
    const uint32_t nbits = __float_as_uint(n);
    const uint32_t s = (nbits >> 16) & 0x8000u, e = (nbits >> 16) & 0x7f80u, m = nbits & 0x7fffffu;
    if (e != 0x7f80u) {
        const int mshift = (int)(m >> 16), masked = (int)(m & 0xffff), cmp = masked - 0x8000;
        const int m1 = cmp > 0 ? mshift + 1 : (cmp < 0 ? mshift : ((mshift & 1) ? mshift + 1 : mshift));
        return (uint16_t)(s | (e + (uint32_t)m1));
    }
    return m != 0 ? (uint16_t)0x7fc0 : (uint16_t)(nbits >> 16);
}

// Q8_0 block quantiser (Q8ByteBufferTensor.java:47-90), warp-collective: lane l holds element l of one 32-element block and gets its
// int8 value back; *scale = the block's scale.  max from Float.MIN_VALUE, iscale = 127 / max, q = (byte)Math.round(x * iscale),
// scale = 1 / iscale.  Used by the weight quantiser (jl_elementwise.cu) and by the appends to I8 KV pages.
__device__ __forceinline__ int8_t q8_block_quantize(float v, float &scale) {
    float mx = fmaxf(warp_max(fabsf(v)), 1.401298464e-45f); // 'absv > max' never replaces max with NaN
    const float iscale = __fdiv_rn(127.0f, mx);
    scale = iscale != 0.0f ? __fdiv_rn(1.0f, iscale) : 0.0f;
    const float f0 = __fmul_rn(v, iscale);
    // Math.round(float) = floor(f0 + 1/2) evaluated exactly; NaN -> 0; (int) saturates, (byte) wraps
    int r;
    if (f0 != f0) r = 0;
    else {
        const double t = floor((double)f0 + 0.5);
        r = t >= 2147483647.0 ? 2147483647 : (t <= -2147483648.0 ? (int)0x80000000 : (int)t);
    }
    return (int8_t)r;
}
// Warp-collective append of one block to an I8 KV row: lane l holds element e0 + l (e0 a multiple of 32).  Returns the lane's
// value as stored, which the appending step uses for its own scores and P.V, as a later read of the page would.
__device__ __forceinline__ float kv_q8_append(char *row, size_t kv_len, int e0, float v) {
    const int lane = threadIdx.x & 31;
    float s;
    const int8_t q = q8_block_quantize(v, s);
    row[e0 + lane] = (char)q;
    if (lane == 0) *(float *)(row + kv_q8_scale_off(kv_len, e0)) = s;
    return __fmul_rn((float)q, s);
}
// Element j (0 <= j < 2 * hp) of a KV head's rotated key (CausalSelfAttention.java:279-285): k = the head's raw key, f = its RoPE
// table row.  The same products as the pairwise rotation of the F32 / BF16 appends.
__device__ __forceinline__ float rope_key_elem(const float *k, const float2 *f, int j, int hp) {
    if (j < hp) {
        const float2 c = __ldg(f + j);
        return __fsub_rn(__fmul_rn(__ldcg(k + j), c.x), __fmul_rn(__ldcg(k + j + hp), c.y));
    }
    const float2 c = __ldg(f + j - hp);
    return __fadd_rn(__fmul_rn(__ldcg(k + j - hp), c.y), __fmul_rn(__ldcg(k + j), c.x));
}

// jafama-equivalent activation in double, cast to float (ActivationFunction.java:29-37)
__device__ __forceinline__ float silu_ref(float x) { return (float)((double)x * (1.0 / (1.0 + exp(-(double)x)))); }

template <typename K, typename... Args>
static inline cudaError_t jl_launch_kernel(K kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    return cudaLaunchKernelEx(&cfg, kernel, args...);
}
