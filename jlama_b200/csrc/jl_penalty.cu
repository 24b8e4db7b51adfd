// Frequency, presence and repetition penalties and logit bias on logits rows: the rule of DESIGN §3.14.
//
// Per row, with c_t = the count of token t among the generated part of the row's history and s_t = whether t occurs anywhere in it:
//   b = l + bias_t;  if s_t: b = b < 0 ? b * repetition : b / repetition;  b = b - (float)c_t * frequency;  if c_t > 0: b = b - presence
// in float32, one correctly rounded operation per step (__fadd_rn / __fmul_rn / __fdiv_rn: the build contracts a*b+c into FMA otherwise).
//
// Two launches cover all rows of a call.  The mark kernel (one CTA per row) turns the row's history and bias list into a dense per-row
// word per token: bits 0..29 count the generated occurrences (atomicAdd), bit 30 flags a bias entry (whose value goes to a dense bias
// row), bit 31 flags a prompt occurrence (atomicOr).  Integer atomics on disjoint bit fields commute, so the words are exact whatever the
// order of the atomics.  The apply kernel (vocabulary slices x rows) reads each logit and its word, writes the processed logit, and
// clears the words it found set, so nothing is cleared per call.  Unpenalised rows are copied.  The logits are read-only.
//
// Allowed-token masks (DESIGN §3.18) ride the same apply pass: a row with a mask (PenaltyRow::mask >= 0) reads one mask word per 32
// tokens (the lanes of a warp share it) and writes -inf for every token whose bit is clear, after its penalties.  A call without a
// masked row passes no mask and runs exactly as before.
#include "jl_common.cuh"

#include <math.h>

#include <algorithm>
#include <vector>

namespace {

constexpr int PEN_THREADS = 256;
constexpr int PEN_SLICE = 8192;
constexpr unsigned PEN_PROMPT = 0x80000000u;
constexpr unsigned PEN_BIAS = 0x40000000u;
constexpr unsigned PEN_COUNT = 0x3fffffffu;
constexpr int64_t PEN_MAX_HIST = PEN_COUNT; // a count never carries into the flag bits

__global__ void __launch_bounds__(PEN_THREADS) penalty_mark_kernel(const PenaltyRow *rows, const int32_t *hist, const int32_t *bias_ids,
                                                                   const float *bias_vals, int vocab, unsigned *cnt, float *bias) {
    const PenaltyRow r = rows[blockIdx.x];
    if (!r.on) return;
    unsigned *c = cnt + (size_t)blockIdx.x * vocab;
    float *bs = bias + (size_t)blockIdx.x * vocab;
    for (int j = r.hist0 + (int)threadIdx.x; j < r.hist1; j += PEN_THREADS) {
        const int t = hist[j];
        if (j < r.prompt1) atomicOr(c + t, PEN_PROMPT);
        else atomicAdd(c + t, 1u);
    }
    for (int j = r.bias0 + (int)threadIdx.x; j < r.bias1; j += PEN_THREADS) {
        const int t = bias_ids[j]; // distinct within the row
        bs[t] = bias_vals[j];
        atomicOr(c + t, PEN_BIAS);
    }
}

__global__ void __launch_bounds__(PEN_THREADS) penalty_apply_kernel(const float *logits, int64_t ld, int vocab, const PenaltyRow *rows,
                                                                    unsigned *cnt, const float *bias, const uint32_t *mask, float *out) {
    const int row = blockIdx.y;
    const PenaltyRow r = rows[row];
    const float *l = logits + (size_t)row * ld;
    float *o = out + (size_t)row * vocab;
    unsigned *c = cnt + (size_t)row * vocab;
    const float *bs = bias + (size_t)row * vocab;
    const uint32_t *mk = mask && r.mask >= 0 ? mask + (size_t)r.mask * (size_t)((vocab + 31) / 32) : nullptr;
    const int i1 = min(vocab, (int)(blockIdx.x + 1) * PEN_SLICE);
    for (int i = blockIdx.x * PEN_SLICE + (int)threadIdx.x; i < i1; i += PEN_THREADS) {
        float v = l[i];
        if (r.on) {
            const unsigned w = c[i];
            if (w) c[i] = 0u;
            const unsigned k = w & PEN_COUNT;
            v = __fadd_rn(v, (w & PEN_BIAS) ? bs[i] : 0.0f);
            if (w & (PEN_PROMPT | PEN_COUNT)) v = v < 0.0f ? __fmul_rn(v, r.repetition) : __fdiv_rn(v, r.repetition);
            v = __fsub_rn(v, __fmul_rn((float)k, r.frequency));
            if (k) v = __fsub_rn(v, r.presence);
        }
        if (mk && !((mk[i >> 5] >> (i & 31)) & 1u)) v = -INFINITY;
        o[i] = v;
    }
}

bool finite_in(float v, float lo, float hi) { return isfinite(v) && v >= lo && v <= hi; }

} // namespace

int jl_penalty_check(jl_ctx *ctx, const char *who, int n, int vocab, const jl_penalties *pen, PenaltyPlan *plan) {
    *plan = PenaltyPlan();
    if (!pen) return JL_OK;
    auto offsets = [&](const int32_t *off, const char *what) -> int {
        if (!off) return JL_OK;
        for (int i = 0; i <= n; i++) {
            if (off[i] < 0) return jl_set_error(ctx, JL_ERR_INVALID, "%s: %s_off[%d] = %d is negative", who, what, i, off[i]);
            if (i > 0 && off[i] < off[i - 1]) return jl_set_error(ctx, JL_ERR_INVALID, "%s: %s_off decreases at %d", who, what, i);
        }
        return JL_OK;
    };
    int rc = offsets(pen->hist_off, "hist");
    if (rc == JL_OK) rc = offsets(pen->bias_off, "bias");
    if (rc != JL_OK) return rc;
    const int64_t n_hist = pen->hist_off ? (int64_t)pen->hist_off[n] - pen->hist_off[0] : 0;
    const int64_t n_bias = pen->bias_off ? (int64_t)pen->bias_off[n] - pen->bias_off[0] : 0;
    if (n_hist > 0 && !pen->hist_ids) return jl_set_error(ctx, JL_ERR_INVALID, "%s: history entries without hist_ids", who);
    if (n_bias > 0 && (!pen->bias_ids || !pen->bias_vals)) return jl_set_error(ctx, JL_ERR_INVALID, "%s: bias entries without ids or values", who);
    if (n_hist > PEN_MAX_HIST || n_bias > PEN_MAX_HIST) return jl_set_error(ctx, JL_ERR_INVALID, "%s: too many history or bias entries", who);
    std::vector<int32_t> ids;
    for (int i = 0; i < n; i++) {
        const float pr = pen->presence ? pen->presence[i] : 0.0f, fr = pen->frequency ? pen->frequency[i] : 0.0f;
        const float rp = pen->repetition ? pen->repetition[i] : 1.0f;
        if (!finite_in(pr, -2.0f, 2.0f)) return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: presence %g outside [-2, 2]", who, i, (double)pr);
        if (!finite_in(fr, -2.0f, 2.0f)) return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: frequency %g outside [-2, 2]", who, i, (double)fr);
        if (!finite_in(rp, 0.0f, 100.0f) || rp == 0.0f)
            return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: repetition %g outside (0, 100]", who, i, (double)rp);
        const int h0 = pen->hist_off ? pen->hist_off[i] : 0, h1 = pen->hist_off ? pen->hist_off[i + 1] : 0;
        const int np = pen->hist_prompt ? pen->hist_prompt[i] : 0;
        if (np < 0 || np > h1 - h0) return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: hist_prompt %d outside [0, %d]", who, i, np, h1 - h0);
        for (int j = h0; j < h1; j++)
            if (pen->hist_ids[j] < 0 || pen->hist_ids[j] >= vocab)
                return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: history id %d outside [0, %d)", who, i, pen->hist_ids[j], vocab);
        const int b0 = pen->bias_off ? pen->bias_off[i] : 0, b1 = pen->bias_off ? pen->bias_off[i + 1] : 0;
        ids.assign(pen->bias_ids ? pen->bias_ids + b0 : nullptr, pen->bias_ids ? pen->bias_ids + b1 : nullptr);
        for (int j = b0; j < b1; j++) {
            if (pen->bias_ids[j] < 0 || pen->bias_ids[j] >= vocab)
                return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: bias id %d outside [0, %d)", who, i, pen->bias_ids[j], vocab);
            if (!finite_in(pen->bias_vals[j], -100.0f, 100.0f))
                return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: bias %g outside [-100, 100]", who, i, (double)pen->bias_vals[j]);
        }
        std::sort(ids.begin(), ids.end());
        if (std::adjacent_find(ids.begin(), ids.end()) != ids.end())
            return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: bias id %d listed twice", who, i, *std::adjacent_find(ids.begin(), ids.end()));
        plan->n_on += pr != 0.0f || fr != 0.0f || rp != 1.0f || b1 > b0;
    }
    plan->n_hist = (int)n_hist, plan->n_bias = (int)n_bias;
    plan->bytes = (size_t)n * sizeof(PenaltyRow) + (size_t)n_hist * 4 + (size_t)n_bias * 8;
    return JL_OK;
}

void jl_penalty_pack(const jl_penalties *pen, int n, const PenaltyPlan &plan, void *tab) {
    PenaltyRow *rows = (PenaltyRow *)tab;
    int32_t *hist = (int32_t *)(rows + n), *bias_ids = hist + plan.n_hist;
    float *bias_vals = (float *)(bias_ids + plan.n_bias);
    const int hb = pen->hist_off ? pen->hist_off[0] : 0, bb = pen->bias_off ? pen->bias_off[0] : 0;
    if (plan.n_hist) memcpy(hist, pen->hist_ids + hb, (size_t)plan.n_hist * 4);
    if (plan.n_bias) memcpy(bias_ids, pen->bias_ids + bb, (size_t)plan.n_bias * 4), memcpy(bias_vals, pen->bias_vals + bb, (size_t)plan.n_bias * 4);
    for (int i = 0; i < n; i++) {
        PenaltyRow &r = rows[i];
        r.presence = pen->presence ? pen->presence[i] : 0.0f;
        r.frequency = pen->frequency ? pen->frequency[i] : 0.0f;
        r.repetition = pen->repetition ? pen->repetition[i] : 1.0f;
        r.hist0 = pen->hist_off ? pen->hist_off[i] - hb : 0;
        r.hist1 = pen->hist_off ? pen->hist_off[i + 1] - hb : 0;
        r.prompt1 = r.hist0 + (pen->hist_prompt ? pen->hist_prompt[i] : 0);
        r.bias0 = pen->bias_off ? pen->bias_off[i] - bb : 0;
        r.bias1 = pen->bias_off ? pen->bias_off[i + 1] - bb : 0;
        r.on = r.presence != 0.0f || r.frequency != 0.0f || r.repetition != 1.0f || r.bias1 > r.bias0;
        r.mask = -1;
    }
}

int jl_launch_penalties(jl_ctx *ctx, cudaStream_t st, const float *logits, int64_t ld, int vocab, int n, const void *tab,
                        const PenaltyPlan &plan, unsigned *cnt, float *bias, const uint32_t *mask, float *out) {
    if (n <= 0) return JL_OK;
    if (vocab < 1 || n > 65535) return jl_set_error(ctx, JL_ERR_INVALID, "penalties: %d rows of vocabulary %d", n, vocab);
    const PenaltyRow *rows = (const PenaltyRow *)tab;
    const int32_t *hist = (const int32_t *)(rows + n), *bias_ids = hist + plan.n_hist;
    const float *bias_vals = (const float *)(bias_ids + plan.n_bias);
    if (!mask || plan.n_on > 0) { // a masked call without a penalised row has nothing to mark
        penalty_mark_kernel<<<n, PEN_THREADS, 0, st>>>(rows, hist, bias_ids, bias_vals, vocab, cnt, bias);
        ctx->launches++;
        JL_CUDA_CHECK(ctx, cudaGetLastError());
    }
    penalty_apply_kernel<<<dim3((vocab + PEN_SLICE - 1) / PEN_SLICE, n), PEN_THREADS, 0, st>>>(logits, ld, vocab, rows, cnt, bias, mask, out);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

int jl_constraint_check(jl_ctx *ctx, const char *who, int n, int vocab, int n_allow, const uint32_t *allow, const int32_t *allow_row,
                        int *n_on) {
    *n_on = 0;
    if (!allow_row) return JL_OK;
    if (n_allow < 0) return jl_set_error(ctx, JL_ERR_INVALID, "%s: n_allow = %d is negative", who, n_allow);
    if (n_allow > 0 && !allow) return jl_set_error(ctx, JL_ERR_INVALID, "%s: %d mask rows without allow", who, n_allow);
    const size_t words = (size_t)(vocab + 31) / 32;
    std::vector<char> seen((size_t)n_allow, 0); // 1: checked and not empty
    for (int i = 0; i < n; i++) {
        const int a = allow_row[i];
        if (a < -1 || a >= n_allow) return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: allow_row %d outside [-1, %d)", who, i, a, n_allow);
        if (a < 0) continue;
        if (!seen[(size_t)a]) {
            const uint32_t *w = allow + (size_t)a * words;
            bool any = false;
            for (size_t k = 0; k < words && !any; k++) {
                const int left = vocab - (int)(k * 32); // bits at or above vocab do not count
                any = (left >= 32 ? w[k] : w[k] & ((1u << left) - 1u)) != 0u;
            }
            if (!any) return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: mask row %d allows no token below %d", who, i, a, vocab);
            seen[(size_t)a] = 1;
        }
        ++*n_on;
    }
    return JL_OK;
}

int jl_constraint_pack(int n, int vocab, int n_allow, const uint32_t *allow, const int32_t *allow_row, void *tab, uint32_t *dst) {
    PenaltyRow *rows = (PenaltyRow *)tab;
    const size_t words = (size_t)(vocab + 31) / 32;
    std::vector<int> slot((size_t)n_allow, -1);
    int c = 0;
    for (int i = 0; i < n; i++) {
        const int a = allow_row[i];
        if (a >= 0 && slot[(size_t)a] < 0) {
            slot[(size_t)a] = c;
            memcpy(dst + (size_t)c++ * words, allow + (size_t)a * words, words * 4);
        }
        rows[i].mask = a >= 0 ? slot[(size_t)a] : -1;
    }
    return c;
}

// HOST-buffer entry point for crafted rows
extern "C" int jl_apply_penalties(jl_ctx *ctx, int n, int vocab, const float *logits, int64_t ld, const jl_penalties *pen, float *out) {
    if (!ctx) return JL_ERR_INVALID;
    if (n < 1 || n > 65535 || vocab < 1 || ld < vocab || !logits || !out)
        return jl_set_error(ctx, JL_ERR_INVALID, "apply_penalties: bad arguments (n=%d, vocab=%d, ld=%lld)", n, vocab, (long long)ld);
    PenaltyPlan plan;
    const int crc = jl_penalty_check(ctx, "apply_penalties", n, vocab, pen, &plan);
    if (crc != JL_OK) return crc;
    const jl_penalties none = {};
    std::vector<char> tab(plan.bytes ? plan.bytes : (size_t)n * sizeof(PenaltyRow));
    PenaltyPlan p = plan;
    p.bytes = tab.size();
    jl_penalty_pack(pen ? pen : &none, n, p, tab.data());
    std::lock_guard<std::mutex> lk(ctx->mu);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    const size_t lb = ((size_t)(n - 1) * ld + vocab) * 4, rb = (size_t)n * vocab * 4, tb = (tab.size() + 15) & ~(size_t)15;
    float *dl = (float *)jl_scratch(ctx, 0, lb);
    char *dw = (char *)jl_scratch(ctx, 1, 2 * rb + tb);
    float *dout = (float *)jl_scratch(ctx, 2, rb);
    if (!dl || !dw || !dout) return JL_ERR_OOM;
    unsigned *dcnt = (unsigned *)dw;
    float *dbias = (float *)(dw + rb);
    void *dtab = dw + 2 * rb;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dl, logits, lb, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemsetAsync(dcnt, 0, rb, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dtab, tab.data(), tab.size(), cudaMemcpyHostToDevice, ctx->stream));
    const int rc = jl_launch_penalties(ctx, ctx->stream, dl, ld, vocab, n, dtab, p, dcnt, dbias, nullptr, dout);
    if (rc != JL_OK) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(out, dout, rb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}
