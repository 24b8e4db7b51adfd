// Token log-probabilities of logits rows: the rule of DESIGN §3.13.
//
// Per row l[0..V), with m = max l and Z = sum_i exp((double) l_i - (double) m) in double:
//   lp_i = (float) (((double) l_i - (double) m) - log(Z))
// for the row's target token and for its top-N tokens (the N largest l, by l descending then index ascending; N <= JL_MAX_LOGPROBS).
//
// The grid is (vocabulary slices of LP_SLICE tokens) x (rows).  Each CTA stages its slice in shared memory and computes the slice max
// m_s, Z_s = sum exp(l - m_s) in double and its top-N candidates (N rounds of a block arg-max: after a round only the thread that held
// the winner rescans its elements).  The last CTA of a row to arrive merges the slices in slice order: M = max m_s,
// Z = sum_s Z_s * exp(m_s - M), then the N best of the slices' sorted candidate lists.  The split of a row depends on V alone and every
// reduction runs in a fixed order, so the bits depend only on the row: not on the number of rows in the launch or the row's slot.
// The logits are read-only.
#include "jl_common.cuh"

#include <math.h>

namespace {

constexpr int LP_THREADS = 256;
constexpr int LP_SLICE = 8192;
constexpr int LP_PER = LP_SLICE / LP_THREADS;
constexpr int LP_WARPS = LP_THREADS / 32;
constexpr int LP_NONE = 0x7fffffff;
constexpr int LP_MAX_SLICES = JL_LOGPROBS_MAX_VOCAB / LP_SLICE;
// the merge reuses the slice buffer: candidates at [0, S*N) and [LP_SLICE/2, LP_SLICE/2 + S*N), slice maxima and list heads below each
static_assert(LP_MAX_SLICES * JL_MAX_LOGPROBS <= LP_SLICE / 2 - LP_MAX_SLICES, "merge does not fit the slice buffer");
static_assert(JL_LOGPROBS_MAX_VOCAB % LP_SLICE == 0, "whole slices");

// one (row, slice) of the workspace
struct LpSlice {
    float m;
    float cl[JL_MAX_LOGPROBS]; // candidate logits, best first
    int ci[JL_MAX_LOGPROBS];   // candidate token ids (-1: the slice has no more)
    double z;
};

__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

// arg-max of (v, i) over the block (ties: lowest index) through LP_WARPS slots of red_v / red_i; callers alternate between two slot
// buffers so that one barrier per call suffices
__device__ __forceinline__ void block_argmax(float &v, int &i, float *red_v, int *red_i) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (better(ov, oi, v, i)) v = ov, i = oi;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) red_v[warp] = v, red_i[warp] = i;
    __syncthreads();
    v = red_v[0], i = red_i[0];
#pragma unroll
    for (int w = 1; w < LP_WARPS; w++)
        if (better(red_v[w], red_i[w], v, i)) v = red_v[w], i = red_i[w];
}

__global__ void __launch_bounds__(LP_THREADS)
    logprobs_kernel(const float *__restrict__ logits, int64_t ld, int vocab, const LogprobRow *__restrict__ rows,
                    const int32_t *__restrict__ targets, LpSlice *__restrict__ ws, unsigned *__restrict__ cnt, LogprobOut *__restrict__ out) {
    __shared__ float v[LP_SLICE];
    __shared__ float red_v[2][LP_WARPS];
    __shared__ int red_i[2][LP_WARPS];
    __shared__ double red_d[LP_WARPS];
    __shared__ bool last;
    const LogprobRow R = rows[blockIdx.y];
    const int S = gridDim.x, s = blockIdx.x, base = s * LP_SLICE;
    const int len = vocab - base < LP_SLICE ? vocab - base : LP_SLICE;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float *row = logits + (size_t)R.row * ld;
    LpSlice *slices = ws + (size_t)blockIdx.y * S;

    // ---- stage the slice (element j * LP_THREADS + tid belongs to thread tid; NaN marks "not a candidate") + slice max ----
    float mx = -INFINITY;
#pragma unroll 8
    for (int j = 0; j < LP_PER; j++) {
        const int i = j * LP_THREADS + tid;
        const float x = i < len ? row[base + i] : NAN;
        v[i] = x;
        if (i < len) mx = fmaxf(mx, x);
    }
    {
        int dummy = 0;
        block_argmax(mx, dummy, red_v[0], red_i[0]);
    }
    // ---- Z_s = sum exp(l - m_s) in double (an all -inf slice contributes 0) ----
    double z = 0.0;
    if (mx != -INFINITY) {
        const double dm = (double)mx;
#pragma unroll 8
        for (int j = 0; j < LP_PER; j++) {
            const int i = j * LP_THREADS + tid;
            if (i < len) z += exp((double)v[i] - dm);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    if (lane == 0) red_d[warp] = z;
    __syncthreads();
    if (tid == 0) {
        double t = red_d[0];
        for (int w = 1; w < LP_WARPS; w++) t += red_d[w];
        slices[s].m = mx;
        slices[s].z = t;
    }

    // ---- top-N candidates of the slice ----
    const int N = R.top_n;
    float bv = -INFINITY;
    int bi = LP_NONE;
    auto rescan = [&]() {
        bv = -INFINITY, bi = LP_NONE;
        for (int j = 0; j < LP_PER; j++) {
            const int i = j * LP_THREADS + tid;
            const float x = v[i];
            if (better(x, i, bv, bi)) bv = x, bi = i;
        }
    };
    if (N > 0) rescan();
    for (int r = 0; r < N; r++) {
        float wv = bv;
        int wi = bi;
        block_argmax(wv, wi, red_v[(r + 1) & 1], red_i[(r + 1) & 1]);
        if (tid == 0) slices[s].cl[r] = wv, slices[s].ci[r] = wi == LP_NONE ? -1 : base + wi;
        if (wi != LP_NONE && (wi % LP_THREADS) == tid) {
            v[wi] = NAN;
            rescan();
        }
    }

    // ---- the last CTA of the row merges ----
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        const unsigned old = atomicAdd(&cnt[blockIdx.y], 1u);
        last = old == (unsigned)(S - 1);
        if (last) cnt[blockIdx.y] = 0; // every slice has arrived: reset for the next launch
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    // slice candidates -> shared memory (cl at v[0..S*N), ci at v[LP_SLICE/2..)), heads of the sorted lists after them
    float *cl = v;
    int *ci = (int *)(v + LP_SLICE / 2);
    float *sm = v + LP_SLICE / 2 - LP_MAX_SLICES; // slice maxima
    int *head = (int *)(v + LP_SLICE - LP_MAX_SLICES);
    for (int k = tid; k < S * N; k += LP_THREADS) {
        const int ss = k / N, r = k - ss * N;
        cl[k] = __ldcg(&slices[ss].cl[r]);
        ci[k] = __ldcg(&slices[ss].ci[r]);
    }
    for (int k = tid; k < S; k += LP_THREADS) sm[k] = __ldcg(&slices[k].m), head[k] = 0;
    __syncthreads(); // slice maxima, list heads and candidates are read by other threads below
    if (tid == 0) {
        float M = sm[0];
        for (int k = 1; k < S; k++) M = fmaxf(M, sm[k]);
        double Z = 0.0;
        for (int k = 0; k < S; k++) // slice order
            if (sm[k] != -INFINITY) Z += __ldcg(&slices[k].z) * exp((double)sm[k] - (double)M);
        red_d[0] = (double)M, red_d[1] = log(Z);
    }
    __syncthreads();
    const double M = red_d[0], logZ = red_d[1];
    LogprobOut &o = out[R.row];
    if (tid == 0) {
        const int t = targets ? targets[R.row] : -1;
        o.lp = t >= 0 && t < vocab ? (float)(((double)row[t] - M) - logZ) : NAN;
    }
    if (warp == 0) {
        for (int r = 0; r < JL_MAX_LOGPROBS; r++) {
            float wv = -INFINITY;
            int wi = LP_NONE, wsl = -1;
            for (int k = lane; r < N && k < S; k += 32) {
                const int h = head[k];
                if (h < N && ci[k * N + h] >= 0 && better(cl[k * N + h], ci[k * N + h], wv, wi)) wv = cl[k * N + h], wi = ci[k * N + h], wsl = k;
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, wv, off);
                const int oi = __shfl_xor_sync(0xffffffffu, wi, off);
                const int os = __shfl_xor_sync(0xffffffffu, wsl, off);
                if (better(ov, oi, wv, wi)) wv = ov, wi = oi, wsl = os;
            }
            if (lane == 0) {
                const bool have = wi != LP_NONE;
                o.ids[r] = have ? wi : -1;
                o.lps[r] = have ? (float)(((double)wv - M) - logZ) : NAN;
                if (have) head[wsl]++;
            }
            __syncwarp();
        }
    }
}

} // namespace

int jl_logprobs_slices(int vocab) { return (vocab + LP_SLICE - 1) / LP_SLICE; }

size_t jl_logprobs_ws_bytes(int vocab, int rows) { return (size_t)rows * jl_logprobs_slices(vocab) * sizeof(LpSlice); }

int jl_launch_logprobs(jl_ctx *ctx, cudaStream_t st, const float *logits, int64_t ld, int vocab, const LogprobRow *rows, int n,
                       const int32_t *targets, void *ws, unsigned *cnt, LogprobOut *out) {
    if (n <= 0) return JL_OK;
    if (vocab < 1 || vocab > JL_LOGPROBS_MAX_VOCAB || n > 65535)
        return jl_set_error(ctx, JL_ERR_INVALID, "logprobs: %d rows of vocabulary %d", n, vocab);
    logprobs_kernel<<<dim3(jl_logprobs_slices(vocab), n), LP_THREADS, 0, st>>>(logits, ld, vocab, rows, targets, (LpSlice *)ws, cnt, out);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

void jl_logprobs_unpack(const LogprobOut *o, const int32_t *top_n, int n, float *lp_out, int32_t *top_ids_out, float *top_lp_out) {
    for (int i = 0; i < n; i++) {
        const bool on = top_n && top_n[i] >= 0; // top_n NULL: every row without logprobs
        if (lp_out) lp_out[i] = on ? o[i].lp : NAN;
        for (int r = 0; r < JL_MAX_LOGPROBS; r++) {
            const bool slot = on && r < top_n[i];
            if (top_ids_out) top_ids_out[(size_t)i * JL_MAX_LOGPROBS + r] = slot ? o[i].ids[r] : -1;
            if (top_lp_out) top_lp_out[(size_t)i * JL_MAX_LOGPROBS + r] = slot ? o[i].lps[r] : NAN;
        }
    }
}

int jl_logprobs_check(jl_ctx *ctx, const char *who, int n, int vocab, const int32_t *top_n, int *n_on) {
    int k = 0;
    for (int i = 0; i < n; i++) {
        const int t = top_n ? top_n[i] : -1;
        if (t < -1 || t > JL_MAX_LOGPROBS) return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: top_n %d (-1..%d)", who, i, t, JL_MAX_LOGPROBS);
        k += t >= 0;
    }
    if (k > 0 && vocab > JL_LOGPROBS_MAX_VOCAB)
        return jl_set_error(ctx, JL_ERR_INVALID, "%s: vocabulary of %d above %d", who, vocab, JL_LOGPROBS_MAX_VOCAB);
    if (n_on) *n_on = k;
    return JL_OK;
}

// HOST-buffer entry point for crafted rows
extern "C" int jl_logprobs(jl_ctx *ctx, int n, int vocab, const float *logits, int64_t ld, const int32_t *targets, const int32_t *top_n,
                           float *lp_out, int32_t *top_ids_out, float *top_lp_out) {
    if (!ctx) return JL_ERR_INVALID;
    if (n < 1 || vocab < 1 || ld < vocab || !logits || !top_n || !lp_out)
        return jl_set_error(ctx, JL_ERR_INVALID, "logprobs: bad arguments (n=%d, vocab=%d, ld=%lld)", n, vocab, (long long)ld);
    int n_on = 0;
    const int crc = jl_logprobs_check(ctx, "logprobs", n, vocab, top_n, &n_on);
    if (crc != JL_OK) return crc;
    for (int i = 0; i < n; i++) {
        if (targets && (targets[i] < -1 || targets[i] >= vocab))
            return jl_set_error(ctx, JL_ERR_INVALID, "logprobs: row %d: target %d outside [-1, %d)", i, targets[i], vocab);
        const float *l = logits + (size_t)i * ld;
        bool finite = false;
        for (int k = 0; k < vocab; k++) {
            if (isnan(l[k]) || l[k] == INFINITY) return jl_set_error(ctx, JL_ERR_INVALID, "logprobs: row %d: NaN or +inf at %d", i, k);
            finite = finite || l[k] != -INFINITY;
        }
        if (!finite) return jl_set_error(ctx, JL_ERR_INVALID, "logprobs: row %d has no finite logit", i);
    }
    std::vector<LogprobRow> hr;
    for (int i = 0; i < n; i++)
        if (top_n[i] >= 0) hr.push_back(LogprobRow{i, top_n[i]});
    std::vector<LogprobOut> ho((size_t)n);
    if (n_on > 0) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
        const size_t lb = ((size_t)(n - 1) * ld + vocab) * 4;
        const size_t wsb = jl_logprobs_ws_bytes(vocab, n_on), cb = (size_t)n_on * 4, rb = (size_t)n_on * sizeof(LogprobRow), tb = (size_t)n * 4;
        float *dl = (float *)jl_scratch(ctx, 0, lb);
        char *dw = (char *)jl_scratch(ctx, 1, wsb + cb + rb + tb + 64);
        LogprobOut *dout = (LogprobOut *)jl_scratch(ctx, 2, (size_t)n * sizeof(LogprobOut));
        if (!dl || !dw || !dout) return JL_ERR_OOM;
        unsigned *dcnt = (unsigned *)(dw + wsb);
        LogprobRow *drows = (LogprobRow *)(dw + wsb + cb);
        int32_t *dtgt = (int32_t *)(dw + wsb + cb + rb);
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dl, logits, lb, cudaMemcpyHostToDevice, ctx->stream));
        JL_CUDA_CHECK(ctx, cudaMemsetAsync(dcnt, 0, cb, ctx->stream));
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(drows, hr.data(), rb, cudaMemcpyHostToDevice, ctx->stream));
        if (targets) JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dtgt, targets, tb, cudaMemcpyHostToDevice, ctx->stream));
        const int rc = jl_launch_logprobs(ctx, ctx->stream, dl, ld, vocab, drows, n_on, targets ? dtgt : nullptr, dw, dcnt, dout);
        if (rc != JL_OK) return rc;
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(ho.data(), dout, (size_t)n * sizeof(LogprobOut), cudaMemcpyDeviceToHost, ctx->stream));
        JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    }
    jl_logprobs_unpack(ho.data(), top_n, n, lp_out, top_ids_out, top_lp_out);
    return JL_OK;
}
