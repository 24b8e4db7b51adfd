// Concurrent-session scheduler: iteration-level ("continuous") batching of generation requests into the batched decode step.
//
// The reference serves concurrent requests with one thread per request, each running AbstractModel.generate() on its own KvBuffer
// (core/tensor/KvBufferCache.java:58-60; jlama-net/.../openai/OpenAIChatService.java:64-74,107-160): the weights are streamed once
// per thread per token.  On the GPU the unit that shares one weight stream is the *decode step over N sessions* (jl_model_decode,
// csrc/jl_gemm8.cu), so concurrency becomes a queue in front of that step:
//
//   every jl_sched_step():   admit queued requests into free session slots (FIFO)            KvBufferCache.getKvBuffer
//                            forward prompt chunks of the admitted requests (token budget)    AbstractModel.batchForward :295-312
//                              in ONE batch_forward_multi call when a batch backend is installed
//                            sample their first token when a prompt is complete               AbstractModel.generate :576
//                            ONE decode step for every generating request, <= max_rows rows   AbstractModel.generate :590-600
//                              per call, requests of different lengths side by side
//                            retire requests that hit a stop token / their token limit        :604-608, FinishReason
//                            -> their slots are free for the next step's admissions
//
// The scheduler is pure host logic above four backend calls (reset_session / batch_forward / sample / decode).  jl_sched_create
// binds them to a jl_model; jl_sched_create_backend takes them as function pointers, which is how the CPU tests drive the very same
// policy code with the oracle as the "device" (tests/test_scheduler.py) and how a host that owns its own model object would plug in.
// Kept sessions and host spill: a finished JL_SCHED_KEEP_SESSION request holds its slot and KV for a follow-up turn.  When a request
// finds no free slot and the backend can offload (jl_model_kv_offload), the least recently finished kept session is moved to host
// memory and its slot is reused; its continuation later restores the pages into whatever slot is free (jl_model_kv_restore).
// Locking: `step_mu` serialises steps; `mu` guards the request table and is NOT held across backend calls, so submit / result /
// cancel from other threads never wait for GPU work.
#include <algorithm>
#include <chrono>
#include <deque>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include "../../include/jlama_b200.h"

void jl_model_limits(jl_model *m, int out[6]); // jl_model.cu: {max_sessions, max_context, max_batch, max rows per decode call, ctx_per_page,
                                               // vocab_size}

namespace {

// the penalties of a request (DESIGN §3.14); its history is built per call from its prompt and generated tokens
struct Penalty {
    float presence = 0.0f, frequency = 0.0f, repetition = 1.0f;
    std::vector<int32_t> bias_ids;
    std::vector<float> bias_vals;
    bool on() const { return presence != 0.0f || frequency != 0.0f || repetition != 1.0f || !bias_ids.empty(); }
};

struct Request {
    int64_t id = 0;
    std::vector<int32_t> prompt;
    std::vector<int32_t> stop;
    int max_new = 0;
    int flags = 0;
    float temperature = 0.0f;
    int top_k = 0;      // top-k / top-p filter of a request with temperature > 0 (filtered() decides whether it applies)
    float top_p = 1.0f;
    int logprobs = -1;  // -1: none; else the top alternatives per generated token (0..JL_MAX_LOGPROBS)
    std::vector<float> lp, top_lp;   // per generated token: its logprob, [JL_MAX_LOGPROBS] alternatives' logprobs
    std::vector<int32_t> top_ids;    // [JL_MAX_LOGPROBS] per generated token
    Penalty pen;
    uint64_t rng = 0; // splitmix64 state: the k-th sampled token of a request uses its k-th draw, however the steps were batched
    int state = JL_SCHED_QUEUED;
    int reason = JL_FINISH_NONE;
    int session = -1;
    int start_pos = 0;  // context position of prompt[0] (> 0 when the request continues a kept session)
    int prefilled = 0;  // prompt tokens already forwarded
    int forwarded = 0;  // generated tokens already fed back through a decode step
    int cached = 0;     // prompt tokens attached from the prefix cache instead of forwarded
    bool cancel = false;
    int64_t parent = -1;     // finished request whose kept session (and KV) this request continues
    int64_t child = -1;      // pending / admitted continuation of this request
    // n completions of one prompt (jl_sched_submit_n): the leader forwards the prompt, then its session is forked into the siblings'
    int64_t leader = -1;            // sibling still waiting for the fork: its group's leader
    std::vector<int64_t> siblings;  // leader: the siblings still waiting for the fork
    bool spilling = false;   // chosen as the victim of this step's offload; `spill` is set when the backend call returns
    int64_t spill = -1;      // backend handle of this finished request's KV after it was offloaded to host memory (session == -1 then)
    std::vector<int32_t> out;
    uint64_t submit_step = 0, first_token_step = 0, finish_step = 0;
    // host clock, like Generator.Response's promptTimeMs / generateTimeMs (AbstractModel.java:561-568,589,623): queued -> admitted ->
    // first token -> finished
    std::chrono::steady_clock::time_point t_submit, t_admit, t_first, t_finish;
    bool admitted = false;
    int next_pos() const { return start_pos + (int)prompt.size() + forwarded; } // position the next decode step writes
    bool filtered() const { return temperature > 0.0f && (top_k > 0 || top_p < 1.0f); }
};

// a cached prefix (DESIGN §3.17): the backend handle retaining the KV of `tokens` (a whole number of pages) at positions [0, tokens.size())
struct PrefixEntry {
    int64_t handle = -1;
    std::vector<int32_t> tokens;
    std::vector<uint64_t> hashes; // hash of tokens[0, (k + 1) * ctx_per_page) per page k: its keys in the index
    uint64_t last_use = 0;        // step of the last insert or hit
    int pins = 0;                 // jobs of the current step that attach from it: neither evicted nor replaced until they have
};

// the running hash of a token prefix at every page boundary, over the first `pages` pages
std::vector<uint64_t> page_hashes(const int32_t *t, int pages, int cpp) {
    std::vector<uint64_t> out((size_t)pages);
    uint64_t h = 1469598103934665603ull;
    for (int k = 0; k < pages; k++) {
        for (int i = k * cpp; i < (k + 1) * cpp; i++) h = (h ^ (uint64_t)(uint32_t)t[i]) * 1099511628211ull;
        out[(size_t)k] = h;
    }
    return out;
}

} // namespace

struct jl_sched {
    jl_sched_backend be;
    jl_sched_batch_backend bb = {}; // optional: all prompt chunks of a step in one call
    jl_sched_topkp_backend tb = {}; // optional: calls with a top-k / top-p filtered row
    jl_sched_logprob_backend lb = {}; // optional: calls with a logprob request
    jl_sched_penalty_backend pb = {}; // optional: calls with a penalised request
    jl_sched_constraint_backend cb = {}; // optional: calls with a constrained request, with the mask provider below
    jl_sched_mask_fn *mask_fn = nullptr;
    void *mask_user = nullptr;
    jl_sched_fork_backend fb = {};    // optional: n completions of one prompt
    jl_model *model = nullptr;        // jl_sched_create: the model behind the backend
    // prefix cache (DESIGN §3.17), on when prefix_max_pages > 0; entries and index change under `mu`, their handles outside it
    jl_sched_prefix_backend xb = {};
    int prefix_max_pages = 0;
    std::map<int64_t, PrefixEntry> prefix;              // entry id (insertion order) -> entry
    std::unordered_multimap<uint64_t, int64_t> prefix_index; // page-boundary hash -> entries whose tokens start with that prefix
    int64_t next_entry = 1;
    jl_sched_prefix_stats_t pstats = {};
    struct PendingRetain {
        int session;
        std::vector<int32_t> tokens;
    };
    std::vector<PendingRetain> retains; // finished fresh requests whose KV is retained before their slot is reused
    void *user = nullptr;
    int n_sessions = 0, max_rows = 0, max_context = 0, prefill_budget = 0;
    std::mutex mu, step_mu;
    std::unordered_map<int64_t, Request> reqs;
    std::deque<int64_t> queue;        // admission order
    std::vector<int64_t> active;      // admitted, unfinished requests in admission order
    std::vector<int64_t> slot_owner;  // session slot -> request id, -1 = free; a kept session stays owned by its finished request
    int64_t next_id = 1;
    uint64_t step_no = 0;
    std::string last_error;
    jl_sched_stats totals = {};
    std::vector<int64_t> discards; // spill handles of released requests, dropped by the next step (backend calls never run under `mu`)
};

static int sched_error(jl_sched *s, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    s->last_error = buf;
    return code;
}

// ThreadLocalRandom.current().nextFloat() of AbstractModel.generate (:576, :594): 24 random bits / 2^24 in [0, 1), from a per-request
// splitmix64 stream so that a (seed, prompt) pair reproduces its tokens.
static float next_uniform(Request &r) {
    uint64_t z = (r.rng += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    return (float)(z >> 40) * (1.0f / 16777216.0f);
}

// ---- jl_model backend ---------------------------------------------------------------------------------------------------------
static int mb_reset(void *u, int session) { return jl_model_reset_session((jl_model *)u, session); }
static int mb_forward(void *u, int session, const int32_t *tokens, int n, int start_pos) {
    return jl_model_batch_forward((jl_model *)u, session, tokens, n, start_pos);
}
static int mb_sample(void *u, int session, float temperature, float uniform, int32_t *token) {
    return jl_model_sample((jl_model *)u, session, temperature, uniform, token, nullptr);
}
static int mb_decode(void *u, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions, const float *temperatures,
                     const float *uniforms, int32_t *next) {
    return jl_model_decode_sample((jl_model *)u, n, sessions, tokens, positions, temperatures, uniforms, next, nullptr);
}

// weak: the policy code also links on its own, without the model (tests/native builds it that way)
extern "C" int jl_model_batch_forward_multi(jl_model *, int, const int32_t *, const int32_t *, const int32_t *, const int32_t *) __attribute__((weak));
extern "C" int jl_model_sample_multi(jl_model *, int, const int32_t *, const float *, const float *, int32_t *, float *) __attribute__((weak));
static int mb_forward_multi(void *u, int n_seg, const int32_t *sessions, const int32_t *start_pos, const int32_t *lengths, const int32_t *tokens) {
    return jl_model_batch_forward_multi((jl_model *)u, n_seg, sessions, start_pos, lengths, tokens);
}
static int mb_sample_multi(void *u, int n, const int32_t *sessions, const float *temperatures, const float *uniforms, int32_t *tokens) {
    return jl_model_sample_multi((jl_model *)u, n, sessions, temperatures, uniforms, tokens, nullptr);
}
extern "C" int jl_model_decode_sample_topkp(jl_model *, int, const int32_t *, const int32_t *, const int32_t *, const float *, const int32_t *,
                                            const float *, const float *, int32_t *, float *) __attribute__((weak));
extern "C" int jl_model_sample_multi_topkp(jl_model *, int, const int32_t *, const float *, const int32_t *, const float *, const float *,
                                           int32_t *, float *) __attribute__((weak));
extern "C" int jl_model_decode_logprobs(jl_model *, int, const int32_t *, const int32_t *, const int32_t *, const float *, const int32_t *,
                                        const float *, const float *, const int32_t *, int32_t *, float *, int32_t *, float *, float *)
    __attribute__((weak));
extern "C" int jl_model_sample_multi_logprobs(jl_model *, int, const int32_t *, const float *, const int32_t *, const float *, const float *,
                                              const int32_t *, int32_t *, float *, int32_t *, float *, float *) __attribute__((weak));
static int mb_decode_logprobs(void *u, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions, const float *temperatures,
                              const int32_t *top_k, const float *top_p, const float *uniforms, const int32_t *top_n, int32_t *next, float *lp,
                              int32_t *top_ids, float *top_lp) {
    return jl_model_decode_logprobs((jl_model *)u, n, sessions, tokens, positions, temperatures, top_k, top_p, uniforms, top_n, next, lp, top_ids,
                                    top_lp, nullptr);
}
static int mb_sample_multi_logprobs(void *u, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k, const float *top_p,
                                    const float *uniforms, const int32_t *top_n, int32_t *tokens, float *lp, int32_t *top_ids, float *top_lp) {
    return jl_model_sample_multi_logprobs((jl_model *)u, n, sessions, temperatures, top_k, top_p, uniforms, top_n, tokens, lp, top_ids, top_lp,
                                          nullptr);
}
extern "C" int jl_model_decode_penalized(jl_model *, int, const int32_t *, const int32_t *, const int32_t *, const float *, const int32_t *,
                                         const float *, const float *, const int32_t *, const jl_penalties *, int32_t *, float *, int32_t *, float *,
                                         float *) __attribute__((weak));
extern "C" int jl_model_sample_multi_penalized(jl_model *, int, const int32_t *, const float *, const int32_t *, const float *, const float *,
                                               const int32_t *, const jl_penalties *, int32_t *, float *, int32_t *, float *, float *)
    __attribute__((weak));
static int mb_decode_penalized(void *u, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions, const float *temperatures,
                               const int32_t *top_k, const float *top_p, const float *uniforms, const int32_t *top_n, const jl_penalties *pen,
                               int32_t *next, float *lp, int32_t *top_ids, float *top_lp) {
    return jl_model_decode_penalized((jl_model *)u, n, sessions, tokens, positions, temperatures, top_k, top_p, uniforms, top_n, pen, next, lp,
                                     top_ids, top_lp, nullptr);
}
static int mb_sample_multi_penalized(void *u, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                     const float *top_p, const float *uniforms, const int32_t *top_n, const jl_penalties *pen, int32_t *tokens,
                                     float *lp, int32_t *top_ids, float *top_lp) {
    return jl_model_sample_multi_penalized((jl_model *)u, n, sessions, temperatures, top_k, top_p, uniforms, top_n, pen, tokens, lp, top_ids,
                                           top_lp, nullptr);
}
static int mb_decode_topkp(void *u, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions, const float *temperatures,
                           const int32_t *top_k, const float *top_p, const float *uniforms, int32_t *next) {
    return jl_model_decode_sample_topkp((jl_model *)u, n, sessions, tokens, positions, temperatures, top_k, top_p, uniforms, next, nullptr);
}
static int mb_sample_multi_topkp(void *u, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k, const float *top_p,
                                 const float *uniforms, int32_t *tokens) {
    return jl_model_sample_multi_topkp((jl_model *)u, n, sessions, temperatures, top_k, top_p, uniforms, tokens, nullptr);
}

extern "C" int jl_model_decode_constrained(jl_model *, int, const int32_t *, const int32_t *, const int32_t *, const float *, const int32_t *,
                                           const float *, const float *, const int32_t *, const jl_penalties *, int, const uint32_t *,
                                           const int32_t *, int32_t *, float *, int32_t *, float *, float *) __attribute__((weak));
extern "C" int jl_model_sample_multi_constrained(jl_model *, int, const int32_t *, const float *, const int32_t *, const float *, const float *,
                                                 const int32_t *, const jl_penalties *, int, const uint32_t *, const int32_t *, int32_t *, float *,
                                                 int32_t *, float *, float *) __attribute__((weak));
static int mb_decode_constrained(void *u, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                                 const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms, const int32_t *top_n,
                                 const jl_penalties *pen, int n_allow, const uint32_t *allow, const int32_t *allow_row, int32_t *next, float *lp,
                                 int32_t *top_ids, float *top_lp) {
    return jl_model_decode_constrained((jl_model *)u, n, sessions, tokens, positions, temperatures, top_k, top_p, uniforms, top_n, pen, n_allow,
                                       allow, allow_row, next, lp, top_ids, top_lp, nullptr);
}
static int mb_sample_multi_constrained(void *u, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                       const float *top_p, const float *uniforms, const int32_t *top_n, const jl_penalties *pen, int n_allow,
                                       const uint32_t *allow, const int32_t *allow_row, int32_t *tokens, float *lp, int32_t *top_ids,
                                       float *top_lp) {
    return jl_model_sample_multi_constrained((jl_model *)u, n, sessions, temperatures, top_k, top_p, uniforms, top_n, pen, n_allow, allow,
                                             allow_row, tokens, lp, top_ids, top_lp, nullptr);
}

extern "C" int jl_model_kv_fork(jl_model *, int, int, int, const int32_t *) __attribute__((weak));
static int mb_fork(void *u, int src, int positions, int n, const int32_t *dst) { return jl_model_kv_fork((jl_model *)u, src, positions, n, dst); }

static int mb_offload(void *u, int session, int64_t *handle) {
    const int64_t h = jl_model_kv_offload((jl_model *)u, session);
    if (h < 0) return (int)h;
    *handle = h;
    return JL_OK;
}
static int mb_restore(void *u, int session, int64_t handle) { return jl_model_kv_restore((jl_model *)u, session, handle); }
static int mb_discard(void *u, int64_t handle) { return jl_model_kv_discard((jl_model *)u, handle); }

extern "C" int64_t jl_model_kv_retain(jl_model *, int, int) __attribute__((weak));
extern "C" int jl_model_kv_attach(jl_model *, int64_t, int, int) __attribute__((weak));
extern "C" int jl_model_kv_release(jl_model *, int64_t) __attribute__((weak));
extern "C" int jl_model_kv_retained(jl_model *, int64_t *, int64_t *) __attribute__((weak));
static int mb_retain(void *u, int session, int positions, int64_t *handle) {
    const int64_t h = jl_model_kv_retain((jl_model *)u, session, positions);
    if (h < 0) return (int)h;
    *handle = h;
    return JL_OK;
}
static int mb_attach(void *u, int64_t handle, int positions, int session) { return jl_model_kv_attach((jl_model *)u, handle, positions, session); }
static int mb_release(void *u, int64_t handle) { return jl_model_kv_release((jl_model *)u, handle); }
static int mb_retained(void *u, int64_t *handles, int64_t *pages) { return jl_model_kv_retained((jl_model *)u, handles, pages); }

extern "C" int jl_sched_create_backend(const jl_sched_backend *be, void *user, int n_sessions, int max_rows, int max_context,
                                       int prefill_tokens_per_step, jl_sched **out) {
    if (!be || !out || !be->reset_session || !be->batch_forward || !be->sample || !be->decode || n_sessions <= 0 || max_rows <= 0 ||
        max_context <= 1)
        return JL_ERR_INVALID;
    if ((be->offload != nullptr) != (be->restore != nullptr) || (be->offload != nullptr) != (be->discard != nullptr))
        return JL_ERR_INVALID; // host spill is all three calls or none
    jl_sched *s = new jl_sched();
    s->be = *be;
    s->user = user;
    s->n_sessions = n_sessions;
    s->max_rows = max_rows;
    s->max_context = max_context;
    s->prefill_budget = prefill_tokens_per_step > 0 ? prefill_tokens_per_step : 0;
    s->slot_owner.assign((size_t)n_sessions, -1);
    *out = s;
    return JL_OK;
}

extern "C" int jl_sched_create(jl_model *m, int max_active, int prefill_tokens_per_step, jl_sched **out) {
    if (!m || !out) return JL_ERR_INVALID;
    int lim[6] = {0, 0, 0, 0, 0, 0};
    jl_model_limits(m, lim);
    if (lim[0] <= 0) return JL_ERR_INVALID; // not finalized
    const int n = max_active > 0 && max_active < lim[0] ? max_active : lim[0];
    static const jl_sched_backend be = {mb_reset, mb_forward, mb_sample, mb_decode, mb_offload, mb_restore, mb_discard};
    const int rc = jl_sched_create_backend(&be, m, n, lim[3], lim[1], prefill_tokens_per_step, out);
    if (rc == JL_OK && jl_model_batch_forward_multi && jl_model_sample_multi) (*out)->bb = {mb_forward_multi, mb_sample_multi};
    if (rc == JL_OK && jl_model_decode_sample_topkp && jl_model_sample_multi_topkp) (*out)->tb = {mb_decode_topkp, mb_sample_multi_topkp};
    if (rc == JL_OK && jl_model_decode_logprobs && jl_model_sample_multi_logprobs) (*out)->lb = {mb_decode_logprobs, mb_sample_multi_logprobs};
    if (rc == JL_OK && jl_model_decode_penalized && jl_model_sample_multi_penalized)
        (*out)->pb = {mb_decode_penalized, mb_sample_multi_penalized};
    if (rc == JL_OK && jl_model_decode_constrained && jl_model_sample_multi_constrained)
        (*out)->cb = {mb_decode_constrained, mb_sample_multi_constrained, lim[5]};
    if (rc == JL_OK && jl_model_kv_fork) (*out)->fb = {mb_fork};
    if (rc == JL_OK) (*out)->model = m;
    return rc;
}

extern "C" int jl_sched_set_batch_backend(jl_sched *s, const jl_sched_batch_backend *bb) {
    if (!s || (bb && (!bb->forward_multi || !bb->sample_multi))) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> a(s->step_mu);
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->step_no > 0) return sched_error(s, JL_ERR_INVALID, "set_batch_backend: the scheduler has already stepped");
    s->bb = bb ? *bb : jl_sched_batch_backend{};
    return JL_OK;
}

extern "C" int jl_sched_set_topkp_backend(jl_sched *s, const jl_sched_topkp_backend *tb) {
    if (!s || !tb || !tb->decode_topkp || !tb->sample_multi_topkp) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> a(s->step_mu);
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->step_no > 0) return sched_error(s, JL_ERR_INVALID, "set_topkp_backend: the scheduler has already stepped");
    s->tb = *tb;
    return JL_OK;
}

extern "C" int jl_sched_set_logprob_backend(jl_sched *s, const jl_sched_logprob_backend *lb) {
    if (!s || !lb || !lb->decode_logprobs || !lb->sample_multi_logprobs) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> a(s->step_mu);
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->step_no > 0) return sched_error(s, JL_ERR_INVALID, "set_logprob_backend: the scheduler has already stepped");
    s->lb = *lb;
    return JL_OK;
}

extern "C" int jl_sched_set_penalty_backend(jl_sched *s, const jl_sched_penalty_backend *pb) {
    if (!s || !pb || !pb->decode_penalized || !pb->sample_multi_penalized) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> a(s->step_mu);
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->step_no > 0) return sched_error(s, JL_ERR_INVALID, "set_penalty_backend: the scheduler has already stepped");
    s->pb = *pb;
    return JL_OK;
}

extern "C" int jl_sched_set_constraint_backend(jl_sched *s, const jl_sched_constraint_backend *cb) {
    if (!s || !cb || !cb->decode_constrained || !cb->sample_multi_constrained || cb->vocab < 1) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> a(s->step_mu);
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->step_no > 0) return sched_error(s, JL_ERR_INVALID, "set_constraint_backend: the scheduler has already stepped");
    s->cb = *cb;
    return JL_OK;
}

extern "C" int jl_sched_set_mask_provider(jl_sched *s, jl_sched_mask_fn *fn, void *user) {
    if (!s) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> a(s->step_mu);
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->step_no > 0) return sched_error(s, JL_ERR_INVALID, "set_mask_provider: the scheduler has already stepped");
    s->mask_fn = fn, s->mask_user = fn ? user : nullptr;
    return JL_OK;
}

extern "C" int jl_sched_set_fork_backend(jl_sched *s, const jl_sched_fork_backend *fb) {
    if (!s || !fb || !fb->fork) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> a(s->step_mu);
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->step_no > 0) return sched_error(s, JL_ERR_INVALID, "set_fork_backend: the scheduler has already stepped");
    s->fb = *fb;
    return JL_OK;
}

extern "C" int jl_sched_set_prefix_cache(jl_sched *s, const jl_sched_prefix_backend *pb, int max_pages) {
    if (!s || max_pages < 0) return JL_ERR_INVALID;
    jl_sched_prefix_backend xb = {};
    if (pb) {
        if (!pb->retain || !pb->attach || !pb->release || !pb->retained || pb->ctx_per_page < 1) return JL_ERR_INVALID;
        xb = *pb;
    } else if (s->model && jl_model_kv_retain) {
        int lim[6] = {0, 0, 0, 0, 0, 0};
        jl_model_limits(s->model, lim);
        xb = {mb_retain, mb_attach, mb_release, mb_retained, lim[4]};
    }
    std::lock_guard<std::mutex> a(s->step_mu);
    {
        std::lock_guard<std::mutex> lk(s->mu);
        if (s->step_no > 0) return sched_error(s, JL_ERR_INVALID, "set_prefix_cache: the scheduler has already stepped");
        if (!xb.retain) return sched_error(s, JL_ERR_INVALID, "set_prefix_cache: a backend scheduler needs the prefix calls");
        if (max_pages == 0) {
            s->xb = {}, s->prefix_max_pages = 0;
            return JL_OK;
        }
    }
    const int rc = xb.retained(s->user, nullptr, nullptr); // a model under tensor parallelism refuses
    std::lock_guard<std::mutex> lk(s->mu);
    if (rc != JL_OK) return sched_error(s, rc, "set_prefix_cache: the backend refuses retained prefixes (%d)", rc);
    s->xb = xb, s->prefix_max_pages = max_pages;
    return JL_OK;
}

extern "C" int jl_sched_prefix_stats(jl_sched *s, jl_sched_prefix_stats_t *out) {
    if (!s || !out) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(s->mu);
    *out = s->pstats;
    out->entries = (int64_t)s->prefix.size();
    return JL_OK;
}

extern "C" int jl_sched_request_cached(jl_sched *s, int64_t request) {
    if (!s) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(s->mu);
    auto it = s->reqs.find(request);
    if (it == s->reqs.end()) return sched_error(s, JL_ERR_INVALID, "request_cached: unknown request %lld", (long long)request);
    return it->second.cached;
}

// must hold s->mu.  Forget entry `it` (its handle is the caller's to release, table unlocked).
static int64_t prefix_erase(jl_sched *s, std::map<int64_t, PrefixEntry>::iterator it) {
    for (uint64_t h : it->second.hashes) {
        auto r = s->prefix_index.equal_range(h);
        for (auto i = r.first; i != r.second; ++i)
            if (i->second == it->first) {
                s->prefix_index.erase(i);
                break;
            }
    }
    const int64_t handle = it->second.handle;
    s->prefix.erase(it);
    return handle;
}

// must hold s->mu.  The most recently used entry whose tokens start with t[0, pages * ctx_per_page) (hash hit confirmed by the tokens),
// or prefix.end(); with `exact`, only an entry of exactly that length.
static std::map<int64_t, PrefixEntry>::iterator prefix_find(jl_sched *s, const int32_t *t, int pages, uint64_t hash, bool exact) {
    const size_t n = (size_t)pages * (size_t)s->xb.ctx_per_page;
    auto best = s->prefix.end();
    auto r = s->prefix_index.equal_range(hash);
    for (auto i = r.first; i != r.second; ++i) {
        auto e = s->prefix.find(i->second);
        if (e == s->prefix.end() || e->second.tokens.size() < n || (exact && e->second.tokens.size() != n)) continue;
        if (!std::equal(t, t + n, e->second.tokens.begin())) continue;
        if (best == s->prefix.end() || e->second.last_use > best->second.last_use ||
            (e->second.last_use == best->second.last_use && e->first > best->first))
            best = e;
    }
    return best;
}

// release the least recently used entry no job of this step attaches from (table unlocked); false when there is none
static bool prefix_evict(jl_sched *s) {
    int64_t handle = -1;
    {
        std::lock_guard<std::mutex> lk(s->mu);
        auto victim = s->prefix.end();
        for (auto it = s->prefix.begin(); it != s->prefix.end(); ++it)
            if (!it->second.pins && (victim == s->prefix.end() || it->second.last_use < victim->second.last_use)) victim = it; // ids ascend
        if (victim == s->prefix.end()) return false;
        handle = prefix_erase(s, victim);
        s->pstats.evictions++;
    }
    s->xb.release(s->user, handle);
    return true;
}

// a backend call that may run out of device memory: with the prefix cache on, release least recently used entries and retry until it
// succeeds or nothing is left to release, so the cache never fails a call that would succeed without it (table unlocked)
template <class F> static int evicting(jl_sched *s, F &&call) {
    int rc = call();
    while (rc == JL_ERR_OOM && s->prefix_max_pages > 0 && prefix_evict(s)) rc = call();
    return rc;
}

// retain the KV of `tokens` (whole pages) that `session` holds at positions [0, tokens.size()) (table unlocked).  A prefix an entry
// already holds only refreshes that entry; a new entry replaces the entries it extends.
static void prefix_retain(jl_sched *s, int session, const std::vector<int32_t> &tokens) {
    const int cpp = s->xb.ctx_per_page, pages = (int)tokens.size() / cpp;
    if (pages < 1) return;
    const std::vector<uint64_t> hashes = page_hashes(tokens.data(), pages, cpp);
    {
        std::lock_guard<std::mutex> lk(s->mu);
        auto e = prefix_find(s, tokens.data(), pages, hashes.back(), false);
        if (e != s->prefix.end()) {
            e->second.last_use = s->step_no;
            return;
        }
    }
    int64_t handle = -1;
    if (s->xb.retain(s->user, session, pages * cpp, &handle) != JL_OK) return; // the cache is best effort: the request is unaffected
    std::vector<int64_t> replaced;
    {
        std::lock_guard<std::mutex> lk(s->mu);
        for (int k = 0; k < pages - 1; k++) {
            auto e = prefix_find(s, tokens.data(), k + 1, hashes[(size_t)k], true);
            if (e != s->prefix.end() && !e->second.pins) replaced.push_back(prefix_erase(s, e));
        }
        const int64_t id = s->next_entry++;
        PrefixEntry &n = s->prefix[id];
        n.handle = handle, n.tokens.assign(tokens.begin(), tokens.begin() + (long)pages * cpp), n.hashes = hashes, n.last_use = s->step_no;
        for (uint64_t h : hashes) s->prefix_index.emplace(h, id);
    }
    for (int64_t h : replaced) s->xb.release(s->user, h);
}

// the retains of requests that finished since the last call, before their slots are reused (table unlocked)
static void prefix_flush(jl_sched *s) {
    std::vector<jl_sched::PendingRetain> todo;
    {
        std::lock_guard<std::mutex> lk(s->mu);
        todo.swap(s->retains);
    }
    for (const auto &p : todo) prefix_retain(s, p.session, p.tokens);
}

extern "C" int jl_sched_free(jl_sched *s) {
    if (!s) return JL_ERR_INVALID;
    {
        std::lock_guard<std::mutex> a(s->step_mu); // a step in flight finishes first
    }
    // host copies of spilled sessions nobody will restore any more
    if (s->be.discard) {
        for (int64_t h : s->discards) s->be.discard(s->user, h);
        for (auto &kv : s->reqs)
            if (kv.second.spill >= 0) s->be.discard(s->user, kv.second.spill);
    }
    for (auto &kv : s->prefix) s->xb.release(s->user, kv.second.handle);
    delete s;
    return JL_OK;
}

// a copy the calling thread owns (the shared string is rewritten under `mu` by whichever thread fails next)
extern "C" const char *jl_sched_last_error(jl_sched *s) {
    static thread_local std::string mine;
    if (!s) return "null scheduler";
    std::lock_guard<std::mutex> lk(s->mu);
    mine = s->last_error;
    return mine.c_str();
}

static bool finite_in(float v, float lo, float hi) { return v == v && v >= lo && v <= hi; } // NaN and +-inf fail

// must hold s->mu.  The checked request of submit's arguments, without its id; JL_OK or -1 with the error set.
static int make_request(jl_sched *s, Request &r, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens, int n_stop,
                        int flags, int64_t continue_request, float temperature, int top_k, float top_p, uint64_t seed, int logprobs,
                        float presence, float frequency, float repetition, int n_bias, const int32_t *bias_ids, const float *bias_vals) {
    if (!prompt || n_prompt <= 0 || max_new <= 0 || n_stop < 0 || (n_stop > 0 && !stop_tokens) || !(temperature >= 0.0f))
        return sched_error(s, -1, "submit: bad arguments (n_prompt=%d, max_new=%d, temperature=%g)", n_prompt, max_new, (double)temperature);
    if (top_k < 0 || !(top_p > 0.0f && top_p <= 1.0f))
        return sched_error(s, -1, "submit: bad filter (top_k=%d, top_p=%g)", top_k, (double)top_p);
    if (logprobs < -1 || logprobs > JL_MAX_LOGPROBS) return sched_error(s, -1, "submit: logprobs %d (-1..%d)", logprobs, JL_MAX_LOGPROBS);
    if (!finite_in(presence, -2.0f, 2.0f) || !finite_in(frequency, -2.0f, 2.0f) || !finite_in(repetition, 0.0f, 100.0f) || repetition == 0.0f)
        return sched_error(s, -1, "submit: bad penalties (presence=%g, frequency=%g, repetition=%g)", (double)presence, (double)frequency,
                           (double)repetition);
    if (n_bias < 0 || (n_bias > 0 && (!bias_ids || !bias_vals))) return sched_error(s, -1, "submit: bad logit bias (%d entries)", n_bias);
    r.temperature = temperature, r.top_k = top_k, r.top_p = top_p, r.logprobs = logprobs;
    r.pen.presence = presence, r.pen.frequency = frequency, r.pen.repetition = repetition;
    r.pen.bias_ids.assign(bias_ids, bias_ids + n_bias);
    r.pen.bias_vals.assign(bias_vals, bias_vals + n_bias);
    {
        std::vector<int32_t> ids = r.pen.bias_ids;
        std::sort(ids.begin(), ids.end());
        for (int j = 0; j < n_bias; j++) {
            if (bias_ids[j] < 0 || !finite_in(bias_vals[j], -100.0f, 100.0f))
                return sched_error(s, -1, "submit: logit bias entry %d (id %d, value %g)", j, bias_ids[j], (double)bias_vals[j]);
            if (j > 0 && ids[(size_t)j] == ids[(size_t)j - 1]) return sched_error(s, -1, "submit: logit bias lists id %d twice", ids[(size_t)j]);
        }
    }
    if (r.pen.on() && !s->pb.decode_penalized)
        return sched_error(s, -1, "submit: penalties need the penalty backend (jl_sched_set_penalty_backend)");
    if (r.filtered() && !s->tb.decode_topkp)
        return sched_error(s, -1, "submit: top_k / top_p need the top-k / top-p backend (jl_sched_set_topkp_backend)");
    if (logprobs >= 0 && !s->lb.decode_logprobs)
        return sched_error(s, -1, "submit: logprobs need the logprob backend (jl_sched_set_logprob_backend)");
    if ((flags & JL_SCHED_CONSTRAINED) && (!s->mask_fn || !s->cb.decode_constrained))
        return sched_error(s, -1, "submit: constrained requests need a mask provider and the constraint backend (jl_sched_set_mask_provider, "
                                  "jl_sched_set_constraint_backend)");
    if (continue_request >= 0) {
        // AbstractModel.generate :533 startPos = kvmem.getCurrentContextPosition(): a follow-up on the same session appends to its KV
        auto it = s->reqs.find(continue_request);
        if (it == s->reqs.end() || it->second.state != JL_SCHED_FINISHED || !(it->second.flags & JL_SCHED_KEEP_SESSION) ||
            (it->second.session < 0 && it->second.spill < 0 && !it->second.spilling))
            return sched_error(s, -1, "submit: request %lld is not a finished request that kept its session", (long long)continue_request);
        if (it->second.child >= 0)
            return sched_error(s, -1, "submit: request %lld already has a continuation", (long long)continue_request);
        r.start_pos = it->second.next_pos();
        r.parent = continue_request;
    }
    // Preconditions :530: the prompt must leave room for at least the token sampled from it
    if (r.start_pos + n_prompt >= s->max_context)
        return sched_error(s, -1, "submit: prompt of %d tokens at position %d exceeds the context of %d", n_prompt, r.start_pos,
                           s->max_context);
    r.prompt.assign(prompt, prompt + n_prompt);
    if (n_stop > 0) r.stop.assign(stop_tokens, stop_tokens + n_stop);
    r.max_new = max_new;
    r.flags = flags;
    r.rng = seed;
    r.submit_step = s->step_no;
    r.t_submit = r.t_admit = r.t_first = r.t_finish = std::chrono::steady_clock::now();
    r.out.reserve((size_t)(max_new < 4096 ? max_new : 4096));
    return JL_OK;
}

// must hold s->mu.  Queue a checked request; returns its id.
static int64_t enqueue(jl_sched *s, Request &&r) {
    r.id = s->next_id++;
    const int64_t id = r.id;
    if (r.parent >= 0) s->reqs[r.parent].child = id;
    s->reqs.emplace(id, std::move(r));
    s->queue.push_back(id);
    return id;
}

extern "C" int64_t jl_sched_submit_penalized(jl_sched *s, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens,
                                             int n_stop, int flags, int64_t continue_request, float temperature, int top_k, float top_p,
                                             uint64_t seed, int logprobs, float presence, float frequency, float repetition, int n_bias,
                                             const int32_t *bias_ids, const float *bias_vals) {
    if (!s) return -1;
    std::lock_guard<std::mutex> lk(s->mu);
    Request r;
    if (make_request(s, r, prompt, n_prompt, max_new, stop_tokens, n_stop, flags, continue_request, temperature, top_k, top_p, seed, logprobs,
                     presence, frequency, repetition, n_bias, bias_ids, bias_vals) != JL_OK)
        return -1;
    return enqueue(s, std::move(r));
}

extern "C" int jl_sched_submit_n(jl_sched *s, int n, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens, int n_stop,
                                 int flags, int64_t continue_request, float temperature, int top_k, float top_p, uint64_t seed, int logprobs,
                                 float presence, float frequency, float repetition, int n_bias, const int32_t *bias_ids, const float *bias_vals,
                                 int64_t *ids_out) {
    if (!s || !ids_out) return JL_ERR_INVALID;
    if (n == 1) {
        const int64_t id = jl_sched_submit_penalized(s, prompt, n_prompt, max_new, stop_tokens, n_stop, flags, continue_request, temperature,
                                                     top_k, top_p, seed, logprobs, presence, frequency, repetition, n_bias, bias_ids, bias_vals);
        if (id < 0) return JL_ERR_INVALID;
        ids_out[0] = id;
        return JL_OK;
    }
    std::lock_guard<std::mutex> lk(s->mu);
    if (n < 1 || n > s->n_sessions) return sched_error(s, JL_ERR_INVALID, "submit_n: n = %d (1..%d session slots)", n, s->n_sessions);
    if (!s->fb.fork) return sched_error(s, JL_ERR_INVALID, "submit_n: n > 1 needs the fork backend (jl_sched_set_fork_backend)");
    Request r;
    if (make_request(s, r, prompt, n_prompt, max_new, stop_tokens, n_stop, flags, continue_request, temperature, top_k, top_p, seed, logprobs,
                     presence, frequency, repetition, n_bias, bias_ids, bias_vals) != JL_OK)
        return JL_ERR_INVALID;
    // member j draws from the stream seeded with seed + j; the siblings start where the leader does and fork its session
    for (int j = 0; j < n; j++) {
        Request m = r;
        m.rng = seed + (uint64_t)j;
        if (j > 0) m.parent = -1, m.leader = ids_out[0];
        ids_out[j] = enqueue(s, std::move(m));
    }
    s->reqs[ids_out[0]].siblings.assign(ids_out + 1, ids_out + n);
    return JL_OK;
}

extern "C" int64_t jl_sched_submit_logprobs(jl_sched *s, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens,
                                            int n_stop, int flags, int64_t continue_request, float temperature, int top_k, float top_p,
                                            uint64_t seed, int logprobs) {
    return jl_sched_submit_penalized(s, prompt, n_prompt, max_new, stop_tokens, n_stop, flags, continue_request, temperature, top_k, top_p, seed,
                                     logprobs, 0.0f, 0.0f, 1.0f, 0, nullptr, nullptr);
}

extern "C" int64_t jl_sched_submit_topkp(jl_sched *s, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens,
                                         int n_stop, int flags, int64_t continue_request, float temperature, int top_k, float top_p,
                                         uint64_t seed) {
    return jl_sched_submit_logprobs(s, prompt, n_prompt, max_new, stop_tokens, n_stop, flags, continue_request, temperature, top_k, top_p, seed, -1);
}

extern "C" int64_t jl_sched_submit(jl_sched *s, const int32_t *prompt, int n_prompt, int max_new, const int32_t *stop_tokens,
                                   int n_stop, int flags, int64_t continue_request, float temperature, uint64_t seed) {
    return jl_sched_submit_topkp(s, prompt, n_prompt, max_new, stop_tokens, n_stop, flags, continue_request, temperature, 0, 1.0f, seed);
}

extern "C" int jl_sched_cancel(jl_sched *s, int64_t request) {
    if (!s) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(s->mu);
    auto it = s->reqs.find(request);
    if (it == s->reqs.end()) return sched_error(s, JL_ERR_INVALID, "cancel: unknown request %lld", (long long)request);
    if (it->second.state == JL_SCHED_FINISHED || it->second.state == JL_SCHED_FAILED) return JL_OK;
    it->second.cancel = true; // takes effect at the next step boundary
    return JL_OK;
}

extern "C" int jl_sched_result_logprobs(jl_sched *s, int64_t request, int first, int count, float *lp, int32_t *top_ids, float *top_lp,
                                        int *n_available) {
    if (!s || first < 0 || count < 0) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(s->mu);
    auto it = s->reqs.find(request);
    if (it == s->reqs.end()) return sched_error(s, JL_ERR_INVALID, "result_logprobs: unknown request %lld", (long long)request);
    const Request &r = it->second;
    if (r.logprobs < 0) return sched_error(s, JL_ERR_INVALID, "result_logprobs: request %lld was submitted without logprobs", (long long)request);
    const int n = (int)r.lp.size();
    const int k = first >= n ? 0 : (n - first < count ? n - first : count);
    const size_t W = JL_MAX_LOGPROBS;
    if (k > 0 && lp) memcpy(lp, r.lp.data() + first, sizeof(float) * (size_t)k);
    if (k > 0 && top_ids) memcpy(top_ids, r.top_ids.data() + (size_t)first * W, sizeof(int32_t) * (size_t)k * W);
    if (k > 0 && top_lp) memcpy(top_lp, r.top_lp.data() + (size_t)first * W, sizeof(float) * (size_t)k * W);
    if (n_available) *n_available = n;
    return JL_OK;
}

extern "C" int jl_sched_result(jl_sched *s, int64_t request, int32_t *tokens, int cap, int *n_tokens, int *state, int *finish_reason) {
    if (!s || cap < 0 || (cap > 0 && !tokens)) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(s->mu);
    auto it = s->reqs.find(request);
    if (it == s->reqs.end()) return sched_error(s, JL_ERR_INVALID, "result: unknown request %lld", (long long)request);
    const Request &r = it->second;
    const int n = (int)r.out.size();
    if (tokens && cap > 0) memcpy(tokens, r.out.data(), sizeof(int32_t) * (size_t)(n < cap ? n : cap));
    if (n_tokens) *n_tokens = n;
    if (state) *state = r.state;
    if (finish_reason) *finish_reason = r.reason;
    return JL_OK;
}

extern "C" int jl_sched_request_info(jl_sched *s, int64_t request, jl_sched_request_info_t *info) {
    if (!s || !info) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(s->mu);
    auto it = s->reqs.find(request);
    if (it == s->reqs.end()) return sched_error(s, JL_ERR_INVALID, "info: unknown request %lld", (long long)request);
    const Request &r = it->second;
    info->state = r.state, info->finish_reason = r.reason, info->session = r.session, info->start_pos = r.start_pos;
    info->n_prompt = (int)r.prompt.size(), info->n_prefilled = r.prefilled, info->n_generated = (int)r.out.size();
    info->next_position = r.next_pos();
    info->spilled = r.spill >= 0 ? 1 : 0;
    info->submit_step = (int64_t)r.submit_step, info->first_token_step = (int64_t)r.first_token_step;
    info->finish_step = (int64_t)r.finish_step;
    // phases that have not ended yet are measured up to now
    const auto now = std::chrono::steady_clock::now();
    auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
        return std::chrono::duration<double, std::milli>(b - a).count();
    };
    const bool admitted = r.admitted;
    const bool has_first = !r.out.empty();
    const bool done = r.state == JL_SCHED_FINISHED || r.state == JL_SCHED_FAILED;
    info->queue_ms = ms(r.t_submit, admitted ? r.t_admit : (done ? r.t_finish : now));
    info->prompt_ms = admitted ? ms(r.t_admit, has_first ? r.t_first : (done ? r.t_finish : now)) : 0.0;
    info->generate_ms = has_first ? ms(r.t_first, done ? r.t_finish : now) : 0.0;
    return JL_OK;
}

// free the slot a finished request kept (or drop its bookkeeping)
extern "C" int jl_sched_release(jl_sched *s, int64_t request) {
    if (!s) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(s->mu);
    auto it = s->reqs.find(request);
    if (it == s->reqs.end()) return sched_error(s, JL_ERR_INVALID, "release: unknown request %lld", (long long)request);
    Request &r = it->second;
    if (r.state != JL_SCHED_FINISHED && r.state != JL_SCHED_FAILED)
        return sched_error(s, JL_ERR_INVALID, "release: request %lld is still running (cancel it first)", (long long)request);
    if (r.child >= 0) {
        auto ch = s->reqs.find(r.child);
        if (ch != s->reqs.end() && ch->second.state == JL_SCHED_QUEUED)
            return sched_error(s, JL_ERR_INVALID, "release: request %lld has a queued continuation", (long long)request);
        if (ch != s->reqs.end()) ch->second.parent = -1;
    }
    if (r.parent >= 0) {
        auto pa = s->reqs.find(r.parent);
        if (pa != s->reqs.end()) pa->second.child = -1;
    }
    if (r.session >= 0 && s->slot_owner[(size_t)r.session] == request) s->slot_owner[(size_t)r.session] = -1;
    if (r.spill >= 0) s->discards.push_back(r.spill);
    s->reqs.erase(it);
    return JL_OK;
}

extern "C" int jl_sched_counts(jl_sched *s, int *queued, int *active, int *free_slots) {
    if (!s) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(s->mu);
    if (queued) *queued = (int)s->queue.size();
    if (active) *active = (int)s->active.size();
    if (free_slots) {
        int f = 0;
        for (int64_t o : s->slot_owner) f += o < 0;
        *free_slots = f;
    }
    return JL_OK;
}

// must hold s->mu
static void finish(jl_sched *s, Request &r, int state, int reason) {
    r.state = state;
    r.reason = reason;
    r.finish_step = s->step_no;
    r.t_finish = std::chrono::steady_clock::now();
    if (r.leader >= 0) { // a sibling that ends before the fork leaves its group
        std::vector<int64_t> &sib = s->reqs[r.leader].siblings;
        sib.erase(std::remove(sib.begin(), sib.end(), r.id), sib.end());
        r.leader = -1;
    }
    for (size_t i = 0; i < s->active.size(); i++)
        if (s->active[i] == r.id) {
            s->active.erase(s->active.begin() + (long)i);
            break;
        }
    // prefix cache: a fresh request that ends without an error leaves the whole pages of every position whose KV it wrote (its forwarded
    // prompt, then the generated tokens fed back), retained before its slot can be reused
    const int written = r.prefilled + r.forwarded, cpp = s->xb.ctx_per_page;
    if (s->prefix_max_pages > 0 && state == JL_SCHED_FINISHED && r.admitted && r.start_pos == 0 && r.session >= 0 && written >= cpp) {
        jl_sched::PendingRetain p{r.session, std::vector<int32_t>(r.prompt.begin(), r.prompt.begin() + r.prefilled)};
        p.tokens.insert(p.tokens.end(), r.out.begin(), r.out.begin() + r.forwarded);
        p.tokens.resize((size_t)(written / cpp * cpp));
        s->retains.push_back(std::move(p));
    }
    if (r.session >= 0) {
        const bool keep = state == JL_SCHED_FINISHED && (r.flags & JL_SCHED_KEEP_SESSION) && reason != JL_FINISH_CANCELLED;
        if (keep) {
            s->slot_owner[(size_t)r.session] = r.id; // the finished request holds the KV until released or continued
        } else if (s->slot_owner[(size_t)r.session] == r.id) {
            s->slot_owner[(size_t)r.session] = -1;
        }
    }
}

// must hold s->mu.  After a token was appended: AbstractModel.generate's exits (:590 position limit, :604-608 stop token).
static void check_done(jl_sched *s, Request &r, bool stop_check) {
    const int32_t t = r.out.back();
    if (stop_check)
        for (int32_t e : r.stop)
            if (e == t) return finish(s, r, JL_SCHED_FINISHED, JL_FINISH_STOP_TOKEN);
    if ((int)r.out.size() >= r.max_new || r.next_pos() >= s->max_context) finish(s, r, JL_SCHED_FINISHED, JL_FINISH_MAX_TOKENS);
}

namespace {
struct SlotJob { // what has to happen to a session slot before its new owner's first prompt chunk
    int64_t victim = -1; // kept request whose KV is offloaded out of the slot first
    int64_t restore_from = -1; // request whose spilled KV is restored into the slot (continuation of a spilled session)
    bool reset = false;        // fresh request: zero the slot
    int64_t entry = -1;        // fresh request with a cached prefix: attach `attach` positions of this prefix entry instead of the reset
    int64_t handle = -1;
    int attach = 0;
};
// how the token of one row of a sampling call is chosen
struct Select {
    float temperature = 0.0f, uniform = 0.0f;
    int32_t top_k = 0;
    float top_p = 1.0f;
    bool filtered = false;
    int32_t logprobs = -1;
    const Penalty *pen = nullptr; // penalised request: its penalties, history = hist, whose first n_prompt tokens are its prompt
    std::vector<int32_t> hist;
    int n_prompt = 0;
    bool constrained = false;     // JL_SCHED_CONSTRAINED request: `allow` is its provider's mask for this selection
    std::vector<uint32_t> allow;
};
struct PrefillJob {
    int64_t id;
    int session, n, pos;
    bool last;
    bool sibling = false;      // n-completion sibling: no prompt tokens; with `last` its first token is sampled after the leader's fork
    bool cancelled = false;    // leader cancelled before the fork: it forwards the prompt for its siblings but samples nothing
    bool dropped = false;      // the prefix attach failed: the slot was reset and the request is planned again from position 0
    uint64_t rng = 0;          // the request's uniform stream before the first-token draw, restored when the job is dropped
    std::vector<int32_t> retain; // prefix cache: the whole pages of a fresh prompt whose last chunk this job forwards
    std::vector<size_t> sibs;  // leader: the jobs of its siblings in this step
    Select sel;                // for the token sampled from the prompt's last row
    SlotJob slot;
    std::vector<int32_t> tokens;
    int rc = JL_OK;            // status of the job's backend calls
    std::string mask_error;    // the mask provider refused its first token
    size_t call = 0, row = 0;  // its first token: row `row` of its group's first-token call `call`
};

// the jl_penalties of one backend call, row by row; rows without a Penalty are unpenalised with empty histories
struct PenCall {
    std::vector<float> presence, frequency, repetition, bias_vals;
    std::vector<int32_t> hist_off{0}, hist_prompt, hist_ids, bias_off{0}, bias_ids;
    void add(const Penalty *p, const std::vector<int32_t> &hist, int n_prompt) {
        presence.push_back(p ? p->presence : 0.0f), frequency.push_back(p ? p->frequency : 0.0f), repetition.push_back(p ? p->repetition : 1.0f);
        if (p) {
            hist_ids.insert(hist_ids.end(), hist.begin(), hist.end());
            bias_ids.insert(bias_ids.end(), p->bias_ids.begin(), p->bias_ids.end());
            bias_vals.insert(bias_vals.end(), p->bias_vals.begin(), p->bias_vals.end());
        }
        hist_off.push_back((int32_t)hist_ids.size()), hist_prompt.push_back(p ? n_prompt : 0), bias_off.push_back((int32_t)bias_ids.size());
    }
    jl_penalties get() const {
        return jl_penalties{presence.data(), frequency.data(), repetition.data(), hist_off.data(), hist_prompt.data(), hist_ids.data(),
                            bias_off.data(), bias_ids.data(), bias_vals.data()};
    }
};

// the backend pair that serves a sampling call: the constraint pair when one of its rows is constrained, else the penalty pair when one
// is penalised, else the logprob pair when one wants logprobs, else the top-k / top-p pair when one is filtered, else the plain calls
enum Tier { PLAIN, TOPKP, LOGPROB, PENALTY, CONSTRAINED };
Tier tier_of(const Select &x) {
    return x.constrained ? CONSTRAINED : x.pen ? PENALTY : x.logprobs >= 0 ? LOGPROB : x.filtered ? TOPKP : PLAIN;
}

// the arguments and outputs of one sampling call (first tokens, or a decode step with its tokens and positions), row by row
struct Call {
    std::vector<int32_t> sessions, tokens, positions, top_k, top_n;
    std::vector<float> temperatures, uniforms, top_p;
    PenCall pc;
    std::vector<uint32_t> allow;    // the mask rows of the constrained rows, one each
    std::vector<int32_t> allow_row; // row -> its mask row, -1 = unconstrained
    int n_allow = 0;
    Tier tier = PLAIN;
    std::vector<int32_t> next, top_ids; // the tokens; logprob and penalty calls also fill lp, top_ids and top_lp
    std::vector<float> lp, top_lp;
    explicit Call(size_t n) : next(n), top_ids(n * JL_MAX_LOGPROBS), lp(n), top_lp(n * JL_MAX_LOGPROBS) {}
    void add(int32_t session, const Select &x) {
        sessions.push_back(session), temperatures.push_back(x.temperature), uniforms.push_back(x.uniform);
        top_k.push_back(x.top_k), top_p.push_back(x.top_p), top_n.push_back(x.logprobs);
        pc.add(x.pen, x.hist, x.n_prompt);
        allow_row.push_back(x.constrained ? n_allow++ : -1);
        if (x.constrained) allow.insert(allow.end(), x.allow.begin(), x.allow.end());
        tier = std::max(tier, tier_of(x));
    }
    // row i's logprobs -> the request's streams
    void append_lp(Request &r, size_t i) const {
        const size_t W = JL_MAX_LOGPROBS;
        r.lp.push_back(lp[i]);
        r.top_ids.insert(r.top_ids.end(), top_ids.begin() + (long)(i * W), top_ids.begin() + (long)((i + 1) * W));
        r.top_lp.insert(r.top_lp.end(), top_lp.begin() + (long)(i * W), top_lp.begin() + (long)((i + 1) * W));
    }
};

// the work and outcome of one jl_sched_step
struct Step {
    jl_sched_stats st = {};
    int first_error = JL_OK;
    std::vector<PrefillJob> jobs;
    std::vector<int64_t> discards; // spill handles of requests released since the last step
};
} // namespace

// must hold s->mu.  A slot for a request that needs one: a free slot, else (backend permitting) the slot of the kept session that
// finished longest ago -- sessions whose follow-up is already queued go last.  *victim = the request to offload, or -1.
static int take_slot(jl_sched *s, int64_t *victim) {
    *victim = -1;
    for (int k = 0; k < s->n_sessions; k++)
        if (s->slot_owner[(size_t)k] < 0) return k;
    if (!s->be.offload) return -1;
    int best = -1;
    for (int k = 0; k < s->n_sessions; k++) {
        auto it = s->reqs.find(s->slot_owner[(size_t)k]);
        if (it == s->reqs.end() || it->second.state != JL_SCHED_FINISHED || it->second.session != k) continue; // running, not kept
        if (best < 0) {
            best = k;
            continue;
        }
        const Request &a = it->second, &b = s->reqs[s->slot_owner[(size_t)best]];
        const bool a_waits = a.child >= 0, b_waits = b.child >= 0;
        if (a_waits != b_waits ? !a_waits : a.finish_step < b.finish_step) best = k;
    }
    if (best >= 0) *victim = s->slot_owner[(size_t)best];
    return best;
}

// the slot preparation of a job before its first prompt chunk (table unlocked): offload the kept session it displaces, then restore the
// continued session's spilled KV or zero the slot.  A failed offload only drops the victim's kept KV; the job's status is returned.
static int prepare_slot(jl_sched *s, PrefillJob &j, int *first_error) {
    if (j.slot.victim >= 0) {
        int64_t handle = -1;
        const int orc = s->be.offload(s->user, j.session, &handle);
        std::lock_guard<std::mutex> lk(s->mu);
        auto v = s->reqs.find(j.slot.victim);
        if (v != s->reqs.end()) v->second.spilling = false;
        if (orc == JL_OK && v != s->reqs.end()) v->second.spill = handle;
        else if (orc == JL_OK) s->discards.push_back(handle); // released meanwhile
        else {
            // the KV of the kept session could not be saved: it can no longer be continued; the slot is reused regardless
            if (v != s->reqs.end()) v->second.flags &= ~JL_SCHED_KEEP_SESSION;
            if (*first_error == JL_OK) *first_error = sched_error(s, orc, "offload of kept request %lld failed (%d): its session is dropped", (long long)j.slot.victim, orc);
        }
    }
    if (j.slot.restore_from >= 0) {
        int64_t handle = -1;
        {
            std::lock_guard<std::mutex> lk(s->mu);
            auto pa = s->reqs.find(j.slot.restore_from);
            if (pa != s->reqs.end()) handle = pa->second.spill, pa->second.spill = -1;
        }
        return handle >= 0 ? s->be.restore(s->user, j.session, handle) : JL_ERR_INVALID;
    }
    if (j.slot.entry >= 0) {
        // a failed attach never fails the request: the slot is reset and the prompt forwarded from position 0 from the next step on
        const int rc = evicting(s, [&] { return s->xb.attach(s->user, j.slot.handle, j.slot.attach, j.session); });
        {
            std::lock_guard<std::mutex> lk(s->mu);
            auto e = s->prefix.find(j.slot.entry);
            if (e != s->prefix.end()) e->second.pins--;
            if (rc == JL_OK) s->pstats.hits++, s->pstats.cached_tokens += j.slot.attach;
        }
        if (rc == JL_OK) return JL_OK;
        j.dropped = true;
    }
    if (j.slot.reset || j.dropped) return s->be.reset_session(s->user, j.session);
    return JL_OK;
}

// must hold s->mu.  Admit queued request `r`: into its parent's slot when the parent still holds its KV there (always possible), else, when
// `may_take`, into a slot from take_slot, whose kept session is offloaded first.  False, with nothing changed, when it gets no slot.
static bool admit(jl_sched *s, Request &r, bool may_take, std::unordered_map<int64_t, SlotJob> &slot_jobs, jl_sched_stats &st) {
    SlotJob sj;
    auto pa = r.parent >= 0 ? s->reqs.find(r.parent) : s->reqs.end();
    if (pa != s->reqs.end() && pa->second.session >= 0) {
        r.session = pa->second.session; // the parent's slot with its KV; ownership moves to the continuation
        pa->second.session = -1;
    } else {
        int64_t victim = -1;
        const int slot = may_take ? take_slot(s, &victim) : -1;
        if (slot < 0) return false;
        if (victim >= 0) {
            Request &v = s->reqs[victim];
            v.session = -1; // its KV leaves the device in this step (spill handle set when the offload returns)
            v.spilling = true;
            sj.victim = victim;
            st.spilled++;
        }
        r.session = slot;
        if (pa != s->reqs.end()) sj.restore_from = r.parent; // continuation of a spilled session
        else sj.reset = true;
    }
    if (sj.reset && r.leader < 0 && s->prefix_max_pages > 0) {
        // the longest cached whole-page prefix of the prompt that leaves its last token to forward, most recently used first (a
        // sibling gets the leader's KV from the fork instead)
        const int cpp = s->xb.ctx_per_page, pages = ((int)r.prompt.size() - 1) / cpp;
        const std::vector<uint64_t> hashes = page_hashes(r.prompt.data(), pages, cpp);
        s->pstats.lookups++;
        for (int k = pages; k >= 1; k--) {
            auto e = prefix_find(s, r.prompt.data(), k, hashes[(size_t)k - 1], false);
            if (e == s->prefix.end()) continue;
            e->second.last_use = s->step_no, e->second.pins++;
            sj.reset = false, sj.entry = e->first, sj.handle = e->second.handle, sj.attach = k * cpp;
            r.prefilled = r.cached = k * cpp;
            break;
        }
    }
    s->slot_owner[(size_t)r.session] = r.id;
    r.state = JL_SCHED_PREFILL;
    r.t_admit = r.leader >= 0 ? s->reqs[r.leader].t_admit : std::chrono::steady_clock::now(); // a group is admitted at one time
    r.admitted = true;
    s->active.push_back(r.id);
    s->queue.erase(std::find(s->queue.begin(), s->queue.end(), r.id));
    slot_jobs[r.id] = sj;
    st.admitted++;
    return true;
}

// must hold s->mu.  The step's plan: cancellations, admissions, and the prompt job of every prefilling request.
static void plan(jl_sched *s, Step &p) {
    jl_sched_stats &st = p.st;
    std::vector<PrefillJob> &jobs = p.jobs;
    s->step_no++;
    p.discards.swap(s->discards);
    // a cancelled leader still forwards the prompt for its siblings; the second pass ends it once they are all cancelled too
    for (int pass = 0; pass < 2; pass++)
        for (size_t i = 0; i < s->active.size();) {
            Request &r = s->reqs[s->active[i]];
            if (r.cancel && r.siblings.empty()) finish(s, r, JL_SCHED_FINISHED, JL_FINISH_CANCELLED), st.finished++;
            else i++;
        }
    // FIFO admission.  A continuation whose parent still sits in its slot returns to that slot (always possible); every other
    // request needs a slot from take_slot, and the first one that finds none blocks the slot-seeking requests behind it.
    // An n-completion group is admitted whole, at its leader's place: its siblings wait behind it.
    std::unordered_map<int64_t, SlotJob> slot_jobs; // admitted this step: request id -> slot preparation
    bool blocked = false;
    for (size_t qi = 0; qi < s->queue.size();) {
        Request &r = s->reqs[s->queue[qi]];
        if (r.leader >= 0) { // its leader is blocked
            qi++;
            continue;
        }
        for (size_t b = 0; b < r.siblings.size();) {
            Request &sb = s->reqs[r.siblings[b]];
            if (!sb.cancel) {
                b++;
                continue;
            }
            s->queue.erase(std::find(s->queue.begin(), s->queue.end(), sb.id)); // behind qi
            finish(s, sb, JL_SCHED_FINISHED, JL_FINISH_CANCELLED), st.finished++;
        }
        auto pa = r.parent >= 0 ? s->reqs.find(r.parent) : s->reqs.end();
        if (!r.siblings.empty()) {
            // all or nothing: the slots the group needs against the free slots and the kept sessions take_slot may spill
            const int need = (int)r.siblings.size() + (pa != s->reqs.end() && pa->second.session >= 0 ? 0 : 1);
            int avail = 0;
            for (int k = 0; k < s->n_sessions; k++) {
                const int64_t o = s->slot_owner[(size_t)k];
                if (o < 0) avail++;
                else if (s->be.offload && o != r.parent) {
                    auto it = s->reqs.find(o);
                    avail += it != s->reqs.end() && it->second.state == JL_SCHED_FINISHED && it->second.session == k;
                }
            }
            if (blocked || need > avail) {
                blocked = true;
                qi++;
                continue;
            }
        }
        if (r.cancel && r.siblings.empty()) {
            if (pa != s->reqs.end()) pa->second.child = -1; // the parent still holds the KV and may be continued again
            finish(s, r, JL_SCHED_FINISHED, JL_FINISH_CANCELLED), st.finished++;
            s->queue.erase(s->queue.begin() + (long)qi);
            continue;
        }
        if (!admit(s, r, !blocked, slot_jobs, st)) {
            blocked = true;
            qi++;
            continue;
        }
        for (int64_t bid : r.siblings) admit(s, s->reqs[bid], true, slot_jobs, st); // the slots were counted above
    }
    int budget = s->prefill_budget > 0 ? s->prefill_budget : 0x7fffffff;
    std::unordered_map<int64_t, size_t> leader_job; // group leader -> its job of this step
    for (int64_t id : s->active) {
        Request &r = s->reqs[id];
        if (r.state != JL_SCHED_PREFILL) continue;
        auto sj = slot_jobs.find(id);
        PrefillJob j;
        j.id = id, j.session = r.session, j.pos = r.start_pos + r.prefilled, j.sibling = r.leader >= 0;
        if (sj != slot_jobs.end()) j.slot = sj->second; // the slot is prepared in the admission step even if the budget is spent
        if (j.sibling) { // its slot preparation, and its first token in the step of the leader's last chunk
            auto lj = leader_job.find(r.leader);
            j.n = 0, j.last = lj != leader_job.end() && jobs[lj->second].last;
            if (!j.last && sj == slot_jobs.end()) continue;
            if (j.last) jobs[lj->second].sibs.push_back(jobs.size());
        } else {
            if (budget <= 0 && sj == slot_jobs.end()) continue;
            const int left = (int)r.prompt.size() - r.prefilled;
            j.n = left < budget ? left : (budget > 0 ? budget : 0);
            j.last = j.n > 0 && r.prefilled + j.n == (int)r.prompt.size();
            if (j.last && s->prefix_max_pages > 0 && r.start_pos == 0)
                j.retain.assign(r.prompt.begin(), r.prompt.begin() + (long)(r.prompt.size() / (size_t)s->xb.ctx_per_page * (size_t)s->xb.ctx_per_page));
            j.cancelled = r.cancel;
            j.tokens.assign(r.prompt.begin() + r.prefilled, r.prompt.begin() + r.prefilled + j.n);
            if (!r.siblings.empty()) leader_job[id] = jobs.size();
            budget -= j.n;
        }
        if (j.last) { // the token sampled from the prompt's last row (or, for a sibling, from the forked copy of it)
            j.rng = r.rng;
            if (r.temperature != 0.0f) j.sel.temperature = r.temperature, j.sel.uniform = next_uniform(r);
            if (r.filtered()) j.sel.top_k = r.top_k, j.sel.top_p = r.top_p, j.sel.filtered = true;
            j.sel.logprobs = r.logprobs;
            if (r.pen.on()) j.sel.pen = &r.pen, j.sel.hist = r.prompt, j.sel.n_prompt = (int)r.prompt.size();
            j.sel.constrained = (r.flags & JL_SCHED_CONSTRAINED) != 0;
        }
        jobs.push_back(std::move(j));
    }
}

// after a leader's prompt forward (table unlocked): its siblings fail with it, or get its session's KV for the prompt's positions
static void fork_group(jl_sched *s, Step &p, size_t k) {
    const PrefillJob &j = p.jobs[k];
    if (j.dropped) return;
    std::vector<int32_t> dst;
    for (size_t b : j.sibs)
        if (j.rc != JL_OK) p.jobs[b].rc = j.rc;
        else if (p.jobs[b].rc == JL_OK) dst.push_back(p.jobs[b].session);
    if (dst.empty()) return;
    const int rc = evicting(s, [&] { return s->fb.fork(s->user, j.session, j.pos + j.n, (int)dst.size(), dst.data()); });
    if (rc == JL_OK) return;
    for (size_t b : j.sibs) p.jobs[b].rc = rc; // a failed fork fails the siblings only
    std::lock_guard<std::mutex> lk(s->mu);
    if (p.first_error == JL_OK) p.first_error = sched_error(s, rc, "request %lld: fork into %zu siblings failed (%d)", (long long)j.id, dst.size(), rc);
}

// the provider's mask for one selection of a constrained request (table unlocked: the provider may call back into the scheduler);
// false with the reason when it fails or allows no token below the vocabulary
static bool mask_for(jl_sched *s, int64_t id, const std::vector<int32_t> &generated, std::vector<uint32_t> &allow, std::string &why) {
    const int V = s->cb.vocab;
    allow.assign((size_t)(V + 31) / 32, 0u);
    const int rc = s->mask_fn(s->mask_user, id, generated.data(), (int)generated.size(), allow.data());
    if (rc != 0) {
        why = "the mask provider failed (" + std::to_string(rc) + ")";
        return false;
    }
    for (size_t k = 0; k < allow.size(); k++) {
        const int left = V - (int)(k * 32);
        if ((left >= 32 ? allow[k] : allow[k] & ((1u << left) - 1u)) != 0u) return true;
    }
    why = "the mask provider allowed no token";
    return false;
}

// must hold s->mu.  A constrained request whose provider refused its selection fails alone.
static void mask_failed(jl_sched *s, Step &p, Request &r, const std::string &why) {
    const int rc = sched_error(s, JL_ERR_INVALID, "request %lld: %s", (long long)r.id, why.c_str());
    if (p.first_error == JL_OK) p.first_error = rc;
    finish(s, r, JL_SCHED_FAILED, JL_FINISH_ERROR), p.st.finished++;
}

// the first tokens of completed prompts (table unlocked); without a batch backend a plain call has one row
static int sample_first(jl_sched *s, Call &c) {
    const int n = (int)c.sessions.size();
    const jl_penalties pen = c.pc.get();
    if (c.tier == CONSTRAINED)
        return s->cb.sample_multi_constrained(s->user, n, c.sessions.data(), c.temperatures.data(), c.top_k.data(), c.top_p.data(),
                                              c.uniforms.data(), c.top_n.data(), &pen, c.n_allow, c.allow.data(), c.allow_row.data(),
                                              c.next.data(), c.lp.data(), c.top_ids.data(), c.top_lp.data());
    if (c.tier == PENALTY)
        return s->pb.sample_multi_penalized(s->user, n, c.sessions.data(), c.temperatures.data(), c.top_k.data(), c.top_p.data(), c.uniforms.data(),
                                            c.top_n.data(), &pen, c.next.data(), c.lp.data(), c.top_ids.data(), c.top_lp.data());
    if (c.tier == LOGPROB)
        return s->lb.sample_multi_logprobs(s->user, n, c.sessions.data(), c.temperatures.data(), c.top_k.data(), c.top_p.data(), c.uniforms.data(),
                                           c.top_n.data(), c.next.data(), c.lp.data(), c.top_ids.data(), c.top_lp.data());
    if (c.tier == TOPKP)
        return s->tb.sample_multi_topkp(s->user, n, c.sessions.data(), c.temperatures.data(), c.top_k.data(), c.top_p.data(), c.uniforms.data(),
                                        c.next.data());
    if (s->bb.sample_multi) return s->bb.sample_multi(s->user, n, c.sessions.data(), c.temperatures.data(), c.uniforms.data(), c.next.data());
    return s->be.sample(s->user, c.sessions[0], c.temperatures[0], c.uniforms[0], c.next.data());
}

// must hold s->mu.  The outcome of a prompt job's calls -> its request; `calls` are the first-token calls of its group.
static void apply(jl_sched *s, Step &p, const PrefillJob &j, const std::vector<Call> &calls) {
    jl_sched_stats &st = p.st;
    Request &r = s->reqs[j.id];
    if (j.sibling && r.state != JL_SCHED_PREFILL) return; // failed with its leader
    if (j.rc != JL_OK) {
        if (p.first_error == JL_OK) p.first_error = sched_error(s, j.rc, "request %lld: prompt forward failed (%d)", (long long)j.id, j.rc);
        const std::vector<int64_t> sib = r.siblings; // a failed prompt fails the group
        for (int64_t b : sib) finish(s, s->reqs[b], JL_SCHED_FAILED, JL_FINISH_ERROR), st.finished++;
        finish(s, r, JL_SCHED_FAILED, JL_FINISH_ERROR), st.finished++;
        return;
    }
    if (j.dropped) { // the prefix attach failed: the next step plans the prompt from position 0 (a sibling keeps waiting)
        if (!j.sibling) r.prefilled = r.cached = 0;
        if (j.last) r.rng = j.rng; // the first token is drawn again, from the same place in the stream
        return;
    }
    r.prefilled += j.n;
    st.prefill_tokens += j.n;
    if (!j.last) return;
    if (j.sibling) r.prefilled = (int)r.prompt.size();
    for (int64_t b : r.siblings) s->reqs[b].leader = -1; // forked: from now on every member is an ordinary request
    r.siblings.clear();
    if (j.cancelled) {
        finish(s, r, JL_SCHED_FINISHED, JL_FINISH_CANCELLED), st.finished++;
        return;
    }
    if (!j.mask_error.empty()) return mask_failed(s, p, r, j.mask_error);
    const Call &c = calls[j.call];
    r.out.push_back(c.next[j.row]);
    if (r.logprobs >= 0) c.append_lp(r, j.row);
    r.first_token_step = s->step_no;
    r.t_first = std::chrono::steady_clock::now();
    r.state = JL_SCHED_DECODING;
    // the token sampled from the prompt is not stop-checked by the reference (AbstractModel.java:576-589)
    check_done(s, r, false);
    if (r.state != JL_SCHED_DECODING) st.finished++;
}

// the prompt sequence of jobs [b, e) (table unlocked): prepare their slots, ONE forward call over the chunks whose slot is ready, forks
// and retains in job order, the first tokens of the completed prompts max_rows per call, then the outcomes.  A failed forward_multi or
// batched first-token call is reported as the call's error; a lone job's failed call as its request's, by apply.
static void run_group(jl_sched *s, Step &p, size_t b, size_t e) {
    std::vector<PrefillJob> &jobs = p.jobs;
    const bool batched = s->bb.forward_multi != nullptr;
    std::vector<size_t> fw; // the chunks whose slot is ready
    std::vector<int32_t> sess, pos, len, toks;
    for (size_t k = b; k < e; k++) {
        PrefillJob &j = jobs[k];
        if (!j.sibling) j.rc = prepare_slot(s, j, &p.first_error);
        if (j.dropped)
            for (size_t x : j.sibs) jobs[x].dropped = true;
        if (j.rc != JL_OK || j.n == 0 || j.dropped) continue;
        fw.push_back(k), sess.push_back(j.session), pos.push_back(j.pos), len.push_back(j.n);
        toks.insert(toks.end(), j.tokens.begin(), j.tokens.end());
    }
    if (!fw.empty()) {
        const int rc = evicting(s, [&] {
            return batched ? s->bb.forward_multi(s->user, (int)fw.size(), sess.data(), pos.data(), len.data(), toks.data())
                           : s->be.batch_forward(s->user, sess[0], toks.data(), len[0], pos[0]);
        });
        for (size_t k : fw) jobs[k].rc = rc;
        if (rc != JL_OK && batched) {
            std::lock_guard<std::mutex> lk(s->mu);
            if (p.first_error == JL_OK) p.first_error = sched_error(s, rc, "prompt forward of %zu requests failed (%d)", fw.size(), rc);
        }
    }
    std::vector<size_t> done; // the completed prompts: a leader's fork has settled its siblings' status before they are reached
    for (size_t k = b; k < e; k++) {
        fork_group(s, p, k);
        const PrefillJob &j = jobs[k];
        if (j.rc == JL_OK && !j.dropped && !j.retain.empty()) prefix_retain(s, j.session, j.retain);
        if (j.rc == JL_OK && j.last && !j.cancelled && !j.dropped) done.push_back(k);
    }
    // the masks of the constrained first tokens (n_generated 0); a refused one leaves the call
    const std::vector<int32_t> none;
    done.erase(std::remove_if(done.begin(), done.end(),
                              [&](size_t k) {
                                  PrefillJob &j = jobs[k];
                                  return j.sel.constrained && !mask_for(s, j.id, none, j.sel.allow, j.mask_error);
                              }),
               done.end());
    std::vector<Call> calls;
    for (size_t g = 0; g < done.size(); g += (size_t)s->max_rows) {
        const size_t n = std::min(done.size() - g, (size_t)s->max_rows);
        Call c(n);
        for (size_t i = 0; i < n; i++) {
            PrefillJob &j = jobs[done[g + i]];
            c.add(j.session, j.sel);
            j.call = calls.size(), j.row = i;
        }
        const int rc = sample_first(s, c);
        for (size_t i = 0; i < n; i++) jobs[done[g + i]].rc = rc;
        if (rc != JL_OK && batched) {
            std::lock_guard<std::mutex> lk(s->mu);
            if (p.first_error == JL_OK) p.first_error = sched_error(s, rc, "first-token sample of %zu requests failed (%d)", n, rc);
        }
        calls.push_back(std::move(c));
    }
    std::lock_guard<std::mutex> lk(s->mu);
    for (size_t k = b; k < e; k++) apply(s, p, jobs[k], calls);
}

// the step's prompt jobs (table unlocked): with a batch backend one group of every job, else one group per job, in job order
static void run_prompts(jl_sched *s, Step &p) {
    prefix_flush(s); // requests cancelled in the plan: their KV is retained before their slots are prepared for others
    for (int64_t h : p.discards) s->be.discard(s->user, h);
    // siblings' slots are ready before any fork writes into them
    for (PrefillJob &j : p.jobs)
        if (j.sibling) j.rc = prepare_slot(s, j, &p.first_error);
    const size_t group = s->bb.forward_multi ? p.jobs.size() : 1;
    for (size_t b = 0; b < p.jobs.size(); b += group) run_group(s, p, b, b + group);
}

// one decode step over a call's rows (table unlocked)
static int decode_call(jl_sched *s, Call &c) {
    const int n = (int)c.sessions.size();
    const jl_penalties pen = c.pc.get();
    if (c.tier == CONSTRAINED)
        return s->cb.decode_constrained(s->user, n, c.sessions.data(), c.tokens.data(), c.positions.data(), c.temperatures.data(), c.top_k.data(),
                                        c.top_p.data(), c.uniforms.data(), c.top_n.data(), &pen, c.n_allow, c.allow.data(), c.allow_row.data(),
                                        c.next.data(), c.lp.data(), c.top_ids.data(), c.top_lp.data());
    if (c.tier == PENALTY)
        return s->pb.decode_penalized(s->user, n, c.sessions.data(), c.tokens.data(), c.positions.data(), c.temperatures.data(), c.top_k.data(),
                                      c.top_p.data(), c.uniforms.data(), c.top_n.data(), &pen, c.next.data(), c.lp.data(), c.top_ids.data(),
                                      c.top_lp.data());
    if (c.tier == LOGPROB)
        return s->lb.decode_logprobs(s->user, n, c.sessions.data(), c.tokens.data(), c.positions.data(), c.temperatures.data(), c.top_k.data(),
                                     c.top_p.data(), c.uniforms.data(), c.top_n.data(), c.next.data(), c.lp.data(), c.top_ids.data(),
                                     c.top_lp.data());
    if (c.tier == TOPKP)
        return s->tb.decode_topkp(s->user, n, c.sessions.data(), c.tokens.data(), c.positions.data(), c.temperatures.data(), c.top_k.data(),
                                  c.top_p.data(), c.uniforms.data(), c.next.data());
    return s->be.decode(s->user, n, c.sessions.data(), c.tokens.data(), c.positions.data(), c.temperatures.data(), c.uniforms.data(), c.next.data());
}

// one decode step for every generating request, max_rows rows per backend call
static void run_decode(jl_sched *s, Step &p) {
    jl_sched_stats &st = p.st;
    const size_t M = (size_t)s->max_rows;
    struct Row {
        int64_t id;
        int32_t session, token, position;
        Select x;
        std::vector<int32_t> generated; // constrained: a copy for the mask provider
        std::string refused;
    };
    std::vector<Row> rows;
    {
        std::lock_guard<std::mutex> lk(s->mu);
        for (int64_t id : s->active) {
            Request &r = s->reqs[id];
            if (r.state != JL_SCHED_DECODING) continue;
            Select x{r.temperature, r.temperature != 0.0f ? next_uniform(r) : 0.0f, r.top_k, r.top_p, r.filtered(), r.logprobs};
            if (r.pen.on()) { // the prompt, then every generated token including the one this step feeds
                x.pen = &r.pen, x.n_prompt = (int)r.prompt.size();
                x.hist = r.prompt;
                x.hist.insert(x.hist.end(), r.out.begin(), r.out.end());
            }
            x.constrained = (r.flags & JL_SCHED_CONSTRAINED) != 0;
            rows.push_back(Row{id, r.session, r.out.back(), r.next_pos(), std::move(x), {}, {}});
            if (rows.back().x.constrained) rows.back().generated = r.out;
        }
    }
    // the masks of the constrained rows; a refused row fails its request and leaves the step
    bool refused = false;
    for (Row &w : rows)
        if (w.x.constrained && !mask_for(s, w.id, w.generated, w.x.allow, w.refused)) refused = true;
    if (refused) {
        std::lock_guard<std::mutex> lk(s->mu);
        for (const Row &w : rows)
            if (!w.refused.empty()) mask_failed(s, p, s->reqs[w.id], w.refused);
    }
    std::vector<Call> calls;
    std::vector<int64_t> ids; // request of row i of call g: ids[g * max_rows + i]
    for (const Row &w : rows) {
        if (!w.refused.empty()) continue;
        if (ids.size() % M == 0) calls.emplace_back(M);
        Call &c = calls.back();
        c.add(w.session, w.x), c.tokens.push_back(w.token), c.positions.push_back(w.position);
        ids.push_back(w.id);
    }
    for (size_t g = 0; g < calls.size(); g++) {
        Call &c = calls[g];
        const int n = (int)c.sessions.size();
        const int rc = evicting(s, [&] { return decode_call(s, c); });
        st.decode_calls++;
        std::lock_guard<std::mutex> lk(s->mu);
        for (int i = 0; i < n; i++) {
            Request &r = s->reqs[ids[g * M + (size_t)i]];
            if (rc != JL_OK) {
                if (p.first_error == JL_OK) p.first_error = sched_error(s, rc, "decode step of %d sessions failed (%d)", n, rc);
                finish(s, r, JL_SCHED_FAILED, JL_FINISH_ERROR), st.finished++;
                continue;
            }
            r.forwarded++;
            r.out.push_back(c.next[(size_t)i]);
            if (r.logprobs >= 0) c.append_lp(r, (size_t)i);
            st.decode_rows++;
            check_done(s, r, true);
            if (r.state != JL_SCHED_DECODING) st.finished++;
        }
    }
}

// the step's finished requests are retained, then least recently used entries go until the cache alone holds max_pages pages
static void prefix_upkeep(jl_sched *s) {
    if (s->prefix_max_pages <= 0) return;
    prefix_flush(s);
    for (;;) {
        int64_t only = 0;
        if (s->xb.retained(s->user, nullptr, &only) != JL_OK) break;
        {
            std::lock_guard<std::mutex> lk(s->mu);
            s->pstats.pages_retained_only = only;
        }
        if (only <= s->prefix_max_pages || !prefix_evict(s)) break;
    }
}

// the counts of `st` added to `sum`; active and queued are levels, taken as they are
static void add_stats(jl_sched_stats &sum, const jl_sched_stats &st) {
    sum.admitted += st.admitted, sum.prefill_tokens += st.prefill_tokens, sum.decode_rows += st.decode_rows;
    sum.decode_calls += st.decode_calls, sum.finished += st.finished, sum.spilled += st.spilled;
    sum.active = st.active, sum.queued = st.queued;
}

// the levels after the step, and the step's counts added to the scheduler's totals
static void record_stats(jl_sched *s, jl_sched_stats &st) {
    std::lock_guard<std::mutex> lk(s->mu);
    st.active = (int)s->active.size();
    st.queued = (int)s->queue.size();
    add_stats(s->totals, st);
}

extern "C" int jl_sched_step(jl_sched *s, jl_sched_stats *stats) {
    if (!s) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> step_lock(s->step_mu);
    Step p;
    {
        std::lock_guard<std::mutex> lk(s->mu);
        plan(s, p);
    }
    run_prompts(s, p);
    run_decode(s, p);
    prefix_upkeep(s);
    record_stats(s, p.st);
    if (stats) *stats = p.st;
    return p.first_error;
}

extern "C" int jl_sched_run(jl_sched *s, int max_steps, jl_sched_stats *totals) {
    if (!s) return JL_ERR_INVALID;
    int rc_all = JL_OK;
    jl_sched_stats sum = {};
    for (int i = 0; max_steps <= 0 || i < max_steps; i++) {
        jl_sched_stats st;
        const int rc = jl_sched_step(s, &st);
        if (rc != JL_OK && rc_all == JL_OK) rc_all = rc;
        add_stats(sum, st);
        if (st.active == 0 && st.queued == 0) break;
        // nothing admitted, forwarded or decoded although work is queued: every slot is held by a kept session
        if (st.admitted == 0 && st.prefill_tokens == 0 && st.decode_rows == 0 && st.finished == 0) {
            if (rc_all == JL_OK) rc_all = sched_error(s, JL_ERR_INVALID, "run: %d queued requests but no session slot can be freed", st.queued);
            break;
        }
    }
    if (totals) *totals = sum;
    return rc_all;
}
