// Sanitizer harness for constrained requests in the session scheduler (DESIGN §3.18): jlama_b200/csrc/jl_sched.cu is compiled with
// -fsanitize=address,undefined and again with -fsanitize=thread and driven by producer threads that submit constrained and plain
// requests while the main thread steps.  The mask provider runs on the stepping thread without the scheduler's lock and calls back
// into it: jl_sched_result on every call, jl_sched_cancel on some requests, and it fails others.  At the end every constrained token
// must be allowed by the mask it was selected under, and the provider must have been called exactly once per selection.
// Built and run by tests/test_sched_mask_sanitizers.py; exit code 0 = clean.
#include "../../jlama_b200/csrc/jl_sched.cu"

#include <atomic>
#include <map>
#include <random>
#include <thread>

// the jl_model backend of jl_sched_create is not under test here: satisfy the linker
extern "C" {
int jl_model_reset_session(jl_model *, int) { return JL_ERR_INVALID; }
int jl_model_batch_forward(jl_model *, int, const int32_t *, int, int) { return JL_ERR_INVALID; }
int jl_model_sample(jl_model *, int, float, float, int32_t *, float *) { return JL_ERR_INVALID; }
int jl_model_decode_sample(jl_model *, int, const int32_t *, const int32_t *, const int32_t *, const float *, const float *, int32_t *, float *) {
    return JL_ERR_INVALID;
}
int64_t jl_model_kv_offload(jl_model *, int) { return JL_ERR_INVALID; }
int jl_model_kv_restore(jl_model *, int, int64_t) { return JL_ERR_INVALID; }
int jl_model_kv_discard(jl_model *, int64_t) { return JL_ERR_INVALID; }
}
void jl_model_limits(jl_model *, int out[6]) { out[0] = out[1] = out[2] = out[3] = out[4] = out[5] = 0; }

static const int VOCAB = 70, WORDS = (VOCAB + 31) / 32, CONTEXT = 64;
#define REQUIRE(cond)                                                              \
    do {                                                                           \
        if (!(cond)) {                                                             \
            fprintf(stderr, "REQUIRE failed: %s (%s:%d)\n", #cond, __FILE__, __LINE__); \
            abort();                                                               \
        }                                                                          \
    } while (0)

// the allowed set of request `id` after `gen`: a function of both, never empty
static bool allowed(int64_t id, const int32_t *gen, int n, int32_t t) {
    uint64_t x = (uint64_t)id * 0x9E3779B97F4A7C15ull + (uint64_t)n * 1099511628211ull + (n ? (uint64_t)gen[n - 1] : 0u);
    if ((int32_t)(x % VOCAB) == t) return true;
    return ((x >> (t % 60)) ^ (uint64_t)t * 2654435761ull) % 3 == 0;
}

static int32_t toy_next(const std::vector<int32_t> &h) {
    uint64_t x = 1469598103934665603ull;
    for (int32_t t : h) x = (x ^ (uint64_t)(t + 1)) * 1099511628211ull;
    return (int32_t)(x % VOCAB);
}

// the first token at or after toy_next(h) (cyclically) whose bit is set
static int32_t masked_next(const std::vector<int32_t> &h, const uint32_t *mask) {
    const int32_t t0 = toy_next(h);
    for (int d = 0; d < VOCAB; d++) {
        const int32_t t = (t0 + d) % VOCAB;
        if (mask[t / 32] >> (t % 32) & 1u) return t;
    }
    REQUIRE(false);
    return -1;
}

struct Toy {
    std::vector<std::vector<int32_t>> hist;
    int max_rows;
    static int reset(void *u, int s) {
        ((Toy *)u)->hist[(size_t)s].clear();
        return JL_OK;
    }
    static int forward(void *u, int s, const int32_t *tok, int n, int start) {
        Toy *t = (Toy *)u;
        REQUIRE(start == (int)t->hist[(size_t)s].size());
        t->hist[(size_t)s].insert(t->hist[(size_t)s].end(), tok, tok + n);
        return JL_OK;
    }
    static int sample(void *u, int s, float, float, int32_t *out) {
        *out = toy_next(((Toy *)u)->hist[(size_t)s]);
        return JL_OK;
    }
    static int decode(void *u, int n, const int32_t *sess, const int32_t *tok, const int32_t *pos, const float *, const float *, int32_t *next) {
        Toy *t = (Toy *)u;
        REQUIRE(n >= 1 && n <= t->max_rows);
        for (int i = 0; i < n; i++) {
            auto &h = t->hist[(size_t)sess[i]];
            REQUIRE(pos[i] == (int)h.size() && pos[i] < CONTEXT);
            h.push_back(tok[i]);
            next[i] = toy_next(h);
        }
        return JL_OK;
    }
    static int rows(Toy *t, int n, const int32_t *sess, int n_allow, const uint32_t *allow, const int32_t *allow_row, int32_t *out) {
        REQUIRE(n >= 1 && n <= t->max_rows);
        int seen = 0;
        for (int i = 0; i < n; i++) {
            const auto &h = t->hist[(size_t)sess[i]];
            REQUIRE(allow_row[i] >= -1 && allow_row[i] < n_allow);
            if (allow_row[i] < 0) {
                out[i] = toy_next(h);
                continue;
            }
            REQUIRE(allow_row[i] == seen++); // one mask row per constrained row, in row order
            out[i] = masked_next(h, allow + (size_t)allow_row[i] * WORDS);
        }
        REQUIRE(seen == n_allow);
        return JL_OK;
    }
    static int decode_constrained(void *u, int n, const int32_t *sess, const int32_t *tok, const int32_t *pos, const float *, const int32_t *,
                                  const float *, const float *, const int32_t *, const jl_penalties *, int n_allow, const uint32_t *allow,
                                  const int32_t *allow_row, int32_t *next, float *, int32_t *, float *) {
        Toy *t = (Toy *)u;
        for (int i = 0; i < n; i++) {
            auto &h = t->hist[(size_t)sess[i]];
            REQUIRE(pos[i] == (int)h.size() && pos[i] < CONTEXT);
            h.push_back(tok[i]);
        }
        return rows(t, n, sess, n_allow, allow, allow_row, next);
    }
    static int sample_multi_constrained(void *u, int n, const int32_t *sess, const float *, const int32_t *, const float *, const float *,
                                        const int32_t *, const jl_penalties *, int n_allow, const uint32_t *allow, const int32_t *allow_row,
                                        int32_t *out, float *, int32_t *, float *) {
        return rows((Toy *)u, n, sess, n_allow, allow, allow_row, out);
    }
};

struct Provider {
    jl_sched *s = nullptr;
    std::mutex mu;
    std::map<int64_t, int> calls; // selections seen per request
    std::map<int64_t, int> failed; // requests the provider failed
    static int fn(void *u, int64_t id, const int32_t *gen, int n, uint32_t *out) {
        Provider *p = (Provider *)u;
        // streaming read of the request from inside the provider: it must see exactly the tokens it was handed
        std::vector<int32_t> buf(64);
        int nt = 0, state = 0, reason = 0;
        REQUIRE(jl_sched_result(p->s, id, buf.data(), (int)buf.size(), &nt, &state, &reason) == JL_OK);
        REQUIRE(nt == n && state != JL_SCHED_FINISHED && state != JL_SCHED_FAILED);
        for (int i = 0; i < n; i++) REQUIRE(buf[(size_t)i] == gen[i]);
        {
            std::lock_guard<std::mutex> lk(p->mu);
            p->calls[id]++;
        }
        if (id % 7 == 3 && n == 2) jl_sched_cancel(p->s, id); // ends after this selection, at the next step boundary
        if (id % 11 == 5 && n == 1) {
            std::lock_guard<std::mutex> lk(p->mu);
            p->failed[id] = 1;
            return 1;
        }
        for (int w = 0; w < WORDS; w++) REQUIRE(out[w] == 0u);
        for (int32_t t = 0; t < VOCAB; t++)
            if (allowed(id, gen, n, t)) out[t / 32] |= 1u << (t % 32);
        return 0;
    }
};

int main() {
    const int SLOTS = 4;
    Toy toy;
    toy.hist.resize(SLOTS), toy.max_rows = 3;
    jl_sched_backend be = {Toy::reset, Toy::forward, Toy::sample, Toy::decode, nullptr, nullptr, nullptr};
    jl_sched *s = nullptr;
    REQUIRE(jl_sched_create_backend(&be, &toy, SLOTS, 3, CONTEXT, 6, &s) == JL_OK);
    const jl_sched_constraint_backend cb = {Toy::decode_constrained, Toy::sample_multi_constrained, VOCAB};
    Provider prov;
    prov.s = s;
    const int32_t p0 = 1;
    REQUIRE(jl_sched_submit(s, &p0, 1, 2, nullptr, 0, JL_SCHED_CONSTRAINED, -1, 0.0f, 0) == -1); // no provider, no backend yet
    REQUIRE(jl_sched_set_constraint_backend(s, &cb) == JL_OK);
    REQUIRE(jl_sched_set_mask_provider(s, Provider::fn, &prov) == JL_OK);

    std::mutex meta_mu;
    std::map<int64_t, bool> meta; // request -> constrained
    std::atomic<int> producers_done{0};
    auto producer = [&](unsigned seed) {
        std::mt19937 rng(seed);
        for (int it = 0; it < 80; it++) {
            std::vector<int32_t> prompt;
            const int n = 1 + (int)(rng() % 6);
            for (int i = 0; i < n; i++) prompt.push_back((int32_t)(rng() % VOCAB));
            const bool con = rng() % 3 != 0;
            const int64_t id = jl_sched_submit(s, prompt.data(), n, 1 + (int)(rng() % 8), nullptr, 0, con ? JL_SCHED_CONSTRAINED : 0, -1, 0.0f,
                                               rng());
            REQUIRE(id > 0);
            std::lock_guard<std::mutex> lk(meta_mu);
            meta[id] = con;
            if (it % 8 == 0) std::this_thread::yield();
        }
    };
    std::vector<std::thread> threads;
    for (unsigned p = 0; p < 3; p++)
        threads.emplace_back([&, p] {
            producer(2000u + p);
            producers_done++;
        });
    while (producers_done.load() < 3) {
        jl_sched_stats st;
        jl_sched_step(s, &st);
        REQUIRE(st.active <= SLOTS);
    }
    for (auto &t : threads) t.join();
    jl_sched_stats totals;
    jl_sched_run(s, 0, &totals);

    int checked = 0, cancelled = 0, failed = 0;
    for (auto &kv : meta) {
        std::vector<int32_t> buf(64);
        int n = 0, state = 0, reason = 0;
        REQUIRE(jl_sched_result(s, kv.first, buf.data(), 64, &n, &state, &reason) == JL_OK);
        REQUIRE(state == JL_SCHED_FINISHED || state == JL_SCHED_FAILED);
        const int calls = prov.calls.count(kv.first) ? prov.calls[kv.first] : 0;
        if (!kv.second) {
            REQUIRE(calls == 0 && state == JL_SCHED_FINISHED);
            continue;
        }
        const bool refused = prov.failed.count(kv.first) > 0;
        REQUIRE(calls == n + (refused ? 1 : 0));
        REQUIRE(refused == (state == JL_SCHED_FAILED));
        for (int i = 0; i < n; i++) REQUIRE(allowed(kv.first, buf.data(), i, buf[(size_t)i]));
        checked++, cancelled += reason == JL_FINISH_CANCELLED, failed += refused;
    }
    REQUIRE(checked >= 60 && cancelled > 0 && failed > 0);
    for (auto &kv : meta) jl_sched_release(s, kv.first);
    REQUIRE(jl_sched_free(s) == JL_OK);
    printf("ok: %d requests, %d constrained checked, %d cancelled by the provider, %d failed by it\n", (int)meta.size(), checked, cancelled,
           failed);
    return 0;
}
