// Device-resident host driver: the C++ mirror of AbstractModel / LlamaModel / TransformerBlock /
// CausalSelfAttention / MLPBlock (core/model/AbstractModel.java:295-329,443-491,516-646;
// core/model/llama/LlamaModel.java:68-184; core/model/TransformerBlock.java:158-215;
// core/model/CausalSelfAttention.java:145-385; core/model/MLPBlock.java:106-166).
// It replays generate()'s exact call sequence; every layer op is a CUDA kernel on activations that
// never leave HBM, KV lives in device pages shaped like KvBufferCache's, and the per-token decode
// step is captured once into a CUDA graph with programmatic dependent launch between kernels.
#include "jl_common.cuh"
#include <string>
#include "jl_pdecode.cuh"

#include <chrono>
#include <map>
#include <math.h>
#include <new>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unordered_map>
#include <vector>

int jl_comm_allreduce_dev(jl_ctx *ctx, cudaStream_t stream, float *buf, size_t count);
int jl_comm_allgather_dev(jl_ctx *ctx, cudaStream_t stream, const void *send, void *recv, size_t bytes_per_rank);

struct jl_model {
    jl_ctx *ctx = nullptr;
    // serialises the entry points that use the model stream and its staging buffers: the reference calls generate() from one thread per
    // request (OpenAIChatService.java:107-160); recursive because generate() is built from the other entry points
    std::recursive_mutex mu;
    jl_model_config cfg;
    jl_dctx d;
    cudaStream_t stream = nullptr;
    bool finalized = false;
    DevTensor g[3];
    bool g_set[3] = {false, false, false};
    std::vector<DevTensor> l; // [layers][9]
    std::vector<char> l_set;
    std::vector<int64_t> bound_ids; // registry ids whose refs this model holds (one entry per set_tensor call)
    int group = 1, attn_seg = 0, kv_seg = 0, h_seg = 0, heads_local = 0, kv_heads_local = 0;
    // rope
    float *rope = nullptr;
    // KV pages
    KvLayout kv;
    void **page_table_dev = nullptr;
    std::vector<void *> page_table_host;
    // shared pages (jl_model_kv_fork): page -> the number of page-table entries that hold it, for the pages more than one entry holds; a
    // page not listed belongs to its one entry.  Empty in a model that never forked, which then does no other per-call work.
    std::unordered_map<void *, int> page_refs;
    KvCopy *d_copy_tab = nullptr; // the page copies of one launch (jl_kv_copy.cu), staged through h_pinned (copy_cap entries)
    int copy_cap = 0;
    size_t page_bytes = 0;
    int max_context = 0;
    // scratch
    int maxB = 0;
    float *x = nullptr, *xb = nullptr, *q = nullptr, *k = nullptr, *v = nullptr, *att = nullptr, *hbuf = nullptr,
          *partial = nullptr, *logits = nullptr, *attn_ws = nullptr, *last_hidden = nullptr, *ln = nullptr, *hbuf2 = nullptr;
    uint16_t *abf = nullptr; // bf16 activations for the tensor-core prefill GEMMs
    bool tc_ok = false;
    // workspaces of the many-row decode GEMM (jl_gemm64.cu); allocated when a decode step can have more than GEMV_MAX_M rows
    void *wide_act = nullptr;
    float *wide_part = nullptr;
    unsigned *wide_cnt = nullptr;
    int max_splits = 32;
    int32_t *d_tokens = nullptr, *d_positions = nullptr, *d_sessions = nullptr, *d_next = nullptr, *d_hist = nullptr,
            *d_counter = nullptr;
    void *argmax_scratch = nullptr;
    int32_t *h_pinned = nullptr; // pinned staging: tokens | positions | sessions | next [maxB each] | attention block table | copy_rows rows
    // multi-session prefill (jl_model_batch_forward_multi): CTA block table of the tiled attention (pa_tab_cap entries) and the
    // (pass row, session) pairs whose rows become last_hidden [2][max_sessions]
    int4 *d_pa_tab = nullptr;
    int32_t *d_rows = nullptr;
    int pa_tab_cap = 0;
    // top-k / top-p sampling (jl_sample.cu): the exponentials of up to min(max_sessions, JL_MAX_DECODE_ROWS) rows, and the row table
    float *topkp_ex = nullptr;
    TopkpRow *d_topkp = nullptr, *h_topkp = nullptr;
    // token logprobs (jl_logprobs.cu): the decode / first-token buffers (allocated at finalize) and the prompt-scoring ones (allocated
    // by the first jl_model_score_multi, with a 64-row logits buffer when max_sessions is smaller)
    struct LpBufs {
        void *ws = nullptr;
        unsigned *cnt = nullptr;
        LogprobRow *d_rows = nullptr, *h_rows = nullptr;
        LogprobOut *d_out = nullptr, *h_out = nullptr;
        int32_t *d_idx = nullptr, *h_idx = nullptr; // scoring: [cap] gathered pass rows, then [cap] their target tokens
        int cap = 0;
    } lp, lp_score;
    float *score_logits = nullptr;
    // penalties (jl_penalty.cu), allocated by the first call with a penalised row: the processed rows, the per-row token words and bias
    // rows of min(max_sessions, JL_MAX_DECODE_ROWS) rows, and the penalty table (grown to the largest call's)
    float *pen_out = nullptr, *pen_bias = nullptr;
    unsigned *pen_cnt = nullptr;
    void *d_pen_tab = nullptr, *h_pen_tab = nullptr;
    size_t pen_tab_cap = 0;
    // allowed-token masks (DESIGN §3.18), allocated by the first call with a constrained row: min(max_sessions, JL_MAX_DECODE_ROWS) rows
    // of (vocab + 31) / 32 words on the device and in pinned staging
    uint32_t *d_mask = nullptr, *h_mask = nullptr;
    int hist_cap = 0;
    // graphs keyed by (n, splits, resident)
    std::map<long long, cudaGraphExec_t> graphs;
    std::map<long long, long long> graph_launches; // kernels per graph replay
    // event timing of the last decode call
    cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
    double last_total_ms = 0;
    int64_t weight_bytes = 0;
    unsigned *fda_done = nullptr;
    // mixture of experts (MoEBlock.java): router + per-expert w1 / w2 / w3, device pointer tables for the indirect GEMV launches
    // GPT-2 family (cfg.arch == JL_ARCH_GPT2): biases per layer [layers][8], wpe and ln_f.bias
    std::vector<DevTensor> aux;
    std::vector<char> aux_set;
    DevTensor gaux[2];
    bool gaux_set[2] = {false, false};
    int n_exp = 0, exp_k = 0;
    std::vector<DevTensor> moe_gate; // [layers]
    std::vector<DevTensor> moe_w;    // [layers][n_exp][3]
    std::vector<char> moe_set;       // [layers][1 + n_exp * 3]
    void **moe_wtab = nullptr;       // device [layers][3][n_exp] weight pointers
    float **moe_stab = nullptr;      // device [layers][3][n_exp] scale pointers
    float *moe_logits = nullptr;     // [maxB][n_exp]
    int32_t *moe_sel = nullptr;      // [maxB][exp_k]
    // grouped expert GEMMs (forward_rows, M >= 2): Q8 rows of xb (gate/up) and of h (down_proj), each pair's down_proj output
    // [maxB * exp_k][E], and the grouping of jl_launch_moe_group (one allocation, moe_grp.tiles first)
    void *moe_qa = nullptr, *moe_qh = nullptr;
    float *moe_dout = nullptr;
    MoeGroups moe_grp = {};
    // persistent decode kernel (jl_pdecode.cu)
    bool pd_ok = false;
    int pd_wdtype = JL_Q4;
    std::vector<PdLayer> pd_layers; // host copy; uploaded to constant memory by jl_launch_pdecode
    unsigned long long *pd_sync = nullptr, *pd_slots = nullptr, *pd_trace = nullptr;
    unsigned *pd_att_done = nullptr;
    int pd_vocab0 = 0, pd_vocab_rows = 0;
    // tensor-parallel exchange buffers: local allocations + every rank's copy opened through CUDA IPC
    uint4 *ll_o = nullptr, *ll_d = nullptr, *ll_a = nullptr;
    // sessions spilled to host memory (jl_model_kv_offload): handle -> (layer page, context page, page bytes) per allocated page
    struct KvSpill {
        std::vector<std::pair<int, int>> pages;
        std::vector<char> bytes;
    };
    std::map<int64_t, KvSpill> spills;
    int64_t next_spill = 1;
    // retained prefixes (jl_model_kv_retain): handle -> the pages [layer page][context page] below `positions` it holds; each page it
    // holds counts one reference in page_refs, exactly like a page-table entry
    struct KvRetained {
        int positions = 0;
        std::vector<void *> pages;
    };
    std::map<int64_t, KvRetained> retained;
    int64_t next_retained = 1;
    uint4 *peer_ll_o[PD_MAX_TP] = {}, *peer_ll_d[PD_MAX_TP] = {}, *peer_ll_a[PD_MAX_TP] = {};
    float *peer_logits[PD_MAX_TP] = {};
    std::vector<void *> ipc_opened;
};

#define M_CHECK(expr)                 \
    do {                              \
        int _rc = (expr);             \
        if (_rc != JL_OK) return _rc; \
    } while (0)

static bool use_graph(const jl_model *m) { return !(m->cfg.flags & JL_MODEL_NO_GRAPH); }
static bool use_pd(const jl_model *m) { return m->pd_ok && !(m->cfg.flags & (JL_MODEL_NO_PERSISTENT | JL_MODEL_NO_GRAPH)); }

// one more page-table entry holds page p
static void add_ref(jl_model *m, void *p) {
    auto it = m->page_refs.find(p);
    if (it == m->page_refs.end()) m->page_refs.emplace(p, 2);
    else it->second++;
}
// an entry lets go of page p: true if p was shared (the others keep it; the last one left owns it alone), false if p was the entry's own
static bool drop_ref(jl_model *m, void *p) {
    if (m->page_refs.empty()) return false;
    auto it = m->page_refs.find(p);
    if (it == m->page_refs.end()) return false;
    if (--it->second == 1) m->page_refs.erase(it);
    return true;
}
static bool is_shared(const jl_model *m, void *p) { return !m->page_refs.empty() && m->page_refs.count(p); }

extern "C" int jl_model_config_size(void) { return (int)sizeof(jl_model_config); }

extern "C" int jl_model_create(jl_ctx *ctx, const jl_model_config *cfg, jl_model **out) {
    if (!ctx || !cfg || !out) return JL_ERR_INVALID;
    *out = nullptr;
    const jl_model_config &c = *cfg;
    if (c.embedding_length <= 0 || c.num_heads <= 0 || c.num_kv_heads <= 0 || c.num_layers <= 0 || c.vocab_size <= 0 ||
        c.hidden_length <= 0 || c.context_length <= 0 || c.num_heads % c.num_kv_heads)
        return jl_set_error(ctx, JL_ERR_INVALID, "model_create: bad config");
    jl_model *m = new jl_model();
    m->ctx = ctx;
    m->cfg = c;
    if (m->cfg.head_size <= 0) m->cfg.head_size = c.embedding_length / c.num_heads; // Config.java:254
    if (m->cfg.max_batch <= 0) m->cfg.max_batch = 256;
    if (m->cfg.max_sessions <= 0) m->cfg.max_sessions = 1;
    if (m->cfg.tp_size <= 0) m->cfg.tp_size = 1;
    if (m->cfg.rope_scaling == 0.0) m->cfg.rope_scaling = 1.0;
    if (m->cfg.working_qtype != JL_I8 && m->cfg.working_qtype != JL_F32)
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_create: working_qtype must be JL_I8 or JL_F32"), delete m, JL_ERR_UNSUPPORTED;
    if (m->cfg.kv_dtype != JL_F32 && m->cfg.kv_dtype != JL_BF16 && m->cfg.kv_dtype != JL_I8)
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_create: kv_dtype must be JL_F32, JL_BF16 or JL_I8"), delete m, JL_ERR_UNSUPPORTED;
    const int hs = m->cfg.head_size;
    // I8 pages: whole 32-element blocks per KV head, and no per-op tensor-parallel path yet
    if (m->cfg.kv_dtype == JL_I8 && (hs % QBLOCK || m->cfg.tp_size > 1))
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_create: kv_dtype JL_I8 needs head_size %% 32 == 0 and tp_size 1 (head_size %d, tp_size %d)", hs,
                            m->cfg.tp_size), delete m, JL_ERR_UNSUPPORTED;
    m->group = c.num_heads / c.num_kv_heads;
    // jlama-net limits model shards to the number of KV heads (JlamaService.java:65-68)
    if (m->cfg.tp_size > c.num_kv_heads || c.num_kv_heads % m->cfg.tp_size)
        return jl_set_error(ctx, JL_ERR_INVALID, "model_create: tp_size must divide num_kv_heads"), delete m, JL_ERR_INVALID;
    int rc = jl_dctx_build(c.embedding_length, c.num_heads * hs, c.hidden_length, hs, m->group, c.num_layers, m->cfg.tp_rank,
                           m->cfg.tp_size, 0, 1, &m->d);
    if (rc) return delete m, jl_set_error(ctx, rc, "model_create: bad shard config");
    m->attn_seg = m->d.attentionSegmentLength;
    m->kv_seg = m->d.kvSegmentLength;
    m->h_seg = m->d.hiddenSegmentLength;
    m->heads_local = m->attn_seg / hs;
    m->kv_heads_local = m->kv_seg / hs;
    m->l.resize((size_t)c.num_layers * 9);
    m->l_set.assign((size_t)c.num_layers * 9, 0);
    if (c.arch == JL_ARCH_GPT2) {
        if (m->cfg.tp_size != 1 || c.num_experts > 0 || c.num_heads != c.num_kv_heads)
            return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_create: GPT-2 blocks are single-rank, dense, multi-head"), delete m, JL_ERR_UNSUPPORTED;
        m->aux.resize((size_t)c.num_layers * 8);
        m->aux_set.assign((size_t)c.num_layers * 8, 0);
    } else if (c.arch != JL_ARCH_LLAMA)
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_create: unknown arch %d", c.arch), delete m, JL_ERR_UNSUPPORTED;
    if (c.num_experts > 0) {
        if (c.num_experts > 64 || c.experts_per_token < 1 || c.experts_per_token > c.num_experts || (c.num_experts % m->cfg.tp_size))
            return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_create: %d experts / top-%d (max 64 experts, single rank)", c.num_experts,
                                c.experts_per_token),
                   delete m, JL_ERR_UNSUPPORTED;
        m->n_exp = c.num_experts, m->exp_k = c.experts_per_token;
        m->moe_gate.resize(c.num_layers);
        m->moe_w.resize((size_t)c.num_layers * m->n_exp * 3);
        m->moe_set.assign((size_t)c.num_layers * (1 + m->n_exp * 3), 0);
    }
    m->max_context = c.max_context > 0 && c.max_context < c.context_length ? c.max_context : c.context_length;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        ctx->models.push_back(m);
    }
    *out = m;
    return JL_OK;
}

// The registry tensor `tensor_id` for a slot of a model that is not finalized yet (ctx->mu held); null, with the error set, otherwise.
static DevTensor *unbound_tensor(jl_model *m, int64_t tensor_id, const char *who) {
    jl_ctx *ctx = m->ctx;
    if (m->finalized) return jl_set_error(ctx, JL_ERR_INVALID, "%s: model already finalized", who), nullptr;
    auto it = ctx->tensors.find(tensor_id);
    if (it == ctx->tensors.end()) return jl_set_error(ctx, JL_ERR_INVALID, "%s: unknown tensor id", who), nullptr;
    return &it->second;
}

// slot = t (ctx->mu held): the model holds a reference on t and drops the one it held on the tensor the slot had, so that tensor can
// be unregistered again
static void bind_tensor(jl_model *m, DevTensor &slot, DevTensor &t) {
    jl_ctx *ctx = m->ctx;
    if (slot.id) {
        auto old = ctx->tensors.find(slot.id);
        if (old != ctx->tensors.end() && old->second.refs > 0) old->second.refs--;
        for (size_t i = 0; i < m->bound_ids.size(); i++)
            if (m->bound_ids[i] == slot.id) {
                m->bound_ids.erase(m->bound_ids.begin() + i);
                break;
            }
    }
    t.refs++;
    m->bound_ids.push_back(t.id);
    slot = t;
}

extern "C" int jl_model_set_tensor(jl_model *m, int layer, int slot, int64_t tensor_id) {
    if (!m) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DevTensor *tp = unbound_tensor(m, tensor_id, "model_set_tensor");
    if (!tp) return JL_ERR_INVALID;
    const DevTensor &t = *tp;
    const jl_model_config &c = m->cfg;
    const int E = c.embedding_length;
    auto expect = [&](int64_t rows, int64_t cols) {
        return (t.rows == rows && t.cols == cols)
                   ? JL_OK
                   : jl_set_error(ctx, JL_ERR_INVALID, "model_set_tensor: layer %d slot %d expects [%lld,%lld], got [%lld,%lld]",
                                  layer, slot, (long long)rows, (long long)cols, (long long)t.rows, (long long)t.cols);
    };
    if (layer < 0) {
        if (slot < 0 || slot > 2) return jl_set_error(ctx, JL_ERR_INVALID, "bad global slot");
        if (slot == JL_T_OUT_NORM) {
            M_CHECK(expect(1, E));
            if (t.dtype != JL_F32 && t.dtype != JL_BF16) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "norm weights must be F32/BF16");
        } else
            M_CHECK(expect(c.vocab_size, E));
        bind_tensor(m, m->g[slot], *tp);
        m->g_set[slot] = true;
        return JL_OK;
    }
    if (layer >= c.num_layers || slot < 0 || slot > 8) return jl_set_error(ctx, JL_ERR_INVALID, "bad layer slot");
    switch (slot) {
        case JL_L_ATTN_NORM:
        case JL_L_FFN_NORM:
            M_CHECK(expect(1, E));
            if (t.dtype != JL_F32 && t.dtype != JL_BF16) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "norm weights must be F32/BF16");
            break;
        case JL_L_Q: M_CHECK(expect(m->attn_seg, E)); break;
        case JL_L_K:
        case JL_L_V: M_CHECK(expect(m->kv_seg, E)); break;
        case JL_L_O: M_CHECK(expect(E, m->attn_seg)); break;
        case JL_L_GATE:
        case JL_L_UP: M_CHECK(expect(m->h_seg, E)); break;
        case JL_L_DOWN: M_CHECK(expect(E, m->h_seg)); break;
    }
    bind_tensor(m, m->l[(size_t)layer * 9 + slot], *tp);
    m->l_set[(size_t)layer * 9 + slot] = 1;
    return JL_OK;
}

extern "C" int jl_model_set_expert_tensor(jl_model *m, int layer, int expert, int which, int64_t tensor_id) {
    if (!m) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (m->n_exp <= 0) return jl_set_error(ctx, JL_ERR_INVALID, "model_set_expert_tensor: the model has no experts");
    DevTensor *tp = unbound_tensor(m, tensor_id, "model_set_expert_tensor");
    if (!tp) return JL_ERR_INVALID;
    if (layer < 0 || layer >= m->cfg.num_layers || expert < -1 || expert >= m->n_exp || which < 0 || which > 2)
        return jl_set_error(ctx, JL_ERR_INVALID, "model_set_expert_tensor: bad layer / expert / slot");
    const DevTensor &t = *tp;
    const int E = m->cfg.embedding_length, H = m->cfg.hidden_length;
    const int64_t rows = expert < 0 ? m->n_exp : (which == 1 ? E : H), cols = expert < 0 ? E : (which == 1 ? H : E);
    if (t.rows != rows || t.cols != cols)
        return jl_set_error(ctx, JL_ERR_INVALID, "model_set_expert_tensor: expects [%lld,%lld], got [%lld,%lld]", (long long)rows, (long long)cols,
                            (long long)t.rows, (long long)t.cols);
    if (expert < 0) {
        bind_tensor(m, m->moe_gate[layer], *tp);
        m->moe_set[(size_t)layer * (1 + m->n_exp * 3)] = 1;
    } else {
        bind_tensor(m, m->moe_w[((size_t)layer * m->n_exp + expert) * 3 + which], *tp);
        m->moe_set[(size_t)layer * (1 + m->n_exp * 3) + 1 + expert * 3 + which] = 1;
    }
    return JL_OK;
}

extern "C" int jl_model_set_aux_tensor(jl_model *m, int layer, int which, int64_t tensor_id) {
    if (!m) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);
    const jl_model_config &c = m->cfg;
    if (c.arch != JL_ARCH_GPT2) return jl_set_error(ctx, JL_ERR_INVALID, "model_set_aux_tensor: only GPT-2 models take bias / position tensors");
    DevTensor *tp = unbound_tensor(m, tensor_id, "model_set_aux_tensor");
    if (!tp) return JL_ERR_INVALID;
    const DevTensor &t = *tp;
    if (t.dtype != JL_F32 && t.dtype != JL_BF16) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_set_aux_tensor: F32 / BF16 only");
    const int E = c.embedding_length;
    int64_t rows = 1, cols = E;
    if (layer < 0) {
        if (which != JL_AUX_POS_EMBED && which != JL_AUX_OUT_NORM_BIAS) return jl_set_error(ctx, JL_ERR_INVALID, "model_set_aux_tensor: bad global slot");
        if (which == JL_AUX_POS_EMBED) rows = c.context_length;
    } else {
        if (layer >= c.num_layers || which < 0 || which > 7) return jl_set_error(ctx, JL_ERR_INVALID, "model_set_aux_tensor: bad layer slot");
        if (which == JL_AUX_K_BIAS || which == JL_AUX_V_BIAS) cols = m->kv_seg;
        else if (which == JL_AUX_Q_BIAS) cols = m->attn_seg;
        else if (which == JL_AUX_FC_BIAS) cols = m->h_seg;
    }
    if (t.rows != rows || t.cols != cols)
        return jl_set_error(ctx, JL_ERR_INVALID, "model_set_aux_tensor: layer %d slot %d expects [%lld,%lld], got [%lld,%lld]", layer, which,
                            (long long)rows, (long long)cols, (long long)t.rows, (long long)t.cols);
    if (layer < 0) bind_tensor(m, m->gaux[which], *tp), m->gaux_set[which] = true;
    else bind_tensor(m, m->aux[(size_t)layer * 8 + which], *tp), m->aux_set[(size_t)layer * 8 + which] = 1;
    return JL_OK;
}

static int dev_alloc(jl_ctx *ctx, void **p, size_t bytes);

// logprob buffers for `cap` rows per call, `launch` rows per kernel launch (`idx`: the scoring gather / target table)
static int lp_alloc(jl_model *m, jl_model::LpBufs &b, int cap, int launch, bool idx) {
    jl_ctx *ctx = m->ctx;
    M_CHECK(dev_alloc(ctx, &b.ws, jl_logprobs_ws_bytes(m->cfg.vocab_size, launch)));
    M_CHECK(dev_alloc(ctx, (void **)&b.cnt, (size_t)launch * sizeof(unsigned)));
    JL_CUDA_CHECK(ctx, cudaMemset(b.cnt, 0, (size_t)launch * sizeof(unsigned)));
    M_CHECK(dev_alloc(ctx, (void **)&b.d_rows, (size_t)cap * sizeof(LogprobRow)));
    M_CHECK(dev_alloc(ctx, (void **)&b.d_out, (size_t)cap * sizeof(LogprobOut)));
    JL_CUDA_CHECK(ctx, cudaMallocHost((void **)&b.h_rows, (size_t)cap * sizeof(LogprobRow)));
    JL_CUDA_CHECK(ctx, cudaMallocHost((void **)&b.h_out, (size_t)cap * sizeof(LogprobOut)));
    if (idx) {
        M_CHECK(dev_alloc(ctx, (void **)&b.d_idx, (size_t)cap * 2 * 4));
        JL_CUDA_CHECK(ctx, cudaMallocHost((void **)&b.h_idx, (size_t)cap * 2 * 4));
    }
    b.cap = cap;
    return JL_OK;
}

static void lp_free(jl_model::LpBufs &b) {
    for (void *p : {b.ws, (void *)b.cnt, (void *)b.d_rows, (void *)b.d_out, (void *)b.d_idx})
        if (p) cudaFree(p);
    for (void *p : {(void *)b.h_rows, (void *)b.h_out, (void *)b.h_idx})
        if (p) cudaFreeHost(p);
    b = jl_model::LpBufs();
}

static int dev_alloc(jl_ctx *ctx, void **p, size_t bytes) {
    if (cudaMalloc(p, bytes ? bytes : 16) != cudaSuccess) {
        cudaGetLastError();
        return jl_set_error(ctx, JL_ERR_OOM, "out of device memory (%zu bytes)", bytes);
    }
    return JL_OK;
}

extern "C" int jl_model_finalize(jl_model *m) {
    if (!m) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    if (m->finalized) return JL_OK;
    const jl_model_config &c = m->cfg;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    for (int i = 0; i < 2; i++)
        if (!m->g_set[i]) return jl_set_error(ctx, JL_ERR_INVALID, "model_finalize: global tensor %d missing", i);
    for (size_t i = 0; i < m->l_set.size(); i++) {
        const size_t slot = i % 9;
        if (m->n_exp > 0 && (slot == JL_L_GATE || slot == JL_L_DOWN || slot == JL_L_UP)) continue; // experts instead of a dense MLP
        if (c.arch == JL_ARCH_GPT2 && slot == JL_L_UP) continue;                                      // c_fc -> GELU -> c_proj: no up projection
        if (!m->l_set[i]) return jl_set_error(ctx, JL_ERR_INVALID, "model_finalize: layer %zu slot %zu missing", i / 9, slot);
    }
    // expert parallelism (BASELINE config 5: "expert FFN GEMMs sharded one-per-GPU"): rank r holds the experts e with
    // e % tp_size == r (whole, not row-split); the router is replicated.  Tensors of other ranks' experts stay unset.
    for (size_t i = 0; i < m->moe_set.size(); i++) {
        const size_t per = 1 + (size_t)m->n_exp * 3, slot = i % per;
        const bool mine = slot == 0 || (int)((slot - 1) / 3) % c.tp_size == c.tp_rank;
        if (mine && !m->moe_set[i]) return jl_set_error(ctx, JL_ERR_INVALID, "model_finalize: layer %zu expert tensor %zu missing", i / per, slot);
        if (!mine && m->moe_set[i]) return jl_set_error(ctx, JL_ERR_INVALID, "model_finalize: layer %zu expert tensor %zu belongs to another rank", i / per, slot);
    }
    // the fused QKV and gate+up launches decode all their segments with one weight dtype: a checkpoint that mixes
    // precisions inside a fused group (e.g. Q in Q4, K/V left in BF16) must be rejected, not mis-read
    for (int L = 0; L < c.num_layers; L++) {
        const DevTensor *lw = &m->l[(size_t)L * 9];
        if (lw[JL_L_K].dtype != lw[JL_L_Q].dtype || lw[JL_L_V].dtype != lw[JL_L_Q].dtype)
            return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_finalize: layer %d q/k/v weights must share one dtype (got %d/%d/%d)", L,
                                lw[JL_L_Q].dtype, lw[JL_L_K].dtype, lw[JL_L_V].dtype);
        if (m->n_exp == 0 && c.arch != JL_ARCH_GPT2 && lw[JL_L_UP].dtype != lw[JL_L_GATE].dtype)
            return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_finalize: layer %d gate/up weights must share one dtype (got %d/%d)", L,
                                lw[JL_L_GATE].dtype, lw[JL_L_UP].dtype);
        // gate/up run fused with SiLU * up, which only the quantised GEMVs implement: refuse F32 / BF16 gate/up here rather than
        // fail at the first token
        if (m->n_exp == 0 && c.arch != JL_ARCH_GPT2 && lw[JL_L_GATE].dtype != JL_Q4 && lw[JL_L_GATE].dtype != JL_I8)
            return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_finalize: layer %d slot %d (gate) and slot %d (up): dtype %d, SiLU * up needs Q4 or I8 weights",
                                L, JL_L_GATE, JL_L_UP, lw[JL_L_GATE].dtype);
    }
    // the experts' w1 / w3 run fused with SiLU * up the same way, and every expert GEMV decodes one quantised dtype
    for (int L = 0; L < c.num_layers && m->n_exp > 0; L++)
        for (int e = c.tp_rank; e < m->n_exp; e += c.tp_size)
            for (int w = 0; w < 3; w++) {
                const int dt = m->moe_w[((size_t)L * m->n_exp + e) * 3 + w].dtype;
                if (dt != JL_Q4 && dt != JL_I8)
                    return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_finalize: layer %d expert %d weight %d (w%d): dtype %d, expert GEMVs need Q4 or I8",
                                        L, e, w, w + 1, dt);
            }
    if (c.arch == JL_ARCH_GPT2) {
        for (size_t i = 0; i < m->aux_set.size(); i++)
            if (!m->aux_set[i]) return jl_set_error(ctx, JL_ERR_INVALID, "model_finalize: layer %zu bias slot %zu missing", i / 8, i % 8);
        if (!m->gaux_set[0] || !m->gaux_set[1]) return jl_set_error(ctx, JL_ERR_INVALID, "model_finalize: wpe / ln_f.bias missing");
    }
    const int E = c.embedding_length, hs = c.head_size;
    JL_CUDA_CHECK(ctx, cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
    // RoPE table (Config.java:271-276) padded by 2*kv_heads positions: head h reads position pos+2*kvh
    // (CausalSelfAttention.java:260-268); the reference would throw past the end of its table.
    {
        const int positions = c.context_length + 2 * c.num_kv_heads;
        std::vector<float> tbl((size_t)positions * (hs / 2) * 2);
        if (c.arch == JL_ARCH_GPT2) // no rotary embedding: the identity rotation (cos 1, sin 0) leaves q and k bit for bit
            for (size_t i = 0; i < tbl.size(); i += 2) tbl[i] = 1.0f, tbl[i + 1] = 0.0f;
        else jl_precompute_freqs_cis(hs, positions, c.rope_theta, c.rope_scaling, tbl.data());
        M_CHECK(dev_alloc(ctx, (void **)&m->rope, tbl.size() * 4));
        JL_CUDA_CHECK(ctx, cudaMemcpy(m->rope, tbl.data(), tbl.size() * 4, cudaMemcpyHostToDevice));
    }
    // KV geometry (KvBufferCache.java:99-112,224-280).  I8 pages have no reference geometry, and the solver would pick a layer split
    // that leaves a nearly empty second layer page (30 + 2 layers for Llama-3-8B): they take the largest divisor of num_layers whose
    // K and V rows of one position fit 8 MiB, and as many positions as then fit (DESIGN §3.16).
    const size_t kv_row = kv_row_bytes(c.kv_dtype, (size_t)m->kv_seg);
    int lpp = 0, cpp = 0;
    if (c.kv_dtype == JL_I8) {
        const size_t cap = (size_t)1 << 23;
        for (int d = c.num_layers; d >= 1 && !lpp; d--)
            if (c.num_layers % d == 0 && (size_t)d * 2 * kv_row <= cap) lpp = d;
        if (!lpp) return jl_set_error(ctx, JL_ERR_INVALID, "kv page geometry: a %zu-byte row does not fit an 8 MiB page", kv_row);
        const size_t fit = cap / ((size_t)lpp * 2 * kv_row);
        cpp = (int)(fit < (size_t)c.context_length ? fit : (size_t)c.context_length);
    } else if (jl_kv_page_geometry(c.num_layers, c.context_length, m->kv_seg, (int)(kv_row / m->kv_seg), 1 << 23, &lpp, &cpp))
        return jl_set_error(ctx, JL_ERR_INVALID, "kv page geometry");
    m->kv.layers_per_page = lpp;
    m->kv.ctx_per_page = cpp;
    m->kv.kv_len = m->kv_seg;
    m->kv.n_layer_pages = (c.num_layers + lpp - 1) / lpp;
    m->kv.n_ctx_pages = (m->max_context + cpp - 1) / cpp;
    m->kv.kv_dtype = c.kv_dtype;
    m->page_bytes = (size_t)lpp * 2 * cpp * kv_row;
    const size_t nent = (size_t)c.max_sessions * m->kv.n_layer_pages * m->kv.n_ctx_pages;
    m->page_table_host.assign(nent, nullptr);
    M_CHECK(dev_alloc(ctx, (void **)&m->page_table_dev, nent * sizeof(void *)));
    JL_CUDA_CHECK(ctx, cudaMemset(m->page_table_dev, 0, nent * sizeof(void *)));
    m->kv.page_table = m->page_table_dev;
    // scratch
    m->maxB = c.max_batch > c.max_sessions ? c.max_batch : c.max_sessions;
    const size_t B = m->maxB;
    M_CHECK(dev_alloc(ctx, (void **)&m->x, B * E * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->xb, B * E * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->q, B * m->attn_seg * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->k, B * m->kv_seg * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->v, B * m->kv_seg * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->att, B * m->attn_seg * 4));
    // experts are held whole (expert parallelism), so their hidden activations need the full hidden length; each (row, selected
    // expert) keeps its own h row, so every phase of every row can be read back after a step
    M_CHECK(dev_alloc(ctx, (void **)&m->hbuf, B * (size_t)(m->n_exp > 0 ? (size_t)m->exp_k * c.hidden_length : m->h_seg) * 4));
    if (m->n_exp > 0) {
        M_CHECK(dev_alloc(ctx, (void **)&m->moe_logits, B * m->n_exp * 4));
        M_CHECK(dev_alloc(ctx, (void **)&m->moe_sel, B * m->exp_k * 4));
        const size_t ne = (size_t)c.num_layers * 3 * m->n_exp;
        std::vector<void *> wt(ne);
        std::vector<float *> st(ne);
        int wd0 = m->moe_w[(size_t)c.tp_rank * 3].dtype; // expert tp_rank is the first one this rank holds
        for (int L = 0; L < c.num_layers; L++)
            for (int w = 0; w < 3; w++)
                for (int e = 0; e < m->n_exp; e++) {
                    const DevTensor &t = m->moe_w[((size_t)L * m->n_exp + e) * 3 + w];
                    if (e % c.tp_size != c.tp_rank) { // another rank's expert: null table entries, the GEMV contributes nothing
                        wt[((size_t)L * 3 + w) * m->n_exp + e] = nullptr;
                        st[((size_t)L * 3 + w) * m->n_exp + e] = nullptr;
                        continue;
                    }
                    if (t.dtype != wd0 || (wd0 != JL_Q4 && wd0 != JL_I8))
                        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "model_finalize: expert weights must share one quantised dtype (Q4 or I8)");
                    wt[((size_t)L * 3 + w) * m->n_exp + e] = t.data;
                    st[((size_t)L * 3 + w) * m->n_exp + e] = t.scales;
                }
        M_CHECK(dev_alloc(ctx, (void **)&m->moe_wtab, ne * sizeof(void *)));
        M_CHECK(dev_alloc(ctx, (void **)&m->moe_stab, ne * sizeof(float *)));
        JL_CUDA_CHECK(ctx, cudaMemcpy(m->moe_wtab, wt.data(), ne * sizeof(void *), cudaMemcpyHostToDevice));
        JL_CUDA_CHECK(ctx, cudaMemcpy(m->moe_stab, st.data(), ne * sizeof(float *), cudaMemcpyHostToDevice));
        // grouped expert GEMMs: at most maxB * k + n_exp tiles for any tile height
        const size_t H = c.hidden_length, P = B * m->exp_k, T = P + m->n_exp;
        M_CHECK(dev_alloc(ctx, &m->moe_qa, jl_gemm64_q8_bytes((int)B, E)));
        M_CHECK(dev_alloc(ctx, &m->moe_qh, jl_gemm64_q8_bytes((int)P, (int)H)));
        M_CHECK(dev_alloc(ctx, (void **)&m->moe_dout, P * E * 4));
        char *gb = nullptr;
        M_CHECK(dev_alloc(ctx, (void **)&gb, T * sizeof(int4) + (P + 2 * (size_t)m->n_exp + 1) * 4));
        m->moe_grp.tiles = (int4 *)gb, m->moe_grp.pairs = (int32_t *)(gb + T * sizeof(int4));
        m->moe_grp.counts = m->moe_grp.pairs + P, m->moe_grp.offsets = m->moe_grp.counts + m->n_exp;
        m->moe_grp.ntiles = m->moe_grp.offsets + m->n_exp;
    }
    M_CHECK(dev_alloc(ctx, (void **)&m->partial, B * E * 4));
    if (c.arch == JL_ARCH_GPT2) M_CHECK(dev_alloc(ctx, (void **)&m->ln, B * E * 4)); // LayerNorm output (its own tensor in the reference too)
    if (c.prefill_tensor_core && c.arch == JL_ARCH_LLAMA) {
        size_t kmax = E > m->h_seg ? E : m->h_seg;
        if ((size_t)m->attn_seg > kmax) kmax = m->attn_seg;
        M_CHECK(dev_alloc(ctx, (void **)&m->ln, B * E * 4));
        M_CHECK(dev_alloc(ctx, (void **)&m->hbuf2, B * m->h_seg * 4));
        M_CHECK(dev_alloc(ctx, (void **)&m->abf, B * kmax * 2));
        bool ok = m->n_exp == 0 && c.arch == JL_ARCH_LLAMA && c.tp_size == 1 && (E % 128) == 0 && (m->h_seg % 128) == 0 && (m->attn_seg % 128) == 0 &&
                  (m->kv_seg % 128) == 0;
        for (int L = 0; L < c.num_layers && ok; L++)
            for (int sl : {JL_L_Q, JL_L_K, JL_L_V, JL_L_O, JL_L_GATE, JL_L_DOWN, JL_L_UP}) {
                const int dt = m->l[(size_t)L * 9 + sl].dtype;
                ok = ok && (dt == JL_Q4 || dt == JL_I8); // both block formats are dequantised into the BF16 weight tile
            }
        m->tc_ok = ok;
    }
    if (c.max_sessions > GEMV_MAX_M) {
        int kmax = E > m->h_seg ? E : m->h_seg;
        if (m->attn_seg > kmax) kmax = m->attn_seg;
        M_CHECK(dev_alloc(ctx, &m->wide_act, jl_gemm64_act_bytes(kmax)));
        M_CHECK(dev_alloc(ctx, (void **)&m->wide_part, jl_gemm64_part_floats(ctx->sm_count) * 4));
        M_CHECK(dev_alloc(ctx, (void **)&m->wide_cnt, (size_t)ctx->sm_count * sizeof(unsigned)));
        JL_CUDA_CHECK(ctx, cudaMemset(m->wide_cnt, 0, (size_t)ctx->sm_count * sizeof(unsigned)));
    }
    M_CHECK(dev_alloc(ctx, (void **)&m->logits, (size_t)c.max_sessions * c.vocab_size * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->last_hidden, (size_t)c.max_sessions * E * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->attn_ws, B * m->heads_local * m->max_splits * (hs + 2) * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->d_tokens, B * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->d_positions, B * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->d_sessions, B * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->d_next, B * 4));
    m->hist_cap = 1 << 16;
    M_CHECK(dev_alloc(ctx, (void **)&m->d_hist, (size_t)m->hist_cap * 4));
    M_CHECK(dev_alloc(ctx, (void **)&m->d_counter, 4));
    M_CHECK(dev_alloc(ctx, &m->argmax_scratch, jl_argmax_scratch_bytes(c.max_sessions)));
    M_CHECK(dev_alloc(ctx, (void **)&m->fda_done, (size_t)m->maxB * m->kv_heads_local * sizeof(unsigned)));
    JL_CUDA_CHECK(ctx, cudaMemset(m->fda_done, 0, (size_t)m->maxB * m->kv_heads_local * sizeof(unsigned)));
    m->pa_tab_cap = (int)(B / 16) + c.max_sessions;
    M_CHECK(dev_alloc(ctx, (void **)&m->d_pa_tab, (size_t)m->pa_tab_cap * sizeof(int4)));
    M_CHECK(dev_alloc(ctx, (void **)&m->d_rows, (size_t)c.max_sessions * 2 * 4));
    // a fork's partial pages (one per layer page and destination) or one session's copy-on-write pages fit one launch
    m->copy_cap = m->kv.n_layer_pages * (c.max_sessions > m->kv.n_ctx_pages ? c.max_sessions : m->kv.n_ctx_pages);
    M_CHECK(dev_alloc(ctx, (void **)&m->d_copy_tab, (size_t)m->copy_cap * sizeof(KvCopy)));
    JL_CUDA_CHECK(ctx, cudaMallocHost((void **)&m->h_pinned, (B * 4 + (size_t)m->pa_tab_cap * 4 + (size_t)c.max_sessions * 2) * 4 +
                                                                 (size_t)m->copy_cap * sizeof(KvCopy)));
    {
        const int rows = c.max_sessions < JL_MAX_DECODE_ROWS ? c.max_sessions : JL_MAX_DECODE_ROWS;
        M_CHECK(dev_alloc(ctx, (void **)&m->topkp_ex, (size_t)rows * c.vocab_size * 4));
        M_CHECK(dev_alloc(ctx, (void **)&m->d_topkp, (size_t)rows * sizeof(TopkpRow)));
        JL_CUDA_CHECK(ctx, cudaMallocHost((void **)&m->h_topkp, (size_t)rows * sizeof(TopkpRow)));
    }
    {
        const int rows = c.max_sessions < JL_MAX_DECODE_ROWS ? c.max_sessions : JL_MAX_DECODE_ROWS;
        M_CHECK(lp_alloc(m, m->lp, rows, rows, false));
    }
    JL_CUDA_CHECK(ctx, cudaEventCreate(&m->ev_begin));
    JL_CUDA_CHECK(ctx, cudaEventCreate(&m->ev_end));
    // algorithmic decode bytes per token on this rank (SURVEY 8d): every linear weight once + lm_head
    auto tb = [](const DevTensor &t) { return (int64_t)t.bytes; };
    int64_t wb = 0;
    for (int L = 0; L < c.num_layers; L++)
        for (int s : {JL_L_Q, JL_L_K, JL_L_V, JL_L_O, JL_L_GATE, JL_L_DOWN, JL_L_UP})
            if (m->l_set[(size_t)L * 9 + s]) wb += tb(m->l[(size_t)L * 9 + s]);
    // mixture of experts: the router plus the experts_per_token selected experts are streamed per token
    for (int L = 0; L < c.num_layers && m->n_exp > 0; L++) {
        wb += tb(m->moe_gate[L]);
        // expert parallel: on average experts_per_token / tp_size of them live on this rank
        for (int w = 0; w < 3; w++) wb += (int64_t)m->exp_k * tb(m->moe_w[((size_t)L * m->n_exp + c.tp_rank) * 3 + w]) / c.tp_size;
    }
    wb += tb(m->g_set[JL_T_LM_HEAD] ? m->g[JL_T_LM_HEAD] : m->g[JL_T_EMBED]);
    m->weight_bytes = wb;
    // ---- persistent decode kernel eligibility: Q8 activations, every linear weight (and the lm_head) in ONE quantised dtype ----
    {
        const DevTensor &head = m->g_set[JL_T_LM_HEAD] ? m->g[JL_T_LM_HEAD] : m->g[JL_T_EMBED];
        const int wd = m->l[JL_L_Q].dtype;
        // I8 KV pages: one-session decode takes the per-op graph.  The persistent kernel's attention (attention_flat<HS, PD_NT> with
        // KVDT -1) addresses F32 / BF16 rows only and would misread I8 rows: do not relax this without an I8 instantiation of it.
        bool ok = m->n_exp == 0 && c.arch == JL_ARCH_LLAMA && c.working_qtype == JL_I8 && (wd == JL_Q4 || wd == JL_I8) && head.dtype == wd &&
                  c.kv_dtype != JL_I8;
        for (int L = 0; L < c.num_layers && ok; L++)
            for (int sl : {JL_L_Q, JL_L_K, JL_L_V, JL_L_O, JL_L_GATE, JL_L_DOWN, JL_L_UP}) ok = ok && m->l[(size_t)L * 9 + sl].dtype == wd;
        // lm_head rows of this rank (vocabulary-sharded under tensor parallelism: SURVEY 8e; the reference computes the
        // full GEMV on the coordinator, AbstractModel.java:444-449)
        const int W = c.tp_size, V = c.vocab_size;
        m->pd_vocab0 = (int)(((long long)V * c.tp_rank) / W);
        m->pd_vocab_rows = (int)(((long long)V * (c.tp_rank + 1)) / W) - m->pd_vocab0;
        if (ok && W > 1 && !ctx->nccl_comm) ok = false; // the IPC handles travel over the communicator
        if (ok) {
            PdParams probe = {};
            probe.layers = c.num_layers, probe.E = E, probe.H = m->h_seg, probe.attn_seg = m->attn_seg, probe.kv_seg = m->kv_seg;
            probe.heads = m->heads_local, probe.kv_heads = m->kv_heads_local, probe.head_size = hs, probe.world = W;
            ok = jl_pdecode_supported(probe, wd, ctx->sm_count);
            // flat decode attention: at most 1024 positions per (kv head, split) task
            int cap = ctx->sm_count / (m->kv_heads_local > 0 ? m->kv_heads_local : 1);
            if (cap > m->max_splits) cap = m->max_splits;
            if (cap < 1 || (m->max_context + cap - 1) / cap > 1024 - 32) ok = false;
        }
        if (ok) {
            std::vector<PdLayer> pl(c.num_layers);
            const int order[7] = {JL_L_Q, JL_L_K, JL_L_V, JL_L_O, JL_L_GATE, JL_L_UP, JL_L_DOWN};
            for (int L = 0; L < c.num_layers; L++) {
                for (int i = 0; i < 7; i++) {
                    pl[L].w[i] = (const uint8_t *)m->l[(size_t)L * 9 + order[i]].data;
                    pl[L].s[i] = m->l[(size_t)L * 9 + order[i]].scales;
                }
                pl[L].attn_norm = m->l[(size_t)L * 9 + JL_L_ATTN_NORM].data;
                pl[L].attn_norm_dt = m->l[(size_t)L * 9 + JL_L_ATTN_NORM].dtype;
                pl[L].ffn_norm = m->l[(size_t)L * 9 + JL_L_FFN_NORM].data;
                pl[L].ffn_norm_dt = m->l[(size_t)L * 9 + JL_L_FFN_NORM].dtype;
            }
            m->pd_layers = pl;
            M_CHECK(dev_alloc(ctx, (void **)&m->pd_sync, PD_SYNC_WORDS * 8));
            JL_CUDA_CHECK(ctx, cudaMemset(m->pd_sync, 0, PD_SYNC_WORDS * 8));
            M_CHECK(dev_alloc(ctx, (void **)&m->pd_slots, (size_t)ctx->sm_count * 8));
            M_CHECK(dev_alloc(ctx, (void **)&m->pd_att_done, (size_t)m->kv_heads_local * sizeof(unsigned)));
            JL_CUDA_CHECK(ctx, cudaMemset(m->pd_att_done, 0, (size_t)m->kv_heads_local * sizeof(unsigned)));
            m->pd_wdtype = wd;
            if (W > 1) {
                // LL receive buffers of this rank and the peers' copies (cudaIpc: one process per GPU)
                const size_t lines = (size_t)W * E / 2 + 8;
                M_CHECK(dev_alloc(ctx, (void **)&m->ll_o, lines * 16));
                M_CHECK(dev_alloc(ctx, (void **)&m->ll_d, lines * 16));
                M_CHECK(dev_alloc(ctx, (void **)&m->ll_a, (size_t)PD_MAX_TP * 16));
                JL_CUDA_CHECK(ctx, cudaMemset(m->ll_o, 0, lines * 16));
                JL_CUDA_CHECK(ctx, cudaMemset(m->ll_d, 0, lines * 16));
                JL_CUDA_CHECK(ctx, cudaMemset(m->ll_a, 0, (size_t)PD_MAX_TP * 16));
                void *local[4] = {m->ll_o, m->ll_d, m->ll_a, m->logits};
                cudaIpcMemHandle_t mine[4];
                for (int i = 0; i < 4; i++) JL_CUDA_CHECK(ctx, cudaIpcGetMemHandle(&mine[i], local[i]));
                cudaIpcMemHandle_t *d_send = nullptr, *d_recv = nullptr;
                M_CHECK(dev_alloc(ctx, (void **)&d_send, sizeof mine));
                M_CHECK(dev_alloc(ctx, (void **)&d_recv, sizeof mine * W));
                JL_CUDA_CHECK(ctx, cudaMemcpy(d_send, mine, sizeof mine, cudaMemcpyHostToDevice));
                int rc = jl_comm_allgather_dev(ctx, m->stream, d_send, d_recv, sizeof mine);
                if (rc == JL_OK && cudaStreamSynchronize(m->stream) != cudaSuccess) rc = jl_set_error(ctx, JL_ERR_CUDA, "handle exchange failed");
                std::vector<cudaIpcMemHandle_t> all((size_t)4 * W);
                if (rc == JL_OK) JL_CUDA_CHECK(ctx, cudaMemcpy(all.data(), d_recv, sizeof mine * W, cudaMemcpyDeviceToHost));
                cudaFree(d_send);
                cudaFree(d_recv);
                if (rc != JL_OK) return rc;
                for (int r = 0; r < W; r++) {
                    void *ptrs[4];
                    for (int i = 0; i < 4; i++) {
                        if (r == c.tp_rank) {
                            ptrs[i] = local[i];
                        } else {
                            cudaError_t e = cudaIpcOpenMemHandle(&ptrs[i], all[(size_t)r * 4 + i], cudaIpcMemLazyEnablePeerAccess);
                            if (e != cudaSuccess)
                                return jl_set_error(ctx, JL_ERR_CUDA, "cudaIpcOpenMemHandle(rank %d): %s (peer access over NVLink is required)", r,
                                                    cudaGetErrorString(e));
                            m->ipc_opened.push_back(ptrs[i]);
                        }
                    }
                    m->peer_ll_o[r] = (uint4 *)ptrs[0], m->peer_ll_d[r] = (uint4 *)ptrs[1], m->peer_ll_a[r] = (uint4 *)ptrs[2];
                    m->peer_logits[r] = (float *)ptrs[3];
                }
            }
            if (getenv("JL_PD_TRACE")) {
                M_CHECK(dev_alloc(ctx, (void **)&m->pd_trace, ((size_t)c.num_layers * 16 + 32) * 8));
                JL_CUDA_CHECK(ctx, cudaMemset(m->pd_trace, 0, ((size_t)c.num_layers * 16 + 32) * 8));
            }
            m->pd_ok = true;
            // per-token stream of this rank: the lm_head is vocabulary-sharded on the persistent path
            if (W > 1) m->weight_bytes += -tb(head) + (int64_t)((double)tb(head) * m->pd_vocab_rows / V);
        }
    }
    m->finalized = true;
    return JL_OK;
}

extern "C" int64_t jl_model_weight_bytes(jl_model *m) { return m ? m->weight_bytes : -1; }

int jl_model_num_experts(jl_model *m) { return m ? m->n_exp : 0; } // jl_model_load_safetensors

// limits the session scheduler (jl_sched.cu) plans against: {max_sessions, reserved context, max_batch, rows per decode call,
// ctx_per_page, vocab_size}
void jl_model_limits(jl_model *m, int out[6]) {
    out[0] = out[1] = out[2] = out[3] = out[4] = out[5] = 0;
    if (!m || !m->finalized) return;
    out[0] = m->cfg.max_sessions, out[1] = m->max_context, out[2] = m->cfg.max_batch;
    out[3] = m->cfg.max_sessions < JL_MAX_DECODE_ROWS ? m->cfg.max_sessions : JL_MAX_DECODE_ROWS;
    out[4] = m->kv.ctx_per_page, out[5] = m->cfg.vocab_size;
}

// The timeline buffer was replaced (jl_debug_ktrace): drop every captured decode graph, they are re-captured on demand.
void jl_models_invalidate_graphs(jl_ctx *ctx) {
    for (jl_model *m : ctx->models) {
        if (m->stream) cudaStreamSynchronize(m->stream);
        for (auto &kv : m->graphs) cudaGraphExecDestroy(kv.second);
        m->graphs.clear();
        m->graph_launches.clear();
    }
}

extern "C" int jl_model_free(jl_model *m) {
    if (!m) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    cudaSetDevice(ctx->device);
    if (m->stream) cudaStreamSynchronize(m->stream);
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        for (int64_t id : m->bound_ids) {
            auto it = ctx->tensors.find(id);
            if (it != ctx->tensors.end() && it->second.refs > 0) it->second.refs--;
        }
        for (size_t i = 0; i < ctx->models.size(); i++)
            if (ctx->models[i] == m) {
                ctx->models.erase(ctx->models.begin() + i);
                break;
            }
    }
    jl_pdecode_forget(ctx->device, m);
    for (auto &kv : m->graphs) cudaGraphExecDestroy(kv.second);
    for (void *p : m->ipc_opened) cudaIpcCloseMemHandle(p);
    for (void *p : m->page_table_host) // a shared page is freed by the last entry or retained prefix that holds it
        if (p && !drop_ref(m, p)) cudaFree(p);
    for (const auto &r : m->retained)
        for (void *p : r.second.pages)
            if (!drop_ref(m, p)) cudaFree(p);
    void *bufs[] = {m->d_copy_tab,m->ln, m->hbuf2, m->abf, m->rope, m->page_table_dev, m->x, m->xb, m->q, m->k, m->v, m->att, m->hbuf, m->partial, m->logits,
                    m->last_hidden, m->attn_ws, m->d_tokens, m->d_positions, m->d_sessions, m->d_next, m->d_hist, m->d_counter,
                    m->argmax_scratch, m->fda_done, m->moe_wtab, m->moe_stab, m->moe_logits, m->moe_sel, m->moe_qa, m->moe_qh, m->moe_dout, m->moe_grp.tiles, m->pd_sync, m->pd_slots, m->pd_att_done, m->pd_trace, m->ll_o, m->ll_d, m->ll_a, m->wide_act, m->wide_part, m->wide_cnt, m->d_pa_tab, m->d_rows, m->topkp_ex, m->d_topkp,
                    m->score_logits, m->pen_out, m->pen_bias, m->pen_cnt, m->d_pen_tab, m->d_mask};
    for (void *p : bufs)
        if (p) cudaFree(p);
    lp_free(m->lp);
    lp_free(m->lp_score);
    if (m->h_pen_tab) cudaFreeHost(m->h_pen_tab);
    if (m->h_mask) cudaFreeHost(m->h_mask);
    if (m->h_pinned) cudaFreeHost(m->h_pinned);
    if (m->h_topkp) cudaFreeHost(m->h_topkp);
    if (m->ev_begin) cudaEventDestroy(m->ev_begin);
    if (m->ev_end) cudaEventDestroy(m->ev_end);
    if (m->stream) cudaStreamDestroy(m->stream);
    delete m;
    return JL_OK;
}

// page table entry of (session, layer page lp, context page cp)
static size_t page_index(const jl_model *m, int session, int lp, int cp) {
    return ((size_t)session * m->kv.n_layer_pages + lp) * m->kv.n_ctx_pages + cp;
}

extern "C" int jl_model_reset_session(jl_model *m, int session) {
    if (!m || !m->finalized || session < 0 || session >= m->cfg.max_sessions) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    // pages stay allocated (a KvBuffer keeps its pages until close); contents are dead once positions restart.
    // Zero them so a fresh session starts from the reference's zero-initialised page (TensorCache.java:105).
    // A shared page (jl_model_kv_fork) is detached instead: the entry is cleared and the other sessions keep the page.
    const size_t per = (size_t)m->kv.n_layer_pages * m->kv.n_ctx_pages, base = page_index(m, session, 0, 0);
    bool detached = false;
    for (size_t i = 0; i < per; i++) {
        void *p = m->page_table_host[base + i];
        if (p && drop_ref(m, p)) m->page_table_host[base + i] = nullptr, detached = true;
        else if (p) JL_CUDA_CHECK(ctx, cudaMemsetAsync(p, 0, m->page_bytes, m->stream));
    }
    if (detached)
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->page_table_dev + base, m->page_table_host.data() + base, per * sizeof(void *),
                                           cudaMemcpyHostToDevice, m->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    return JL_OK;
}

// page table entry idx = p on the host, and on the device through a copy queued on the model stream: the caller synchronises the
// stream before that host entry changes again
static int publish_page(jl_model *m, size_t idx, void *p) {
    m->page_table_host[idx] = p;
    JL_CUDA_CHECK(m->ctx, cudaMemcpyAsync(&m->page_table_dev[idx], &m->page_table_host[idx], sizeof(void *), cudaMemcpyHostToDevice,
                                          m->stream));
    return JL_OK;
}

// the page copies of `cp` on the model stream, copy_cap entries per launch, their table staged after the other areas of h_pinned; the
// caller synchronises before the staging is reused
static int run_page_copies(jl_model *m, const std::vector<KvCopy> &cp) {
    jl_ctx *ctx = m->ctx;
    KvCopy *staged = (KvCopy *)(m->h_pinned + 4 * (size_t)m->maxB + 4 * (size_t)m->pa_tab_cap + 2 * (size_t)m->cfg.max_sessions);
    const int row_bytes = (int)kv_row_bytes(m->kv.kv_dtype, m->kv.kv_len);
    for (size_t i = 0; i < cp.size(); i += (size_t)m->copy_cap) {
        if (i) JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
        const int n = (int)(cp.size() - i < (size_t)m->copy_cap ? cp.size() - i : (size_t)m->copy_cap);
        memcpy(staged, cp.data() + i, (size_t)n * sizeof(KvCopy));
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->d_copy_tab, staged, (size_t)n * sizeof(KvCopy), cudaMemcpyHostToDevice, m->stream));
        M_CHECK(jl_launch_kv_copy(ctx, m->stream, m->d_copy_tab, n, m->page_bytes, m->kv.ctx_per_page, row_bytes));
    }
    return JL_OK;
}

// a new page for entry idx, zeroed on the model stream like the reference's fresh page (TensorCache.java:105), and published
static int alloc_page(jl_model *m, size_t idx) {
    void *p = nullptr;
    M_CHECK(dev_alloc(m->ctx, &p, m->page_bytes));
    JL_CUDA_CHECK(m->ctx, cudaMemsetAsync(p, 0, m->page_bytes, m->stream));
    return publish_page(m, idx, p);
}

// make sure pages for positions [p0, p1] of `session` exist (KvBufferCache.java:307-318 lazy pages) and are its own: a shared page in the
// range is copied on write first, the copy holding the rows below p0 (the lowest position this call writes in it) and zeros above.
// Every new page is allocated before any entry changes, so running out of memory returns JL_ERR_OOM with the session as it was (the
// scheduler's prefix cache retries such a call after releasing retained pages, DESIGN §3.17).
static int ensure_pages(jl_model *m, int session, int p0, int p1) {
    jl_ctx *ctx = m->ctx;
    if (p1 >= m->max_context)
        return jl_set_error(ctx, JL_ERR_INVALID, "position %d exceeds reserved context %d", p1, m->max_context);
    const int cpp = m->kv.ctx_per_page;
    std::vector<size_t> todo; // entries that get a new page, in order
    for (int cp = p0 / cpp; cp <= p1 / cpp; cp++)
        for (int lp = 0; lp < m->kv.n_layer_pages; lp++) {
            const size_t idx = page_index(m, session, lp, cp);
            void *p = m->page_table_host[idx];
            if (!p || is_shared(m, p)) todo.push_back(idx);
        }
    if (todo.empty()) return JL_OK;
    std::vector<void *> fresh(todo.size(), nullptr);
    for (size_t i = 0; i < todo.size(); i++) {
        const int rc = dev_alloc(ctx, &fresh[i], m->page_bytes);
        if (rc != JL_OK) {
            for (size_t k = 0; k < i; k++) cudaFree(fresh[k]);
            return rc;
        }
    }
    std::vector<KvCopy> cow;
    for (size_t i = 0; i < todo.size(); i++) {
        const size_t idx = todo[i];
        void *p = m->page_table_host[idx], *q = fresh[i];
        if (!p) {
            JL_CUDA_CHECK(ctx, cudaMemsetAsync(q, 0, m->page_bytes, m->stream));
        } else {
            const int cp = (int)(idx % (size_t)m->kv.n_ctx_pages);
            cow.push_back(KvCopy{q, p, cp == p0 / cpp ? p0 - cp * cpp : 0, 0});
            drop_ref(m, p);
        }
        M_CHECK(publish_page(m, idx, q));
    }
    if (!cow.empty()) M_CHECK(run_page_copies(m, cow));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream)); // host staging of the pointer must outlive the copy
    return JL_OK;
}

// one quantised/dense GEMM call site; M f32 rows of `a` ([M, p.lda]) against W; splits M into GEMV_MAX_M chunks.
// `wide` (decode steps): more than GEMV_MAX_M rows go to the many-row GEMM in one weight pass where it covers the launch
// (Q4 / Q8_0 weights with Q8 activations, or with F32 activations for the lm_head); other combinations keep the chunks.
static int run_gemm(jl_model *m, GemvParams p, int prologue, int epilogue, int M, bool wide = false) {
    jl_ctx *ctx = m->ctx;
    if (wide && M > GEMV_MAX_M) {
        GemvParams c = p;
        c.M = M;
        c.wide_act = m->wide_act, c.wide_part = m->wide_part, c.wide_cnt = m->wide_cnt;
        if (jl_gemm64_supported(c, prologue, epilogue)) return jl_launch_gemv(ctx, m->stream, c, prologue, epilogue);
    }
    // rows per launch: as many as the staged activations allow (F32 activations at K = 14336 fit 2 rows, Q8 all 8)
    const int chunk = jl_gemv_max_m(p.w_dtype, prologue, p.K);
    if (chunk < 1) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemm: K=%d does not fit shared memory", p.K);
    for (int m0 = 0; m0 < M; m0 += chunk) {
        GemvParams c = p;
        c.M = M - m0 < chunk ? M - m0 : chunk;
        c.a = (const float *)p.a + (size_t)m0 * p.lda;
        for (int s = 0; s < c.nseg; s++) c.seg[s].out = p.seg[s].out + (size_t)m0 * p.seg[s].out_ld;
        if (c.residual) c.residual = p.residual + (size_t)m0 * p.res_ld;
        M_CHECK(jl_launch_gemv(ctx, m->stream, c, prologue, epilogue));
    }
    return JL_OK;
}

static void set_w(GemvParams &p, int seg, const DevTensor &t, float *out, int out_ld) {
    p.seg[seg].w = t.data;
    p.seg[seg].ws = t.scales;
    p.seg[seg].out = out;
    p.seg[seg].rows = (int)t.rows;
    p.seg[seg].out_ld = out_ld;
    p.seg[seg].out_off = 0;
}

// GEMM of weight w (segment 0; callers add the other segments of a fused launch) against f32 activation rows `a` of width K;
// total_rows = output rows of the launch.  Every other field stays value-initialised.
static GemvParams gemv_params(const DevTensor &w, float *out, int out_ld, const float *a, int K, int total_rows) {
    GemvParams p = {};
    p.nseg = 1;
    set_w(p, 0, w, out, out_ld);
    p.w_dtype = w.dtype;
    p.ldw = K, p.K = K;
    p.a = a, p.lda = K;
    p.total_rows = total_rows;
    return p;
}

// the RMSNorm prologue with norm weight w (norm_adj stays 0)
static void set_norm(GemvParams &p, const DevTensor &w, const jl_model *m) {
    p.norm_w = w.data, p.norm_w_dtype = w.dtype, p.norm_eps = m->cfg.layer_norm_eps, p.norm_E = m->cfg.embedding_length;
}

// attention of layer L over M rows whose sessions / positions are on the device, q / k / v -> att
static AttnParams attn_params(const jl_model *m, int L, int M, int splits) {
    AttnParams ap = {};
    ap.kv = m->kv, ap.layer = L, ap.heads = m->heads_local, ap.kv_heads = m->kv_heads_local, ap.head_size = m->cfg.head_size;
    ap.head0_global = m->d.headStart, ap.kv_head0_global = m->d.groupHeadStart;
    ap.q = m->q, ap.k = m->k, ap.v = m->v, ap.q_ld = m->attn_seg, ap.kv_ld = m->kv_seg, ap.out = m->att, ap.rope = m->rope;
    ap.rows = M, ap.sessions = m->d_sessions, ap.positions = m->d_positions;
    ap.scale = (float)(1.0 / sqrt((double)m->cfg.head_size)); // CausalSelfAttention.java:134
    ap.ws = m->attn_ws, ap.splits = splits;
    return ap;
}

// ---- KV append + RoPE, attention (CausalSelfAttention.java:199-356) of layer L for forward_rows / forward_rows_gpt2 ----
// decode (one row per session): one fused kernel, `splits` = about one per 64 positions.  The launch may be replayed from a graph
// for every context of its split bucket (run_decode), so the kernel is chosen by the largest position the bucket can see, not by
// the current one.
static int attention(jl_model *m, int L, int M, int splits, bool decode) {
    const AttnParams ap = attn_params(m, L, M, splits);
    if (decode) {
        const int bound = splits >= m->max_splits ? m->max_context - 1 : splits * 64 * M - 1;
        return jl_launch_fused_decode_attention(m->ctx, m->stream, ap, m->fda_done, bound);
    }
    M_CHECK(jl_launch_rope_kv_append(m->ctx, m->stream, ap, m->q));
    return jl_launch_paged_attention(m->ctx, m->stream, ap);
}

// AbstractModel.forward (:314-329) over M rows whose tokens/positions/sessions are already on the device.
static int forward_rows_gpt2(jl_model *m, int M, int splits, bool distinct_sessions);

static int forward_rows(jl_model *m, int M, int splits, bool distinct_sessions = false) {
    if (m->cfg.arch == JL_ARCH_GPT2) return forward_rows_gpt2(m, M, splits, distinct_sessions);
    jl_ctx *ctx = m->ctx;
    const jl_model_config &c = m->cfg;
    const int E = c.embedding_length;
    const bool q8 = c.working_qtype == JL_I8;
    M_CHECK(jl_launch_embed(ctx, m->stream, m->g[JL_T_EMBED], m->d_tokens, M, m->x, E));
    for (int L = 0; L < c.num_layers; L++) {
        const DevTensor *lw = &m->l[(size_t)L * 9];
        // Q8 activations only pair with Q4/I8 weights (AbstractModel.java:119-176)
        auto act_q = [&](const DevTensor &w) { return q8 && (w.dtype == JL_Q4 || w.dtype == JL_I8); };
        // ---- pre-norm + quantise + QKV (TransformerBlock.java:170-175, CausalSelfAttention.java:161-171) ----
        {
            GemvParams p = gemv_params(lw[JL_L_Q], m->q, m->attn_seg, m->x, E, m->attn_seg + 2 * m->kv_seg);
            p.nseg = 3;
            // k and v outputs are indexed by their own local row: out col = local
            set_w(p, 1, lw[JL_L_K], m->k, m->kv_seg);
            set_w(p, 2, lw[JL_L_V], m->v, m->kv_seg);
            set_norm(p, lw[JL_L_ATTN_NORM], m);
            M_CHECK(run_gemm(m, p, act_q(lw[JL_L_Q]) ? PRO_RMSNORM_QUANT : PRO_RMSNORM_F32, EPI_STORE, M, distinct_sessions));
        }
        M_CHECK(attention(m, L, M, splits, distinct_sessions));
        // ---- o_proj (+ reducer) + residual (CausalSelfAttention.java:363-378, TransformerBlock.java:185) ----
        {
            const bool tp = c.tp_size > 1;
            GemvParams p = gemv_params(lw[JL_L_O], tp ? m->partial : m->xb, E, m->att, m->attn_seg, E);
            p.residual = m->x;
            p.res_ld = E;
            M_CHECK(run_gemm(m, p, act_q(lw[JL_L_O]) ? PRO_F32_QUANT : PRO_F32, tp ? EPI_STORE : EPI_ADD_RESIDUAL, M, distinct_sessions));
            if (tp) {
                M_CHECK(jl_comm_allreduce_dev(ctx, m->stream, m->partial, (size_t)M * E));
                // xb = reduced + x
                JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->xb, m->partial, (size_t)M * E * 4, cudaMemcpyDeviceToDevice, m->stream));
                M_CHECK(jl_launch_accumulate(ctx, m->stream, m->xb, M, E, JL_F32, m->x, nullptr, M, E, 0, E));
            }
        }
        if (m->n_exp > 0) {
            // ---- mixture of experts (MoEBlock.java:73-149); the grouped path below, else one row at a time: router GEMV -> softmax + top-k on the device ->
            // per selected expert gate/up (SiLU*up fused) and down_proj through the expert pointer tables; the expert results
            // are summed UNWEIGHTED in selection order (:139-143), then the residual is added (TransformerBlock.java:203).
            // Row b of the result is the sum over row b's experts (the reference's copy of expert 0's result into row 0 for
            // every batch row, MoEBlock.java:141, is a bug we do not reproduce; with one row per call they coincide).
            // Expert parallel (tp_size > 1): every rank routes identically (replicated router), a selected expert held by another
            // rank has a null table entry and its launches only write zeros / pass the running sum through (gemv_absent); the
            // per-rank sums then meet in one all-reduce.  With two experts per token that sum is exact in any order.
            const int NE = m->n_exp, KE = m->exp_k, H = c.hidden_length;
            void **wt = m->moe_wtab + (size_t)L * 3 * NE;
            float **st = m->moe_stab + (size_t)L * 3 * NE;
            const size_t own = ((size_t)L * NE + c.tp_rank) * 3; // first expert held by this rank: shapes / dtype of every expert
            const bool aq = act_q(m->moe_w[own]);
            // grouped (M >= 2, Q8 activations, one rank): the router over all M rows, the rows grouped by expert on the device,
            // and each selected expert streamed once per launch for all of its rows (jl_launch_gemm64_grouped); a fixed number
            // of launches whatever M is, sized from the tile bound because the selections are only known on the device
            const int R = jl_gemm64_group_rows(M);
            GemvParams gu = gemv_params(m->moe_w[own], m->hbuf, H, m->xb, E, H), dn = gemv_params(m->moe_w[own + 1], m->moe_dout, E, m->hbuf, H, E);
            {
                gu.nseg = 2; // output rows: pair b * k + i of hbuf / moe_dout
                set_w(gu, 1, m->moe_w[own], m->hbuf, H);
                gu.w_tab[0] = (const void *const *)(wt + 0 * NE), gu.ws_tab[0] = (const float *const *)(st + 0 * NE); // w1
                gu.w_tab[1] = (const void *const *)(wt + 2 * NE), gu.ws_tab[1] = (const float *const *)(st + 2 * NE); // w3
                set_norm(gu, lw[JL_L_FFN_NORM], m);
                gu.M = M, gu.wide_act = m->moe_qa, gu.g_div = KE;
                dn.w_tab[0] = (const void *const *)(wt + 1 * NE), dn.ws_tab[0] = (const float *const *)(st + 1 * NE); // w2
                dn.M = M * KE, dn.wide_act = m->moe_qh, dn.g_div = 1;
                for (GemvParams *q : {&gu, &dn}) q->g_tiles = m->moe_grp.tiles, q->g_ntiles = m->moe_grp.ntiles, q->g_pairs = m->moe_grp.pairs;
            }
            if (M >= 2 && aq && c.tp_size == 1 && jl_gemm64_grouped_supported(gu, PRO_RMSNORM_QUANT, EPI_SILU_MUL, R) &&
                jl_gemm64_grouped_supported(dn, PRO_F32_QUANT, EPI_STORE, R)) {
                GemvParams p = gemv_params(m->moe_gate[L], m->moe_logits, NE, m->xb, E, NE);
                set_norm(p, lw[JL_L_FFN_NORM], m);
                M_CHECK(run_gemm(m, p, act_q(m->moe_gate[L]) ? PRO_RMSNORM_QUANT : PRO_RMSNORM_F32, EPI_STORE, M, distinct_sessions));
                M_CHECK(jl_launch_moe_route(ctx, m->stream, m->moe_logits, M, NE, KE, m->moe_sel));
                M_CHECK(jl_launch_moe_group(ctx, m->stream, m->moe_sel, M, NE, KE, R, m->moe_grp));
                const int tiles = jl_moe_tile_bound(M * KE, NE, R);
                M_CHECK(jl_launch_gemm64_grouped(ctx, m->stream, gu, PRO_RMSNORM_QUANT, EPI_SILU_MUL, R, tiles));
                M_CHECK(jl_launch_gemm64_grouped(ctx, m->stream, dn, PRO_F32_QUANT, EPI_STORE, R, tiles));
                M_CHECK(jl_launch_moe_combine(ctx, m->stream, m->moe_dout, M, KE, E, m->xb, m->x));
                continue;
            }
            for (int b = 0; b < M; b++) {
                {
                    GemvParams p = gemv_params(m->moe_gate[L], m->moe_logits + (size_t)b * NE, NE, m->xb + (size_t)b * E, E, NE);
                    set_norm(p, lw[JL_L_FFN_NORM], m);
                    M_CHECK(run_gemm(m, p, act_q(m->moe_gate[L]) ? PRO_RMSNORM_QUANT : PRO_RMSNORM_F32, EPI_STORE, 1));
                }
                M_CHECK(jl_launch_moe_route(ctx, m->stream, m->moe_logits + (size_t)b * NE, 1, NE, KE, m->moe_sel + (size_t)b * KE));
                for (int i = 0; i < KE; i++) {
                    const DevTensor &proto = m->moe_w[own];
                    float *h = m->hbuf + ((size_t)b * KE + i) * H; // row b's expert i
                    GemvParams p = gemv_params(proto, h, H, m->xb + (size_t)b * E, E, H);
                    p.nseg = 2;
                    set_w(p, 1, proto, h, H);
                    p.sel = m->moe_sel + (size_t)b * KE + i;
                    p.w_tab[0] = (const void *const *)(wt + 0 * NE), p.ws_tab[0] = (const float *const *)(st + 0 * NE); // w1
                    p.w_tab[1] = (const void *const *)(wt + 2 * NE), p.ws_tab[1] = (const float *const *)(st + 2 * NE); // w3
                    set_norm(p, lw[JL_L_FFN_NORM], m);
                    M_CHECK(run_gemm(m, p, aq ? PRO_RMSNORM_QUANT : PRO_RMSNORM_F32, EPI_SILU_MUL, 1));
                    GemvParams d = gemv_params(m->moe_w[own + 1], m->x + (size_t)b * E, E, h, H, E);
                    d.sel = p.sel;
                    d.w_tab[0] = (const void *const *)(wt + 1 * NE), d.ws_tab[0] = (const float *const *)(st + 1 * NE); // w2
                    d.residual = m->x + (size_t)b * E, d.res_ld = E; // expert i > 0 accumulates onto the sum so far
                    M_CHECK(run_gemm(m, d, aq ? PRO_F32_QUANT : PRO_F32, i == 0 ? EPI_STORE : EPI_ADD_RESIDUAL, 1));
                }
            }
            if (c.tp_size > 1) M_CHECK(jl_comm_allreduce_dev(ctx, m->stream, m->x, (size_t)M * E));
            M_CHECK(jl_launch_accumulate(ctx, m->stream, m->x, M, E, JL_F32, m->xb, nullptr, M, E, 0, E)); // + residual
            continue;
        }
        // ---- pre-FF norm + quantise + gate/up + SiLU*up (TransformerBlock.java:187-196, MLPBlock.java:117-141) ----
        {
            GemvParams p = gemv_params(lw[JL_L_GATE], m->hbuf, m->h_seg, m->xb, E, m->h_seg);
            p.nseg = 2;
            set_w(p, 1, lw[JL_L_UP], m->hbuf, m->h_seg);
            set_norm(p, lw[JL_L_FFN_NORM], m);
            M_CHECK(run_gemm(m, p, act_q(lw[JL_L_GATE]) ? PRO_RMSNORM_QUANT : PRO_RMSNORM_F32, EPI_SILU_MUL, M, distinct_sessions));
        }
        // ---- down_proj (+ reducer) + residual (MLPBlock.java:144-160, TransformerBlock.java:203) ----
        {
            const bool tp = c.tp_size > 1;
            GemvParams p = gemv_params(lw[JL_L_DOWN], tp ? m->partial : m->x, E, m->hbuf, m->h_seg, E);
            p.residual = m->xb;
            p.res_ld = E;
            M_CHECK(run_gemm(m, p, act_q(lw[JL_L_DOWN]) ? PRO_F32_QUANT : PRO_F32, tp ? EPI_STORE : EPI_ADD_RESIDUAL, M, distinct_sessions));
            if (tp) {
                M_CHECK(jl_comm_allreduce_dev(ctx, m->stream, m->partial, (size_t)M * E));
                JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->x, m->partial, (size_t)M * E * 4, cudaMemcpyDeviceToDevice, m->stream));
                M_CHECK(jl_launch_accumulate(ctx, m->stream, m->x, M, E, JL_F32, m->xb, nullptr, M, E, 0, E));
            }
        }
    }
    return JL_OK;
}

// staging areas of h_pinned: the tokens a step returns, then those after the four [maxB] arrays
static int32_t *pinned_next(jl_model *m) { return m->h_pinned + 3 * (size_t)m->maxB; }
static int4 *pinned_pa_tab(jl_model *m) { return (int4 *)(m->h_pinned + 4 * (size_t)m->maxB); }
static int32_t *pinned_rows(jl_model *m) { return m->h_pinned + 4 * (size_t)m->maxB + 4 * (size_t)m->pa_tab_cap; }

// (token, position, session) of rows [0, n) of the next pass -> pinned staging -> d_tokens / d_positions / d_sessions
static int stage_rows(jl_model *m, int n, const int32_t *tokens, const int32_t *positions, const int32_t *sessions) {
    jl_ctx *ctx = m->ctx;
    int32_t *hp = m->h_pinned;
    const size_t B = m->maxB, bytes = (size_t)n * 4;
    memcpy(hp, tokens, bytes);
    memcpy(hp + B, positions, bytes);
    memcpy(hp + 2 * B, sessions, bytes);
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->d_tokens, hp, bytes, cudaMemcpyHostToDevice, m->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->d_positions, hp + B, bytes, cudaMemcpyHostToDevice, m->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->d_sessions, hp + 2 * B, bytes, cudaMemcpyHostToDevice, m->stream));
    return JL_OK;
}

// Prefill chunks on the tensor cores: the same op sequence as forward_rows with every weight GEMM on wgmma
// (BF16 operands, F32 accumulate; jl_gemm_tc.cu).  Norms, RoPE, attention, SiLU stay f32.
// segs[i] = {session, pos0, first row, rows} (HOST): the M rows are nseg runs of consecutive positions, one per session.  Every op but
// the attention works row by row; one segment takes the single-session tiled attention, several take its block-table variant.
static int forward_rows_tc(jl_model *m, int M, int splits, const int4 *segs, int nseg) {
    jl_ctx *ctx = m->ctx;
    const jl_model_config &c = m->cfg;
    const int E = c.embedding_length, H = m->h_seg;
    int ntab = 0;
    M_CHECK(jl_launch_embed(ctx, m->stream, m->g[JL_T_EMBED], m->d_tokens, M, m->x, E));
    for (int L = 0; L < c.num_layers; L++) {
        const DevTensor *lw = &m->l[(size_t)L * 9];
        M_CHECK(jl_launch_rmsnorm_bf16(ctx, m->stream, m->x, M, E, lw[JL_L_ATTN_NORM].dtype, lw[JL_L_ATTN_NORM].data, 0.0f, c.layer_norm_eps, E,
                                       m->abf, E));
        M_CHECK(jl_launch_gemm_tc(ctx, m->stream, m->abf, E, M, lw[JL_L_Q], m->attn_seg, 0, E, m->q, m->attn_seg, 0, nullptr, 0));
        M_CHECK(jl_launch_gemm_tc(ctx, m->stream, m->abf, E, M, lw[JL_L_K], m->kv_seg, 0, E, m->k, m->kv_seg, 0, nullptr, 0));
        M_CHECK(jl_launch_gemm_tc(ctx, m->stream, m->abf, E, M, lw[JL_L_V], m->kv_seg, 0, E, m->v, m->kv_seg, 0, nullptr, 0));
        const AttnParams ap = attn_params(m, L, M, splits);
        M_CHECK(jl_launch_rope_kv_append(ctx, m->stream, ap, m->q));
        // rows = consecutive positions pos0.. of one session per segment: tiled tensor-core attention (jl_attn_prefill.cu)
        if (!jl_prefill_attention_supported(ap)) {
            M_CHECK(jl_launch_paged_attention(ctx, m->stream, ap));
        } else if (nseg == 1) {
            M_CHECK(jl_launch_prefill_attention(ctx, m->stream, ap, segs[0].x, segs[0].y));
        } else {
            if (L == 0) { // the block table depends on the pass only; the caller synchronises before the staging is reused
                ntab = jl_prefill_attention_table(ctx, ap, segs, nseg, pinned_pa_tab(m));
                JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->d_pa_tab, pinned_pa_tab(m), (size_t)ntab * sizeof(int4), cudaMemcpyHostToDevice, m->stream));
            }
            M_CHECK(jl_launch_prefill_attention_table(ctx, m->stream, ap, m->d_pa_tab, ntab));
        }
        M_CHECK(jl_launch_quantize_bf16(ctx, m->stream, m->att, M, m->attn_seg, 0, m->attn_seg, m->abf));
        M_CHECK(jl_launch_gemm_tc(ctx, m->stream, m->abf, m->attn_seg, M, lw[JL_L_O], E, 0, m->attn_seg, m->xb, E, 0, m->x, E));
        M_CHECK(jl_launch_rmsnorm_bf16(ctx, m->stream, m->xb, M, E, lw[JL_L_FFN_NORM].dtype, lw[JL_L_FFN_NORM].data, 0.0f, c.layer_norm_eps, E,
                                       m->abf, E));
        M_CHECK(jl_launch_gemm_tc(ctx, m->stream, m->abf, E, M, lw[JL_L_GATE], H, 0, E, m->hbuf, H, 0, nullptr, 0));
        M_CHECK(jl_launch_gemm_tc(ctx, m->stream, m->abf, E, M, lw[JL_L_UP], H, 0, E, m->hbuf2, H, 0, nullptr, 0));
        M_CHECK(jl_launch_silu_mul_bf16(ctx, m->stream, m->hbuf, m->hbuf2, M, H, H, m->abf, H));
        M_CHECK(jl_launch_gemm_tc(ctx, m->stream, m->abf, H, M, lw[JL_L_DOWN], E, 0, H, m->x, E, 0, m->xb, E));
    }
    return JL_OK;
}

// GPT-2 blocks (core/model/gpt2/GPT2Model.java:54-129) on the same per-op kernels: x = wte[token] + wpe[position]; per layer
//   ln1 = LayerNorm(x) -> q,k,v = ln1 . W^T + bias -> attention (no rotary: identity table) -> xb = (att . Wo^T + bo) + x
//   ln2 = LayerNorm(xb) -> h = gelu(ln2 . Wfc^T + bfc) -> x = (h . Wproj^T + bproj) + xb
// in the order TransformerBlock.forward / CausalSelfAttention.forward / MLPBlock.forward apply them (bias after the reducer,
// residual last: CausalSelfAttention.java:363-380, MLPBlock.java:126-160, TransformerBlock.java:185,203).
static int forward_rows_gpt2(jl_model *m, int M, int splits, bool distinct_sessions) {
    jl_ctx *ctx = m->ctx;
    const jl_model_config &c = m->cfg;
    const int E = c.embedding_length, H = m->h_seg;
    const bool q8 = c.working_qtype == JL_I8;
    auto act_q = [&](const DevTensor &w) { return q8 && (w.dtype == JL_Q4 || w.dtype == JL_I8); };
    auto bias = [&](float *a, int lda, const DevTensor &b, int n) {
        return jl_launch_accumulate(ctx, m->stream, a, M, lda, b.dtype, b.data, nullptr, 1, (int)b.cols, 0, n);
    };
    // a projection without a norm prologue (the LayerNorms have their own launches)
    auto gemm = [&](const GemvParams &p, const DevTensor &w) {
        return run_gemm(m, p, act_q(w) ? PRO_F32_QUANT : PRO_F32, EPI_STORE, M, distinct_sessions);
    };
    M_CHECK(jl_launch_embed(ctx, m->stream, m->g[JL_T_EMBED], m->d_tokens, M, m->x, E));
    M_CHECK(jl_launch_pos_embed_add(ctx, m->stream, m->x, M, E, m->gaux[JL_AUX_POS_EMBED], m->d_positions));
    for (int L = 0; L < c.num_layers; L++) {
        const DevTensor *lw = &m->l[(size_t)L * 9];
        const DevTensor *ax = &m->aux[(size_t)L * 8];
        M_CHECK(jl_launch_layernorm(ctx, m->stream, m->x, M, E, lw[JL_L_ATTN_NORM].dtype, lw[JL_L_ATTN_NORM].data, ax[JL_AUX_ATTN_NORM_BIAS].dtype,
                                    ax[JL_AUX_ATTN_NORM_BIAS].data, c.layer_norm_eps, E, 0, E, m->ln));
        {
            GemvParams p = gemv_params(lw[JL_L_Q], m->q, m->attn_seg, m->ln, E, m->attn_seg + 2 * m->kv_seg);
            p.nseg = 3;
            set_w(p, 1, lw[JL_L_K], m->k, m->kv_seg);
            set_w(p, 2, lw[JL_L_V], m->v, m->kv_seg);
            M_CHECK(gemm(p, lw[JL_L_Q]));
        }
        M_CHECK(bias(m->q, m->attn_seg, ax[JL_AUX_Q_BIAS], m->attn_seg));
        M_CHECK(bias(m->k, m->kv_seg, ax[JL_AUX_K_BIAS], m->kv_seg));
        M_CHECK(bias(m->v, m->kv_seg, ax[JL_AUX_V_BIAS], m->kv_seg));
        M_CHECK(attention(m, L, M, splits, distinct_sessions));
        M_CHECK(gemm(gemv_params(lw[JL_L_O], m->xb, E, m->att, m->attn_seg, E), lw[JL_L_O]));
        M_CHECK(bias(m->xb, E, ax[JL_AUX_O_BIAS], E));
        M_CHECK(jl_launch_accumulate(ctx, m->stream, m->xb, M, E, JL_F32, m->x, nullptr, M, E, 0, E)); // + residual
        M_CHECK(jl_launch_layernorm(ctx, m->stream, m->xb, M, E, lw[JL_L_FFN_NORM].dtype, lw[JL_L_FFN_NORM].data, ax[JL_AUX_FFN_NORM_BIAS].dtype,
                                    ax[JL_AUX_FFN_NORM_BIAS].data, c.layer_norm_eps, E, 0, E, m->ln));
        M_CHECK(gemm(gemv_params(lw[JL_L_GATE], m->hbuf, H, m->ln, E, H), lw[JL_L_GATE]));
        M_CHECK(bias(m->hbuf, H, ax[JL_AUX_FC_BIAS], H));
        M_CHECK(jl_launch_activation(ctx, m->stream, JL_ACT_GELU, m->hbuf, M, H, 0, H));
        M_CHECK(gemm(gemv_params(lw[JL_L_DOWN], m->x, E, m->hbuf, H, E), lw[JL_L_DOWN]));
        M_CHECK(bias(m->x, E, ax[JL_AUX_PROJ_BIAS], E));
        M_CHECK(jl_launch_accumulate(ctx, m->stream, m->x, M, E, JL_F32, m->xb, nullptr, M, E, 0, E)); // + residual
    }
    return JL_OK;
}

// AbstractModel.sample (:443-473) up to the logits: `n` hidden rows [n, E] -> final norm -> lm_head -> logits [n, vocab].  More than
// GEMV_MAX_M rows take one weight pass where run_gemm's wide mode can (Q4 / Q8_0 lm_head).
static int lm_head_rows(jl_model *m, const float *hidden, int n, float *logits) {
    jl_ctx *ctx = m->ctx;
    const jl_model_config &c = m->cfg;
    const int E = c.embedding_length, V = c.vocab_size;
    const DevTensor &w = m->g_set[JL_T_LM_HEAD] ? m->g[JL_T_LM_HEAD] : m->g[JL_T_EMBED];
    GemvParams p = gemv_params(w, logits, V, hidden, E, V);
    // lm_head uses un-quantised F32 activations (AbstractModel.java:444-449)
    int prologue = PRO_RMSNORM_F32;
    if (c.arch == JL_ARCH_GPT2) { // ln_f is a LayerNorm with bias (GPT2Model.java:112-128), the logits weights are wte
        M_CHECK(jl_launch_layernorm(ctx, m->stream, hidden, n, E, m->g[JL_T_OUT_NORM].dtype, m->g[JL_T_OUT_NORM].data, m->gaux[JL_AUX_OUT_NORM_BIAS].dtype,
                                    m->gaux[JL_AUX_OUT_NORM_BIAS].data, c.layer_norm_eps, E, 0, E, m->ln));
        p.a = m->ln;
        prologue = PRO_F32;
    } else {
        set_norm(p, m->g[JL_T_OUT_NORM], m);
    }
    return run_gemm(m, p, prologue, EPI_STORE, n, true);
}

// AbstractModel.sample (:443-473) for `n` hidden rows -> m->logits -> argmax tokens in m->d_next
static int sample_rows(jl_model *m, const float *hidden, int n) {
    M_CHECK(lm_head_rows(m, hidden, n, m->logits));
    return jl_launch_argmax(m->ctx, m->stream, m->logits, n, m->cfg.vocab_size, m->cfg.vocab_size, m->d_next, m->argmax_scratch);
}

static int pick_splits(const jl_model *m, int max_pos, int rows) {
    // enough CTAs to cover the SMs, at most one split per 128 positions
    int want = (max_pos + 1 + 127) / 128;
    int fill = (m->ctx->sm_count * 2) / (m->kv_heads_local * rows > 0 ? m->kv_heads_local * rows : 1);
    if (fill < 1) fill = 1;
    int s = want < fill ? want : fill;
    if (s > m->max_splits) s = m->max_splits;
    if (s < 1) s = 1;
    // bucket to powers of two so few graphs are needed
    int b = 1;
    while (b < s) b <<= 1;
    return b > m->max_splits ? m->max_splits : b;
}

// row i of dst (dst_rows ? dst_rows[i] : i) = row of src (src_rows ? src_rows[i] : i); rows of E floats, one CTA per row
__global__ void __launch_bounds__(256) copy_rows_kernel(float *dst, const int32_t *dst_rows, const float *src, const int32_t *src_rows, int E) {
    const int i = blockIdx.x;
    float *d = dst + (size_t)(dst_rows ? dst_rows[i] : i) * E;
    const float *a = src + (size_t)(src_rows ? src_rows[i] : i) * E;
    for (int k = threadIdx.x; k < E; k += blockDim.x) d[k] = a[k];
}

static int copy_rows(jl_model *m, float *dst, const int32_t *dst_rows, const float *src, const int32_t *src_rows, int n) {
    jl_ctx *ctx = m->ctx;
    JL_CUDA_CHECK(ctx, jl_launch_kernel(copy_rows_kernel, dim3(n), dim3(256), 0, m->stream, dst, dst_rows, src, src_rows,
                                        m->cfg.embedding_length));
    ctx->launches++;
    return JL_OK;
}

namespace {
struct PrefillChunk { // rows consecutive prompt positions pos.. of one session: a max_batch-row chunk of a segment or its remainder
    int session, pos, rows;
    const int32_t *tokens;
    bool last; // the segment's last chunk
    int entry; // scoring: the output entry of the chunk's first token
};

// prompt scoring outputs of a jl_model_score_multi call (entries laid out like its tokens)
struct ScoreOut {
    int top_n;
    float *lp;
    int32_t *ids;
    float *tlp;
};
} // namespace

// the scoring buffers (first jl_model_score_multi): 64-row lm_head groups whatever max_sessions is, so the logits buffer and the
// many-row GEMM workspaces are added when the model's own are smaller
static int score_alloc(jl_model *m) {
    jl_ctx *ctx = m->ctx;
    const jl_model_config &c = m->cfg;
    if (c.max_sessions < JL_MAX_DECODE_ROWS && !m->score_logits) M_CHECK(dev_alloc(ctx, (void **)&m->score_logits, (size_t)JL_MAX_DECODE_ROWS * c.vocab_size * 4));
    if (!m->wide_act) {
        const int E = c.embedding_length;
        M_CHECK(dev_alloc(ctx, &m->wide_act, jl_gemm64_act_bytes(E)));
        M_CHECK(dev_alloc(ctx, (void **)&m->wide_part, jl_gemm64_part_floats(ctx->sm_count) * 4));
        M_CHECK(dev_alloc(ctx, (void **)&m->wide_cnt, (size_t)ctx->sm_count * sizeof(unsigned)));
        JL_CUDA_CHECK(ctx, cudaMemset(m->wide_cnt, 0, (size_t)ctx->sm_count * sizeof(unsigned)));
    }
    return lp_alloc(m, m->lp_score, m->maxB, JL_MAX_DECODE_ROWS, true);
}

// Scoring of one forwarded pass: every row with a target (the next token of its segment: all rows but a segment's last) is gathered
// into xb, 64 rows per group, and goes through the final norm + lm_head + one logprob launch per group.  The outputs land in the
// pinned staging; the caller synchronises and scatters them (score_scatter).
static int score_pass(jl_model *m, const std::vector<PrefillChunk> &ch, int top_n) {
    jl_ctx *ctx = m->ctx;
    jl_model::LpBufs &b = m->lp_score;
    const int V = m->cfg.vocab_size;
    float *logits = m->score_logits ? m->score_logits : m->logits;
    int k = 0, r0 = 0;
    for (const PrefillChunk &c : ch) {
        for (int j = 0; j < c.rows - (c.last ? 1 : 0); j++, k++)
            b.h_idx[k] = r0 + j, b.h_idx[b.cap + k] = c.tokens[j + 1], b.h_rows[k] = LogprobRow{k % JL_MAX_DECODE_ROWS, top_n};
        r0 += c.rows;
    }
    if (k == 0) return JL_OK;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(b.d_idx, b.h_idx, (size_t)k * 4, cudaMemcpyHostToDevice, m->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(b.d_idx + b.cap, b.h_idx + b.cap, (size_t)k * 4, cudaMemcpyHostToDevice, m->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(b.d_rows, b.h_rows, (size_t)k * sizeof(LogprobRow), cudaMemcpyHostToDevice, m->stream));
    for (int g = 0; g < k; g += JL_MAX_DECODE_ROWS) {
        const int n = k - g < JL_MAX_DECODE_ROWS ? k - g : JL_MAX_DECODE_ROWS;
        M_CHECK(copy_rows(m, m->xb, nullptr, m->x, b.d_idx + g, n));
        M_CHECK(lm_head_rows(m, m->xb, n, logits));
        M_CHECK(jl_launch_logprobs(ctx, m->stream, logits, V, V, b.d_rows + g, n, b.d_idx + b.cap + g, b.ws, b.cnt, b.d_out + g));
    }
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(b.h_out, b.d_out, (size_t)k * sizeof(LogprobOut), cudaMemcpyDeviceToHost, m->stream));
    return JL_OK;
}

// after the pass's synchronise: the staged outputs of score_pass -> the caller's entries (row j of a chunk scores its token j + 1)
static void score_scatter(jl_model *m, const std::vector<PrefillChunk> &ch, const ScoreOut &so) {
    const LogprobOut *o = m->lp_score.h_out;
    for (const PrefillChunk &c : ch)
        for (int j = 0; j < c.rows - (c.last ? 1 : 0); j++, o++) {
            const size_t e = (size_t)c.entry + j + 1;
            jl_logprobs_unpack(o, &so.top_n, 1, so.lp + e, so.ids ? so.ids + e * JL_MAX_LOGPROBS : nullptr,
                               so.tlp ? so.tlp + e * JL_MAX_LOGPROBS : nullptr);
        }
}

// One forward pass over chunks of distinct sessions, their rows back to back (at most maxB), [scoring: the logprobs of its rows,]
// then the last row of every chunk -> last_hidden[session] in one launch.
static int forward_chunks(jl_model *m, const std::vector<PrefillChunk> &ch, bool tc, const ScoreOut *so) {
    jl_ctx *ctx = m->ctx;
    const int n = (int)ch.size(), S = m->cfg.max_sessions;
    int32_t *rows = pinned_rows(m);
    std::vector<int4> segs((size_t)n);
    std::vector<int32_t> tokens, positions, sessions;
    int M = 0, max_pos = 0;
    for (int i = 0; i < n; i++) {
        const PrefillChunk &c = ch[(size_t)i];
        tokens.insert(tokens.end(), c.tokens, c.tokens + c.rows);
        for (int j = 0; j < c.rows; j++) positions.push_back(c.pos + j), sessions.push_back(c.session);
        segs[(size_t)i] = make_int4(c.session, c.pos, M, c.rows);
        M += c.rows;
        rows[i] = M - 1, rows[S + i] = c.session;
        if (c.pos + c.rows - 1 > max_pos) max_pos = c.pos + c.rows - 1;
    }
    M_CHECK(stage_rows(m, M, tokens.data(), positions.data(), sessions.data()));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->d_rows, rows, (size_t)(S + n) * 4, cudaMemcpyHostToDevice, m->stream));
    const int splits = pick_splits(m, max_pos, M);
    if (tc) M_CHECK(forward_rows_tc(m, M, splits, segs.data(), n));
    else M_CHECK(forward_rows(m, M, splits));
    if (so) M_CHECK(score_pass(m, ch, so->top_n));
    M_CHECK(copy_rows(m, m->last_hidden, m->d_rows + S, m->x, m->d_rows, n));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream)); // pinned staging is reused by the next pass
    if (so) score_scatter(m, ch, *so);
    return JL_OK;
}

// chunks of one path, packed greedily in order into passes of at most maxB rows
static int forward_packed(jl_model *m, const std::vector<PrefillChunk> &ch, bool tc, const ScoreOut *so) {
    std::vector<PrefillChunk> pass;
    int rows = 0;
    for (const PrefillChunk &c : ch) {
        if (rows + c.rows > m->maxB) {
            M_CHECK(forward_chunks(m, pass, tc, so));
            pass.clear(), rows = 0;
        }
        pass.push_back(c), rows += c.rows;
    }
    return pass.empty() ? JL_OK : forward_chunks(m, pass, tc, so);
}

// Segment i is cut into max_batch-row chunks (AbstractModel.java:304), and each chunk takes the tensor cores when tc_ok and it has
// >= 16 rows, else the exact path.  Round r forwards the r-th chunk of every segment, so a chunk sees the KV of its session's earlier
// chunks; within a round the chunks of each path share passes of up to maxB rows.  A lone segment (jl_model_batch_forward) thus gets
// one pass per chunk, and the single-session attention kernel.
// `so` (scoring, nullable): the logprobs of every forwarded token, see jl_model_score_multi.
static int forward_multi(jl_model *m, const char *who, int n_seg, const int32_t *sessions, const int32_t *start_pos, const int32_t *lengths,
                         const int32_t *tokens, const ScoreOut *so) {
    if (!m || !m->finalized) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    const jl_model_config &c = m->cfg;
    if (!sessions || !start_pos || !lengths || !tokens) return jl_set_error(ctx, JL_ERR_INVALID, "%s: null argument", who);
    if (n_seg < 1 || n_seg > c.max_sessions)
        return jl_set_error(ctx, JL_ERR_INVALID, "%s: %d segments (1..%d)", who, n_seg, c.max_sessions);
    std::vector<char> seen((size_t)c.max_sessions, 0);
    for (int i = 0; i < n_seg; i++) {
        if (sessions[i] < 0 || sessions[i] >= c.max_sessions)
            return jl_set_error(ctx, JL_ERR_INVALID, "%s: segment %d: session %d out of range", who, i, sessions[i]);
        if (seen[(size_t)sessions[i]]) return jl_set_error(ctx, JL_ERR_INVALID, "%s: session %d appears twice", who, sessions[i]);
        seen[(size_t)sessions[i]] = 1;
        if (lengths[i] < 1 || start_pos[i] < 0)
            return jl_set_error(ctx, JL_ERR_INVALID, "%s: segment %d: length %d at position %d", who, i, lengths[i], start_pos[i]);
        if ((int64_t)start_pos[i] + lengths[i] > m->max_context)
            return jl_set_error(ctx, JL_ERR_INVALID, "%s: segment %d ends past the reserved context %d", who, i, m->max_context);
    }
    if (so) {
        if (c.tp_size > 1) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "%s: logprobs under tensor parallelism", who);
        if (!so->lp) return jl_set_error(ctx, JL_ERR_INVALID, "%s: null lp_out", who);
        if (so->top_n < 0 || so->top_n > JL_MAX_LOGPROBS) return jl_set_error(ctx, JL_ERR_INVALID, "%s: top_n %d (0..%d)", who, so->top_n, JL_MAX_LOGPROBS);
        M_CHECK(jl_logprobs_check(ctx, who, 1, c.vocab_size, &so->top_n, nullptr));
    }
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    if (so && !m->lp_score.cap) M_CHECK(score_alloc(m));
    std::vector<size_t> off((size_t)n_seg);
    for (int i = 0; i < n_seg; i++) {
        M_CHECK(ensure_pages(m, sessions[i], start_pos[i], start_pos[i] + lengths[i] - 1));
        off[(size_t)i] = i ? off[(size_t)i - 1] + (size_t)lengths[i - 1] : 0;
    }
    for (int r0 = 0;; r0 += c.max_batch) {
        std::vector<PrefillChunk> tc, ex;
        for (int i = 0; i < n_seg; i++) {
            if (lengths[i] <= r0) continue;
            const int cnt = lengths[i] - r0 < c.max_batch ? lengths[i] - r0 : c.max_batch;
            (m->tc_ok && cnt >= 16 ? tc : ex).push_back(PrefillChunk{sessions[i], start_pos[i] + r0, cnt, tokens + off[(size_t)i] + r0,
                                                                        r0 + cnt == lengths[i], (int)off[(size_t)i] + r0});
        }
        if (tc.empty() && ex.empty()) break;
        M_CHECK(forward_packed(m, tc, true, so));
        M_CHECK(forward_packed(m, ex, false, so));
    }
    return JL_OK;
}

extern "C" int jl_model_batch_forward_multi(jl_model *m, int n_seg, const int32_t *sessions, const int32_t *start_pos, const int32_t *lengths,
                                            const int32_t *tokens) {
    return forward_multi(m, "batch_forward_multi", n_seg, sessions, start_pos, lengths, tokens, nullptr);
}

extern "C" int jl_model_batch_forward(jl_model *m, int session, const int32_t *tokens, int n, int start_pos) {
    return jl_model_batch_forward_multi(m, 1, &session, &start_pos, &n, tokens);
}

// Prompt scoring: forward_multi with the logprob of every token after a segment's first.  Entry 0 of a segment has no row before it in
// this call (last_hidden follows prompt forwards only, so it need not hold the row before a continuing segment): NaN, id -1.
extern "C" int jl_model_score_multi(jl_model *m, int n_seg, const int32_t *sessions, const int32_t *start_pos, const int32_t *lengths,
                                    const int32_t *tokens, int top_n, float *lp_out, int32_t *top_ids_out, float *top_lp_out) {
    const ScoreOut so{top_n, lp_out, top_ids_out, top_lp_out};
    M_CHECK(forward_multi(m, "score_multi", n_seg, sessions, start_pos, lengths, tokens, &so));
    const int32_t none = -1;
    for (int i = 0, e = 0; i < n_seg; e += lengths[i++])
        jl_logprobs_unpack(nullptr, &none, 1, lp_out + e, top_ids_out ? top_ids_out + (size_t)e * JL_MAX_LOGPROBS : nullptr,
                           top_lp_out ? top_lp_out + (size_t)e * JL_MAX_LOGPROBS : nullptr);
    return JL_OK;
}

extern "C" int jl_model_score(jl_model *m, int session, const int32_t *tokens, int n, int start_pos, int top_n, float *lp_out,
                              int32_t *top_ids_out, float *top_lp_out) {
    return jl_model_score_multi(m, 1, &session, &start_pos, &n, tokens, top_n, lp_out, top_ids_out, top_lp_out);
}

// exp((l-max)/T) then the first index whose running sum reaches `uniform` (AbstractModel.java:475-489).
// Sequential prefix order is part of the semantics, so one thread walks the normalised values.
// The exponentials go to `ex`: the logits row itself for the reference's in-place behaviour, or a scratch row when the raw logits must
// survive the draw (the logprob calls).
__global__ void __launch_bounds__(256) softmax_sample_kernel(const float *logits, float *ex, int vocab, float temperature, float uniform,
                                                             int32_t *out) {
    __shared__ float red[32];
    __shared__ float bc;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    float mx = -INFINITY;
    for (int i = tid; i < vocab; i += blockDim.x) mx = fmaxf(mx, logits[i]);
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    if (tid == 0) {
        float t = red[0];
        for (int i = 1; i < nw; i++) t = fmaxf(t, red[i]);
        bc = t;
    }
    __syncthreads();
    mx = bc;
    float sum = 0.0f;
    for (int i = tid; i < vocab; i += blockDim.x) {
        const float e = (float)exp(((double)logits[i] - (double)mx) / (double)temperature);
        ex[i] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    __syncthreads();
    if (lane == 0) red[warp] = sum;
    __syncthreads();
    if (tid == 0) {
        float t = 0.0f;
        for (int i = 0; i < nw; i++) t += red[i];
        float acc = 0.0f;
        int pick = vocab - 1;
        for (int i = 0; i < vocab; i++) {
            acc += ex[i] / t;
            if (acc >= uniform) {
                pick = i;
                break;
            }
        }
        *out = pick;
    }
}

// device-side bookkeeping at the end of a resident decode step: feed the sampled token back, advance
// the position, append to the history ring.
__global__ void advance_kernel(int32_t *tokens, int32_t *positions, const int32_t *next, int32_t *hist, int32_t *counter,
                               int n, int cap) {
    const int i = threadIdx.x;
    const int cnt = *counter;
    if (i < n) {
        tokens[i] = next[i];
        positions[i] += 1;
        if (cnt * n + i < cap) hist[cnt * n + i] = next[i];
    }
    __syncthreads();
    if (i == 0) *counter = cnt + 1;
}

static int decode_body(jl_model *m, int n, int splits, bool resident) {
    jl_ctx *ctx = m->ctx;
    M_CHECK(forward_rows(m, n, splits, true));
    M_CHECK(sample_rows(m, m->x, n));
    if (resident) {
        JL_CUDA_CHECK(ctx, jl_launch_kernel(advance_kernel, dim3(1), dim3(256), 0, m->stream, m->d_tokens, m->d_positions,
                                            (const int32_t *)m->d_next, m->d_hist, m->d_counter, n, m->hist_cap));
        ctx->launches++;
    }
    return JL_OK;
}

static void fill_pd(jl_model *m, int max_pos, bool resident, bool want_logits, PdParams &p) {
    const jl_model_config &c = m->cfg;
    p = PdParams();
    p.layers = c.num_layers, p.E = c.embedding_length, p.H = m->h_seg, p.attn_seg = m->attn_seg, p.kv_seg = m->kv_seg;
    p.heads = m->heads_local, p.kv_heads = m->kv_heads_local, p.head_size = c.head_size;
    p.vocab = c.vocab_size, p.vocab_rows = m->pd_vocab_rows, p.vocab0 = m->pd_vocab0;
    p.head0_global = m->d.headStart, p.kv_head0_global = m->d.groupHeadStart;
    p.eps = c.layer_norm_eps;
    p.attn_scale = (float)(1.0 / sqrt((double)c.head_size)); // CausalSelfAttention.java:134
    p.lw = nullptr;
    p.embed_dt = m->g[JL_T_EMBED].dtype, p.embed_w = m->g[JL_T_EMBED].data, p.embed_s = m->g[JL_T_EMBED].scales;
    p.out_norm = m->g[JL_T_OUT_NORM].data, p.out_norm_dt = m->g[JL_T_OUT_NORM].dtype;
    const DevTensor &head = m->g_set[JL_T_LM_HEAD] ? m->g[JL_T_LM_HEAD] : m->g[JL_T_EMBED];
    const size_t rb = (size_t)c.embedding_length / 32 * (head.dtype == JL_Q4 ? 16 : 32);
    p.lm_w = (const uint8_t *)head.data + (size_t)m->pd_vocab0 * rb;
    p.lm_s = head.scales + (size_t)m->pd_vocab0 * (c.embedding_length / 32);
    p.x = m->x, p.xb = m->xb, p.q = m->q, p.k = m->k, p.v = m->v, p.att = m->att, p.h = m->hbuf, p.logits = m->logits;
    p.attn_ws = m->attn_ws;
    p.rope = m->rope;
    p.kv = m->kv;
    p.tokens = m->d_tokens, p.positions = m->d_positions, p.next = m->d_next, p.sessions = m->d_sessions;
    p.hist = m->d_hist, p.counter = m->d_counter, p.hist_cap = m->hist_cap, p.resident = resident ? 1 : 0;
    p.sync = m->pd_sync, p.argmax_slots = m->pd_slots, p.att_done = m->pd_att_done;
    // one context split per 64 positions, bounded by the CTAs available for (kv head, split) tasks
    int s = (max_pos + 1 + 63) / 64;
    const int cap = m->ctx->sm_count / m->kv_heads_local;
    if (s > cap) s = cap;
    if (s > m->max_splits) s = m->max_splits;
    if (s < 1) s = 1;
    p.splits = s;
    p.split_cap = cap < m->max_splits ? cap : m->max_splits;
    p.ntok = 1;
    p.world = c.tp_size, p.rank = c.tp_rank;
    for (int r = 0; r < c.tp_size && r < PD_MAX_TP; r++)
        p.ll_o[r] = m->peer_ll_o[r], p.ll_d[r] = m->peer_ll_d[r], p.ll_a[r] = m->peer_ll_a[r], p.logits_peer[r] = m->peer_logits[r];
    p.want_logits = want_logits && c.tp_size > 1 ? 1 : 0;
    p.trace = m->pd_trace;
}

// after a synchronise: did the last persistent launches drain on a timeout?  Resets the protocol state if so.
static int pd_check(jl_model *m) {
    if (!m->pd_ok) return JL_OK;
    unsigned long long st[2] = {0, 0};
    if (cudaMemcpy(st, m->pd_sync, sizeof st, cudaMemcpyDeviceToHost) != cudaSuccess) return jl_set_error(m->ctx, JL_ERR_CUDA, "decode status read failed");
    if (st[1] == 0) return JL_OK;
    cudaMemset(m->pd_sync, 0, PD_SYNC_WORDS * 8);
    cudaMemset(m->pd_att_done, 0, (size_t)m->kv_heads_local * sizeof(unsigned));
    return jl_set_error(m->ctx, JL_ERR_CUDA, "persistent decode kernel timed out waiting on counter %llu (token %llu); state reset", st[1], st[0]);
}

// context-split buckets of the per-op decode step: one CUDA graph per bucket
static const int SPLIT_BUCKETS[] = {1, 2, 3, 4, 6, 8, 12, 16, 24, 32};
// tokens per cooperative launch of the persistent kernel in jl_model_decode_resident
static const int PD_TOKENS_PER_LAUNCH = 16;

// run the decode body through the persistent kernel (one session), a cached CUDA graph, or eagerly
static int run_decode(jl_model *m, int n, int max_pos, bool resident, bool want_logits = false, int ntok = 1) {
    jl_ctx *ctx = m->ctx;
    if (n == 1 && use_pd(m)) {
        PdParams pp;
        fill_pd(m, max_pos, resident, want_logits, pp);
        pp.ntok = resident ? ntok : 1;
        return jl_launch_pdecode(ctx, m->stream, pp, m->pd_layers.data(), m, m->pd_wdtype);
    }
    // fused decode attention: one split per 64 positions (per 64 * n with n sessions in the step: the rows already fill the grid),
    // bucketed so that few graphs are captured
    int splits = (max_pos + 1 + 63) / 64;
    if (n > 1) splits = (splits + n - 1) / n;
    {
        int b = 32;
        for (int v : SPLIT_BUCKETS)
            if (v >= splits) {
                b = v;
                break;
            }
        splits = b > m->max_splits ? m->max_splits : b;
    }
    if (!use_graph(m)) return decode_body(m, n, splits, resident);
    const long long key = ((long long)n << 32) | ((long long)splits << 1) | (resident ? 1 : 0);
    auto it = m->graphs.find(key);
    if (it == m->graphs.end()) {
        // First decode of this (sessions, resident) kind: capture the graph of EVERY context-split bucket now, so that a
        // generation never pays a capture + instantiate (~8 ms) when its context crosses a bucket boundary later.
        // Capturing records launches only; nothing executes and no KV page is touched.
        for (int b : SPLIT_BUCKETS) {
            const int sp = b > m->max_splits ? m->max_splits : b;
            const long long k2 = ((long long)n << 32) | ((long long)sp << 1) | (resident ? 1 : 0);
            if (m->graphs.count(k2)) continue;
            cudaGraph_t graph = nullptr;
            const long long before = ctx->launches;
            const int before_trace = ctx->ktrace_n;
            JL_CUDA_CHECK(ctx, cudaStreamBeginCapture(m->stream, cudaStreamCaptureModeThreadLocal));
            int rc = decode_body(m, n, sp, resident);
            cudaError_t ce = cudaStreamEndCapture(m->stream, &graph);
            const long long per_graph = ctx->launches - before;
            ctx->launches = before;
            if (sp != splits) ctx->ktrace_n = before_trace; // timeline slots only for the graph that is about to run
            if (rc != JL_OK) {
                if (graph) cudaGraphDestroy(graph);
                return rc;
            }
            if (ce != cudaSuccess) return jl_set_error(ctx, JL_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(ce));
            cudaGraphExec_t exec = nullptr;
            ce = cudaGraphInstantiate(&exec, graph, 0);
            cudaGraphDestroy(graph);
            if (ce != cudaSuccess) return jl_set_error(ctx, JL_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(ce));
            m->graphs[k2] = exec;
            m->graph_launches[k2] = per_graph;
        }
        it = m->graphs.find(key);
        if (it == m->graphs.end()) return jl_set_error(ctx, JL_ERR_INVALID, "decode: no graph for %d splits", splits);
    }
    JL_CUDA_CHECK(ctx, cudaGraphLaunch(it->second, m->stream));
    ctx->launches += m->graph_launches[key];
    return JL_OK;
}

// One selection call: its nullable per-row inputs (HOST [n] each) and, after select_check, what they imply.  `topkp` and `logprobs` mark
// the entry points that take those arguments (the *_constrained ones are topkp calls); the plain entry points skip the top-k / top-p
// checks, so a negative temperature reaches the reference rule there.  Penalties (DESIGN §3.14) and masks (DESIGN §3.18) are on when
// `pen` / `allow_row` are set; a call without a penalised or constrained row runs exactly as the narrower call.
struct Selection {
    const float *temperatures = nullptr, *uniforms = nullptr;
    bool topkp = false;
    const int32_t *top_k = nullptr;
    const float *top_p = nullptr;
    bool logprobs = false;
    const int32_t *top_n = nullptr; // nullable = all -1
    float *lp = nullptr;            // logprob outputs, each nullable
    int32_t *ids = nullptr;
    float *tlp = nullptr;
    const jl_penalties *pen = nullptr;
    int n_allow = 0;
    const uint32_t *allow = nullptr;    // [n_allow][words]
    const int32_t *allow_row = nullptr; // -1 = unconstrained
    // derived by select_check
    bool sampled = false;       // a row with temperature != 0
    std::vector<char> filtered; // [n], topkp calls only: the rows the top-k / top-p kernel draws
    int n_filtered = 0;
    int n_lp = 0; // rows with top_n >= 0
    PenaltyPlan plan;
    int n_con = 0; // constrained rows
    bool processed() const { return plan.n_on > 0 || n_con > 0; }
    // the table of the processed rows: the penalties' own, or one unpenalised PenaltyRow per row for a call with masks only
    size_t tab_bytes(int n) const { return pen ? plan.bytes : (size_t)n * sizeof(PenaltyRow); }
};

// The checks of one selection call, before any device work: uniforms for the sampled rows, top-k / top-p, logprobs, penalties, masks.
// Logprobs, penalties and masks are refused under tensor parallelism (`tp`).  A constrained row with temperature > 0 then joins the
// filtered rows: the top-k / top-p kernel draws it (its integer rule gives a banned token weight 0 and never draws one), whatever its
// filter.
static int select_check(jl_ctx *ctx, const char *who, int n, int vocab, bool tp, Selection &s) {
    s.sampled = false, s.n_filtered = s.n_lp = s.n_con = 0, s.plan = PenaltyPlan();
    for (int i = 0; s.temperatures && i < n; i++) s.sampled = s.sampled || s.temperatures[i] != 0.0f;
    if (s.sampled && !s.uniforms) return jl_set_error(ctx, JL_ERR_INVALID, "%s: temperatures without uniform samples", who);
    if (s.topkp) {
        s.filtered.assign((size_t)n, 0);
        M_CHECK(jl_topkp_check(ctx, who, n, vocab, s.temperatures, s.top_k, s.top_p, s.uniforms, s.filtered.data(), &s.n_filtered));
    }
    if (s.logprobs) {
        if (tp) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "%s: logprobs under tensor parallelism", who);
        M_CHECK(jl_logprobs_check(ctx, who, n, vocab, s.top_n, &s.n_lp));
    }
    if (s.pen) {
        if (tp) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "%s: penalties under tensor parallelism", who);
        M_CHECK(jl_penalty_check(ctx, who, n, vocab, s.pen, &s.plan));
    }
    if (!s.allow_row) return JL_OK;
    if (tp) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "%s: constrained rows under tensor parallelism", who);
    M_CHECK(jl_constraint_check(ctx, who, n, vocab, s.n_allow, s.allow, s.allow_row, &s.n_con));
    for (int i = 0; i < n; i++) {
        if (s.allow_row[i] < 0 || !s.temperatures || !(s.temperatures[i] > 0.0f) || s.filtered[(size_t)i]) continue;
        if (!(s.uniforms[i] >= 0.0f && s.uniforms[i] <= 1.0f))
            return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: uniform %g (in [0, 1])", who, i, (double)s.uniforms[i]);
        if (vocab > JL_TOPKP_MAX_VOCAB) return jl_set_error(ctx, JL_ERR_INVALID, "%s: vocabulary of %d above %d", who, vocab, JL_TOPKP_MAX_VOCAB);
        s.filtered[(size_t)i] = 1, s.n_filtered++;
    }
    return JL_OK;
}

// The buffers of one selection pass, DEVICE unless h_: proc, cnt (zero, and left zero), bias and ex hold n rows of vocab words; the
// tables hold the call's; next holds the arg-max of the raw rows on entry and the tokens on return.
struct SelectBufs {
    float *proc;
    unsigned *cnt;
    float *bias;
    void *d_tab, *h_tab;
    uint32_t *d_mask, *h_mask;
    TopkpRow *d_topkp, *h_topkp;
    float *ex;
    int32_t *next;
    void *argmax;
};

// The selection of a checked call on `rows` (DEVICE [n][vocab]): penalties and masks turn them into the processed rows (two launches,
// one without a penalised row) and the arg-max runs again on those; the filtered rows are drawn in one launch of the top-k / top-p
// kernel, the other sampled rows by the reference's prefix-sum rule (AbstractModel.java:475-489), whose exponentials overwrite their
// row unless the logprobs still read the raw rows.  The tables ride the stream, one copy each.
static int select_pass(jl_ctx *ctx, cudaStream_t st, int n, int V, float *rows, const Selection &s, const SelectBufs &b) {
    float *src = rows;
    if (s.processed()) {
        const jl_penalties none = {};
        jl_penalty_pack(s.pen ? s.pen : &none, n, s.plan, b.h_tab);
        const uint32_t *mask = nullptr;
        if (s.n_con > 0) {
            const int mr = jl_constraint_pack(n, V, s.n_allow, s.allow, s.allow_row, b.h_tab, b.h_mask);
            JL_CUDA_CHECK(ctx, cudaMemcpyAsync(b.d_mask, b.h_mask, (size_t)mr * ((V + 31) / 32) * 4, cudaMemcpyHostToDevice, st));
            mask = b.d_mask;
        }
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(b.d_tab, b.h_tab, s.tab_bytes(n), cudaMemcpyHostToDevice, st));
        M_CHECK(jl_launch_penalties(ctx, st, rows, V, V, n, b.d_tab, s.plan, b.cnt, b.bias, mask, b.proc));
        M_CHECK(jl_launch_argmax(ctx, st, b.proc, n, V, V, b.next, b.argmax));
        src = b.proc;
    }
    if (s.n_filtered > 0) {
        int c = 0;
        for (int i = 0; i < n; i++)
            if (s.filtered[(size_t)i])
                b.h_topkp[c++] = TopkpRow{i, s.temperatures[i], s.top_k ? s.top_k[i] : 0, s.top_p ? s.top_p[i] : 1.0f, s.uniforms[i]};
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(b.d_topkp, b.h_topkp, (size_t)c * sizeof(TopkpRow), cudaMemcpyHostToDevice, st));
        M_CHECK(jl_launch_sample_topkp(ctx, st, src, V, V, b.d_topkp, c, b.ex, b.next));
    }
    for (int i = 0; s.sampled && i < n; i++) {
        if (s.temperatures[i] == 0.0f) continue; // :471-473 short-circuit: the arg-max stands
        if (s.n_filtered > 0 && s.filtered[(size_t)i]) continue;
        float *row = src + (size_t)i * V;
        softmax_sample_kernel<<<1, 256, 0, st>>>(row, s.n_lp > 0 ? b.ex + (size_t)i * V : row, V, s.temperatures[i], s.uniforms[i], b.next + i);
        ctx->launches++;
        JL_CUDA_CHECK(ctx, cudaGetLastError());
    }
    return JL_OK;
}

// the model's buffers of a call with processed rows and a penalty table of `tab` bytes, with `masks` the mask rows too (model lock
// held).  The count words are zeroed in stream order.
static int select_alloc(jl_model *m, size_t tab, bool masks) {
    jl_ctx *ctx = m->ctx;
    const int S = m->cfg.max_sessions, rows = S < JL_MAX_DECODE_ROWS ? S : JL_MAX_DECODE_ROWS;
    if (!m->pen_out) {
        const size_t rb = (size_t)rows * m->cfg.vocab_size * 4;
        M_CHECK(dev_alloc(ctx, (void **)&m->pen_out, rb));
        M_CHECK(dev_alloc(ctx, (void **)&m->pen_bias, rb));
        M_CHECK(dev_alloc(ctx, (void **)&m->pen_cnt, rb));
        JL_CUDA_CHECK(ctx, cudaMemsetAsync(m->pen_cnt, 0, rb, m->stream));
    }
    if (tab > m->pen_tab_cap) {
        size_t cap = 4096;
        while (cap < tab) cap *= 2;
        if (m->d_pen_tab) cudaFree(m->d_pen_tab), m->d_pen_tab = nullptr;
        if (m->h_pen_tab) cudaFreeHost(m->h_pen_tab), m->h_pen_tab = nullptr;
        m->pen_tab_cap = 0;
        M_CHECK(dev_alloc(ctx, &m->d_pen_tab, cap));
        JL_CUDA_CHECK(ctx, cudaMallocHost(&m->h_pen_tab, cap));
        m->pen_tab_cap = cap;
    }
    if (masks && !m->d_mask) {
        const size_t bytes = (size_t)rows * ((m->cfg.vocab_size + 31) / 32) * 4;
        M_CHECK(dev_alloc(ctx, (void **)&m->d_mask, bytes));
        JL_CUDA_CHECK(ctx, cudaMallocHost((void **)&m->h_mask, bytes));
    }
    return JL_OK;
}

// Everything after the logits of a checked call (m->logits, n rows, their arg-max in m->d_next; model lock held): logits_out gets the raw
// logits before any row is exponentiated, then the selection pass, one logprob launch for the rows with top_n >= 0 (of the raw logits,
// the chosen tokens as targets), and the tokens.  `decode`: the step's end event is recorded, and the persistent kernel's status checked
// after the synchronise.
static int select_tail(jl_model *m, int n, Selection &s, float *logits_out, int32_t *tokens_out, bool decode) {
    jl_ctx *ctx = m->ctx;
    const int V = m->cfg.vocab_size;
    if (logits_out) JL_CUDA_CHECK(ctx, cudaMemcpyAsync(logits_out, m->logits, (size_t)n * V * 4, cudaMemcpyDeviceToHost, m->stream));
    if (s.processed()) M_CHECK(select_alloc(m, s.tab_bytes(n), s.n_con > 0));
    const SelectBufs b{m->pen_out, m->pen_cnt, m->pen_bias, m->d_pen_tab, m->h_pen_tab, m->d_mask, m->h_mask,
                       m->d_topkp, m->h_topkp, m->topkp_ex, m->d_next, m->argmax_scratch};
    M_CHECK(select_pass(ctx, m->stream, n, V, m->logits, s, b));
    jl_model::LpBufs &lb = m->lp;
    if (s.n_lp > 0) {
        int c = 0;
        for (int i = 0; i < n; i++)
            if (s.top_n[i] >= 0) lb.h_rows[c++] = LogprobRow{i, s.top_n[i]};
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(lb.d_rows, lb.h_rows, (size_t)c * sizeof(LogprobRow), cudaMemcpyHostToDevice, m->stream));
        M_CHECK(jl_launch_logprobs(ctx, m->stream, m->logits, V, V, lb.d_rows, c, m->d_next, lb.ws, lb.cnt, lb.d_out));
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(lb.h_out, lb.d_out, (size_t)n * sizeof(LogprobOut), cudaMemcpyDeviceToHost, m->stream));
    }
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(pinned_next(m), m->d_next, (size_t)n * 4, cudaMemcpyDeviceToHost, m->stream));
    if (decode) JL_CUDA_CHECK(ctx, cudaEventRecord(m->ev_end, m->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    if (decode && n == 1 && use_pd(m)) M_CHECK(pd_check(m));
    memcpy(tokens_out, pinned_next(m), (size_t)n * 4);
    if (s.logprobs) jl_logprobs_unpack(lb.h_out, s.top_n, n, s.lp, s.ids, s.tlp);
    return JL_OK;
}

// One decode step of n sessions; `s` selects each row's token from its logits row: the arg-max, or a draw (see Selection).
static int decode_impl(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions, int32_t *next_tokens,
                       float *logits_out, Selection &s) {
    if (!m || !m->finalized || n <= 0 || n > m->cfg.max_sessions || n > JL_MAX_DECODE_ROWS || !sessions || !tokens || !positions ||
        !next_tokens)
        return m ? jl_set_error(m->ctx, JL_ERR_INVALID, "decode: bad arguments (n=%d, max %d)", n, JL_MAX_DECODE_ROWS) : JL_ERR_INVALID;
    M_CHECK(select_check(m->ctx, "decode", n, m->cfg.vocab_size, m->cfg.tp_size > 1, s));
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    int max_pos = 0;
    for (int i = 0; i < n; i++) {
        if (sessions[i] < 0 || sessions[i] >= m->cfg.max_sessions || positions[i] < 0)
            return jl_set_error(ctx, JL_ERR_INVALID, "decode: bad session/position");
        for (int j = 0; j < i; j++) // two rows of one session would append to and read the same KV positions concurrently
            if (sessions[j] == sessions[i]) return jl_set_error(ctx, JL_ERR_INVALID, "decode: session %d appears twice in one step", sessions[i]);
        M_CHECK(ensure_pages(m, sessions[i], positions[i], positions[i]));
        if (positions[i] > max_pos) max_pos = positions[i];
    }
    JL_CUDA_CHECK(ctx, cudaEventRecord(m->ev_begin, m->stream));
    M_CHECK(stage_rows(m, n, tokens, positions, sessions));
    M_CHECK(run_decode(m, n, max_pos, false, logits_out != nullptr || s.sampled || s.processed()));
    M_CHECK(select_tail(m, n, s, logits_out, next_tokens, true));
    float ms = 0;
    cudaEventElapsedTime(&ms, m->ev_begin, m->ev_end);
    m->last_total_ms = ms;
    return JL_OK;
}

// AbstractModel.sample on the last forwarded rows of n distinct sessions (arguments already checked): the rows are gathered in one
// launch and share one lm_head pass (sample_rows' wide mode: one weight pass for 9..64 rows).  logits_out gets the raw logits.
static int sample_sessions(jl_model *m, int n, const int32_t *sessions, int32_t *tokens_out, float *logits_out, Selection &s) {
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    memcpy(pinned_rows(m), sessions, (size_t)n * 4);
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->d_rows, pinned_rows(m), (size_t)n * 4, cudaMemcpyHostToDevice, m->stream));
    M_CHECK(copy_rows(m, m->xb, nullptr, m->last_hidden, m->d_rows, n));
    M_CHECK(sample_rows(m, m->xb, n));
    return select_tail(m, n, s, logits_out, tokens_out, false);
}

extern "C" int jl_model_sample(jl_model *m, int session, float temperature, float uniform, int32_t *token_out,
                               float *logits_out) {
    if (!m || !m->finalized || !token_out || session < 0 || session >= m->cfg.max_sessions) return JL_ERR_INVALID;
    Selection s{&temperature, &uniform};
    M_CHECK(select_check(m->ctx, "sample", 1, m->cfg.vocab_size, m->cfg.tp_size > 1, s));
    // logits_out is written at temperature 0 only
    return sample_sessions(m, 1, &session, token_out, temperature == 0.0f ? logits_out : nullptr, s);
}

static int sample_multi_impl(jl_model *m, int n, const int32_t *sessions, int32_t *tokens_out, float *logits_out, Selection &s) {
    if (!m || !m->finalized) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    const int S = m->cfg.max_sessions, cap = S < JL_MAX_DECODE_ROWS ? S : JL_MAX_DECODE_ROWS;
    if (!sessions || !tokens_out) return jl_set_error(ctx, JL_ERR_INVALID, "sample_multi: null argument");
    if (n < 1 || n > cap) return jl_set_error(ctx, JL_ERR_INVALID, "sample_multi: %d rows (1..%d)", n, cap);
    std::vector<char> seen((size_t)S, 0);
    for (int i = 0; i < n; i++) {
        if (sessions[i] < 0 || sessions[i] >= S) return jl_set_error(ctx, JL_ERR_INVALID, "sample_multi: session %d out of range", sessions[i]);
        if (seen[(size_t)sessions[i]]) return jl_set_error(ctx, JL_ERR_INVALID, "sample_multi: session %d appears twice", sessions[i]);
        seen[(size_t)sessions[i]] = 1;
    }
    M_CHECK(select_check(ctx, "sample_multi", n, m->cfg.vocab_size, m->cfg.tp_size > 1, s));
    return sample_sessions(m, n, sessions, tokens_out, logits_out, s);
}

extern "C" int jl_model_sample_multi(jl_model *m, int n, const int32_t *sessions, const float *temperatures, const float *uniforms,
                                     int32_t *tokens_out, float *logits_out) {
    Selection s{temperatures, uniforms};
    return sample_multi_impl(m, n, sessions, tokens_out, logits_out, s);
}

extern "C" int jl_model_sample_multi_topkp(jl_model *m, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                           const float *top_p, const float *uniforms, int32_t *tokens_out, float *logits_out) {
    Selection s{temperatures, uniforms, true, top_k, top_p};
    return sample_multi_impl(m, n, sessions, tokens_out, logits_out, s);
}

extern "C" int jl_model_decode_sample_topkp(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                                            const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms,
                                            int32_t *next_tokens, float *logits_out) {
    Selection s{temperatures, uniforms, true, top_k, top_p};
    return decode_impl(m, n, sessions, tokens, positions, next_tokens, logits_out, s);
}

extern "C" int jl_model_sample_multi_logprobs(jl_model *m, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                              const float *top_p, const float *uniforms, const int32_t *top_n, int32_t *tokens_out, float *lp_out,
                                              int32_t *top_ids_out, float *top_lp_out, float *logits_out) {
    Selection s{temperatures, uniforms, true, top_k, top_p, true, top_n, lp_out, top_ids_out, top_lp_out};
    return sample_multi_impl(m, n, sessions, tokens_out, logits_out, s);
}

extern "C" int jl_model_decode_logprobs(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                                        const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms,
                                        const int32_t *top_n, int32_t *next_tokens, float *lp_out, int32_t *top_ids_out, float *top_lp_out,
                                        float *logits_out) {
    Selection s{temperatures, uniforms, true, top_k, top_p, true, top_n, lp_out, top_ids_out, top_lp_out};
    return decode_impl(m, n, sessions, tokens, positions, next_tokens, logits_out, s);
}

extern "C" int jl_model_sample_multi_penalized(jl_model *m, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                               const float *top_p, const float *uniforms, const int32_t *top_n, const jl_penalties *pen,
                                               int32_t *tokens_out, float *lp_out, int32_t *top_ids_out, float *top_lp_out, float *logits_out) {
    Selection s{temperatures, uniforms, true, top_k, top_p, true, top_n, lp_out, top_ids_out, top_lp_out, pen};
    return sample_multi_impl(m, n, sessions, tokens_out, logits_out, s);
}

extern "C" int jl_model_decode_penalized(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                                         const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms,
                                         const int32_t *top_n, const jl_penalties *pen, int32_t *next_tokens, float *lp_out, int32_t *top_ids_out,
                                         float *top_lp_out, float *logits_out) {
    Selection s{temperatures, uniforms, true, top_k, top_p, true, top_n, lp_out, top_ids_out, top_lp_out, pen};
    return decode_impl(m, n, sessions, tokens, positions, next_tokens, logits_out, s);
}

extern "C" int jl_model_sample_multi_constrained(jl_model *m, int n, const int32_t *sessions, const float *temperatures, const int32_t *top_k,
                                                 const float *top_p, const float *uniforms, const int32_t *top_n, const jl_penalties *pen,
                                                 int n_allow, const uint32_t *allow, const int32_t *allow_row, int32_t *tokens_out, float *lp_out,
                                                 int32_t *top_ids_out, float *top_lp_out, float *logits_out) {
    Selection s{temperatures, uniforms, true, top_k, top_p, true, top_n, lp_out, top_ids_out, top_lp_out, pen, n_allow, allow, allow_row};
    return sample_multi_impl(m, n, sessions, tokens_out, logits_out, s);
}

extern "C" int jl_model_decode_constrained(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                                           const float *temperatures, const int32_t *top_k, const float *top_p, const float *uniforms,
                                           const int32_t *top_n, const jl_penalties *pen, int n_allow, const uint32_t *allow,
                                           const int32_t *allow_row, int32_t *next_tokens, float *lp_out, int32_t *top_ids_out,
                                           float *top_lp_out, float *logits_out) {
    Selection s{temperatures, uniforms, true, top_k, top_p, true, top_n, lp_out, top_ids_out, top_lp_out, pen, n_allow, allow, allow_row};
    return decode_impl(m, n, sessions, tokens, positions, next_tokens, logits_out, s);
}

// HOST-buffer entry point for crafted rows: the model calls' selection pass (select_pass) on the rows, after the arg-max the model's
// lm_head pass takes.  Every sampled row's uniform must lie in [0, 1].
extern "C" int jl_select_constrained(jl_ctx *ctx, int n, int vocab, const float *logits, int64_t ld, const float *temperatures,
                                     const int32_t *top_k, const float *top_p, const float *uniforms, const jl_penalties *pen, int n_allow,
                                     const uint32_t *allow, const int32_t *allow_row, int32_t *out) {
    if (!ctx) return JL_ERR_INVALID;
    const char *who = "select_constrained";
    if (n < 1 || n > 65535 || vocab < 1 || vocab > JL_TOPKP_MAX_VOCAB || ld < vocab || !logits || !out)
        return jl_set_error(ctx, JL_ERR_INVALID, "%s: bad arguments (n=%d, vocab=%d, ld=%lld)", who, n, vocab, (long long)ld);
    Selection s{temperatures, uniforms, true, top_k, top_p, false, nullptr, nullptr, nullptr, nullptr, pen, n_allow, allow, allow_row};
    M_CHECK(select_check(ctx, who, n, vocab, false, s));
    for (int i = 0; s.sampled && i < n; i++)
        if (temperatures[i] > 0.0f && !(uniforms[i] >= 0.0f && uniforms[i] <= 1.0f))
            return jl_set_error(ctx, JL_ERR_INVALID, "%s: row %d: uniform %g (in [0, 1])", who, i, (double)uniforms[i]);
    std::vector<char> h_tab(s.processed() ? s.tab_bytes(n) : 0);
    std::vector<uint32_t> h_mask(s.n_con > 0 ? (size_t)n * ((vocab + 31) / 32) : 0);
    std::vector<TopkpRow> h_topkp((size_t)s.n_filtered);
    std::lock_guard<std::mutex> lk(ctx->mu);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t rb = al((size_t)n * vocab * 4), tb = al(h_tab.size()), ob = al((size_t)n * 4), kb = al(h_topkp.size() * sizeof(TopkpRow));
    float *rows = (float *)jl_scratch(ctx, 0, rb);
    char *dw = (char *)jl_scratch(ctx, 1, 3 * rb + tb + h_mask.size() * 4);
    float *ex = (float *)jl_scratch(ctx, 2, rb);
    char *dsel = (char *)jl_scratch(ctx, 3, ob + kb + jl_argmax_scratch_bytes(n));
    if (!rows || !dw || !ex || !dsel) return JL_ERR_OOM;
    const SelectBufs b{(float *)(dw + 2 * rb), (unsigned *)dw, (float *)(dw + rb), dw + 3 * rb, h_tab.data(), (uint32_t *)(dw + 3 * rb + tb),
                       h_mask.data(), (TopkpRow *)(dsel + ob), h_topkp.data(), ex, (int32_t *)dsel, dsel + ob + kb};
    cudaStream_t st = ctx->stream;
    JL_CUDA_CHECK(ctx, cudaMemcpy2DAsync(rows, (size_t)vocab * 4, logits, (size_t)ld * 4, (size_t)vocab * 4, n, cudaMemcpyHostToDevice, st));
    if (s.processed()) JL_CUDA_CHECK(ctx, cudaMemsetAsync(b.cnt, 0, (size_t)n * vocab * 4, st));
    M_CHECK(jl_launch_argmax(ctx, st, rows, n, vocab, vocab, b.next, b.argmax));
    M_CHECK(select_pass(ctx, st, n, vocab, rows, s, b));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(out, b.next, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(st));
    return JL_OK;
}

extern "C" int jl_model_decode(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                               int32_t *next_tokens, float *logits_out) {
    Selection s;
    return decode_impl(m, n, sessions, tokens, positions, next_tokens, logits_out, s);
}

extern "C" int jl_model_decode_sample(jl_model *m, int n, const int32_t *sessions, const int32_t *tokens, const int32_t *positions,
                                      const float *temperatures, const float *uniforms, int32_t *next_tokens, float *logits_out) {
    Selection s{temperatures, uniforms};
    return decode_impl(m, n, sessions, tokens, positions, next_tokens, logits_out, s);
}

extern "C" int jl_model_decode_resident(jl_model *m, int session, int32_t first_token, int start_pos, int n_new,
                                        int32_t *out_tokens) {
    if (!m || !m->finalized || session < 0 || session >= m->cfg.max_sessions || n_new <= 0 || !out_tokens || start_pos < 0)
        return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    if (n_new > m->hist_cap) return jl_set_error(ctx, JL_ERR_INVALID, "decode_resident: n_new too large");
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    M_CHECK(ensure_pages(m, session, start_pos, start_pos + n_new - 1));
    M_CHECK(stage_rows(m, 1, &first_token, &start_pos, &session));
    *pinned_next(m) = 0;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->d_counter, pinned_next(m), 4, cudaMemcpyHostToDevice, m->stream));
    JL_CUDA_CHECK(ctx, cudaEventRecord(m->ev_begin, m->stream));
    // persistent kernel: up to PD_TOKENS_PER_LAUNCH tokens per cooperative launch (the fed-back token crosses a grid barrier
    // instead of a kernel boundary); other paths: one graph replay per token
    const int tpl = use_pd(m) ? PD_TOKENS_PER_LAUNCH : 1;
    for (int i = 0; i < n_new; i += tpl) {
        const int nt = n_new - i < tpl ? n_new - i : tpl;
        M_CHECK(run_decode(m, 1, start_pos + i, true, false, nt));
    }
    JL_CUDA_CHECK(ctx, cudaEventRecord(m->ev_end, m->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(out_tokens, m->d_hist, (size_t)n_new * 4, cudaMemcpyDeviceToHost, m->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    if (use_pd(m)) M_CHECK(pd_check(m));
    float ms = 0;
    cudaEventElapsedTime(&ms, m->ev_begin, m->ev_end);
    m->last_total_ms = ms;
    return JL_OK;
}

// diagnostic: CTA 0's phase stamps (globaltimer ns) of the last persistent decode launch; needs JL_PD_TRACE=1 at finalize.
// out[0] = kernel start, out[1 + L*8 + k]: k 0 qkv dependency met, 1 qkv done, 2 attention done (attention CTAs only), 3 o_proj dependency
// met, 4 o_proj done, 5 gate/up dependency met, 6 gate/up done, 7 down dependency met; then lm_head dependency met, token published.
extern "C" int jl_model_debug_trace(jl_model *m, uint64_t *out, int64_t out_words) {
    if (!m || !m->finalized || !out) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    if (!m->pd_trace) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "phase tracing is off (set JL_PD_TRACE=1 before creating the model)");
    const size_t words = (size_t)m->cfg.num_layers * 16 + 32;
    if ((size_t)out_words < words) return jl_set_error(ctx, JL_ERR_INVALID, "trace buffer too small (%zu words needed)", words);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpy(out, m->pd_trace, words * 8, cudaMemcpyDeviceToHost));
    return (int)words;
}

extern "C" int jl_model_decode_mode(jl_model *m, int n) {
    if (!m || !m->finalized) return JL_ERR_INVALID;
    if (n == 1 && use_pd(m)) return 3;
    return use_graph(m) ? 1 : 0;
}

extern "C" int jl_model_last_timing(jl_model *m, double *total_ms, double *gemv_ms) {
    if (!m) return JL_ERR_INVALID;
    if (total_ms) *total_ms = m->last_total_ms;
    if (gemv_ms) *gemv_ms = 0.0;
    return JL_OK;
}

// AbstractModel.generate (:516-646): the prompt, its first token, then one decode step per token.  At temperature 0 every token is the
// arg-max and logits_out (nullable, [n_new, vocab]) gets the raw logits of each step; otherwise uniforms[i] plays
// ThreadLocalRandom.current().nextFloat() of the i-th sample() call (:576, :594), so a caller that passes the same stream gets the same
// tokens.
// `g` holds the one-row selection of every token: g.temperatures points at the temperature, g.uniforms at the uniforms of the tokens,
// and the logprob outputs at token 0's row (token i writes row i).  All arguments are checked before the prompt is forwarded; with
// g.topkp every token is sampled as by jl_model_decode_sample_topkp.  g.pen (nullable, its history ignored): the penalties of every
// token; token i's history is the prompt and the i tokens before it.
static int generate(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, const Selection &g, int32_t *out_tokens,
                    float *logits_out, double *timings_ms) {
    const float temperature = *g.temperatures;
    if (!m || !m->finalized || !prompt || n_prompt <= 0 || n_new <= 0 || !out_tokens || (temperature != 0.0f && !g.uniforms)) return JL_ERR_INVALID;
    for (int i = 0; g.topkp && i < n_new; i++)
        M_CHECK(jl_topkp_check(m->ctx, "generate", 1, m->cfg.vocab_size, g.temperatures, g.top_k, g.top_p, g.uniforms ? g.uniforms + i : nullptr,
                               nullptr, nullptr));
    // the history of token i: the prompt, then out_tokens[0, i) (generated ids come from the model, so checking the prompt's suffices)
    std::vector<int32_t> hist;
    int32_t hoff[2] = {0, n_prompt}, hprompt = n_prompt;
    jl_penalties pen = {};
    Selection s = g;
    float u = temperature != 0.0f ? g.uniforms[0] : 0.0f;
    s.uniforms = &u;
    if (g.pen) {
        hist.assign(prompt, prompt + n_prompt);
        hist.reserve((size_t)n_prompt + n_new);
        pen = *g.pen;
        pen.hist_off = hoff, pen.hist_prompt = &hprompt, pen.hist_ids = hist.data();
        s.pen = &pen;
    }
    M_CHECK(select_check(m->ctx, "generate", 1, m->cfg.vocab_size, m->cfg.tp_size > 1, s));
    auto at = [&](int i) -> Selection & { // token i, after out_tokens[0, i) are known
        u = temperature != 0.0f ? g.uniforms[i] : 0.0f;
        if (g.pen) {
            hist.resize((size_t)n_prompt + i);
            if (i > 0) memcpy(hist.data() + n_prompt, out_tokens, (size_t)i * 4);
            hoff[1] = n_prompt + i;
            pen.hist_ids = hist.data();
        }
        s.lp = g.lp ? g.lp + i : nullptr;
        s.ids = g.ids ? g.ids + (size_t)i * JL_MAX_LOGPROBS : nullptr;
        s.tlp = g.tlp ? g.tlp + (size_t)i * JL_MAX_LOGPROBS : nullptr;
        return s;
    };
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    const int V = m->cfg.vocab_size;
    auto t0 = std::chrono::steady_clock::now();
    M_CHECK(jl_model_reset_session(m, session));
    M_CHECK(jl_model_batch_forward(m, session, prompt, n_prompt, 0));
    int32_t next = 0;
    if (g.topkp)
        M_CHECK(sample_multi_impl(m, 1, &session, &next, nullptr, at(0)));
    else
        M_CHECK(jl_model_sample(m, session, temperature, u, &next, logits_out));
    auto t1 = std::chrono::steady_clock::now();
    out_tokens[0] = next;
    for (int i = 1; i < n_new; i++) {
        const int32_t pos = n_prompt + i - 1;
        int32_t nx = 0;
        M_CHECK(decode_impl(m, 1, &session, &next, &pos, &nx, logits_out ? logits_out + (size_t)i * V : nullptr, at(i)));
        next = nx;
        out_tokens[i] = next;
    }
    auto t2 = std::chrono::steady_clock::now();
    if (timings_ms) {
        timings_ms[0] = std::chrono::duration<double, std::milli>(t1 - t0).count();
        timings_ms[1] = std::chrono::duration<double, std::milli>(t2 - t1).count();
    }
    return JL_OK;
}

extern "C" int jl_model_generate(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, int32_t *out_tokens,
                                 float *logits_out, double *timings_ms) {
    const float greedy = 0.0f;
    return generate(m, session, prompt, n_prompt, n_new, Selection{&greedy}, out_tokens, logits_out, timings_ms);
}

extern "C" int jl_model_generate_sample(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, float temperature,
                                        const float *uniforms, int32_t *out_tokens, double *timings_ms) {
    return generate(m, session, prompt, n_prompt, n_new, Selection{&temperature, uniforms}, out_tokens, nullptr, timings_ms);
}

extern "C" int jl_model_generate_sample_topkp(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, float temperature,
                                              int top_k, float top_p, const float *uniforms, int32_t *out_tokens, double *timings_ms) {
    return generate(m, session, prompt, n_prompt, n_new, Selection{&temperature, uniforms, true, &top_k, &top_p}, out_tokens, nullptr,
                    timings_ms);
}

extern "C" int jl_model_generate_logprobs(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, float temperature, int top_k,
                                          float top_p, const float *uniforms, int top_n, int32_t *out_tokens, float *lp_out, int32_t *top_ids_out,
                                          float *top_lp_out, double *timings_ms) {
    const Selection g{&temperature, uniforms, true, &top_k, &top_p, true, &top_n, lp_out, top_ids_out, top_lp_out};
    return generate(m, session, prompt, n_prompt, n_new, g, out_tokens, nullptr, timings_ms);
}

extern "C" int jl_model_generate_penalized(jl_model *m, int session, const int32_t *prompt, int n_prompt, int n_new, float temperature,
                                           int top_k, float top_p, const float *uniforms, int top_n, float presence, float frequency,
                                           float repetition, int n_bias, const int32_t *bias_ids, const float *bias_vals, int32_t *out_tokens,
                                           float *lp_out, int32_t *top_ids_out, float *top_lp_out, double *timings_ms) {
    if (m && n_bias < 0) return jl_set_error(m->ctx, JL_ERR_INVALID, "generate: %d bias entries", n_bias);
    const int32_t boff[2] = {0, n_bias};
    jl_penalties gp = {};
    gp.presence = &presence, gp.frequency = &frequency, gp.repetition = &repetition;
    gp.bias_off = boff, gp.bias_ids = bias_ids, gp.bias_vals = bias_vals;
    const Selection g{&temperature, uniforms, true, &top_k, &top_p, true, &top_n, lp_out, top_ids_out, top_lp_out, &gp};
    return generate(m, session, prompt, n_prompt, n_new, g, out_tokens, nullptr, timings_ms);
}

// ---- KV persistence (KvBufferCache.KvBufferPage, core/tensor/KvBufferCache.java:121-176): the reference backs every page of a
// non-ephemeral session with the file  <workingDirectory>/<session>-L<layerPage>C<contextPage>.page  holding the raw little-endian
// page ([layersPerPage][2][contextPerPage][kvLength] of the working KV dtype).  Here pages live in HBM; save writes the allocated
// pages of a session in exactly that naming and byte layout, load maps such files back (allocating the pages) so a session can be
// resumed by this library or by the reference.  Returns the number of pages written / read, or a negative status.
extern "C" int jl_model_kv_save(jl_model *m, int session, const char *dir, const char *session_name) {
    if (!m || !m->finalized || !dir || !session_name || session < 0 || session >= m->cfg.max_sessions) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    std::vector<char> host(m->page_bytes);
    int n = 0;
    for (int lp = 0; lp < m->kv.n_layer_pages; lp++)
        for (int cp = 0; cp < m->kv.n_ctx_pages; cp++) {
            const void *page = m->page_table_host[page_index(m, session, lp, cp)];
            if (!page) continue;
            JL_CUDA_CHECK(ctx, cudaMemcpy(host.data(), page, m->page_bytes, cudaMemcpyDeviceToHost));
            const std::string path = std::string(dir) + "/" + session_name + "-L" + std::to_string(lp) + "C" + std::to_string(cp) + ".page";
            FILE *f = fopen(path.c_str(), "wb");
            if (!f) return jl_set_error(ctx, JL_ERR_INVALID, "kv_save: cannot open %s", path.c_str());
            const size_t w = fwrite(host.data(), 1, m->page_bytes, f);
            if (fclose(f) != 0 || w != m->page_bytes) return jl_set_error(ctx, JL_ERR_INVALID, "kv_save: short write to %s", path.c_str());
            n++;
        }
    return n;
}

extern "C" int jl_model_kv_load(jl_model *m, int session, const char *dir, const char *session_name) {
    if (!m || !m->finalized || !dir || !session_name || session < 0 || session >= m->cfg.max_sessions) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    std::vector<char> host(m->page_bytes);
    int n = 0;
    for (int cp = 0; cp < m->kv.n_ctx_pages; cp++)
        for (int lp = 0; lp < m->kv.n_layer_pages; lp++) {
            const std::string path = std::string(dir) + "/" + session_name + "-L" + std::to_string(lp) + "C" + std::to_string(cp) + ".page";
            FILE *f = fopen(path.c_str(), "rb");
            if (!f) continue;
            const size_t r = fread(host.data(), 1, m->page_bytes, f);
            const bool more = fgetc(f) != EOF;
            fclose(f);
            // KvBufferPage re-sizes a file of the wrong length (:148); a page of another geometry cannot be this session's
            if (r != m->page_bytes || more)
                return jl_set_error(ctx, JL_ERR_INVALID, "kv_load: %s is not a %zu-byte page of this model's geometry", path.c_str(), m->page_bytes);
            M_CHECK(ensure_pages(m, session, cp * m->kv.ctx_per_page, cp * m->kv.ctx_per_page)); // allocates every layer page of cp
            void *page = m->page_table_host[page_index(m, session, lp, cp)];
            JL_CUDA_CHECK(ctx, cudaMemcpy(page, host.data(), m->page_bytes, cudaMemcpyHostToDevice));
            n++;
        }
    return n;
}

// ---- host spill of an idle session -----------------------------------------------------------------------------------------------
// The reference's pages are memory-mapped files, so an idle session costs no RAM (KvBufferCache.java:121-176).  Here an idle session
// would pin HBM; offload moves its pages to host memory and returns the slot to the pool, restore brings them back into any slot.
extern "C" int jl_model_kv_pages(jl_model *m, int session) {
    if (!m || !m->finalized || session < 0 || session >= m->cfg.max_sessions) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    const size_t per = (size_t)m->kv.n_layer_pages * m->kv.n_ctx_pages;
    int n = 0;
    for (size_t i = 0; i < per; i++) n += m->page_table_host[page_index(m, session, 0, 0) + i] != nullptr;
    return n;
}

extern "C" int jl_model_kv_page_stats(jl_model *m, int64_t *pages_allocated, int64_t *page_entries) {
    if (!m || !m->finalized) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    int64_t entries = 0, held = 0, extra = 0;
    for (void *p : m->page_table_host) entries += p != nullptr;
    for (const auto &r : m->retained) held += (int64_t)r.second.pages.size();
    for (const auto &r : m->page_refs) extra += r.second - 1; // a page held by k entries and retained prefixes is one allocation
    if (pages_allocated) *pages_allocated = entries + held - extra;
    if (page_entries) *page_entries = entries;
    return JL_OK;
}

// dst's row of the page table becomes the source's pages [0, full) of every layer page (src[lp * src_ld + cp]) and, with part >= 0, a
// private copy of the source's page `part` holding its rows below `positions` (dst's own page there, else one taken from `fresh`).
// dst's other pages are released as by jl_model_reset_session: a shared page is detached, an own page is zeroed.  The row is uploaded
// on the model stream; own pages the shared ones replace go to `freed` and the partial copies to `copies`, for the caller to run and
// free once the stream is done.
static int share_pages(jl_model *m, int dst, void *const *src, size_t src_ld, int full, int part, int positions, std::vector<void *> &fresh,
                       std::vector<KvCopy> &copies, std::vector<void *> &freed) {
    jl_ctx *ctx = m->ctx;
    const int cpp = m->kv.ctx_per_page, nlp = m->kv.n_layer_pages, ncp = m->kv.n_ctx_pages;
    for (int lp = 0; lp < nlp; lp++)
        for (int cp = 0; cp < ncp; cp++) {
            const size_t idx = page_index(m, dst, lp, cp);
            void *old = m->page_table_host[idx];
            if (cp < full) {
                void *sp = src[(size_t)lp * src_ld + cp];
                if (old == sp) continue; // shares it already
                if (old && !drop_ref(m, old)) freed.push_back(old);
                m->page_table_host[idx] = sp;
                add_ref(m, sp);
            } else if (cp == part) {
                void *q = old && !is_shared(m, old) ? old : nullptr;
                if (!q) {
                    if (old) drop_ref(m, old);
                    q = fresh.back();
                    fresh.pop_back();
                }
                m->page_table_host[idx] = q;
                copies.push_back(KvCopy{q, src[(size_t)lp * src_ld + cp], positions - part * cpp, 0});
            } else if (old && drop_ref(m, old)) {
                m->page_table_host[idx] = nullptr;
            } else if (old) {
                JL_CUDA_CHECK(ctx, cudaMemsetAsync(old, 0, m->page_bytes, m->stream));
            }
        }
    const size_t base = page_index(m, dst, 0, 0), per = (size_t)nlp * ncp; // the destination's whole row of the table in one copy
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->page_table_dev + base, m->page_table_host.data() + base, per * sizeof(void *),
                                       cudaMemcpyHostToDevice, m->stream));
    return JL_OK;
}

// ---- fork: sessions that share a prefix's KV pages (DESIGN §3.15) ----------------------------------------------------------------
// Every context page wholly below `positions` is shared (entry -> src's page, no bytes move); a page holding positions - 1 but not
// ending there gets a private copy per destination (rows below positions, zeros above: the page an unforked session would hold).  A
// destination's pages past the prefix are released as by jl_model_reset_session, and its last_hidden becomes src's.
extern "C" int jl_model_kv_fork(jl_model *m, int src, int positions, int n, const int32_t *dst) {
    if (!m || !m->finalized) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    const int S = m->cfg.max_sessions;
    if (m->cfg.tp_size > 1) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "kv_fork: under tensor parallelism");
    if (n < 1 || !dst) return jl_set_error(ctx, JL_ERR_INVALID, "kv_fork: %d destinations", n);
    if (src < 0 || src >= S) return jl_set_error(ctx, JL_ERR_INVALID, "kv_fork: source session %d out of range", src);
    if (positions < 1 || positions > m->max_context)
        return jl_set_error(ctx, JL_ERR_INVALID, "kv_fork: %d positions (1..%d)", positions, m->max_context);
    std::vector<char> seen((size_t)S, 0);
    for (int i = 0; i < n; i++) {
        if (dst[i] < 0 || dst[i] >= S || dst[i] == src || seen[(size_t)dst[i]])
            return jl_set_error(ctx, JL_ERR_INVALID, "kv_fork: destination %d is out of range, the source or repeated", dst[i]);
        seen[(size_t)dst[i]] = 1;
    }
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    const int cpp = m->kv.ctx_per_page, nlp = m->kv.n_layer_pages, ncp = m->kv.n_ctx_pages;
    const int full = positions / cpp, part = positions % cpp ? full : -1; // shared pages [0, full), the partial page
    for (int lp = 0; lp < nlp; lp++)
        for (int cp = 0; cp <= (positions - 1) / cpp; cp++)
            if (!m->page_table_host[page_index(m, src, lp, cp)])
                return jl_set_error(ctx, JL_ERR_INVALID, "kv_fork: session %d has no page for layer page %d, context page %d", src, lp, cp);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    // the partial copies' new pages first (a destination reuses its own page there): running out of memory changes nothing
    std::vector<void *> fresh;
    for (int i = 0; i < n && part >= 0; i++)
        for (int lp = 0; lp < nlp; lp++) {
            void *old = m->page_table_host[page_index(m, dst[i], lp, part)];
            if (old && !is_shared(m, old)) continue;
            void *q = nullptr;
            const int rc = dev_alloc(ctx, &q, m->page_bytes);
            if (rc != JL_OK) {
                for (void *f : fresh) cudaFree(f);
                return rc;
            }
            fresh.push_back(q);
        }
    std::vector<KvCopy> copies;
    std::vector<void *> freed; // destination pages the shared ones replace, freed once the stream is done
    for (int i = 0; i < n; i++) {
        M_CHECK(share_pages(m, dst[i], m->page_table_host.data() + page_index(m, src, 0, 0), (size_t)ncp, full, part, positions, fresh, copies,
                            freed));
        const size_t E = (size_t)m->cfg.embedding_length;
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(m->last_hidden + (size_t)dst[i] * E, m->last_hidden + (size_t)src * E, E * 4,
                                           cudaMemcpyDeviceToDevice, m->stream));
    }
    M_CHECK(run_page_copies(m, copies));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream)); // the staged table rows and copy entries must outlive their copies
    for (void *p : freed) cudaFree(p);
    for (void *p : fresh) cudaFree(p); // a page two destinations shared became the second one's own, and it kept it
    return JL_OK;
}

// ---- retained prefixes: whole pages that outlive their session (the scheduler's prefix cache, DESIGN §3.17) ----------------------
// A handle holds one reference to each page it retains, counted in page_refs like a page-table entry, so copy-on-write (ensure_pages),
// reset_session, kv_offload and kv_load treat a retained page exactly like one another session shares.
extern "C" int64_t jl_model_kv_retain(jl_model *m, int session, int positions) {
    if (!m || !m->finalized) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    if (m->cfg.tp_size > 1) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "kv_retain: under tensor parallelism");
    if (session < 0 || session >= m->cfg.max_sessions) return jl_set_error(ctx, JL_ERR_INVALID, "kv_retain: session %d out of range", session);
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    const int cpp = m->kv.ctx_per_page, nlp = m->kv.n_layer_pages, full = positions / cpp;
    if (positions < cpp || positions % cpp || positions > m->max_context)
        return jl_set_error(ctx, JL_ERR_INVALID, "kv_retain: %d positions (a multiple of %d up to %d)", positions, cpp, m->max_context);
    for (int lp = 0; lp < nlp; lp++)
        for (int cp = 0; cp < full; cp++)
            if (!m->page_table_host[page_index(m, session, lp, cp)])
                return jl_set_error(ctx, JL_ERR_INVALID, "kv_retain: session %d has no page for layer page %d, context page %d", session, lp, cp);
    jl_model::KvRetained r;
    r.positions = positions;
    r.pages.reserve((size_t)nlp * full);
    for (int lp = 0; lp < nlp; lp++)
        for (int cp = 0; cp < full; cp++) {
            void *p = m->page_table_host[page_index(m, session, lp, cp)];
            add_ref(m, p);
            r.pages.push_back(p);
        }
    const int64_t h = m->next_retained++;
    m->retained.emplace(h, std::move(r));
    return h;
}

// `session` becomes what `handle` holds for [0, positions): a page-aligned fork whose source is the handle
extern "C" int jl_model_kv_attach(jl_model *m, int64_t handle, int positions, int session) {
    if (!m || !m->finalized) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    if (m->cfg.tp_size > 1) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "kv_attach: under tensor parallelism");
    if (session < 0 || session >= m->cfg.max_sessions) return jl_set_error(ctx, JL_ERR_INVALID, "kv_attach: session %d out of range", session);
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    auto it = m->retained.find(handle);
    if (it == m->retained.end()) return jl_set_error(ctx, JL_ERR_INVALID, "kv_attach: unknown handle %lld", (long long)handle);
    const int cpp = m->kv.ctx_per_page;
    const jl_model::KvRetained &r = it->second;
    if (positions < cpp || positions % cpp || positions > r.positions)
        return jl_set_error(ctx, JL_ERR_INVALID, "kv_attach: %d positions (a multiple of %d up to the %d retained)", positions, cpp, r.positions);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    std::vector<void *> fresh, freed;
    std::vector<KvCopy> copies; // stays empty: a page-aligned prefix has no partial page
    M_CHECK(share_pages(m, session, r.pages.data(), (size_t)(r.positions / cpp), positions / cpp, -1, positions, fresh, copies, freed));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream)); // the staged table row must outlive its copy
    for (void *p : freed) cudaFree(p);
    return JL_OK;
}

extern "C" int jl_model_kv_release(jl_model *m, int64_t handle) {
    if (!m || !m->finalized) return JL_ERR_INVALID;
    jl_ctx *ctx = m->ctx;
    if (m->cfg.tp_size > 1) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "kv_release: under tensor parallelism");
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    auto it = m->retained.find(handle);
    if (it == m->retained.end()) return jl_set_error(ctx, JL_ERR_INVALID, "kv_release: unknown handle %lld", (long long)handle);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    for (void *p : it->second.pages)
        if (!drop_ref(m, p)) cudaFree(p); // the last holder
    m->retained.erase(it);
    return JL_OK;
}

extern "C" int jl_model_kv_retained(jl_model *m, int64_t *handles, int64_t *pages_retained_only) {
    if (!m || !m->finalized) return JL_ERR_INVALID;
    if (m->cfg.tp_size > 1) return jl_set_error(m->ctx, JL_ERR_UNSUPPORTED, "kv_retained: under tensor parallelism");
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    std::unordered_map<void *, int> held; // page -> references the handles hold
    for (const auto &r : m->retained)
        for (void *p : r.second.pages) held[p]++;
    int64_t only = 0;
    for (const auto &h : held) {
        auto it = m->page_refs.find(h.first);
        only += (it == m->page_refs.end() ? 1 : it->second) == h.second; // every reference is a handle's
    }
    if (handles) *handles = (int64_t)m->retained.size();
    if (pages_retained_only) *pages_retained_only = only;
    return JL_OK;
}

extern "C" int64_t jl_model_kv_offload(jl_model *m, int session) {
    if (!m || !m->finalized || session < 0 || session >= m->cfg.max_sessions) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    jl_model::KvSpill sp;
    for (int lp = 0; lp < m->kv.n_layer_pages; lp++)
        for (int cp = 0; cp < m->kv.n_ctx_pages; cp++)
            if (m->page_table_host[page_index(m, session, lp, cp)]) sp.pages.emplace_back(lp, cp);
    try {
        sp.bytes.resize(sp.pages.size() * m->page_bytes);
    } catch (const std::bad_alloc &) {
        return jl_set_error(ctx, JL_ERR_OOM, "kv_offload: out of host memory for %zu pages", sp.pages.size());
    }
    // copy everything first, free afterwards: a failure leaves the session as it was
    for (size_t i = 0; i < sp.pages.size(); i++) {
        const size_t idx = page_index(m, session, sp.pages[i].first, sp.pages[i].second);
        JL_CUDA_CHECK(ctx, cudaMemcpy(sp.bytes.data() + i * m->page_bytes, m->page_table_host[idx], m->page_bytes, cudaMemcpyDeviceToHost));
    }
    for (size_t i = 0; i < sp.pages.size(); i++) {
        const size_t idx = page_index(m, session, sp.pages[i].first, sp.pages[i].second);
        void *page = m->page_table_host[idx];
        M_CHECK(publish_page(m, idx, nullptr));
        JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream)); // the staged pointer must outlive the copy
        if (!drop_ref(m, page)) cudaFree(page); // a shared page stays with the sessions that still hold it
    }
    const int64_t h = m->next_spill++;
    m->spills.emplace(h, std::move(sp));
    return h;
}

extern "C" int jl_model_kv_restore(jl_model *m, int session, int64_t handle) {
    if (!m || !m->finalized || session < 0 || session >= m->cfg.max_sessions) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    auto it = m->spills.find(handle);
    if (it == m->spills.end()) return jl_set_error(ctx, JL_ERR_INVALID, "kv_restore: unknown spill handle %lld", (long long)handle);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    M_CHECK(jl_model_reset_session(m, session)); // pages the slot still holds from its previous user start from zero
    const jl_model::KvSpill &sp = it->second;
    for (size_t i = 0; i < sp.pages.size(); i++) {
        const size_t idx = page_index(m, session, sp.pages[i].first, sp.pages[i].second);
        if (!m->page_table_host[idx]) {
            M_CHECK(alloc_page(m, idx));
            JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream)); // zeroed and published before the copy below fills it
        }
        JL_CUDA_CHECK(ctx, cudaMemcpy(m->page_table_host[idx], sp.bytes.data() + i * m->page_bytes, m->page_bytes, cudaMemcpyHostToDevice));
    }
    m->spills.erase(it);
    return JL_OK;
}

extern "C" int jl_model_kv_discard(jl_model *m, int64_t handle) {
    if (!m) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    return m->spills.erase(handle) ? JL_OK : jl_set_error(m->ctx, JL_ERR_INVALID, "kv_discard: unknown spill handle %lld", (long long)handle);
}

extern "C" int jl_model_read_kv(jl_model *m, int session, int layer, int position, int which, float *out) {
    if (!m || !m->finalized || !out || session < 0 || session >= m->cfg.max_sessions || layer < 0 ||
        layer >= m->cfg.num_layers || position < 0 || position >= m->max_context || (which != 0 && which != 1))
        return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    const KvLayout &kv = m->kv;
    const int lp = layer / kv.layers_per_page, rl = layer % kv.layers_per_page;
    const int cp = position / kv.ctx_per_page, rc = position % kv.ctx_per_page;
    const char *base = (const char *)m->page_table_host[page_index(m, session, lp, cp)];
    if (!base) return jl_set_error(ctx, JL_ERR_INVALID, "read_kv: page not allocated");
    const size_t rowb = kv_row_bytes(kv.kv_dtype, kv.kv_len);
    const char *row = base + (((size_t)rl * 2 + which) * kv.ctx_per_page + rc) * rowb;
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    if (kv.kv_dtype == JL_F32) {
        JL_CUDA_CHECK(ctx, cudaMemcpy(out, row, rowb, cudaMemcpyDeviceToHost));
    } else if (kv.kv_dtype == JL_I8) { // dequantised: value * its block's scale, rounded once as the kernels read it
        std::vector<char> tmp(rowb);
        JL_CUDA_CHECK(ctx, cudaMemcpy(tmp.data(), row, rowb, cudaMemcpyDeviceToHost));
        for (int i = 0; i < kv.kv_len; i++) {
            float sc;
            memcpy(&sc, tmp.data() + kv_q8_scale_off(kv.kv_len, i), 4);
            out[i] = (float)(int8_t)tmp[i] * sc;
        }
    } else {
        std::vector<uint16_t> tmp(kv.kv_len);
        JL_CUDA_CHECK(ctx, cudaMemcpy(tmp.data(), row, rowb, cudaMemcpyDeviceToHost));
        for (int i = 0; i < kv.kv_len; i++) {
            uint32_t u = ((uint32_t)tmp[i]) << 16;
            memcpy(&out[i], &u, 4);
        }
    }
    return JL_OK;
}

// DistributedContext of this model (which rows / columns of every tensor this rank holds) and its shard count
extern "C" int jl_model_tp_layout(jl_model *m, jl_dctx *out, int *tp_size) {
    if (!m || !out) return JL_ERR_INVALID;
    *out = m->d;
    if (tp_size) *tp_size = m->cfg.tp_size;
    return JL_OK;
}

extern "C" int jl_model_debug_read(jl_model *m, int which, float *out, int64_t n) {
    if (!m || !m->finalized || !out || n <= 0) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    // 8 / 9: the router probabilities (the route kernel overwrites the logits) and the selections (int32 bits) of MoE models;
    // 10 / 11: the up projection and the BF16 operand buffer (uint16 pairs per word) of tensor-core prefill models;
    // 12: the LayerNorm output of GPT-2 models (the input of the projection after a LayerNorm: c_fc after a forward, the lm_head
    // after a sampling call)
    const float *src[13] = {m->x, m->xb, m->q, m->k, m->v, m->att, m->hbuf, m->logits, m->moe_logits, (const float *)m->moe_sel, m->hbuf2,
                            (const float *)m->abf, m->cfg.arch == JL_ARCH_GPT2 ? m->ln : nullptr};
    const size_t B = m->maxB;
    size_t kmax = m->cfg.embedding_length > m->h_seg ? m->cfg.embedding_length : m->h_seg;
    if ((size_t)m->attn_seg > kmax) kmax = m->attn_seg;
    const size_t cap[13] = {B * m->cfg.embedding_length, B * m->cfg.embedding_length, B * m->attn_seg, B * m->kv_seg, B * m->kv_seg,
                            B * m->attn_seg, B * (m->n_exp > 0 ? (size_t)m->exp_k * m->cfg.hidden_length : m->h_seg),
                            (size_t)m->cfg.max_sessions * m->cfg.vocab_size, B * m->n_exp, B * m->exp_k, B * m->h_seg, B * kmax / 2,
                            B * m->cfg.embedding_length};
    if (which < 0 || which > 12 || (size_t)n > cap[which] || !src[which])
        return jl_set_error(ctx, JL_ERR_INVALID, "debug_read: bad buffer / size");
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpy(out, src[which], (size_t)n * 4, cudaMemcpyDeviceToHost));
    return JL_OK;
}

extern "C" int jl_model_read_hidden(jl_model *m, int session, float *out) {
    if (!m || !m->finalized || !out || session < 0 || session >= m->cfg.max_sessions) return JL_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> model_lock(m->mu);
    jl_ctx *ctx = m->ctx;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(m->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpy(out, m->last_hidden + (size_t)session * m->cfg.embedding_length,
                                  (size_t)m->cfg.embedding_length * 4, cudaMemcpyDeviceToHost));
    return JL_OK;
}
