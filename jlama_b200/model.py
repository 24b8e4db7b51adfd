"""Host-side mirror of AbstractModel / LlamaModel (core/model/AbstractModel.java, core/model/llama/LlamaModel.java)
on top of the device-resident C++ driver (csrc/jl_model.cu, C ABI jl_model_*).

    model = LlamaModel(ctx, cfg, weights)            # ModelSupport.loadModel + registerModelTensor
    tokens = model.generate(prompt_ids, n_new)       # AbstractModel.generate at temperature 0

Sharding follows jlama-net: DistributedContext (model/DistributedContext.java:60-98) decides the row
slices of q/k/v/gate/up and the column slices of o/down (LlamaModel.java:120-133; Weights.getLoadOffsets,
safetensors/Weights.java:99-117); the slices are cut on the host and only this rank's part is uploaded.
"""
import collections
import ctypes as C

import numpy as np

from . import native
from .native import BF16, F32, I8, Q4, ptr
from .sampling import MAX_LOGPROBS


class DistributedContext:
    """model/DistributedContext.java:60-98 via the library's pure host function jl_dctx_build."""

    def __init__(self, cfg, model_shard=0, num_model_shards=1, layer_shard=0, num_layer_shards=1):
        hs = cfg["E"] // cfg["heads"]
        d = native.Dctx()
        rc = native.load().jl_dctx_build(cfg["E"], cfg["heads"] * hs, cfg["H"], hs, cfg["heads"] // cfg["kv_heads"],
                                         cfg["layers"], model_shard, num_model_shards, layer_shard, num_layer_shards,
                                         C.byref(d))
        if rc != 0:
            raise ValueError("bad shard configuration")
        for name, _ in native.Dctx._fields_:
            setattr(self, name, getattr(d, name))
        self.model_shard, self.num_model_shards = model_shard, num_model_shards


def _slice_rows(t, start, length):
    dt, data, scales = t
    return (dt, np.ascontiguousarray(data[start:start + length]),
            None if scales is None else np.ascontiguousarray(scales[start:start + length]))


def _slice_cols(t, start, length):
    """AbstractTensor.sparsify columns (core/tensor/AbstractTensor.java:151-172): copy of a column range."""
    dt, data, scales = t
    if dt == Q4:
        assert start % 32 == 0 and length % 32 == 0
        return (dt, np.ascontiguousarray(data[:, start // 2:(start + length) // 2]),
                np.ascontiguousarray(scales[:, start // 32:(start + length) // 32]))
    if dt == I8:
        return (dt, np.ascontiguousarray(data[:, start:start + length]),
                np.ascontiguousarray(scales[:, start // 32:(start + length) // 32]))
    return (dt, np.ascontiguousarray(data[:, start:start + length]), None)


def _filter_arrays(top_k, top_p, n):
    """per-row top_k (int32) / top_p (float32) arrays of a *_topkp call; None stays None (unfiltered)"""
    k = None if top_k is None else np.ascontiguousarray(np.broadcast_to(top_k, (n,)), dtype=np.int32)
    p = None if top_p is None else np.ascontiguousarray(np.broadcast_to(top_p, (n,)), dtype=np.float32)
    return k, p


TokenLogprobs = collections.namedtuple("TokenLogprobs", "lp top_ids top_lp")
TokenLogprobs.__doc__ = """Logprobs of n tokens (DESIGN §3.13): lp [n] float32 (NaN where none was asked), top_ids [n, 20] int32 and top_lp [n, 20]
float32 (the top alternatives, best first; id -1 and NaN past the count asked)."""


def _logprob_arrays(n):
    return TokenLogprobs(np.empty(n, dtype=np.float32), np.empty((n, MAX_LOGPROBS), dtype=np.int32),
                         np.empty((n, MAX_LOGPROBS), dtype=np.float32))


RowPenalty = collections.namedtuple("RowPenalty", "presence frequency repetition logit_bias prompt generated",
                                    defaults=(0.0, 0.0, 1.0, None, (), ()))
RowPenalty.__doc__ = """Penalties of one row (DESIGN §3.14): presence / frequency in [-2, 2], repetition in (0, 100], logit_bias {id: value} (or
(id, value) pairs) with values in [-100, 100], and the row's history: its prompt ids, then its generated ids (in a decode step including
the token fed in that step).  generate_sample takes one without a history."""


def _bias_pairs(logit_bias):
    pairs = list(logit_bias.items()) if isinstance(logit_bias, dict) else list(logit_bias or ())
    return np.asarray([t for t, _ in pairs], dtype=np.int32), np.asarray([v for _, v in pairs], dtype=np.float32)


def _mask_arrays(allowed, n, vocab):
    """per-row allowed sets (None = unconstrained; a bool[vocab] or packed uint32 words, DESIGN §3.18) -> (n_allow, allow
    [n_allow][words] uint32, allow_row int32[n])"""
    from .sampling import mask_words, pack_mask
    assert len(allowed) == n
    words = mask_words(vocab)
    rows, allow_row = [], np.full(n, -1, dtype=np.int32)
    for i, a in enumerate(allowed):
        if a is None:
            continue
        a = np.asarray(a)
        w = pack_mask(a) if a.dtype == bool else np.asarray(a, dtype=np.uint32).reshape(-1)
        assert len(w) == words, (i, len(w), words)
        allow_row[i] = len(rows)
        rows.append(w)
    allow = np.ascontiguousarray(np.concatenate(rows) if rows else np.zeros(words, np.uint32), dtype=np.uint32)
    return len(rows), allow, allow_row


def _penalty_struct(penalties, n):
    """per-row RowPenalty (None = unpenalised) -> (native.Penalties, the arrays it points into, to keep alive for the call)"""
    rows = [RowPenalty() if q is None else RowPenalty(*q) for q in penalties]
    assert len(rows) == n
    hist = [np.concatenate([np.asarray(q.prompt, dtype=np.int32).reshape(-1), np.asarray(q.generated, dtype=np.int32).reshape(-1)]) for q in rows]
    bias = [_bias_pairs(q.logit_bias) for q in rows]
    arrays = [np.asarray([q.presence for q in rows], dtype=np.float32), np.asarray([q.frequency for q in rows], dtype=np.float32),
              np.asarray([q.repetition for q in rows], dtype=np.float32),
              np.concatenate([[0], np.cumsum([len(h) for h in hist])]).astype(np.int32),
              np.asarray([len(q.prompt) for q in rows], dtype=np.int32), np.concatenate(hist + [np.empty(0, np.int32)]).astype(np.int32),
              np.concatenate([[0], np.cumsum([len(b[0]) for b in bias])]).astype(np.int32),
              np.concatenate([b[0] for b in bias] + [np.empty(0, np.int32)]).astype(np.int32),
              np.concatenate([b[1] for b in bias] + [np.empty(0, np.float32)]).astype(np.float32)]
    arrays = [np.ascontiguousarray(a) for a in arrays]
    return native.Penalties(*[a.ctypes.data for a in arrays]), arrays


def _select_args(n, vocab, temperatures, uniforms, top_k, top_p, logprobs, penalties, allowed):
    """The per-row selection arguments of a decode / sample_multi call, converted once for the narrowest entry point they need:
    (its suffix: "_constrained", "_penalized", "_logprobs", "_topkp" or "" for the plain one, its arguments before the token output,
    those between the token output and logits_out, the TokenLogprobs it fills or None, the arrays to keep alive for the call)."""
    t = None if temperatures is None else np.ascontiguousarray(temperatures, dtype=np.float32)
    u = None if uniforms is None else np.ascontiguousarray(uniforms, dtype=np.float32)
    assert (t is None or len(t) == n) and (u is None or len(u) == n)
    if allowed is not None:
        tier = "_constrained"
    elif penalties is not None:
        tier = "_penalized"
    elif logprobs is not None:
        tier = "_logprobs"
    elif top_k is not None or top_p is not None:
        tier = "_topkp"
    else:
        return "", (ptr(t), ptr(u)), (), None, (t, u)
    k, p = _filter_arrays(top_k, top_p, n)
    pre, keep = [ptr(t), ptr(k), ptr(p), ptr(u)], [t, u, k, p]
    if tier == "_topkp":
        return tier, pre, (), None, keep
    tn = np.ascontiguousarray(np.broadcast_to(-1 if logprobs is None else logprobs, (n,)), dtype=np.int32)
    lp = _logprob_arrays(n)
    pre.append(ptr(tn))
    keep += [tn, lp]
    if tier != "_logprobs":
        pen, arrays = _penalty_struct(penalties if penalties is not None else [None] * n, n)
        pre.append(C.addressof(pen))
        keep += [pen, arrays]
    if tier == "_constrained":
        n_allow, allow, allow_row = _mask_arrays(allowed, n, vocab)
        pre += [n_allow, ptr(allow), ptr(allow_row)]
        keep += [allow, allow_row]
    return tier, pre, (ptr(lp.lp), ptr(lp.top_ids), ptr(lp.top_lp)), lp, keep


class LlamaModel:
    def __init__(self, ctx, cfg, weights, working_qtype=I8, kv_dtype=F32, max_batch=256, max_sessions=1, max_context=0,
                 tp_rank=0, tp_size=1, flags=0, prefill_tensor_core=0):
        """kv_dtype: F32, BF16, or I8 for Q8_0 pages (int8 values with one f32 scale per 32 elements, 9/8 byte per element; DESIGN
        §3.16).  An I8 model needs tp_size 1 and decodes one session on the per-op graph rather than the persistent kernel."""
        self.ctx, self.cfg, self.lib = ctx, cfg, ctx.lib
        self.dctx = DistributedContext(cfg, tp_rank, tp_size)
        mc = native.ModelConfig(
            context_length=cfg["ctx"], embedding_length=cfg["E"], hidden_length=cfg["H"], num_heads=cfg["heads"],
            num_kv_heads=cfg["kv_heads"], num_layers=cfg["layers"], vocab_size=cfg["vocab"], head_size=cfg["E"] // cfg["heads"],
            layer_norm_eps=cfg["eps"], rope_theta=cfg["rope_theta"], rope_scaling=cfg.get("rope_scale", 1.0),
            working_qtype=working_qtype, kv_dtype=kv_dtype, max_batch=max_batch, max_sessions=max_sessions,
            max_context=max_context, tp_rank=tp_rank, tp_size=tp_size, prefill_tensor_core=prefill_tensor_core, flags=flags,
            num_experts=cfg.get("experts", 0), experts_per_token=cfg.get("experts_per_token", 0))
        h = C.c_void_p()
        ctx.check(self.lib.jl_model_create(ctx.h, C.byref(mc), C.byref(h)))
        self.h = h
        self._ids = []
        self.max_sessions = max_sessions
        try:
            self._load(ctx, cfg, weights, tp_size)
        except Exception:
            self.close()  # a rejected checkpoint must not leak the half-built model or its tensors
            raise

    @classmethod
    def from_checkpoint(cls, ctx, path, max_context=0, max_sessions=1, tp_rank=0, tp_size=1, working_qtype=I8, kv_dtype=F32,
                        flags=0, prefill_tensor_core=0, max_batch=256):
        """ModelSupport.loadModel: a Jlama checkpoint directory (config.json + model.safetensors[.index.json]) read, sharded
        and bound entirely behind the C ABI (jl_config_from_json, jl_st_open, jl_model_load_safetensors).  kv_dtype: F32, BF16 or
        I8 (Q8_0 pages, tp_size 1), as for the constructor."""
        import os
        from . import safetensors_io as sio
        mc = sio.config_from_json(os.path.join(path, "config.json"))
        mc.working_qtype, mc.kv_dtype, mc.max_batch, mc.max_sessions, mc.max_context = working_qtype, kv_dtype, max_batch, max_sessions, max_context
        mc.tp_rank, mc.tp_size, mc.flags, mc.prefill_tensor_core = tp_rank, tp_size, flags, prefill_tensor_core
        self = cls.__new__(cls)
        self.ctx, self.lib = ctx, ctx.lib
        self.cfg = dict(ctx=mc.context_length, E=mc.embedding_length, H=mc.hidden_length, heads=mc.num_heads, kv_heads=mc.num_kv_heads,
                        layers=mc.num_layers, vocab=mc.vocab_size, eps=mc.layer_norm_eps, rope_theta=mc.rope_theta, name=os.path.basename(path))
        if mc.num_experts:
            self.cfg.update(experts=mc.num_experts, experts_per_token=mc.experts_per_token)
        self.dctx = DistributedContext(self.cfg, tp_rank, tp_size)
        self.max_sessions = max_sessions
        self._ids = []
        h = C.c_void_p()
        ctx.check(self.lib.jl_model_create(ctx.h, C.byref(mc), C.byref(h)))
        self.h = h
        try:
            with sio.SafeTensors(path) as st:
                cap = (16 + 3 * mc.num_experts) * mc.num_layers + 8
                ids = (C.c_int64 * cap)()
                n = C.c_int()
                rc = self.lib.jl_model_load_safetensors(self.h, ctx.h, st.h, ids, cap, C.byref(n))
                self._ids = [ids[i] for i in range(min(n.value, cap))]
                ctx.check(rc)
            ctx.check(self.lib.jl_model_finalize(self.h))
        except Exception:
            self.close()
            raise
        return self

    def _load(self, ctx, cfg, weights, tp_size):
        if callable(weights):
            get = weights
        else:
            get = weights.get
        d = self.dctx

        def put(layer, slot, name, shard=None):
            t = get(name)
            if t is None:
                return False
            if shard == "rows_attn":
                t = _slice_rows(t, d.attentionSegmentStart, d.attentionSegmentLength)
            elif shard == "rows_kv":
                t = _slice_rows(t, d.kvSegmentStart, d.kvSegmentLength)
            elif shard == "rows_hidden":
                t = _slice_rows(t, d.hiddenSegmentStart, d.hiddenSegmentLength)
            elif shard == "cols_attn":
                t = _slice_cols(t, d.attentionSegmentStart, d.attentionSegmentLength)
            elif shard == "cols_hidden":
                t = _slice_cols(t, d.hiddenSegmentStart, d.hiddenSegmentLength)
            dt, data, scales = t
            rows = data.shape[0]
            cols = data.shape[1] * (2 if dt == Q4 else 1)
            tid = self.lib.jl_register_tensor(ctx.h, dt, rows, cols, ptr(data), ptr(scales))
            if tid < 0:
                raise native.JlamaNativeError(-1, self.lib.jl_last_error(ctx.h).decode())
            self._ids.append(tid)
            ctx.check(self.lib.jl_model_set_tensor(self.h, layer, slot, tid))
            return True

        def put_expert(layer, expert, which, name):
            dt, data, scales = get(name)
            rows = data.shape[0]
            cols = data.shape[1] * (2 if dt == Q4 else 1)
            tid = self.lib.jl_register_tensor(ctx.h, dt, rows, cols, ptr(data), ptr(scales))
            if tid < 0:
                raise native.JlamaNativeError(-1, self.lib.jl_last_error(ctx.h).decode())
            self._ids.append(tid)
            ctx.check(self.lib.jl_model_set_expert_tensor(self.h, layer, expert, which, tid))

        sharded = tp_size > 1
        put(-1, native.T_EMBED, "model.embed_tokens.weight")
        put(-1, native.T_OUT_NORM, "model.norm.weight")
        put(-1, native.T_LM_HEAD, "lm_head.weight")
        for i in range(cfg["layers"]):
            b = "model.layers.%d." % i
            put(i, native.L_ATTN_NORM, b + "input_layernorm.weight")
            put(i, native.L_Q, b + "self_attn.q_proj.weight", "rows_attn" if sharded else None)
            put(i, native.L_K, b + "self_attn.k_proj.weight", "rows_kv" if sharded else None)
            put(i, native.L_V, b + "self_attn.v_proj.weight", "rows_kv" if sharded else None)
            put(i, native.L_O, b + "self_attn.o_proj.weight", "cols_attn" if sharded else None)
            put(i, native.L_FFN_NORM, b + "post_attention_layernorm.weight")
            if cfg.get("experts"):  # MixtralModel.java:88-105
                put_expert(i, -1, 0, b + "block_sparse_moe.gate.weight")
                for e in range(cfg["experts"]):
                    if e % tp_size != self.dctx.model_shard:
                        continue  # expert parallelism: expert e lives (whole) on rank e % tp_size
                    for which, nm in ((0, "w1"), (1, "w2"), (2, "w3")):
                        put_expert(i, e, which, b + "block_sparse_moe.experts.%d.%s.weight" % (e, nm))
                continue
            put(i, native.L_GATE, b + "mlp.gate_proj.weight", "rows_hidden" if sharded else None)
            put(i, native.L_DOWN, b + "mlp.down_proj.weight", "cols_hidden" if sharded else None)
            put(i, native.L_UP, b + "mlp.up_proj.weight", "rows_hidden" if sharded else None)
        ctx.check(self.lib.jl_model_finalize(self.h))

    # -- AbstractModel API ---------------------------------------------------------------------------
    def reset_session(self, session=0):
        self.ctx.check(self.lib.jl_model_reset_session(self.h, session))

    def batch_forward(self, tokens, start_pos=0, session=0):
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        self.ctx.check(self.lib.jl_model_batch_forward(self.h, session, ptr(tokens), len(tokens), start_pos))

    def sample(self, session=0, temperature=0.0, uniform=0.0, want_logits=True):
        tok = C.c_int32()
        logits = np.empty(self.cfg["vocab"], dtype=np.float32) if want_logits else None
        self.ctx.check(self.lib.jl_model_sample(self.h, session, C.c_float(temperature), C.c_float(uniform), C.byref(tok),
                                                ptr(logits)))
        return tok.value, logits

    def batch_forward_multi(self, segments):
        """AbstractModel.batchForward for several sessions in shared passes: segments = [(session, tokens, start_pos), ...], sessions
        distinct.  Tensor-core chunks come out bit-identical to batch_forward of the same segment."""
        sessions = np.ascontiguousarray([s for s, _, _ in segments], dtype=np.int32)
        starts = np.ascontiguousarray([p for _, _, p in segments], dtype=np.int32)
        lengths = np.ascontiguousarray([len(t) for _, t, _ in segments], dtype=np.int32)
        tokens = np.ascontiguousarray(np.concatenate([np.asarray(t, dtype=np.int32) for _, t, _ in segments]) if segments else [], dtype=np.int32)
        self.ctx.check(self.lib.jl_model_batch_forward_multi(self.h, len(segments), ptr(sessions), ptr(starts), ptr(lengths), ptr(tokens)))

    def sample_multi(self, sessions, temperatures=None, uniforms=None, want_logits=False, top_k=None, top_p=None, logprobs=None,
                     penalties=None, allowed=None):
        """AbstractModel.sample on the last forwarded row of each session, in one lm_head pass; rows with a temperature other than 0
        draw with the reference's rule from uniforms[i], or with the top-k / top-p rule (DESIGN §3.12) when top_k / top_p (per row)
        filter them.  Returns (tokens, raw logits [n, vocab] or None); with logprobs (an int or one per row: -1 none, 0 the chosen
        token's, up to 20 alternatives; DESIGN §3.13) also a TokenLogprobs of the chosen tokens.  penalties: one RowPenalty (or None)
        per row (DESIGN §3.14); each row is then selected from its processed logits.  allowed: per row None or the allowed-token set
        (a bool[vocab] or packed uint32 words, DESIGN §3.18) the row is selected under; logits and logprobs stay those of the raw logits."""
        sessions = np.ascontiguousarray(sessions, dtype=np.int32)
        n = len(sessions)
        out = np.empty(n, dtype=np.int32)
        logits = np.empty((n, self.cfg["vocab"]), dtype=np.float32) if want_logits else None
        tier, pre, post, lp, _keep = _select_args(n, self.cfg["vocab"], temperatures, uniforms, top_k, top_p, logprobs, penalties, allowed)
        call = getattr(self.lib, "jl_model_sample_multi" + tier)
        self.ctx.check(call(self.h, n, ptr(sessions), *pre, ptr(out), *post, ptr(logits)))
        return (out, logits) if logprobs is None else (out, logits, lp)

    def decode(self, tokens, positions, sessions=None, want_logits=False, temperatures=None, uniforms=None, top_k=None, top_p=None,
               logprobs=None, penalties=None, allowed=None):
        """One decode step for n sessions.  temperatures / uniforms (per row): rows with a temperature other than 0 are sampled with
        AbstractModel.sample's rule (:475-489) from their logits row, the others take the arg-max.  top_k / top_p (per row, optional):
        rows with a temperature above 0 that they filter are drawn with the top-k / top-p rule (DESIGN §3.12) instead.  Returns
        (next tokens, logits or None); with logprobs (an int or one per row, as in sample_multi) also a TokenLogprobs of the chosen
        tokens.  penalties: one RowPenalty (or None) per row (DESIGN §3.14); logits and logprobs stay those of the raw logits.  allowed:
        per row None or the allowed-token set the row is selected under (as in sample_multi; DESIGN §3.18)."""
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        positions = np.ascontiguousarray(positions, dtype=np.int32)
        n = len(tokens)
        sessions = np.arange(n, dtype=np.int32) if sessions is None else np.ascontiguousarray(sessions, dtype=np.int32)
        nxt = np.empty(n, dtype=np.int32)
        logits = np.empty((n, self.cfg["vocab"]), dtype=np.float32) if want_logits else None
        tier, pre, post, lp, _keep = _select_args(n, self.cfg["vocab"], temperatures, uniforms, top_k, top_p, logprobs, penalties, allowed)
        rows = (self.h, n, ptr(sessions), ptr(tokens), ptr(positions))
        if not tier and temperatures is None:
            self.ctx.check(self.lib.jl_model_decode(*rows, ptr(nxt), ptr(logits)))
        else:
            call = getattr(self.lib, "jl_model_decode" + ("_sample" + tier if tier in ("", "_topkp") else tier))
            self.ctx.check(call(*rows, *pre, ptr(nxt), *post, ptr(logits)))
        return (nxt, logits) if logprobs is None else (nxt, logits, lp)

    def score_multi(self, segments, top_n=0):
        """batch_forward_multi that also scores the tokens (DESIGN §3.13): segments = [(session, tokens, start_pos), ...].  Returns one
        TokenLogprobs per segment: entry k is the logprob of tokens[k] given everything before it in the session, with top_n (0..20)
        alternatives; entry 0 is NaN with id -1.  KV and the last hidden rows are exactly those batch_forward_multi leaves."""
        sessions = np.ascontiguousarray([s for s, _, _ in segments], dtype=np.int32)
        starts = np.ascontiguousarray([p for _, _, p in segments], dtype=np.int32)
        lengths = np.ascontiguousarray([len(t) for _, t, _ in segments], dtype=np.int32)
        tokens = np.ascontiguousarray(np.concatenate([np.asarray(t, dtype=np.int32) for _, t, _ in segments]) if segments else [], dtype=np.int32)
        lp = _logprob_arrays(len(tokens))
        self.ctx.check(self.lib.jl_model_score_multi(self.h, len(segments), ptr(sessions), ptr(starts), ptr(lengths), ptr(tokens), int(top_n),
                                                     ptr(lp.lp), ptr(lp.top_ids), ptr(lp.top_lp)))
        cut = np.cumsum(lengths)[:-1]
        return [TokenLogprobs(*parts) for parts in zip(*(np.split(a, cut) for a in lp))]

    def score(self, tokens, start_pos=0, session=0, top_n=0):
        """score_multi of one segment: a TokenLogprobs of the tokens"""
        return self.score_multi([(session, tokens, start_pos)], top_n)[0]

    def decode_resident(self, first_token, start_pos, n_new, session=0):
        out = np.empty(n_new, dtype=np.int32)
        self.ctx.check(self.lib.jl_model_decode_resident(self.h, session, int(first_token), start_pos, n_new, ptr(out)))
        return out

    def generate(self, prompt, n_new, session=0, want_logits=False):
        prompt = np.ascontiguousarray(prompt, dtype=np.int32)
        out = np.empty(n_new, dtype=np.int32)
        logits = np.empty((n_new, self.cfg["vocab"]), dtype=np.float32) if want_logits else None
        tm = (C.c_double * 2)()
        self.ctx.check(self.lib.jl_model_generate(self.h, session, ptr(prompt), len(prompt), n_new, ptr(out), ptr(logits), tm))
        self.last_timings_ms = (tm[0], tm[1])
        return out, logits

    def generate_sample(self, prompt, n_new, temperature, uniforms, session=0, top_k=None, top_p=None, logprobs=None, penalties=None):
        """AbstractModel.generate with a temperature; uniforms[i] stands for the i-th ThreadLocalRandom.nextFloat() of the loop.  With
        top_k / top_p every token is drawn with the top-k / top-p rule (DESIGN §3.12).  With logprobs (one int for every token) returns
        (tokens, TokenLogprobs).  penalties: one RowPenalty (its history ignored) for every token (DESIGN §3.14); token k's history is the
        prompt and the k tokens before it."""
        prompt = np.ascontiguousarray(prompt, dtype=np.int32)
        u = np.ascontiguousarray(uniforms, dtype=np.float32)
        assert len(u) >= n_new
        out = np.empty(n_new, dtype=np.int32)
        lp = _logprob_arrays(n_new)
        head = (self.h, session, ptr(prompt), len(prompt), n_new, C.c_float(temperature))
        filt = (int(top_k or 0), C.c_float(1.0 if top_p is None else top_p), ptr(u))
        lp_out = (ptr(lp.lp), ptr(lp.top_ids), ptr(lp.top_lp))
        top_n = -1 if logprobs is None else int(logprobs)
        if penalties is not None:
            q = RowPenalty(*penalties)
            bi, bv = _bias_pairs(q.logit_bias)
            self.ctx.check(self.lib.jl_model_generate_penalized(*head, *filt, top_n, C.c_float(q.presence), C.c_float(q.frequency),
                                                                C.c_float(q.repetition), len(bi), ptr(bi), ptr(bv), ptr(out), *lp_out, None))
        elif logprobs is not None:
            self.ctx.check(self.lib.jl_model_generate_logprobs(*head, *filt, top_n, ptr(out), *lp_out, None))
        elif top_k is None and top_p is None:
            self.ctx.check(self.lib.jl_model_generate_sample(*head, ptr(u), ptr(out), None))
        else:
            self.ctx.check(self.lib.jl_model_generate_sample_topkp(*head, *filt, ptr(out), None))
        return out if logprobs is None else (out, lp)

    def kv_save(self, directory, session_name, session=0):
        """KvBufferCache.KvBufferPage persistence: <directory>/<session_name>-L<l>C<c>.page files; returns the page count."""
        n = self.lib.jl_model_kv_save(self.h, session, str(directory).encode(), str(session_name).encode())
        if n < 0:
            self.ctx.check(n)
        return n

    def kv_load(self, directory, session_name, session=0):
        n = self.lib.jl_model_kv_load(self.h, session, str(directory).encode(), str(session_name).encode())
        if n < 0:
            self.ctx.check(n)
        return n

    def kv_offload(self, session=0):
        """Move the session's KV pages to host memory and free their HBM; returns the handle kv_restore takes."""
        h = self.lib.jl_model_kv_offload(self.h, session)
        if h < 0:
            self.ctx.check(int(h))
        return h

    def kv_restore(self, handle, session=0):
        self.ctx.check(self.lib.jl_model_kv_restore(self.h, session, handle))

    def kv_discard(self, handle):
        self.ctx.check(self.lib.jl_model_kv_discard(self.h, handle))

    def kv_pages(self, session=0):
        return int(self.lib.jl_model_kv_pages(self.h, session))

    def kv_fork(self, src, dst, positions):
        """Each session in dst becomes what src holds for positions [0, positions): whole pages are shared copy-on-write, the page
        holding positions - 1 is copied, and sampling on dst draws from src's last forwarded row (DESIGN §3.15)."""
        d = np.ascontiguousarray(list(dst), dtype=np.int32)
        self.ctx.check(self.lib.jl_model_kv_fork(self.h, src, positions, len(d), ptr(d)))

    def kv_retain(self, positions, session=0):
        """Hold the session's pages wholly below `positions` (a multiple of ctx_per_page) beyond the session's life; returns the handle
        kv_attach and kv_release take (DESIGN §3.17)."""
        h = self.lib.jl_model_kv_retain(self.h, session, positions)
        if h < 0:
            self.ctx.check(int(h))
        return h

    def kv_attach(self, handle, positions, session=0):
        """The session becomes what `handle` holds for [0, positions): its entries point at the retained pages, no bytes move.  Forward
        at least one token before sampling."""
        self.ctx.check(self.lib.jl_model_kv_attach(self.h, handle, positions, session))

    def kv_release(self, handle):
        self.ctx.check(self.lib.jl_model_kv_release(self.h, handle))

    def kv_retained(self):
        """(handles alive, pages held by handles and by no session)"""
        n, p = C.c_int64(), C.c_int64()
        self.ctx.check(self.lib.jl_model_kv_retained(self.h, C.byref(n), C.byref(p)))
        return n.value, p.value

    def kv_page_stats(self):
        """(pages allocated, page-table entries): a page shared by k sessions counts once in the first and k times in the second"""
        a, e = C.c_int64(), C.c_int64()
        self.ctx.check(self.lib.jl_model_kv_page_stats(self.h, C.byref(a), C.byref(e)))
        return a.value, e.value

    def read_kv(self, layer, position, which, session=0):
        out = np.empty(self.dctx.kvSegmentLength, dtype=np.float32)
        self.ctx.check(self.lib.jl_model_read_kv(self.h, session, layer, position, which, ptr(out)))
        return out

    def read_hidden(self, session=0):
        out = np.empty(self.cfg["E"], dtype=np.float32)
        self.ctx.check(self.lib.jl_model_read_hidden(self.h, session, ptr(out)))
        return out

    def debug_read(self, which, n):
        """Test hook: internal activation buffer of the last forward/decode call (0 x, 1 xb, 2 q, 3 k, 4 v, 5 att, 6 h, 7 logits).
        Mixture-of-experts models: h holds one row per (row, selected expert), expert i of row b at row b * experts_per_token + i;
        8 is the router probabilities [rows, experts] and 9 the selected experts [rows, experts_per_token] (int32 bits: .view(np.int32)).
        Tensor-core prefill models (prefill_tensor_core=1): 10 is the up projection [rows, H] (h holds the gate projection there),
        and 11 the BF16 operand buffer of the last GEMM, n float words of two BF16 each (.view(np.uint16)); after a tensor-core pass
        it holds bf16(silu(gate) * up) of the last layer [rows, H], down_proj's input.  Other models refuse 10 and 11.
        GPT-2 models: 12 is the LayerNorm output [rows, E]; after batch_forward / batch_forward_multi it holds ln_2 of the last layer
        (the c_fc input), after decode / sample / sample_multi ln_f of the sampled rows (the lm_head input).  Other models refuse 12."""
        out = np.empty(n, dtype=np.float32)
        self.ctx.check(self.lib.jl_model_debug_read(self.h, which, ptr(out), n))
        return out

    def decode_mode(self, n=1):
        return int(self.lib.jl_model_decode_mode(self.h, n))

    def weight_bytes(self):
        return int(self.lib.jl_model_weight_bytes(self.h))

    def last_timing(self):
        a, b = C.c_double(), C.c_double()
        self.lib.jl_model_last_timing(self.h, C.byref(a), C.byref(b))
        return a.value, b.value

    def close(self):
        if self.h:
            self.lib.jl_model_free(self.h)
            self.h = None
            for tid in self._ids:
                self.lib.jl_unregister_tensor(self.ctx.h, tid)
            self._ids = []


class GPT2Model(LlamaModel):
    """core/model/gpt2/GPT2Model.java:54-129 behind the same C ABI (jl_model_config.arch = JL_ARCH_GPT2): wte + wpe embeddings, LayerNorm
    with bias, biased projections, GELU MLP, no rotary embedding, logits over wte.  `weights` holds the checkpoint in its file layout
    (Hugging Face Conv1D: c_attn / c_fc / c_proj weights are [in, out]); like the reference's loader this class transposes them and
    splits c_attn into q, k, v (GPT2Model.java:79-80).  BASELINE config 1 (GPT-2-small F32).  kv_dtype: F32, BF16 or I8 (Q8_0 pages,
    DESIGN §3.16)."""

    def __init__(self, ctx, cfg, weights, working_qtype=native.F32, kv_dtype=F32, max_batch=256, max_sessions=1, max_context=0, flags=0):
        self.ctx, self.cfg, self.lib = ctx, cfg, ctx.lib
        self.dctx = DistributedContext(cfg, 0, 1)
        mc = native.ModelConfig(
            context_length=cfg["ctx"], embedding_length=cfg["E"], hidden_length=cfg["H"], num_heads=cfg["heads"], num_kv_heads=cfg["heads"],
            num_layers=cfg["layers"], vocab_size=cfg["vocab"], head_size=cfg["E"] // cfg["heads"], layer_norm_eps=cfg["eps"], rope_theta=10000.0,
            rope_scaling=1.0, working_qtype=working_qtype, kv_dtype=kv_dtype, max_batch=max_batch, max_sessions=max_sessions,
            max_context=max_context, tp_rank=0, tp_size=1, prefill_tensor_core=0, flags=flags, num_experts=0, experts_per_token=0,
            arch=native.ARCH_GPT2)
        h = C.c_void_p()
        ctx.check(self.lib.jl_model_create(ctx.h, C.byref(mc), C.byref(h)))
        self.h = h
        self._ids = []
        self.max_sessions = max_sessions
        try:
            self._load_gpt2(ctx, cfg, weights)
        except Exception:
            self.close()
            raise

    def _load_gpt2(self, ctx, cfg, weights):
        get = weights if callable(weights) else weights.get
        E = cfg["E"]

        def reg(a):
            a = np.ascontiguousarray(a, dtype=np.float32)
            a = a.reshape(1, -1) if a.ndim == 1 else a
            tid = self.lib.jl_register_tensor(ctx.h, F32, a.shape[0], a.shape[1], ptr(a), None)
            if tid < 0:
                raise native.JlamaNativeError(-1, self.lib.jl_last_error(ctx.h).decode())
            self._ids.append(tid)
            return tid

        def w(name):
            return get(name)[1]  # (dtype, data, scales)

        ctx.check(self.lib.jl_model_set_tensor(self.h, -1, native.T_EMBED, reg(w("wte.weight"))))
        ctx.check(self.lib.jl_model_set_aux_tensor(self.h, -1, native.AUX_POS_EMBED, reg(w("wpe.weight"))))
        ctx.check(self.lib.jl_model_set_tensor(self.h, -1, native.T_OUT_NORM, reg(w("ln_f.weight"))))
        ctx.check(self.lib.jl_model_set_aux_tensor(self.h, -1, native.AUX_OUT_NORM_BIAS, reg(w("ln_f.bias"))))
        for i in range(cfg["layers"]):
            b = "h.%d." % i
            st, sa = (lambda slot, a: ctx.check(self.lib.jl_model_set_tensor(self.h, i, slot, reg(a)))), \
                     (lambda slot, a: ctx.check(self.lib.jl_model_set_aux_tensor(self.h, i, slot, reg(a))))
            st(native.L_ATTN_NORM, w(b + "ln_1.weight"))
            sa(native.AUX_ATTN_NORM_BIAS, w(b + "ln_1.bias"))
            wq, wk, wv = np.split(w(b + "attn.c_attn.weight").T, 3, axis=0)  # .transpose().split(3, 0)
            bq, bk, bv = np.split(w(b + "attn.c_attn.bias").reshape(-1), 3)    # .split(3, 1)
            st(native.L_Q, wq), st(native.L_K, wk), st(native.L_V, wv)
            sa(native.AUX_Q_BIAS, bq), sa(native.AUX_K_BIAS, bk), sa(native.AUX_V_BIAS, bv)
            st(native.L_O, w(b + "attn.c_proj.weight").T)
            sa(native.AUX_O_BIAS, w(b + "attn.c_proj.bias"))
            st(native.L_FFN_NORM, w(b + "ln_2.weight"))
            sa(native.AUX_FFN_NORM_BIAS, w(b + "ln_2.bias"))
            st(native.L_GATE, w(b + "mlp.c_fc.weight").T)
            sa(native.AUX_FC_BIAS, w(b + "mlp.c_fc.bias"))
            st(native.L_DOWN, w(b + "mlp.c_proj.weight").T)
            sa(native.AUX_PROJ_BIAS, w(b + "mlp.c_proj.bias"))
        ctx.check(self.lib.jl_model_finalize(self.h))
