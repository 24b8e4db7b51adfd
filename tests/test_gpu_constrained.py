"""Constrained decoding on the GPU (allowed-token masks in csrc/jl_penalty.cu's apply pass, DESIGN §3.18) against the numpy statement of
the rule (jlama_b200/sampling.apply_mask / select_constrained): the selection on crafted rows through jl_select_constrained (token for
token), the decode and first-token calls on the rows they hand back as logits_out, and the scheduler against one-row replays.
Importing this file does not load the CUDA library."""
import ctypes as C

import numpy as np
import pytest

from jlama_b200.native import JL_ERR_INVALID
from jlama_b200.sampling import apply_mask, apply_penalties, pack_mask, sample_topkp, select_constrained

pytestmark = [pytest.mark.gpu, pytest.mark.late]


def _rule_row(row, q):
    return row if q is None else apply_penalties(row, q.prompt, q.generated, q.presence, q.frequency, q.repetition, q.logit_bias)


def _select(ctx, rows, T, k, p, u, pens, allowed):
    from jlama_b200.model import _mask_arrays, _penalty_struct
    from jlama_b200.native import ptr
    n, V = rows.shape
    out = np.full(n, -7, np.int32)
    pen, _keep = _penalty_struct(pens if pens is not None else [None] * n, n)
    n_allow, allow, allow_row = _mask_arrays(allowed, n, V)
    rc = ctx.lib.jl_select_constrained(ctx.h, n, V, ptr(np.ascontiguousarray(rows)), V, ptr(T), ptr(k), ptr(p), ptr(u), C.addressof(pen),
                                       n_allow, ptr(allow), ptr(allow_row), ptr(out))
    return rc, out


def _want(row, q, a, T, k, p, u):
    """the token of the rule, for a constrained row or an unconstrained row at T = 0 or filtered"""
    b = _rule_row(row, q)
    if a is not None:
        return select_constrained(b, a, T, k, p, u)
    return sample_topkp(b, T, k, p, u)


# ---- 1. the selection on crafted rows -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [1, 33, 4097, 128256])
def test_select_constrained_equals_the_rule(cuda_ctx, V):
    from jlama_b200.model import RowPenalty
    rng = np.random.default_rng(V)
    singles = sorted({0, V - 1} | {e for e in (31, 32, 63, 64, 4095, 4096) if e < V})
    rows, allowed, T, k, p, u, pens = [], [], [], [], [], [], []

    def add(row, a, t=0.0, kk=0, pp=1.0, uu=0.0, q=None):
        rows.append(row), allowed.append(a), T.append(t), k.append(kk), p.append(pp), u.append(uu), pens.append(q)

    for e in singles:  # one allowed token, at the ends and at word edges, under every selection
        a = np.zeros(V, bool)
        a[e] = True
        for t, kk, pp, uu in ((0.0, 0, 1.0, 0.0), (0.9, 0, 1.0, 0.0), (0.9, 0, 1.0, 1.0), (1.3, 5, 0.5, 0.7)):
            add((rng.standard_normal(V) * 4).astype(np.float32), a, t, kk, pp, uu)
    for _ in range(6):
        row = (rng.standard_normal(V) * 4).astype(np.float32)
        a = rng.random(V) < 0.4
        a[rng.integers(0, V)] = True
        idx = np.flatnonzero(a)
        row[idx[::2]] = row[idx].max() + 1.0  # ties among the allowed tokens, above every banned one but one
        row[np.flatnonzero(~a)[:1]] = row.max() + 5.0
        n_ok = int(a.sum())
        add(row, a)                                        # greedy: the first of the tied allowed tokens
        add(row, a, 0.8, 0, 1.0, 0.0)                      # u = 0 and 1 with the integer rule
        add(row, a, 0.8, 0, 1.0, 1.0)
        add(row, a, 1.1, n_ok + 5, 1.0, float(rng.random()))  # top_k above the allowed count
        add(row, a, 0.7, 3, 0.8, float(rng.random()))
        q = RowPenalty(0.5, 0.7, 1.3, {int(idx[0]): 100.0, int(rng.integers(0, V)): -100.0}, rng.integers(0, V, 9), rng.integers(0, V, 12))
        add(row, a, 0.0, q=q)                              # penalties and bias before the mask
        add(row, a, 0.9, 0, 0.95, float(rng.random()), q=q)
        add(row, None)                                     # unconstrained neighbours: greedy and filtered
        add(row, None, 0.9, 4, 1.0, float(rng.random()), q=q)
    rows = np.stack(rows)
    T, k, p, u = (np.asarray(x, dt) for x, dt in ((T, np.float32), (k, np.int32), (p, np.float32), (u, np.float32)))
    # junk above the vocabulary in every mask word array, and rows sharing mask rows
    packed = [None if a is None else pack_mask(a) for a in allowed]
    for w in packed:
        if w is not None and V % 32:
            w[-1] |= np.uint32(~((1 << (V % 32)) - 1) & 0xFFFFFFFF)
    rc, out = _select(cuda_ctx, rows, T, k, p, u, pens, packed)
    assert rc == 0, cuda_ctx.lib.jl_last_error(cuda_ctx.h)
    for i in range(len(rows)):
        want = _want(rows[i], pens[i], allowed[i], float(T[i]), int(k[i]), float(p[i]), float(u[i]))
        assert out[i] == want, (V, i, out[i], want)
        if allowed[i] is not None:
            assert allowed[i][out[i]], (V, i)
    # the same mask row shared by many rows
    n = 9
    a = rng.random(V) < 0.5
    a[0] = True
    rows2 = (rng.standard_normal((n, V)) * 3).astype(np.float32)
    T2 = np.array([0.0, 0.9] * 4 + [0.0], np.float32)
    u2 = rng.random(n).astype(np.float32)
    rc, out = _select(cuda_ctx, rows2, T2, np.zeros(n, np.int32), np.ones(n, np.float32), u2, None, [a] * n)
    assert rc == 0 and [int(x) for x in out] == [select_constrained(rows2[i], a, float(T2[i]), 0, 1.0, float(u2[i])) for i in range(n)]


def test_select_constrained_refuses_bad_masks(cuda_ctx):
    from jlama_b200.native import ptr
    V, n = 40, 2
    rows = np.zeros((n, V), np.float32)
    z = np.zeros(n, np.float32)
    out = np.zeros(n, np.int32)
    allow = np.zeros(2 * 2, np.uint32)
    allow[2] = 1  # row 1 allows token 0; row 0 allows nothing
    allow[1] = np.uint32(0xFFFFFF00)  # bits at or above 40 only: still empty
    for n_allow, al, rows_of in ((2, allow, [0, 1]), (2, allow, [1, 2]), (2, allow, [-2, 1]), (1, None, [0, 0]), (-1, allow, [-1, -1])):
        ar = np.asarray(rows_of, np.int32)
        rc = cuda_ctx.lib.jl_select_constrained(cuda_ctx.h, n, V, ptr(rows), V, ptr(z), None, None, ptr(z), None, n_allow, ptr(al), ptr(ar),
                                                ptr(out))
        assert rc == JL_ERR_INVALID, (n_allow, rows_of)


# ---- 2. decode and first-token calls ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def models(cuda_ctx):
    """Llama `small` with Q4 and with Q8_0 weights, 64 session slots, every session prefilled; per session its prompt and first token"""
    from jlama_b200 import synth
    from jlama_b200.model import LlamaModel
    from jlama_b200.native import I8, Q4
    out = {}
    cfg = synth.get_config("small")
    for name, wdt in (("Q4", Q4), ("Q8_0", I8)):
        m = LlamaModel(cuda_ctx, cfg, synth.make_weights(cfg, wdtype=wdt), max_sessions=64, max_context=128)
        prompts, firsts = [], []
        for s in range(64):
            pr = synth.random_prompt(cfg, 3 + s % 5, seed=700 + s)
            m.reset_session(s)
            m.batch_forward(pr, 0, session=s)
            firsts.append(m.sample(session=s, want_logits=False)[0])
            prompts.append(np.asarray(pr, np.int32))
        out[name] = (m, prompts, np.array(firsts, np.int32))
    yield out
    for m, _, _ in out.values():
        m.close()


def _rows_of(n, V, seed):
    """per-row (T, k, p, u, top_n, allowed, penalty): greedy, reference-rule T, top-k / top-p rows; two in three constrained"""
    from jlama_b200.model import RowPenalty
    rng = np.random.default_rng(seed)
    T = np.array([(0.0, 0.8, 0.7, 1.2, 0.0, 0.5)[i % 6] for i in range(n)], np.float32)
    k = np.array([(0, 0, 40, 0, 5, V - 1)[i % 6] for i in range(n)], np.int32)
    p = np.array([(1.0, 1.0, 0.9, 0.5, 0.3, 0.999)[i % 6] for i in range(n)], np.float32)
    u = rng.random(n).astype(np.float32)
    tn = np.array([(5, -1, 0, 3)[i % 4] for i in range(n)], np.int32)
    allowed, pens = [], []
    for i in range(n):
        a = None
        if i % 3 != 2:
            a = rng.random(V) < (0.5, 0.02, 0.9)[i % 3]
            a[rng.integers(0, V)] = True
        allowed.append(a)
        pens.append(RowPenalty(0.4, 0.3, 1.2, {int(rng.integers(0, V)): 3.0}) if i % 4 == 1 else None)
    return T, k, p, u, tn, allowed, pens


def _check(m, toks, lg, lp, ref, ref_lg, ref_lp, T, k, p, u, allowed, pens, where):
    assert np.array_equal(lg.view(np.int32), ref_lg.view(np.int32)), where  # logits_out: the raw logits
    for i in range(len(toks)):
        w = where + (i,)
        if allowed[i] is None:  # unconstrained: the _penalized call's token and logprobs, bit for bit
            assert toks[i] == ref[i], w
            assert lp.lp[i].view(np.int32) == ref_lp.lp[i].view(np.int32), w
        else:
            assert allowed[i][toks[i]], w
            assert toks[i] == select_constrained(_rule_row(lg[i], pens[i]), allowed[i], float(T[i]), int(k[i]), float(p[i]), float(u[i])), w
        assert np.array_equal(lp.top_ids[i], ref_lp.top_ids[i]), w  # the alternatives stay those of the raw logits


@pytest.mark.parametrize("wdt", ["Q4", "Q8_0"])
@pytest.mark.parametrize("n", [1, 8, 64])
def test_decode_constrained_rows_follow_the_rule(models, wdt, n):
    m, prompts, firsts = models[wdt]
    V = m.cfg["vocab"]
    T, k, p, u, tn, allowed, pens = _rows_of(max(n, 6), V, n)
    if n == 1:
        assert wdt != "Q4" or m.decode_mode(1) == 3  # the persistent one-row path: a greedy constrained row
    T, k, p, u, tn, allowed, pens = T[:n], k[:n], p[:n], u[:n], tn[:n], allowed[:n], pens[:n]
    sess = np.arange(n, dtype=np.int32)
    pos = np.array([len(prompts[s]) for s in range(n)], np.int32)
    args = dict(sessions=sess, want_logits=True, temperatures=T, uniforms=u, top_k=k, top_p=p, logprobs=tn, penalties=pens)
    ref, ref_lg, ref_lp = m.decode(firsts[:n], pos, **args)
    toks, lg, lp = m.decode(firsts[:n], pos, allowed=allowed, **args)
    _check(m, toks, lg, lp, ref, ref_lg, ref_lp, T, k, p, u, allowed, pens, ("decode", wdt, n))
    if n == 1:  # the constraint acts on the one-row path: ban the unconstrained pick
        a = np.ones(V, bool)
        a[ref[0]] = False
        t1, lg1 = m.decode(firsts[:1], pos, sessions=sess, want_logits=True, allowed=[a])
        assert t1[0] != ref[0] and t1[0] == int(np.argmax(apply_mask(lg1[0], a)))


@pytest.mark.parametrize("wdt", ["Q4", "Q8_0"])
@pytest.mark.parametrize("n", [1, 8, 64])
def test_sample_multi_constrained_rows_follow_the_rule(models, wdt, n):
    m, prompts, firsts = models[wdt]
    V = m.cfg["vocab"]
    T, k, p, u, tn, allowed, pens = _rows_of(max(n, 6), V, 50 + n)
    T, k, p, u, tn, allowed, pens = T[:n], k[:n], p[:n], u[:n], tn[:n], allowed[:n], pens[:n]
    sess = np.arange(n, dtype=np.int32)
    ref, ref_lg, ref_lp = m.sample_multi(sess, T, u, want_logits=True, top_k=k, top_p=p, logprobs=tn, penalties=pens)
    toks, lg, lp = m.sample_multi(sess, T, u, want_logits=True, top_k=k, top_p=p, logprobs=tn, penalties=pens, allowed=allowed)
    _check(m, toks, lg, lp, ref, ref_lg, ref_lp, T, k, p, u, allowed, pens, ("sample_multi", wdt, n))


def _decode_raw(m, n, toks, pos, T, u, allow_row):
    """jl_model_decode_constrained with allow_row as given (None = NULL) and no mask rows"""
    from jlama_b200.native import ptr
    nxt = np.zeros(n, np.int32)
    sess = np.arange(n, dtype=np.int32)
    rc = m.lib.jl_model_decode_constrained(m.h, n, ptr(sess), ptr(toks), ptr(pos), ptr(T), None, None, ptr(u), None, None, 0, None,
                                           ptr(allow_row), ptr(nxt), None, None, None, None)
    return rc, nxt


def test_no_constrained_row_is_the_penalized_call_launches_included(models, cuda_ctx):
    from jlama_b200.native import ptr
    m, prompts, firsts = models["Q4"]
    for n in (1, 8, 64):
        pos = np.array([len(prompts[s]) for s in range(n)], np.int32)
        toks = np.ascontiguousarray(firsts[:n])
        T = np.array([(0.0, 0.8, 0.0, 1.1)[i % 4] for i in range(n)], np.float32)
        u = np.random.default_rng(n).random(n).astype(np.float32)
        sess = np.arange(n, dtype=np.int32)
        nxt = np.zeros(n, np.int32)
        m.lib.jl_model_decode_penalized(m.h, n, ptr(sess), ptr(toks), ptr(pos), ptr(T), None, None, ptr(u), None, None, ptr(nxt), None, None,
                                        None, None)
        a = cuda_ctx.kernel_launches()
        assert m.lib.jl_model_decode_penalized(m.h, n, ptr(sess), ptr(toks), ptr(pos), ptr(T), None, None, ptr(u), None, None, ptr(nxt), None,
                                               None, None, None) == 0
        b = cuda_ctx.kernel_launches()
        rc, t_null = _decode_raw(m, n, toks, pos, T, u, None)
        c = cuda_ctx.kernel_launches()
        assert rc == 0 and t_null.tolist() == nxt.tolist() and c - b == b - a, (n, b - a, c - b)
        rc, t_off = _decode_raw(m, n, toks, pos, T, u, np.full(n, -1, np.int32))
        d = cuda_ctx.kernel_launches()
        assert rc == 0 and t_off.tolist() == nxt.tolist() and d - c == b - a, (n, b - a, d - c)


def test_refused_calls_leave_the_kv_untouched(models):
    from jlama_b200.native import JlamaNativeError
    m, prompts, firsts = models["Q8_0"]
    V = m.cfg["vocab"]
    pos = np.array([len(prompts[s]) for s in (0, 1)], np.int32)
    before = [m.read_kv(0, int(pos[s]), w, session=s) for s in (0, 1) for w in (0, 1)]
    nxt = (firsts[:2] + 1) % V
    sess = np.array([0, 1], np.int32)
    empty = np.zeros(V, bool)
    junk = pack_mask(empty)
    if V % 32:
        junk[-1] = np.uint32(~((1 << (V % 32)) - 1) & 0xFFFFFFFF)  # bits past the vocabulary only
    for bad in ([np.ones(V, bool), empty], [junk, None]):
        with pytest.raises(JlamaNativeError) as ei:
            m.decode(nxt, pos, sessions=sess, allowed=bad)
        assert ei.value.code == JL_ERR_INVALID
        with pytest.raises(JlamaNativeError):
            m.sample_multi(sess, allowed=bad)
    for rows in ([0, 1], [-2, -1]):  # a mask row index outside [-1, n_allow) with one mask row
        from jlama_b200.native import ptr
        ar = np.asarray(rows, np.int32)
        allow = pack_mask(np.ones(V, bool))
        out = np.zeros(2, np.int32)
        rc = m.lib.jl_model_decode_constrained(m.h, 2, ptr(sess), ptr(nxt), ptr(pos), None, None, None, None, None, None, 1, ptr(allow), ptr(ar),
                                               ptr(out), None, None, None, None)
        assert rc == JL_ERR_INVALID
    rc, _ = _decode_raw(m, 2, nxt, pos, np.zeros(2, np.float32), np.zeros(2, np.float32), np.array([0, -1], np.int32))  # n_allow 0
    assert rc == JL_ERR_INVALID
    after = [m.read_kv(0, int(pos[s]), w, session=s) for s in (0, 1) for w in (0, 1)]
    assert all(np.array_equal(x, y) for x, y in zip(before, after))


# ---- 3. the scheduler ---------------------------------------------------------------------------------------------------------------
def _grammar(V, key, gen):
    h = (key * 7919 + 104729 * len(gen) + (int(gen[-1]) if len(gen) else 0)) % (1 << 31)
    a = np.random.default_rng(h).random(V) < 0.05
    a[h % V] = True
    return a


def test_scheduler_constrained_requests_equal_one_row_replays(cuda_ctx):
    from jlama_b200 import synth
    from jlama_b200.model import LlamaModel
    from jlama_b200.scheduler import SessionScheduler
    cfg = synth.get_config("small")
    V = cfg["vocab"]
    keys, calls = {}, []

    def provider(r, g):
        calls.append((r, len(g)))
        return _grammar(V, keys[r], g)

    # one slot: every call has one row, exactly the calls of a host loop over the model
    gm = LlamaModel(cuda_ctx, cfg, synth.make_weights(cfg), max_sessions=1)
    prompt = synth.random_prompt(cfg, 10, seed=951)
    with SessionScheduler(gm, mask_provider=provider) as sched:
        a = sched.submit(prompt, 12, constrained=True)
        keys[a] = 3
        sched.run()
        ta = sched.result(a)[0].tolist()
    assert calls == [(a, i) for i in range(12)]
    gm.reset_session(0)
    gm.batch_forward(prompt, 0)
    want = [int(gm.sample_multi([0], allowed=[_grammar(V, 3, [])])[0][0])]
    for i in range(1, 12):
        want.append(int(gm.decode([want[-1]], [len(prompt) + i - 1], allowed=[_grammar(V, 3, want)])[0][0]))
    assert ta == want
    gm.close()

    # eight slots: constrained requests beside unconstrained ones; every token allowed, and each the best allowed token of a one-row
    # replay's logits up to the batched-decode bar of tests/test_gpu_model.py (2e-3 of max|logit|, Q4 weights)
    gm = LlamaModel(cuda_ctx, cfg, synth.make_weights(cfg), max_sessions=8)
    rng = np.random.default_rng(9)
    reqs = []
    with SessionScheduler(gm, mask_provider=provider) as sched:
        ids = []
        for i in range(20):
            pr = synth.random_prompt(cfg, int(rng.integers(2, 8)), seed=2000 + i)
            con = i % 4 != 3
            rid = sched.submit(pr, int(rng.integers(1, 7)), constrained=con)
            keys[rid] = 100 + i
            reqs.append((pr, con, rid))
        sched.run()
        runs = [sched.result(r)[0].tolist() for _, _, r in reqs]
    for j, ((pr, con, rid), toks) in enumerate(zip(reqs, runs)):
        gm.reset_session(0)
        gm.batch_forward(pr, 0, session=0)
        lgs = [gm.sample_multi([0], want_logits=True)[1][0]]
        for i in range(1, len(toks)):
            lgs.append(gm.decode([toks[i - 1]], [len(pr) + i - 1], want_logits=True)[1][0])
        for i, lg in enumerate(lgs):
            b = apply_mask(lg, _grammar(V, 100 + j, toks[:i])) if con else lg
            assert np.isfinite(b[toks[i]]) and b[toks[i]] >= b.max() - 4e-3 * np.abs(lg).max(), (rid, i)
    gm.close()
