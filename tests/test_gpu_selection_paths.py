"""The selection after the logits is one pass behind every sampling entry point (jl_model.cu: select_check, select_pass).  Two things pin
it: jl_select_constrained, the host-buffer hook the edge tests use, picks the tokens a model call picks from the same rows; and each entry
point validates what it takes, so a negative temperature reaches the reference rule on the plain calls and is refused before any kernel
launch on every wider one.  Importing this file does not load the CUDA library."""
import ctypes as C

import numpy as np
import pytest

from jlama_b200.native import JL_ERR_INVALID

pytestmark = pytest.mark.gpu

KINDS = ("greedy", "reference", "filtered", "penalised greedy", "penalised reference", "constrained greedy", "constrained sampled",
         "constrained penalised")


@pytest.fixture(scope="module")
def model(cuda_ctx):
    """Llama `small` (Q4), 64 session slots, every session prefilled; per session its prompt and first token"""
    from jlama_b200 import synth
    from jlama_b200.model import LlamaModel
    cfg = synth.get_config("small")
    m = LlamaModel(cuda_ctx, cfg, synth.make_weights(cfg), max_sessions=64, max_context=128)
    prompts, firsts = [], []
    for s in range(64):
        pr = synth.random_prompt(cfg, 3 + s % 7, seed=1300 + s)
        m.reset_session(s)
        m.batch_forward(pr, 0, session=s)
        firsts.append(m.sample(session=s, want_logits=False)[0])
        prompts.append(np.asarray(pr, np.int32))
    yield m, prompts, np.array(firsts, np.int32)
    m.close()


def _rows(n, V, prompts, firsts, seed):
    """per-row (T, k, p, u, allowed, penalty), row i of kind KINDS[i % 8]"""
    from jlama_b200.model import RowPenalty
    rng = np.random.default_rng(seed)
    T, k, p, allowed, pens = [], [], [], [], []
    for i in range(n):
        kind = KINDS[i % len(KINDS)]
        sampled = kind not in ("greedy", "penalised greedy", "constrained greedy")
        T.append((0.7, 1.1, 0.9)[i % 3] if sampled else 0.0)
        k.append(40 if kind == "filtered" else 0)
        p.append(0.9 if kind == "filtered" else 1.0)
        a = None
        if kind.startswith("constrained"):
            a = rng.random(V) < 0.3
            a[rng.integers(0, V)] = True
        allowed.append(a)
        q = None
        if kind.startswith("penalised") or kind == "constrained penalised":
            q = RowPenalty(0.5, 0.4, 1.3, {int(rng.integers(0, V)): 4.0, int(rng.integers(0, V)): -3.0}, prompts[i], [int(firsts[i])])
        pens.append(q)
    u = rng.random(n).astype(np.float32)
    return np.array(T, np.float32), np.array(k, np.int32), np.array(p, np.float32), u, allowed, pens


def _select_host(ctx, rows, T, k, p, u, pens, allowed):
    from jlama_b200.model import _mask_arrays, _penalty_struct
    from jlama_b200.native import ptr
    n, V = rows.shape
    out = np.full(n, -7, np.int32)
    pen, _keep = _penalty_struct(pens, n)
    n_allow, allow, allow_row = _mask_arrays(allowed, n, V)
    rc = ctx.lib.jl_select_constrained(ctx.h, n, V, ptr(np.ascontiguousarray(rows)), V, ptr(T), ptr(k), ptr(p), ptr(u), C.addressof(pen),
                                       n_allow, ptr(allow), ptr(allow_row), ptr(out))
    return rc, out


@pytest.mark.parametrize("logprobs", [None, 3])
@pytest.mark.parametrize("n", [8, 64])
def test_host_hook_picks_the_tokens_of_the_model_call(model, cuda_ctx, n, logprobs):
    m, prompts, firsts = model
    V = m.cfg["vocab"]
    T, k, p, u, allowed, pens = _rows(n, V, prompts, firsts, 40 + n)
    pos = np.array([len(prompts[s]) for s in range(n)], np.int32)
    res = m.decode(firsts[:n], pos, sessions=np.arange(n, dtype=np.int32), want_logits=True, temperatures=T, uniforms=u, top_k=k,
                   top_p=p, logprobs=logprobs, penalties=pens, allowed=allowed)
    toks, lg = res[0], res[1]
    rc, out = _select_host(cuda_ctx, lg, T, k, p, u, pens, allowed)
    assert rc == 0, cuda_ctx.lib.jl_last_error(cuda_ctx.h)
    bad = [(i, KINDS[i % len(KINDS)], int(toks[i]), int(out[i])) for i in range(n) if toks[i] != out[i]]
    assert not bad, bad
    for i, a in enumerate(allowed):
        if a is not None:
            assert a[toks[i]], i


def test_negative_temperature_reaches_the_plain_calls_only(model, cuda_ctx):
    from jlama_b200.native import JlamaNativeError
    m, prompts, firsts = model
    V = m.cfg["vocab"]
    n = 4
    sess = np.arange(n, dtype=np.int32)
    pos = np.array([len(prompts[s]) for s in range(n)], np.int32)
    T = np.array([0.0, -0.5, 0.8, 0.0], np.float32)
    u = np.array([0.1, 0.6, 0.3, 0.9], np.float32)
    # the plain calls: the reference rule takes the row
    toks, _ = m.decode(firsts[:n], pos, sessions=sess, temperatures=T, uniforms=u)
    assert all(0 <= t < V for t in toks), toks
    toks, _ = m.sample_multi(sess, T, u)
    assert all(0 <= t < V for t in toks), toks
    # every wider call refuses it before any kernel launch
    wider = {"topkp": dict(top_k=np.zeros(n, np.int32)), "logprobs": dict(logprobs=0), "penalized": dict(penalties=[None] * n),
             "constrained": dict(allowed=[np.ones(V, bool)] + [None] * (n - 1))}
    for name, extra in wider.items():
        for call in (lambda: m.decode(firsts[:n], pos, sessions=sess, temperatures=T, uniforms=u, **extra),
                     lambda: m.sample_multi(sess, T, u, **extra)):
            before = cuda_ctx.kernel_launches()
            with pytest.raises(JlamaNativeError) as ei:
                call()
            assert ei.value.code == JL_ERR_INVALID, name
            assert cuda_ctx.kernel_launches() == before, name
