"""Constrained requests in the native scheduler (DESIGN §3.18), on CPU: a toy backend whose tokens follow the rule on the logits of the
history (penalties, then the allowed-token mask), and the CPU oracle as the device.  The mask provider stands in for a grammar engine:
it is called once before every selection of a constrained request with the tokens that request has generated, and every token it
emits must be allowed.  Requests must come out as they would alone, and unconstrained neighbours exactly as without constrained ones."""
import numpy as np
import pytest

from jlama_b200 import native, synth
from jlama_b200.sampling import apply_mask, apply_penalties, pack_mask, sample_topkp
from jlama_b200.scheduler import SessionScheduler

VOCAB = 45  # two mask words, the second one partly past the vocabulary
STOP = 44


def _toy_logits(history):
    h = 1469598103934665603
    for t in history:
        h = ((h ^ (int(t) + 1)) * 1099511628211) % (1 << 64)
    return (np.random.default_rng(h).standard_normal(VOCAB) * 2).astype(np.float32)


def grammar(key, generated):
    """a toy automaton: the allowed set after `generated`, a function of the request's key and its tokens so far.  Key k >= 100 ends after
    k - 100 tokens by allowing only STOP."""
    if key >= 100 and len(generated) >= key - 100:
        a = np.zeros(VOCAB, bool)
        a[STOP] = True
        return a
    h = (key * 1000003 + 7919 * len(generated) + (int(generated[-1]) if len(generated) else 0)) % (1 << 31)
    a = np.random.default_rng(h).random(VOCAB) < 0.3
    a[h % (VOCAB - 1)] = True  # never empty; STOP only as a random member
    return a


class Toy:
    """Sessions are token histories; every selection follows the rule on the toy logits of the session's history."""

    def __init__(self, n_sessions, max_rows):
        self.hist = [None] * n_sessions
        self.max_rows = max_rows
        self.calls, self.spilled = [], {}

    def reset_session(self, s):
        self.hist[s] = []

    def batch_forward(self, s, tokens, start_pos):
        assert start_pos == len(self.hist[s])
        self.hist[s].extend(int(t) for t in tokens)

    def forward_multi(self, sessions, start_pos, lengths, tokens):
        off = 0
        for s, p, n in zip(sessions.tolist(), start_pos.tolist(), lengths.tolist()):
            self.batch_forward(s, tokens[off:off + n], p)
            off += n

    def offload(self, s):
        h = len(self.spilled) + 100
        self.spilled[h] = self.hist[s]
        self.hist[s] = None
        return h

    def restore(self, s, h):
        self.hist[s] = self.spilled.pop(h)

    def discard(self, h):
        self.spilled.pop(h, None)

    def _rows(self, name, sessions, tokens, positions, temps, ks, ps, unis, pens=None, allowed=None):
        n = len(sessions)
        assert 1 <= n <= self.max_rows
        self.calls.append((name, tuple(sessions.tolist())))
        if tokens is not None:
            for s, t, pos in zip(sessions.tolist(), tokens.tolist(), positions.tolist()):
                assert pos == len(self.hist[s])
                self.hist[s].append(t)
        out = []
        for i, s in enumerate(sessions.tolist()):
            b = _toy_logits(self.hist[s])
            q = pens[i] if pens else None
            if q is not None:
                b = apply_penalties(b, q.prompt, q.generated, q.presence, q.frequency, q.repetition, q.logit_bias)
            if allowed is not None and allowed[i] is not None:
                b = apply_mask(b, allowed[i])
            out.append(sample_topkp(b, float(temps[i]), int(ks[i]) if ks is not None else 0, float(ps[i]) if ps is not None else 1.0,
                                    float(unis[i])))
        return out

    def _lp(self, n, toks):
        return toks, np.full(n, np.nan, np.float32), np.full((n, 20), -1, np.int32), np.full((n, 20), np.nan, np.float32)

    def sample(self, s, T, u):
        return self._rows("sample", np.array([s]), None, None, np.array([T]), None, None, np.array([u], np.float32))[0]

    def sample_multi(self, sessions, temps, unis):
        return self._rows("sample_multi", sessions, None, None, temps, None, None, unis)

    def sample_multi_topkp(self, sessions, temps, ks, ps, unis):
        return self._rows("sample_multi_topkp", sessions, None, None, temps, ks, ps, unis)

    def sample_multi_penalized(self, sessions, temps, ks, ps, unis, top_n, pens):
        return self._lp(len(sessions), self._rows("sample_multi_penalized", sessions, None, None, temps, ks, ps, unis, pens))

    def sample_multi_constrained(self, sessions, temps, ks, ps, unis, top_n, pens, allowed):
        return self._lp(len(sessions), self._rows("sample_multi_constrained", sessions, None, None, temps, ks, ps, unis, pens, allowed))

    def decode(self, sessions, tokens, positions, temps, unis):
        return self._rows("decode", sessions, tokens, positions, temps, None, None, unis)

    def decode_topkp(self, sessions, tokens, positions, temps, ks, ps, unis):
        return self._rows("decode_topkp", sessions, tokens, positions, temps, ks, ps, unis)

    def decode_penalized(self, sessions, tokens, positions, temps, ks, ps, unis, top_n, pens):
        return self._lp(len(sessions), self._rows("decode_penalized", sessions, tokens, positions, temps, ks, ps, unis, pens))

    def decode_constrained(self, sessions, tokens, positions, temps, ks, ps, unis, top_n, pens, allowed):
        return self._lp(len(sessions), self._rows("decode_constrained", sessions, tokens, positions, temps, ks, ps, unis, pens, allowed))


class Provider:
    """the grammar engine: request id -> key (set by the test after submit), a log of every call, optional failures"""

    def __init__(self):
        self.keys, self.log = {}, []
        self.fail, self.empty = set(), set()
        self.on_call = None

    def __call__(self, request, generated):
        self.log.append((request, [int(t) for t in generated]))
        if self.on_call:
            self.on_call(request, generated)
        key = self.keys[request]
        if key in self.fail and len(generated) >= 2:
            raise RuntimeError("grammar error")
        if key in self.empty and len(generated) >= 1:
            return np.zeros(VOCAB, bool)
        a = grammar(key, generated)
        return pack_mask(a) if key % 2 else a  # both forms a provider may return


def _sched(n_sessions=3, max_rows=2, batched=True, budget=0, provider=None, constraint_backend=True):
    be = Toy(n_sessions, max_rows)
    kw = dict(decode_topkp=be.decode_topkp, sample_multi_topkp=be.sample_multi_topkp, decode_penalized=be.decode_penalized,
              sample_multi_penalized=be.sample_multi_penalized, offload=be.offload, restore=be.restore, discard=be.discard)
    if batched:
        kw.update(forward_multi=be.forward_multi, sample_multi=be.sample_multi)
    if constraint_backend:
        kw.update(decode_constrained=be.decode_constrained, sample_multi_constrained=be.sample_multi_constrained, vocab=VOCAB)
    if provider is not None:
        kw.update(mask_provider=provider)
    s = SessionScheduler.over_backend(be.reset_session, be.batch_forward, be.sample, be.decode, n_sessions, max_rows, 4096, budget, **kw)
    return be, s


PEN = dict(presence_penalty=0.8, frequency_penalty=0.6, repetition_penalty=1.7, logit_bias={3: -100.0, 11: 4.0})
REQS = [([1, 2, 3, 4, 5, 6, 7], dict(constrained=True), 1),
        ([4, 5], dict(temperature=0.6, seed=9), None),
        ([6], dict(temperature=0.9, seed=2, constrained=True), 2),
        ([7, 8, 9, 10], dict(temperature=1.0, top_k=8, top_p=0.9, seed=3, repetition_penalty=1.4, constrained=True), 3),
        ([11], dict(temperature=0.5, top_p=0.5, seed=5), None),
        ([12, 13, 12, 13, 12], dict(PEN, constrained=True), 4),
        ([2, 2, 2], dict(PEN, temperature=0.7, seed=11), None),
        ([9, 9], dict(temperature=0.8, seed=4, constrained=True), 5)]


def _submit(s, prov, prompt, max_new, kw, key):
    rid = s.submit(prompt, max_new, **kw)
    if key is not None:
        prov.keys[rid] = key
    return rid


def _alone(prompt, max_new, kw, key):
    prov = Provider()
    _, s = _sched(n_sessions=1, max_rows=1, batched=False, provider=prov)
    rid = _submit(s, prov, prompt, max_new, kw, key)
    s.run()
    return s.result(rid)[0].tolist()


def _check_provider_log(prov, rid, toks):
    """one call per selection, in order, with exactly the tokens generated before it"""
    seen = [g for r, g in prov.log if r == rid]
    assert seen == [toks[:i] for i in range(len(toks))], (rid, seen, toks)


@pytest.mark.parametrize("budget", [0, 3])
@pytest.mark.parametrize("batched", [True, False])
@pytest.mark.parametrize("max_rows", [1, 2, 4])
def test_constrained_requests_equal_their_replay_alone_however_batched(batched, max_rows, budget):
    prov = Provider()
    be, s = _sched(n_sessions=3, max_rows=max_rows, batched=batched, budget=budget, provider=prov)
    ids = [_submit(s, prov, p, 8, kw, key) for p, kw, key in REQS]
    s.run()
    for rid, (p, kw, key) in zip(ids, REQS):
        toks, state, _ = s.result(rid)
        toks = toks.tolist()
        assert state == native.SCHED_FINISHED and len(toks) == 8
        assert toks == _alone(p, 8, kw, key), (p, kw)
        if key is not None:
            _check_provider_log(prov, rid, toks)
            for i, t in enumerate(toks):
                assert grammar(key, toks[:i])[t], (rid, i, t)
        else:
            assert all(r != rid for r, _ in prov.log)
    names = [c[0] for c in be.calls]
    assert "decode_constrained" in names and "sample_multi_constrained" in names


def test_unconstrained_neighbours_are_unchanged_by_constrained_requests():
    prov = Provider()
    _, s = _sched(n_sessions=4, max_rows=4, provider=prov)
    ids = [_submit(s, prov, p, 9, kw, key) for p, kw, key in REQS]
    s.run()
    _, s0 = _sched(n_sessions=4, max_rows=4, provider=Provider())
    free = [(p, {k: v for k, v in kw.items() if k != "constrained"}) for p, kw, key in REQS if key is None]
    ids0 = [s0.submit(p, 9, **kw) for p, kw in free]
    s0.run()
    got = [s.result(rid)[0].tolist() for rid, (_, _, key) in zip(ids, REQS) if key is None]
    assert got == [s0.result(rid)[0].tolist() for rid in ids0]
    # and the constraint acts: without it the constrained requests generate other tokens
    assert _alone(REQS[0][0], 8, {}, None) != _alone(REQS[0][0], 8, REQS[0][1], REQS[0][2])


def test_a_finished_grammar_ends_the_request_with_its_stop_token():
    prov = Provider()
    _, s = _sched(provider=prov)
    a = _submit(s, prov, [1, 2, 3], 40, dict(stop=[STOP], constrained=True), 105)  # STOP only from the 6th token on
    b = _submit(s, prov, [4], 40, dict(stop=[STOP], constrained=True, temperature=0.9, seed=3), 100)  # STOP only, from the first token
    s.run()
    ta, state, reason = s.result(a)
    assert state == native.SCHED_FINISHED and reason == native.FINISH_STOP_TOKEN and len(ta) == 6 and ta[-1] == STOP
    assert STOP not in ta[:-1].tolist() or not grammar(105, [])[STOP]
    # the first token is not stop-checked (as the reference's): the STOP-only grammar stops at its second token
    tb, state, reason = s.result(b)
    assert tb.tolist() == [STOP, STOP] and reason == native.FINISH_STOP_TOKEN


def test_a_failing_provider_or_an_empty_mask_fails_only_its_request():
    prov = Provider()
    prov.fail.add(7)
    prov.empty.add(9)
    _, s = _sched(n_sessions=4, max_rows=4, provider=prov)
    bad = _submit(s, prov, [1, 2], 8, dict(constrained=True), 7)
    empty = _submit(s, prov, [3], 8, dict(constrained=True, temperature=0.5, seed=1), 9)
    good = [_submit(s, prov, p, 8, kw, key) for p, kw, key in REQS[:4]]
    s.run(check=False)
    tb, state, reason = s.result(bad)
    assert state == native.SCHED_FAILED and reason == native.FINISH_ERROR and len(tb) == 2
    te, state, reason = s.result(empty)
    assert state == native.SCHED_FAILED and reason == native.FINISH_ERROR and len(te) == 1
    assert any("grammar error" in str(e) for e in s.backend_errors)
    for rid, (p, kw, key) in zip(good, REQS[:4]):
        toks, state, _ = s.result(rid)
        assert state == native.SCHED_FINISHED and toks.tolist() == _alone(p, 8, kw, key)
    # a first token refused by the provider
    prov2 = Provider()
    prov2.on_call = lambda r, g: (_ for _ in ()).throw(RuntimeError("no grammar")) if r == first else None
    _, s2 = _sched(provider=prov2)
    first = _submit(s2, prov2, [5, 6], 4, dict(constrained=True), 1)
    other = _submit(s2, prov2, [5, 6], 4, dict(constrained=True), 1)
    with pytest.raises(native.JlamaNativeError, match="mask provider"):
        s2.run()
    s2.run()
    assert s2.result(first)[1:] == (native.SCHED_FAILED, native.FINISH_ERROR) and len(s2.result(first)[0]) == 0
    assert s2.result(other)[1] == native.SCHED_FINISHED and s2.result(other)[0].tolist() == _alone([5, 6], 4, dict(constrained=True), 1)


def test_constrained_submits_need_a_provider_and_the_backend():
    _, s = _sched(provider=None)
    with pytest.raises(native.JlamaNativeError, match="mask provider"):
        s.submit([1, 2], 4, constrained=True)
    with pytest.raises(native.JlamaNativeError):
        s.submit_n([1, 2], 2, 4, constrained=True)
    _, s = _sched(provider=Provider(), constraint_backend=False)
    with pytest.raises(native.JlamaNativeError, match="constraint backend"):
        s.submit([1, 2], 4, constrained=True)
    assert s.submit([1, 2], 4) > 0  # unconstrained requests do not need either


def test_submit_n_members_get_their_own_provider_calls():
    prov = Provider()
    be = Toy(4, 4)
    fork_calls = []

    def fork(src, positions, dst):
        fork_calls.append(len(dst))
        for d in dst.tolist():
            be.hist[d] = list(be.hist[src][:positions])

    s = SessionScheduler.over_backend(be.reset_session, be.batch_forward, be.sample, be.decode, 4, 4, 4096, 0,
                                      forward_multi=be.forward_multi, sample_multi=be.sample_multi, decode_topkp=be.decode_topkp,
                                      sample_multi_topkp=be.sample_multi_topkp, decode_penalized=be.decode_penalized,
                                      sample_multi_penalized=be.sample_multi_penalized, decode_constrained=be.decode_constrained,
                                      sample_multi_constrained=be.sample_multi_constrained, vocab=VOCAB, fork=fork, mask_provider=prov)
    ids = s.submit_n([1, 2, 3], 3, 6, temperature=0.8, seed=20, constrained=True)
    for j, rid in enumerate(ids):
        prov.keys[rid] = 30 + j
    s.run()
    assert fork_calls == [2]
    for j, rid in enumerate(ids):
        toks = s.result(rid)[0].tolist()
        assert len(toks) == 6
        _check_provider_log(prov, rid, toks)
        assert toks == _alone([1, 2, 3], 6, dict(temperature=0.8, seed=20 + j, constrained=True), 30 + j)


def test_cancel_from_the_provider_and_a_continuation_after_a_spill():
    prov = Provider()
    _, s = _sched(n_sessions=2, max_rows=2, provider=prov)
    # the provider cancels its own request at its third token: it ends at the next step boundary, after that token
    victim = []
    prov.on_call = lambda r, g: s.cancel(r) if r in victim and len(g) == 2 and s.result(r)[1] == native.SCHED_DECODING else None
    a = _submit(s, prov, [1, 2, 3], 5, dict(keep_session=True, constrained=True), 11)
    c = _submit(s, prov, [8, 9], 20, dict(constrained=True), 13)
    victim.append(c)
    s.run()
    ta = s.result(a)[0].tolist()
    assert ta == _alone([1, 2, 3], 5, dict(constrained=True), 11)
    tc, state, reason = s.result(c)
    assert reason == native.FINISH_CANCELLED and len(tc) == 3
    # two fresh requests take both slots, so the kept session of `a` is spilled; its continuation restores it
    x = _submit(s, prov, [4, 4], 3, dict(constrained=True), 15)
    y = _submit(s, prov, [5], 3, {}, None)
    s.run()
    assert s.info(a).spilled == 1
    b = _submit(s, prov, [6, 7], 5, dict(continue_request=a, constrained=True), 17)
    s.run()
    tb = s.result(b)[0].tolist()
    _check_provider_log(prov, b, tb)  # the continuation's own tokens only
    hist = [1, 2, 3] + ta[:-1] + [6, 7]  # the last token of `a` was never fed back
    want = []
    for i in range(5):
        b_row = apply_mask(_toy_logits(hist), grammar(17, want))
        want.append(int(np.argmax(b_row)))
        hist.append(want[-1])
    assert tb == want
    assert s.result(x)[1] == s.result(y)[1] == native.SCHED_FINISHED


@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_as_the_device_every_constrained_request_equals_a_masked_host_loop(oracle, seed):
    """The CPU restatement of the model as the device (one OracleLlama per slot): constrained rows take the rule on the oracle's logits,
    the others the oracle's own selection.  Every request equals a host loop over the oracle alone that applies apply_mask to its
    logits."""
    cfg = synth.get_config("tiny")
    V = cfg["vocab"]
    w = synth.make_weights(cfg)
    n_slots = 3
    slots = [oracle.OracleLlama(cfg, w, act_q8=True) for _ in range(n_slots)]
    hidden = [None] * n_slots

    def gram(key, gen):
        h = (key * 7777 + 31 * len(gen) + (int(gen[-1]) if len(gen) else 0)) % (1 << 31)
        a = np.random.default_rng(h).random(V) < 0.2
        a[h % V] = True
        return a

    def pick(s, hid, T, k, p, u, allow):
        tok, logits = slots[s].sample(hid)
        if allow is None:
            return tok if T == 0.0 else oracle.sample_temperature(logits, T, u)
        return sample_topkp(apply_mask(logits, allow), T, k, p, u)

    def forward_multi(sessions, start_pos, lengths, tokens):
        off = 0
        for s, p, n in zip(sessions.tolist(), start_pos.tolist(), lengths.tolist()):
            hidden[s] = slots[s].batch_forward(tokens[off:off + n], p)
            off += n

    def sample_multi(sessions, temps, unis):
        return [pick(s, hidden[s], T, 0, 1.0, u, None) for s, T, u in zip(sessions.tolist(), temps.tolist(), unis.tolist())]

    def sample_multi_constrained(sessions, temps, ks, ps, unis, top_n, pens, allowed):
        toks = [pick(s, hidden[s], T, k, p, u, a) for s, T, k, p, u, a in zip(sessions.tolist(), temps.tolist(), ks.tolist(), ps.tolist(),
                                                                               unis.tolist(), allowed)]
        return toks, np.full(len(toks), np.nan, np.float32), np.full((len(toks), 20), -1, np.int32), np.full((len(toks), 20), np.nan, np.float32)

    def decode(sessions, tokens, positions, temps, unis):
        return [pick(s, slots[s].batch_forward([t], p), T, 0, 1.0, u, None)
                for s, t, p, T, u in zip(sessions.tolist(), tokens.tolist(), positions.tolist(), temps.tolist(), unis.tolist())]

    def decode_constrained(sessions, tokens, positions, temps, ks, ps, unis, top_n, pens, allowed):
        toks = [pick(s, slots[s].batch_forward([t], p), T, k, pp, u, a)
                for s, t, p, T, k, pp, u, a in zip(sessions.tolist(), tokens.tolist(), positions.tolist(), temps.tolist(), ks.tolist(),
                                                   ps.tolist(), unis.tolist(), allowed)]
        return toks, np.full(len(toks), np.nan, np.float32), np.full((len(toks), 20), -1, np.int32), np.full((len(toks), 20), np.nan, np.float32)

    keys = {}
    sched = SessionScheduler.over_backend(lambda s: slots[s].reset(), None, None, decode, n_slots, 2, cfg["ctx"], prefill_tokens_per_step=16,
                                          forward_multi=forward_multi, sample_multi=sample_multi, decode_constrained=decode_constrained,
                                          sample_multi_constrained=sample_multi_constrained, vocab=V,
                                          mask_provider=lambda r, g: gram(keys[r], g))
    rng = np.random.default_rng(seed)
    reqs = []
    for i in range(7):
        prompt = synth.random_prompt(cfg, 3 + int(rng.integers(0, 12)), seed=500 + 10 * seed + i)
        con = bool(rng.integers(0, 3))
        T = float(rng.choice([0.0, 0.8]))
        sd = int(rng.integers(1, 1 << 30))
        rid = sched.submit(prompt, 2 + int(rng.integers(0, 5)), temperature=T, seed=sd, constrained=con)
        keys[rid] = i
        reqs.append((rid, prompt, con, T, sd))
    sched.run()
    ref = oracle.OracleLlama(cfg, w, act_q8=True)
    n_con = 0
    for rid, prompt, con, T, sd in reqs:
        toks, state, _ = sched.result(rid)
        assert state == native.SCHED_FINISHED
        if not con:
            if T == 0.0:
                want, _ = ref.generate(prompt, len(toks))
                assert toks.tolist() == list(want)
            continue
        n_con += 1
        ref.reset()
        hid = ref.batch_forward(prompt, 0)
        us = _uniforms(sd, len(toks))
        want = []
        for i in range(len(toks)):
            _, logits = ref.sample(hid)
            want.append(sample_topkp(apply_mask(logits, gram(keys[rid], want)), T, 0, 1.0, us[i] if T else 0.0))
            hid = ref.batch_forward([want[-1]], len(prompt) + i)
        assert toks.tolist() == want, (rid, T)
    assert n_con >= 2
    sched.close()
    ref.close()
    for o in slots:
        o.close()


def _uniforms(seed, n):
    """the scheduler's per-request uniform stream (splitmix64, 24 bits)"""
    x, M, out = seed, (1 << 64) - 1, []
    for _ in range(n):
        x = (x + 0x9E3779B97F4A7C15) & M
        z = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        out.append(float(np.float32((z ^ (z >> 31)) >> 40) * np.float32(1.0 / 16777216.0)))
    return out
