"""Host-side mirror of the concurrent-session scheduler (csrc/jl_sched.cu, C ABI jl_sched_*).

The reference serves concurrent requests with one thread per request, each running AbstractModel.generate() on its own KvBuffer
(core/tensor/KvBufferCache.java:58-60, jlama-net/.../openai/OpenAIChatService.java:107-160).  Here requests queue in front of the
batched decode step and are batched per iteration:

    sched = SessionScheduler(model)                       # all of the model's session slots
    a = sched.submit(prompt_a, max_new=64, stop=[eos])
    b = sched.submit(prompt_b, max_new=16)
    sched.run()                                           # or step() from a serving loop while other threads submit
    tokens, state, reason = sched.result(a)

`SessionScheduler.over_backend` runs the same native policy code over Python callables (reset_session / batch_forward / sample /
decode); tests/test_scheduler.py uses it with the CPU oracle standing in for the device.
"""
import ctypes as C

import numpy as np

from . import native


class OutOfMemory(Exception):
    """raised by an over_backend call that ran out of device memory before doing anything: the scheduler sees JL_ERR_OOM"""


def penalty_rows(pen, n):
    """a jl_penalties (ctypes pointer) of n rows -> [model.RowPenalty per row]; logit_bias as a list of (id, value) pairs"""
    from .model import RowPenalty
    q = pen.contents

    def arr(addr, ctype, k, default):
        if not addr:
            return np.full(k, default)
        return np.ctypeslib.as_array(C.cast(addr, C.POINTER(ctype)), shape=(k,)).copy() if k else np.empty(0)

    pres, freq, rep = arr(q.presence, C.c_float, n, 0.0), arr(q.frequency, C.c_float, n, 0.0), arr(q.repetition, C.c_float, n, 1.0)
    hoff, boff = arr(q.hist_off, C.c_int32, n + 1, 0), arr(q.bias_off, C.c_int32, n + 1, 0)
    hp = arr(q.hist_prompt, C.c_int32, n, 0)
    hist = arr(q.hist_ids, C.c_int32, int(hoff[n]), 0)
    bids, bvals = arr(q.bias_ids, C.c_int32, int(boff[n]), 0), arr(q.bias_vals, C.c_float, int(boff[n]), 0.0)
    out = []
    for i in range(n):
        h = hist[hoff[i]:hoff[i + 1]].astype(np.int32)
        out.append(RowPenalty(float(pres[i]), float(freq[i]), float(rep[i]),
                              [(int(t), float(v)) for t, v in zip(bids[boff[i]:boff[i + 1]], bvals[boff[i]:boff[i + 1]])],
                              h[:int(hp[i])], h[int(hp[i]):]))
    return out


def allowed_rows(n_allow, allow, allow_row, n, vocab):
    """the masks of a constrained call (ctypes pointers) -> per row None (unconstrained) or its allowed set as bool[vocab]"""
    from .sampling import mask_words, unpack_mask
    rows = np.ctypeslib.as_array(allow_row, shape=(n,)).copy()
    words = np.ctypeslib.as_array(allow, shape=(n_allow * mask_words(vocab),)).copy() if n_allow else np.empty(0, np.uint32)
    W = mask_words(vocab)
    return [None if r < 0 else unpack_mask(words[r * W:(r + 1) * W], vocab) for r in rows]


def _flags(keep_session, constrained):
    return (native.SCHED_KEEP_SESSION if keep_session else 0) | (native.SCHED_CONSTRAINED if constrained else 0)


class SessionScheduler:
    def __init__(self, model, max_active=0, prefill_tokens_per_step=0, prefix_cache_pages=0, mask_provider=None):
        """prefix_cache_pages > 0: fresh requests reuse the KV pages of earlier prompts that share a whole-page prefix with theirs,
        the cache holding at most that many pages no session holds (DESIGN §3.17).  mask_provider: the grammar engine of constrained
        requests (submit(..., constrained=True); DESIGN §3.18), see _install_mask_provider."""
        self.lib = model.lib
        self._model = model  # the scheduler borrows the model: keep it alive
        self._keep = None
        self.backend_errors = []
        h = C.c_void_p()
        rc = self.lib.jl_sched_create(model.h, max_active, prefill_tokens_per_step, C.byref(h))
        if rc != native.JL_OK:
            raise native.JlamaNativeError(rc, "jl_sched_create failed (is the model finalized?)")
        self.h = h
        try:
            if prefix_cache_pages:
                self._check(self.lib.jl_sched_set_prefix_cache(self.h, None, int(prefix_cache_pages)))
            if mask_provider is not None:
                self._install_mask_provider(mask_provider, int(model.cfg["vocab"]))
        except native.JlamaNativeError:
            self.close()
            raise

    def _install_mask_provider(self, mask_provider, vocab):
        """mask_provider(request, generated: np.int32[k]) -> the allowed set of the request's next token, a bool[vocab] or packed uint32
        words (sampling.pack_mask).  Called once before every selection of a constrained request, with the tokens it has generated so
        far (none for its first token), on the stepping thread; it may call result() / cancel() but must not step.  A raised exception
        fails that request alone (JL_FINISH_ERROR; the exception is kept in backend_errors)."""
        from .sampling import mask_words, pack_mask
        W = mask_words(vocab)

        def _mask(_u, request, generated, n, out):
            try:
                a = np.asarray(mask_provider(int(request), np.ctypeslib.as_array(generated, shape=(n,)).copy() if n else np.empty(0, np.int32)))
                w = pack_mask(a) if a.dtype == bool else np.asarray(a, dtype=np.uint32).reshape(-1)
                if len(w) != W:
                    raise ValueError("mask of %d words for a vocabulary of %d (%d words)" % (len(w), vocab, W))
                np.ctypeslib.as_array(out, shape=(W,))[:] = w
                return native.JL_OK
            except Exception as e:  # noqa: BLE001 -- a Python exception must not unwind through the C caller
                self.backend_errors.append(e)
                return native.JL_ERR_INVALID

        fn = native.SCHED_MASK_FN(_mask)
        self._keep_mask = fn  # the C side keeps the pointer
        self._check(self.lib.jl_sched_set_mask_provider(self.h, fn, None))

    @classmethod
    def over_backend(cls, reset_session, batch_forward, sample, decode, n_sessions, max_rows, max_context, prefill_tokens_per_step=0,
                     offload=None, restore=None, discard=None, forward_multi=None, sample_multi=None, decode_topkp=None,
                     sample_multi_topkp=None, decode_logprobs=None, sample_multi_logprobs=None, decode_penalized=None,
                     sample_multi_penalized=None, fork=None, retain=None, attach=None, release=None, retained=None, ctx_per_page=0,
                     prefix_cache_pages=0, decode_constrained=None, sample_multi_constrained=None, vocab=0, mask_provider=None):
        """reset_session(session); batch_forward(session, tokens: np.int32[n], start_pos); sample(session, temperature, uniform) -> token;
        decode(sessions, tokens, positions: np.int32[n], temperatures, uniforms: np.float32[n]) -> next tokens; optionally the host-spill trio offload(session) -> handle,
        restore(session, handle), discard(handle).  Optionally the batched prompt pair (both or neither):
        forward_multi(sessions, start_pos, lengths, tokens: np.int32) forwards the segments (tokens back to back) in one call, and
        sample_multi(sessions, temperatures, uniforms) -> first tokens; with them a step makes one forward_multi call for all its prompt
        chunks.  Optionally the top-k / top-p pair (both or neither): decode_topkp(sessions, tokens, positions, temperatures, top_k,
        top_p, uniforms) and sample_multi_topkp(sessions, temperatures, top_k, top_p, uniforms) take every call that holds a filtered
        request.  Optionally the logprob pair (both or neither): decode_logprobs(sessions, tokens, positions, temperatures, top_k, top_p,
        uniforms, top_n) and sample_multi_logprobs(sessions, temperatures, top_k, top_p, uniforms, top_n) return (tokens, lp [n],
        top_ids [n, 20], top_lp [n, 20]) and take every call that holds a request with logprobs (top_n -1 for the other rows).
        Optionally the penalty pair (both or neither): decode_penalized and sample_multi_penalized take the logprob pair's arguments plus
        a list of RowPenalty (one per row, with its history; unpenalised rows have empty ones), return what the logprob pair returns, and
        take every call that holds a penalised request.  Optionally fork(src, positions, dst: np.int32[n]) gives the sessions dst the KV
        of src's positions [0, positions) and its last row; submit_n needs it for n > 1.  Optionally the prefix cache (all four with
        ctx_per_page, enabled when prefix_cache_pages > 0): retain(session, positions) -> handle, attach(handle, positions, session),
        release(handle) and retained() -> (handles, pages held only by handles).  Optionally the constraint pair (both or neither, with the
        vocabulary `vocab`): decode_constrained and sample_multi_constrained take the penalty pair's arguments plus a list of allowed
        sets (one per row: None, or a bool[vocab]), return what the penalty pair returns and take every call that holds a constrained
        request; mask_provider is the grammar engine of those requests (see _install_mask_provider).
        A raised exception fails the affected requests (JL_ERR_INVALID), exactly like a backend error code; a raised native.OutOfMemory
        returns JL_ERR_OOM."""
        self = cls.__new__(cls)
        self.lib = native.load()
        self._model = None
        self.backend_errors = []

        def guard(fn):
            def wrapped(*a):
                try:
                    return fn(*a)
                except Exception as e:  # noqa: BLE001 -- a Python exception must not unwind through the C caller
                    self.backend_errors.append(e)
                    return native.JL_ERR_OOM if isinstance(e, OutOfMemory) else native.JL_ERR_INVALID
            return wrapped

        @guard
        def _reset(_u, session):
            reset_session(session)
            return native.JL_OK

        @guard
        def _forward(_u, session, tokens, n, start_pos):
            batch_forward(session, np.ctypeslib.as_array(tokens, shape=(n,)).copy(), start_pos)
            return native.JL_OK

        @guard
        def _sample(_u, session, temperature, uniform, out):
            out[0] = int(sample(session, temperature, uniform))
            return native.JL_OK

        @guard
        def _decode(_u, n, sessions, tokens, positions, temperatures, uniforms, nxt):
            arr = lambda p: np.ctypeslib.as_array(p, shape=(n,)).copy()  # noqa: E731
            res = decode(arr(sessions), arr(tokens), arr(positions), arr(temperatures), arr(uniforms))
            for i in range(n):
                nxt[i] = int(res[i])
            return native.JL_OK

        @guard
        def _offload(_u, session, handle_out):
            handle_out[0] = int(offload(session))
            return native.JL_OK

        @guard
        def _restore(_u, session, handle):
            restore(session, handle)
            return native.JL_OK

        @guard
        def _discard(_u, handle):
            discard(handle)
            return native.JL_OK

        be = native.SchedBackend(native.SCHED_RESET_FN(_reset), native.SCHED_FORWARD_FN(_forward), native.SCHED_SAMPLE_FN(_sample),
                                 native.SCHED_DECODE_FN(_decode))
        if offload is not None:
            be.offload, be.restore, be.discard = native.SCHED_OFFLOAD_FN(_offload), native.SCHED_RESTORE_FN(_restore), native.SCHED_DISCARD_FN(_discard)
        self._keep = be  # the C side copies the struct, the CFUNCTYPE objects must outlive it
        h = C.c_void_p()
        rc = self.lib.jl_sched_create_backend(C.byref(be), None, n_sessions, max_rows, max_context, prefill_tokens_per_step, C.byref(h))
        if rc != native.JL_OK:
            raise native.JlamaNativeError(rc, "jl_sched_create_backend: bad arguments")
        self.h = h
        if (forward_multi is None) != (sample_multi is None):
            self.close()
            raise ValueError("forward_multi and sample_multi come together")
        if forward_multi is not None:
            @guard
            def _forward_multi(_u, n, sessions, start_pos, lengths, tokens):
                arr = lambda p, k: np.ctypeslib.as_array(p, shape=(k,)).copy()  # noqa: E731
                ln = arr(lengths, n)
                forward_multi(arr(sessions, n), arr(start_pos, n), ln, arr(tokens, int(ln.sum())))
                return native.JL_OK

            @guard
            def _sample_multi(_u, n, sessions, temperatures, uniforms, out):
                arr = lambda p: np.ctypeslib.as_array(p, shape=(n,)).copy()  # noqa: E731
                res = sample_multi(arr(sessions), arr(temperatures), arr(uniforms))
                for i in range(n):
                    out[i] = int(res[i])
                return native.JL_OK

            bb = native.SchedBatchBackend(native.SCHED_FORWARD_MULTI_FN(_forward_multi), native.SCHED_SAMPLE_MULTI_FN(_sample_multi))
            self._keep_batch = bb
            self._check(self.lib.jl_sched_set_batch_backend(self.h, C.byref(bb)))
        if (decode_topkp is None) != (sample_multi_topkp is None):
            self.close()
            raise ValueError("decode_topkp and sample_multi_topkp come together")
        if decode_topkp is not None:
            @guard
            def _decode_topkp(_u, n, sessions, tokens, positions, temperatures, top_k, top_p, uniforms, nxt):
                arr = lambda p: np.ctypeslib.as_array(p, shape=(n,)).copy()  # noqa: E731
                res = decode_topkp(arr(sessions), arr(tokens), arr(positions), arr(temperatures), arr(top_k), arr(top_p), arr(uniforms))
                for i in range(n):
                    nxt[i] = int(res[i])
                return native.JL_OK

            @guard
            def _sample_multi_topkp(_u, n, sessions, temperatures, top_k, top_p, uniforms, out):
                arr = lambda p: np.ctypeslib.as_array(p, shape=(n,)).copy()  # noqa: E731
                res = sample_multi_topkp(arr(sessions), arr(temperatures), arr(top_k), arr(top_p), arr(uniforms))
                for i in range(n):
                    out[i] = int(res[i])
                return native.JL_OK

            tb = native.SchedTopkpBackend(native.SCHED_DECODE_TOPKP_FN(_decode_topkp), native.SCHED_SAMPLE_MULTI_TOPKP_FN(_sample_multi_topkp))
            self._keep_topkp = tb
            self._check(self.lib.jl_sched_set_topkp_backend(self.h, C.byref(tb)))
        if (decode_logprobs is None) != (sample_multi_logprobs is None):
            self.close()
            raise ValueError("decode_logprobs and sample_multi_logprobs come together")
        def put(n, res, out, lp, ids, tlp):
            tok, l, i, t = res
            W = native.JL_MAX_LOGPROBS
            np.ctypeslib.as_array(out, shape=(n,))[:] = np.asarray(tok, dtype=np.int32)
            np.ctypeslib.as_array(lp, shape=(n,))[:] = np.asarray(l, dtype=np.float32)
            np.ctypeslib.as_array(ids, shape=(n * W,))[:] = np.asarray(i, dtype=np.int32).reshape(-1)
            np.ctypeslib.as_array(tlp, shape=(n * W,))[:] = np.asarray(t, dtype=np.float32).reshape(-1)
            return native.JL_OK

        if decode_logprobs is not None:

            @guard
            def _decode_logprobs(_u, n, sessions, tokens, positions, temperatures, top_k, top_p, uniforms, top_n, nxt, lp, ids, tlp):
                arr = lambda p: np.ctypeslib.as_array(p, shape=(n,)).copy()  # noqa: E731
                return put(n, decode_logprobs(arr(sessions), arr(tokens), arr(positions), arr(temperatures), arr(top_k), arr(top_p),
                                              arr(uniforms), arr(top_n)), nxt, lp, ids, tlp)

            @guard
            def _sample_multi_logprobs(_u, n, sessions, temperatures, top_k, top_p, uniforms, top_n, out, lp, ids, tlp):
                arr = lambda p: np.ctypeslib.as_array(p, shape=(n,)).copy()  # noqa: E731
                return put(n, sample_multi_logprobs(arr(sessions), arr(temperatures), arr(top_k), arr(top_p), arr(uniforms), arr(top_n)),
                           out, lp, ids, tlp)

            lb = native.SchedLogprobBackend(native.SCHED_DECODE_LOGPROBS_FN(_decode_logprobs),
                                            native.SCHED_SAMPLE_MULTI_LOGPROBS_FN(_sample_multi_logprobs))
            self._keep_logprobs = lb
            self._check(self.lib.jl_sched_set_logprob_backend(self.h, C.byref(lb)))
        if (decode_penalized is None) != (sample_multi_penalized is None):
            self.close()
            raise ValueError("decode_penalized and sample_multi_penalized come together")
        if decode_penalized is not None:
            @guard
            def _decode_penalized(_u, n, sessions, tokens, positions, temperatures, top_k, top_p, uniforms, top_n, pen, nxt, lp, ids, tlp):
                arr = lambda p: np.ctypeslib.as_array(p, shape=(n,)).copy()  # noqa: E731
                return put(n, decode_penalized(arr(sessions), arr(tokens), arr(positions), arr(temperatures), arr(top_k), arr(top_p),
                                               arr(uniforms), arr(top_n), penalty_rows(pen, n)), nxt, lp, ids, tlp)

            @guard
            def _sample_multi_penalized(_u, n, sessions, temperatures, top_k, top_p, uniforms, top_n, pen, out, lp, ids, tlp):
                arr = lambda p: np.ctypeslib.as_array(p, shape=(n,)).copy()  # noqa: E731
                return put(n, sample_multi_penalized(arr(sessions), arr(temperatures), arr(top_k), arr(top_p), arr(uniforms), arr(top_n),
                                                     penalty_rows(pen, n)), out, lp, ids, tlp)

            pb = native.SchedPenaltyBackend(native.SCHED_DECODE_PENALIZED_FN(_decode_penalized),
                                            native.SCHED_SAMPLE_MULTI_PENALIZED_FN(_sample_multi_penalized))
            self._keep_penalties = pb
            self._check(self.lib.jl_sched_set_penalty_backend(self.h, C.byref(pb)))
        if fork is not None:
            @guard
            def _fork(_u, src, positions, n, dst):
                fork(src, positions, np.ctypeslib.as_array(dst, shape=(n,)).copy())
                return native.JL_OK

            fb = native.SchedForkBackend(native.SCHED_FORK_FN(_fork))
            self._keep_fork = fb
            self._check(self.lib.jl_sched_set_fork_backend(self.h, C.byref(fb)))
        if retain is not None:
            @guard
            def _retain(_u, session, positions, handle_out):
                handle_out[0] = int(retain(session, positions))
                return native.JL_OK

            @guard
            def _attach(_u, handle, positions, session):
                attach(handle, positions, session)
                return native.JL_OK

            @guard
            def _release(_u, handle):
                release(handle)
                return native.JL_OK

            @guard
            def _retained(_u, handles, pages):
                n, p = retained()
                if handles:
                    handles[0] = int(n)
                if pages:
                    pages[0] = int(p)
                return native.JL_OK

            xb = native.SchedPrefixBackend(native.SCHED_RETAIN_FN(_retain), native.SCHED_ATTACH_FN(_attach), native.SCHED_RELEASE_FN(_release),
                                           native.SCHED_RETAINED_FN(_retained), int(ctx_per_page))
            self._keep_prefix = xb
            self._check(self.lib.jl_sched_set_prefix_cache(self.h, C.byref(xb), int(prefix_cache_pages)))
        if (decode_constrained is None) != (sample_multi_constrained is None):
            self.close()
            raise ValueError("decode_constrained and sample_multi_constrained come together")
        if decode_constrained is not None:
            @guard
            def _decode_constrained(_u, n, sessions, tokens, positions, temperatures, top_k, top_p, uniforms, top_n, pen, n_allow, allow,
                                    allow_row, nxt, lp, ids, tlp):
                arr = lambda p: np.ctypeslib.as_array(p, shape=(n,)).copy()  # noqa: E731
                return put(n, decode_constrained(arr(sessions), arr(tokens), arr(positions), arr(temperatures), arr(top_k), arr(top_p),
                                                 arr(uniforms), arr(top_n), penalty_rows(pen, n),
                                                 allowed_rows(n_allow, allow, allow_row, n, vocab)), nxt, lp, ids, tlp)

            @guard
            def _sample_multi_constrained(_u, n, sessions, temperatures, top_k, top_p, uniforms, top_n, pen, n_allow, allow, allow_row, out,
                                          lp, ids, tlp):
                arr = lambda p: np.ctypeslib.as_array(p, shape=(n,)).copy()  # noqa: E731
                return put(n, sample_multi_constrained(arr(sessions), arr(temperatures), arr(top_k), arr(top_p), arr(uniforms), arr(top_n),
                                                       penalty_rows(pen, n), allowed_rows(n_allow, allow, allow_row, n, vocab)),
                           out, lp, ids, tlp)

            cb = native.SchedConstraintBackend(native.SCHED_DECODE_CONSTRAINED_FN(_decode_constrained),
                                               native.SCHED_SAMPLE_MULTI_CONSTRAINED_FN(_sample_multi_constrained), int(vocab))
            self._keep_constraints = cb
            self._check(self.lib.jl_sched_set_constraint_backend(self.h, C.byref(cb)))
        if mask_provider is not None:
            self._install_mask_provider(mask_provider, int(vocab))
        return self

    def _check(self, rc):
        if rc != native.JL_OK:
            raise native.JlamaNativeError(rc, self.lib.jl_sched_last_error(self.h).decode())

    def submit(self, prompt, max_new, stop=(), keep_session=False, continue_request=-1, temperature=0.0, seed=0, top_k=0, top_p=1.0,
               logprobs=-1, presence_penalty=0.0, frequency_penalty=0.0, repetition_penalty=1.0, logit_bias=None, constrained=False):
        """temperature 0 = arg-max; otherwise tokens are drawn from a uniform stream seeded with `seed`, with the reference's rule, or
        with the top-k / top-p rule (DESIGN §3.12) when top_k > 0 or top_p < 1.  logprobs >= 0: every generated token also gets its
        logprob and that many top alternatives (DESIGN §3.13), read with result_logprobs.  presence_penalty / frequency_penalty /
        repetition_penalty / logit_bias ({id: value}): every token is selected from its penalised logits (DESIGN §3.14), the history being
        this request's prompt and generated tokens.  constrained: every token is selected under the allowed set the mask provider
        gives for it (DESIGN §3.18)."""
        from .model import _bias_pairs
        prompt = np.ascontiguousarray(prompt, dtype=np.int32)
        stop = np.ascontiguousarray(list(stop), dtype=np.int32)
        bi, bv = _bias_pairs(logit_bias)
        rid = self.lib.jl_sched_submit_penalized(self.h, native.ptr(prompt), len(prompt), max_new, native.ptr(stop) if len(stop) else None,
                                                 len(stop), _flags(keep_session, constrained), continue_request,
                                                 C.c_float(temperature), int(top_k), C.c_float(top_p), C.c_uint64(seed), int(logprobs),
                                                 C.c_float(presence_penalty), C.c_float(frequency_penalty), C.c_float(repetition_penalty),
                                                 len(bi), native.ptr(bi), native.ptr(bv))
        if rid < 0:
            raise native.JlamaNativeError(native.JL_ERR_INVALID, self.lib.jl_sched_last_error(self.h).decode())
        return rid

    def submit_n(self, prompt, n, max_new, stop=(), keep_session=False, continue_request=-1, temperature=0.0, seed=0, top_k=0, top_p=1.0,
                 logprobs=-1, presence_penalty=0.0, frequency_penalty=0.0, repetition_penalty=1.0, logit_bias=None, constrained=False):
        """n completions of one prompt (OpenAI's `n`) -> their request ids.  Member j is the request submit() makes with seed + j; the
        prompt is forwarded once and its KV pages are shared by the members (DESIGN §3.15)."""
        from .model import _bias_pairs
        prompt = np.ascontiguousarray(prompt, dtype=np.int32)
        stop = np.ascontiguousarray(list(stop), dtype=np.int32)
        bi, bv = _bias_pairs(logit_bias)
        ids = np.zeros(max(int(n), 1), dtype=np.int64)
        rc = self.lib.jl_sched_submit_n(self.h, int(n), native.ptr(prompt), len(prompt), max_new, native.ptr(stop) if len(stop) else None,
                                        len(stop), _flags(keep_session, constrained), continue_request, C.c_float(temperature),
                                        int(top_k), C.c_float(top_p), C.c_uint64(seed), int(logprobs), C.c_float(presence_penalty),
                                        C.c_float(frequency_penalty), C.c_float(repetition_penalty), len(bi), native.ptr(bi), native.ptr(bv),
                                        native.ptr(ids))
        if rc != native.JL_OK:
            raise native.JlamaNativeError(rc, self.lib.jl_sched_last_error(self.h).decode())
        return [int(i) for i in ids[:n]]

    def cancel(self, request):
        self._check(self.lib.jl_sched_cancel(self.h, request))

    def step(self, check=True):
        st = native.SchedStats()
        rc = self.lib.jl_sched_step(self.h, C.byref(st))
        if check:
            self._check(rc)
        return st

    def run(self, max_steps=0, check=True):
        st = native.SchedStats()
        rc = self.lib.jl_sched_run(self.h, max_steps, C.byref(st))
        if check:
            self._check(rc)
        return st

    def result(self, request):
        """(tokens generated so far, state, finish reason)"""
        n, state, reason = C.c_int(), C.c_int(), C.c_int()
        self._check(self.lib.jl_sched_result(self.h, request, None, 0, C.byref(n), C.byref(state), C.byref(reason)))
        out = np.empty(n.value, dtype=np.int32)
        if n.value:
            self._check(self.lib.jl_sched_result(self.h, request, native.ptr(out), n.value, C.byref(n), C.byref(state), C.byref(reason)))
        return out[:min(n.value, len(out))], state.value, reason.value

    def result_logprobs(self, request, first=0, count=None):
        """TokenLogprobs of the generated tokens [first, first + count) of a request submitted with logprobs (count None = all there
        are); entry k belongs to the request's k-th generated token."""
        from .model import TokenLogprobs
        avail = C.c_int()
        self._check(self.lib.jl_sched_result_logprobs(self.h, request, 0, 0, None, None, None, C.byref(avail)))
        k = max(0, avail.value - first) if count is None else max(0, min(count, avail.value - first))
        W = native.JL_MAX_LOGPROBS
        lp = TokenLogprobs(np.empty(k, dtype=np.float32), np.empty((k, W), dtype=np.int32), np.empty((k, W), dtype=np.float32))
        if k:
            self._check(self.lib.jl_sched_result_logprobs(self.h, request, first, k, native.ptr(lp.lp), native.ptr(lp.top_ids),
                                                          native.ptr(lp.top_lp), C.byref(avail)))
        return lp

    def info(self, request):
        inf = native.SchedRequestInfo()
        self._check(self.lib.jl_sched_request_info(self.h, request, C.byref(inf)))
        return inf

    def release(self, request):
        self._check(self.lib.jl_sched_release(self.h, request))

    def prefix_stats(self):
        """the prefix cache's SchedPrefixStats: entries, lookups, hits, cached_tokens, evictions, pages_retained_only"""
        st = native.SchedPrefixStats()
        self._check(self.lib.jl_sched_prefix_stats(self.h, C.byref(st)))
        return st

    def cached_tokens(self, request):
        """prompt tokens the request took from the prefix cache instead of forwarding them"""
        n = self.lib.jl_sched_request_cached(self.h, request)
        if n < 0:
            self._check(n)
        return n

    def counts(self):
        q, a, f = C.c_int(), C.c_int(), C.c_int()
        self._check(self.lib.jl_sched_counts(self.h, C.byref(q), C.byref(a), C.byref(f)))
        return q.value, a.value, f.value

    def close(self):
        if self.h:
            self.lib.jl_sched_free(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()
