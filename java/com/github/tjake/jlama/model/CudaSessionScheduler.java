/*
 * Reference-side binding for the concurrent-session scheduler of libjlama_b200.so (include/jlama_b200.h, jl_sched_*).
 *
 * Jlama serves concurrent requests with one thread per request, each inside AbstractModel.generate(UUID session, ...) on its own KvBuffer
 * (core/model/AbstractModel.java:516-646, core/tensor/KvBufferCache.java:58-60, jlama-net/.../openai/OpenAIChatService.java:64-74,107-160).
 * With a device-resident model those threads would serialise on the GPU and stream the weights once per request per token.  This class
 * keeps the call shape -- generate(session, promptTokens, maxNew, eosTokens, onToken) blocks its calling thread and streams tokens to the
 * callback -- but every call only queues a request; ONE stepping thread runs jl_sched_step, which batches all generating requests into
 * one decode step (the weights are read once for all of them), forwards prompt chunks under a token budget and reuses session slots as
 * requests finish.  A session UUID that comes back (the X-Jlama-Session header) continues on its kept KV at
 * kvmem.getCurrentContextPosition() exactly like AbstractModel.java:533.
 *
 * SOURCE ONLY (no JDK in this image): jlama_b200/scheduler.py binds the same entry points and is what tests/test_scheduler.py (CPU,
 * the native policy over the oracle) and tests/test_gpu_scheduler.py exercise.
 */
package com.github.tjake.jlama.model;

import java.lang.foreign.*;
import java.lang.invoke.MethodHandle;
import java.lang.invoke.MethodHandles;
import java.lang.invoke.MethodType;
import java.util.Map;
import java.util.UUID;
import java.util.concurrent.ConcurrentHashMap;
import java.util.function.IntConsumer;

import static java.lang.foreign.ValueLayout.*;

public final class CudaSessionScheduler implements AutoCloseable {
    public static final int QUEUED = 0, PREFILL = 1, DECODING = 2, FINISHED = 3, FAILED = 4;          // JL_SCHED_*
    public static final int MAX_TOKENS = 1, STOP_TOKEN = 2, CANCELLED = 3, ERROR = 4;                    // JL_FINISH_* (Generator.FinishReason)
    private static final int KEEP_SESSION = 1, CONSTRAINED = 2;                                      // JL_SCHED_* submit flags

    private static final Linker LINKER = Linker.nativeLinker();
    private static final SymbolLookup LIB = SymbolLookup.loaderLookup().or(LINKER.defaultLookup());
    private static MethodHandle h(String name, FunctionDescriptor fd) {
        return LINKER.downcallHandle(LIB.find(name).orElseThrow(() -> new UnsatisfiedLinkError(name)), fd);
    }
    private static final MethodHandle jl_sched_create = h("jl_sched_create", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, ADDRESS));
    private static final MethodHandle jl_sched_free = h("jl_sched_free", FunctionDescriptor.of(JAVA_INT, ADDRESS));
    private static final MethodHandle jl_sched_last_error = h("jl_sched_last_error", FunctionDescriptor.of(ADDRESS, ADDRESS));
    private static final MethodHandle jl_sched_submit_penalized =
        h("jl_sched_submit_penalized", FunctionDescriptor.of(JAVA_LONG, ADDRESS, ADDRESS, JAVA_INT, JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, JAVA_LONG,
                                                             JAVA_FLOAT, JAVA_INT, JAVA_FLOAT, JAVA_LONG, JAVA_INT, JAVA_FLOAT, JAVA_FLOAT, JAVA_FLOAT,
                                                             JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle jl_sched_submit_n =
        h("jl_sched_submit_n", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, JAVA_LONG,
                                                     JAVA_FLOAT, JAVA_INT, JAVA_FLOAT, JAVA_LONG, JAVA_INT, JAVA_FLOAT, JAVA_FLOAT, JAVA_FLOAT,
                                                     JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_sched_result_logprobs =
        h("jl_sched_result_logprobs", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_LONG, JAVA_INT, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_sched_cancel = h("jl_sched_cancel", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_LONG));
    private static final MethodHandle jl_sched_step = h("jl_sched_step", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle jl_sched_result =
        h("jl_sched_result", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_LONG, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_sched_release = h("jl_sched_release", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_LONG));
    private static final MethodHandle jl_sched_set_prefix_cache =
        h("jl_sched_set_prefix_cache", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, JAVA_INT));
    private static final MethodHandle jl_sched_set_mask_provider =
        h("jl_sched_set_mask_provider", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_sched_prefix_stats = h("jl_sched_prefix_stats", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));

    private final Arena arena = Arena.ofShared();
    private final MemorySegment sched;
    private final Map<UUID, Long> kept = new ConcurrentHashMap<>(); // session UUID -> its last finished request (holds the KV slot)
    private final Thread stepper;
    private volatile boolean running = true;
    private final Object tick = new Object();

    /** prefillTokensPerStep bounds how long a new prompt may delay the decode step of the running requests (0 = whole prompts). */
    public CudaSessionScheduler(CudaLlamaModel model, int maxActive, int prefillTokensPerStep) {
        this(model, maxActive, prefillTokensPerStep, 0);
    }

    /**
     * The grammar engine of constrained requests (JSON mode, a JSON schema, tool-call arguments, a regex; DESIGN §3.18): the allowed set
     * of the next token of `request` after the tokens it has `generated` (none for its first token), indexed by token id.  Called once
     * before every selection of a constrained request, on the stepping thread; it must not block on generate() of the same scheduler.
     * When the grammar is complete it allows only the request's stop tokens.  Throwing fails that request alone.
     */
    @FunctionalInterface
    public interface MaskProvider {
        boolean[] allowed(long request, int[] generated);
    }

    private MaskProvider maskProvider;
    private int vocab;

    /** jl_sched_mask_fn upcall: the provider's set -> allow_out [(vocab + 31) / 32] (zeroed by the scheduler); non-zero on failure */
    private int mask(MemorySegment user, long request, MemorySegment generated, int n, MemorySegment allowOut) {
        try {
            int[] gen = n == 0 ? new int[0] : generated.reinterpret(4L * n).toArray(JAVA_INT);
            boolean[] a = maskProvider.allowed(request, gen);
            MemorySegment out = allowOut.reinterpret(4L * ((vocab + 31) / 32));
            for (int t = 0; t < vocab && t < a.length; t++)
                if (a[t]) out.setAtIndex(JAVA_INT, t / 32, out.getAtIndex(JAVA_INT, t / 32) | (1 << (t % 32)));
            return 0;
        } catch (Throwable t) {
            return 1; // an exception must not unwind through the native caller
        }
    }


    /**
     * prefixCachePages > 0: requests without a session reuse the KV pages of earlier prompts that share a whole-page prefix with theirs,
     * the cache holding at most that many pages no session holds (DESIGN §3.17).  A stateless chat client that resends its whole
     * conversation then forwards only the new turn.
     */
    public CudaSessionScheduler(CudaLlamaModel model, int maxActive, int prefillTokensPerStep, int prefixCachePages) {
        this(model, maxActive, prefillTokensPerStep, prefixCachePages, null);
    }

    /** A scheduler whose constrained requests (generate(..., constrained = true, ...)) take their allowed sets from maskProvider (nullable). */
    public CudaSessionScheduler(CudaLlamaModel model, int maxActive, int prefillTokensPerStep, int prefixCachePages, MaskProvider maskProvider) {
        try {
            MemorySegment out = arena.allocate(ADDRESS);
            int rc = (int) jl_sched_create.invokeExact(model.handle(), maxActive, prefillTokensPerStep, out);
            if (rc != 0) throw new IllegalStateException("jl_sched_create: " + rc);
            sched = out.get(ADDRESS, 0);
            if (prefixCachePages > 0) {
                rc = (int) jl_sched_set_prefix_cache.invokeExact(sched, MemorySegment.NULL, prefixCachePages);
                if (rc != 0) {
                    int ignored = (int) jl_sched_free.invokeExact(sched);
                    throw new IllegalStateException("jl_sched_set_prefix_cache: " + rc);
                }
            }
            if (maskProvider != null) { // before the stepping thread's first step
                this.maskProvider = maskProvider;
                this.vocab = model.vocabularySize();
                MethodHandle up = MethodHandles.lookup().findVirtual(CudaSessionScheduler.class, "mask",
                        MethodType.methodType(int.class, MemorySegment.class, long.class, MemorySegment.class, int.class, MemorySegment.class)).bindTo(this);
                MemorySegment stub = LINKER.upcallStub(up, FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_LONG, ADDRESS, JAVA_INT, ADDRESS), arena);
                rc = (int) jl_sched_set_mask_provider.invokeExact(sched, stub, MemorySegment.NULL);
                if (rc != 0) {
                    int ignored = (int) jl_sched_free.invokeExact(sched);
                    throw new IllegalStateException("jl_sched_set_mask_provider: " + rc);
                }
            }
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
        stepper = new Thread(this::loop, "jlama-cuda-scheduler");
        stepper.setDaemon(true);
        stepper.start();
    }

    /** The serving loop: step while anything is queued or running, sleep otherwise.  jl_sched_stats = 8 ints ([5] active, [6] queued). */
    private void loop() {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment st = a.allocate(JAVA_INT, 8);
            while (running) {
                int rc = (int) jl_sched_step.invokeExact(sched, st);   // a failing request is marked FAILED; the others go on
                boolean idle = st.getAtIndex(JAVA_INT, 5) == 0 && st.getAtIndex(JAVA_INT, 6) == 0;
                synchronized (tick) {
                    tick.notifyAll();                                  // wake the generate() callers: new tokens may be there
                    if (idle) tick.wait(5);
                }
            }
        } catch (Throwable t) { running = false; synchronized (tick) { tick.notifyAll(); } }
    }

    /**
     * AbstractModel.generate over token ids: blocks until the request finishes, calls onToken for every generated token in order, returns
     * the FinishReason code.  keepSession = the caller sent a session id and may come back with a follow-up prompt.  temperature 0 = arg-max;
     * otherwise every token is drawn with AbstractModel.sample's rule (:475-489) from a stream seeded here (the reference draws
     * ThreadLocalRandom.current().nextFloat() per token, :576,:594).
     */
    public int generate(UUID session, int[] promptTokens, float temperature, int maxNew, int[] eosTokens, boolean keepSession, IntConsumer onToken) {
        return generate(session, promptTokens, temperature, 0, 1.0f, maxNew, eosTokens, keepSession, onToken);
    }

    /**
     * generate() with a token filter (the CLI's --top-p, an OpenAI request's top_p / top_k): with temperature > 0 and topK > 0 or topP < 1
     * every token is drawn with the top-k / top-p rule (DESIGN §3.12) from the request's uniform stream.  topK 0 and topP 1 = no filter.
     */
    public int generate(UUID session, int[] promptTokens, float temperature, int topK, float topP, int maxNew, int[] eosTokens, boolean keepSession,
                        IntConsumer onToken) {
        return generate(session, promptTokens, temperature, topK, topP, maxNew, eosTokens, keepSession, -1,
                        (token, lp, topIds, topLp) -> onToken.accept(token));
    }

    /** A token of completion `index` (0..n-1) of an n-completion request. */
    @FunctionalInterface
    public interface CompletionTokenConsumer {
        void accept(int index, int token);
    }

    /**
     * n completions of one prompt (an OpenAI request's `n`; DESIGN §3.15): the prompt is forwarded once and its KV pages are shared by
     * the completions, completion j drawing from the stream seeded with seed + j.  Blocks until all finish, calls onToken for every
     * generated token of each completion in order, returns their FinishReason codes.  No session is kept.
     */
    public int[] generate(int n, int[] promptTokens, float temperature, int topK, float topP, int maxNew, int[] eosTokens, long seed,
                          CudaLlamaModel.Penalties penalties, CompletionTokenConsumer onToken) {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment pr = a.allocateFrom(JAVA_INT, promptTokens);
            MemorySegment eos = eosTokens.length == 0 ? MemorySegment.NULL : a.allocateFrom(JAVA_INT, eosTokens);
            MemorySegment bi = a.allocateFrom(JAVA_INT, penalties.biasIds()), bv = a.allocateFrom(JAVA_FLOAT, penalties.biasValues());
            MemorySegment ids = a.allocate(JAVA_LONG, Math.max(n, 1));
            int rc = (int) jl_sched_submit_n.invokeExact(sched, n, pr, promptTokens.length, maxNew, eos, eosTokens.length, 0, -1L, temperature,
                                                         topK, topP, seed, -1, penalties.presence(), penalties.frequency(),
                                                         penalties.repetition(), penalties.biasIds().length, bi, bv, ids);
            if (rc != 0) throw new IllegalArgumentException(((MemorySegment) jl_sched_last_error.invokeExact(sched)).reinterpret(512).getString(0));
            synchronized (tick) { tick.notifyAll(); }
            MemorySegment buf = a.allocate(JAVA_INT, maxNew), cnt = a.allocate(JAVA_INT), state = a.allocate(JAVA_INT), reason = a.allocate(JAVA_INT);
            int[] seen = new int[n], why = new int[n];
            boolean[] done = new boolean[n];
            for (int left = n; left > 0;) {
                for (int j = 0; j < n; j++) {
                    if (done[j]) continue;
                    long id = ids.getAtIndex(JAVA_LONG, j);
                    rc = (int) jl_sched_result.invokeExact(sched, id, buf, maxNew, cnt, state, reason);
                    if (rc != 0) throw new IllegalStateException("jl_sched_result: " + rc);
                    for (int have = Math.min(cnt.get(JAVA_INT, 0), maxNew); seen[j] < have; seen[j]++) onToken.accept(j, buf.getAtIndex(JAVA_INT, seen[j]));
                    int s = state.get(JAVA_INT, 0);
                    if (s != FINISHED && s != FAILED) continue;
                    done[j] = true;
                    left--;
                    why[j] = s == FAILED ? ERROR : reason.get(JAVA_INT, 0);
                    int ignored = (int) jl_sched_release.invokeExact(sched, id);
                }
                if (left == 0) break;
                if (!running) throw new IllegalStateException("scheduler stopped");
                synchronized (tick) { tick.wait(2); }
            }
            return why;
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** A generated token with its log-probability and its top alternatives (best first; DESIGN §3.13). */
    @FunctionalInterface
    public interface TokenLogprobConsumer {
        void accept(int token, float logprob, int[] topIds, float[] topLogprobs);
    }

    /**
     * generate() with log-probabilities (an OpenAI chat request's logprobs / top_logprobs): logprobs -1 = none (logprob NaN, empty
     * alternatives), 0 = each token's own, up to 20 alternatives per token.  The tokens are those of the same request without them.
     */
    public int generate(UUID session, int[] promptTokens, float temperature, int topK, float topP, int maxNew, int[] eosTokens, boolean keepSession,
                        int logprobs, TokenLogprobConsumer onToken) {
        return generate(session, promptTokens, temperature, topK, topP, maxNew, eosTokens, keepSession, logprobs,
                        new CudaLlamaModel.Penalties(0f, 0f, 1f, new int[0], new float[0]), onToken);
    }

    /**
     * generate() with penalties (an OpenAI request's presence_penalty / frequency_penalty / logit_bias, a Hugging Face client's
     * repetition_penalty; DESIGN §3.14): every token is selected from its penalised logits, the history being this request's prompt and
     * its generated tokens (for a continued session, this turn's prompt only).  The penalties' own history fields are ignored.
     */
    public int generate(UUID session, int[] promptTokens, float temperature, int topK, float topP, int maxNew, int[] eosTokens, boolean keepSession,
                        int logprobs, CudaLlamaModel.Penalties penalties, TokenLogprobConsumer onToken) {
        return generate(session, promptTokens, temperature, topK, topP, maxNew, eosTokens, keepSession, false, logprobs, penalties, onToken);
    }

    /**
     * generate() under a grammar (DESIGN §3.18): with constrained = true every token is selected under the allowed set the scheduler's
     * MaskProvider gives for it, after the penalties.  A request whose provider throws or allows nothing ends with ERROR.
     */
    public int generate(UUID session, int[] promptTokens, float temperature, int topK, float topP, int maxNew, int[] eosTokens, boolean keepSession,
                        boolean constrained, int logprobs, CudaLlamaModel.Penalties penalties, TokenLogprobConsumer onToken) {
        final int W = CudaLlamaModel.MAX_LOGPROBS;
        try (Arena a = Arena.ofConfined()) {
            MemorySegment pr = a.allocateFrom(JAVA_INT, promptTokens);
            MemorySegment eos = eosTokens.length == 0 ? MemorySegment.NULL : a.allocateFrom(JAVA_INT, eosTokens);
            MemorySegment bi = a.allocateFrom(JAVA_INT, penalties.biasIds()), bv = a.allocateFrom(JAVA_FLOAT, penalties.biasValues());
            Long parent = kept.remove(session);
            long id = (long) jl_sched_submit_penalized.invokeExact(sched, pr, promptTokens.length, maxNew, eos, eosTokens.length,
                                                                    (keepSession ? KEEP_SESSION : 0) | (constrained ? CONSTRAINED : 0),
                                                                    parent == null ? -1L : (long) parent,
                                                                    temperature, topK, topP, java.util.concurrent.ThreadLocalRandom.current().nextLong(),
                                                                    logprobs, penalties.presence(), penalties.frequency(), penalties.repetition(),
                                                                    penalties.biasIds().length, bi, bv);
            if (id < 0) throw new IllegalArgumentException(((MemorySegment) jl_sched_last_error.invokeExact(sched)).reinterpret(512).getString(0));
            synchronized (tick) { tick.notifyAll(); }
            MemorySegment buf = a.allocate(JAVA_INT, maxNew), n = a.allocate(JAVA_INT), state = a.allocate(JAVA_INT), reason = a.allocate(JAVA_INT);
            MemorySegment lp = a.allocate(JAVA_FLOAT, maxNew), ids = a.allocate(JAVA_INT, (long) maxNew * W), tlp = a.allocate(JAVA_FLOAT, (long) maxNew * W);
            MemorySegment avail = a.allocate(JAVA_INT);
            int seen = 0;
            for (;;) {
                int rc = (int) jl_sched_result.invokeExact(sched, id, buf, maxNew, n, state, reason);
                if (rc != 0) throw new IllegalStateException("jl_sched_result: " + rc);
                int have = Math.min(n.get(JAVA_INT, 0), maxNew);
                if (logprobs >= 0 && have > seen) {
                    rc = (int) jl_sched_result_logprobs.invokeExact(sched, id, seen, have - seen, lp.asSlice(seen * 4L),
                                                                    ids.asSlice((long) seen * W * 4), tlp.asSlice((long) seen * W * 4), avail);
                    if (rc != 0) throw new IllegalStateException("jl_sched_result_logprobs: " + rc);
                }
                for (; seen < have; seen++) {
                    if (logprobs < 0) { onToken.accept(buf.getAtIndex(JAVA_INT, seen), Float.NaN, new int[0], new float[0]); continue; }
                    int[] ti = ids.asSlice((long) seen * W * 4, (long) logprobs * 4).toArray(JAVA_INT);
                    float[] tl = tlp.asSlice((long) seen * W * 4, (long) logprobs * 4).toArray(JAVA_FLOAT);
                    onToken.accept(buf.getAtIndex(JAVA_INT, seen), lp.getAtIndex(JAVA_FLOAT, seen), ti, tl);
                }
                int s = state.get(JAVA_INT, 0);
                if (s == FINISHED || s == FAILED) break;
                if (!running) throw new IllegalStateException("scheduler stopped");
                synchronized (tick) { tick.wait(2); }
            }
            int why = reason.get(JAVA_INT, 0);
            if (parent != null) { int ignored = (int) jl_sched_release.invokeExact(sched, (long) parent); } // its slot moved to this request
            if (keepSession && state.get(JAVA_INT, 0) == FINISHED && why != CANCELLED) kept.put(session, id);
            else { int ignored = (int) jl_sched_release.invokeExact(sched, id); }
            if (state.get(JAVA_INT, 0) == FAILED)
                throw new RuntimeException(((MemorySegment) jl_sched_last_error.invokeExact(sched)).reinterpret(512).getString(0));
            return why;
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** KvBufferCache.KvBuffer.close for a kept session: its slot returns to the pool. */
    /** jl_sched_prefix_stats_t: {entries, lookups, hits, cached prompt tokens, evictions, pages held only by the cache}. */
    public long[] prefixStats() {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment st = a.allocate(JAVA_LONG, 6);
            int rc = (int) jl_sched_prefix_stats.invokeExact(sched, st);
            if (rc != 0) throw new IllegalStateException("jl_sched_prefix_stats: " + rc);
            return st.toArray(JAVA_LONG);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    public void closeSession(UUID session) {
        Long id = kept.remove(session);
        if (id != null) try { int rc = (int) jl_sched_release.invokeExact(sched, (long) id); } catch (Throwable ignored) { }
    }

    @Override public void close() {
        running = false;
        synchronized (tick) { tick.notifyAll(); }
        try { stepper.join(1000); int rc = (int) jl_sched_free.invokeExact(sched); } catch (Throwable ignored) { }
        arena.close();
    }
}
