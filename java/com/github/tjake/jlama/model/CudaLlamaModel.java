/*
 * Reference-side binding for the MODEL-LEVEL entry points of libjlama_b200.so (include/jlama_b200.h, jl_model_*): a LlamaModel whose
 * layers live on the GPU.  It keeps AbstractModel's public call shape -- batchForward / sample / generate
 * (core/model/AbstractModel.java:295-329,443-491,516-646) -- and replaces the per-layer Java objects that LlamaModel builds in
 * loadTransformerBlockWeights (core/model/llama/LlamaModel.java:117-143: RMSNorm, CausalSelfAttention, MLPBlock per layer) by one
 * device-resident model: weights are registered once, KV pages, activations and the sampled token stay in HBM, and a decode step is
 * one kernel launch.  Row (f2) of SURVEY.md section 8.
 *
 * SOURCE ONLY: this image has no JDK, so the class is not compiled or tested here.  jlama_b200/model.py (LlamaModel) makes exactly the
 * same calls in the same order and IS tested (tests/test_gpu_model.py, tests/test_gpu_checkpoint.py); INTEGRATION.md section 3
 * shows where a maintainer plugs this class in.
 */
package com.github.tjake.jlama.model;

import com.github.tjake.jlama.safetensors.Config;
import com.github.tjake.jlama.safetensors.DType;
import com.github.tjake.jlama.safetensors.WeightLoader;
import com.github.tjake.jlama.tensor.AbstractTensor;
import com.github.tjake.jlama.tensor.Q4ByteBufferTensor;
import com.github.tjake.jlama.tensor.Q8ByteBufferTensor;
import java.lang.foreign.*;
import java.lang.invoke.MethodHandle;
import java.util.ArrayList;
import java.util.List;

import static java.lang.foreign.ValueLayout.*;

public final class CudaLlamaModel implements AutoCloseable {
    // include/jlama_b200.h
    private static final int JL_F32 = 0, JL_BF16 = 1, JL_Q4 = 2, JL_I8 = 3;
    private static final int T_EMBED = 0, T_OUT_NORM = 1, T_LM_HEAD = 2;
    private static final int L_ATTN_NORM = 0, L_Q = 1, L_K = 2, L_V = 3, L_O = 4, L_FFN_NORM = 5, L_GATE = 6, L_DOWN = 7, L_UP = 8;

    /** jl_model_config, field for field (all 4-byte except the two doubles; natural alignment like the C struct). */
    private static final StructLayout CONFIG = MemoryLayout.structLayout(
        JAVA_INT.withName("context_length"), JAVA_INT.withName("embedding_length"), JAVA_INT.withName("hidden_length"),
        JAVA_INT.withName("num_heads"), JAVA_INT.withName("num_kv_heads"), JAVA_INT.withName("num_layers"),
        JAVA_INT.withName("vocab_size"), JAVA_INT.withName("head_size"), JAVA_FLOAT.withName("layer_norm_eps"),
        MemoryLayout.paddingLayout(4), JAVA_DOUBLE.withName("rope_theta"), JAVA_DOUBLE.withName("rope_scaling"),
        JAVA_INT.withName("working_qtype"), JAVA_INT.withName("kv_dtype"), JAVA_INT.withName("max_batch"),
        JAVA_INT.withName("max_sessions"), JAVA_INT.withName("max_context"), JAVA_INT.withName("tp_rank"), JAVA_INT.withName("tp_size"),
        JAVA_INT.withName("prefill_tensor_core"), JAVA_INT.withName("flags"), JAVA_INT.withName("num_experts"),
        JAVA_INT.withName("experts_per_token"), JAVA_INT.withName("arch") /* 0 = Llama / Mixtral blocks, 1 = GPT-2 blocks */);

    private static final Linker LINKER = Linker.nativeLinker();
    private static final SymbolLookup LIB;
    static {
        System.loadLibrary("jlama_b200");
        LIB = SymbolLookup.loaderLookup().or(LINKER.defaultLookup());
    }
    private static MethodHandle h(String name, FunctionDescriptor fd) {
        return LINKER.downcallHandle(LIB.find(name).orElseThrow(() -> new UnsatisfiedLinkError(name)), fd);
    }
    private static final MethodHandle jl_init = h("jl_init", FunctionDescriptor.of(JAVA_INT, JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle jl_last_error = h("jl_last_error", FunctionDescriptor.of(ADDRESS, ADDRESS));
    private static final MethodHandle jl_register_tensor =
        h("jl_register_tensor", FunctionDescriptor.of(JAVA_LONG, ADDRESS, JAVA_INT, JAVA_LONG, JAVA_LONG, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_create = h("jl_model_create", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_set_tensor =
        h("jl_model_set_tensor", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, JAVA_LONG));
    private static final MethodHandle jl_model_set_expert_tensor =
        h("jl_model_set_expert_tensor", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, JAVA_INT, JAVA_LONG));
    private static final MethodHandle jl_model_finalize = h("jl_model_finalize", FunctionDescriptor.of(JAVA_INT, ADDRESS));
    private static final MethodHandle jl_model_free = h("jl_model_free", FunctionDescriptor.of(JAVA_INT, ADDRESS));
    private static final MethodHandle jl_model_reset_session = h("jl_model_reset_session", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT));
    private static final MethodHandle jl_model_kv_fork =
        h("jl_model_kv_fork", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, JAVA_INT, ADDRESS));
    private static final MethodHandle jl_model_kv_page_stats = h("jl_model_kv_page_stats", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_kv_retain = h("jl_model_kv_retain", FunctionDescriptor.of(JAVA_LONG, ADDRESS, JAVA_INT, JAVA_INT));
    private static final MethodHandle jl_model_kv_attach =
        h("jl_model_kv_attach", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_LONG, JAVA_INT, JAVA_INT));
    private static final MethodHandle jl_model_kv_release = h("jl_model_kv_release", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_LONG));
    private static final MethodHandle jl_model_kv_retained = h("jl_model_kv_retained", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_batch_forward =
        h("jl_model_batch_forward", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT));
    private static final MethodHandle jl_model_sample =
        h("jl_model_sample", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, JAVA_FLOAT, JAVA_FLOAT, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_decode_sample_topkp =
        h("jl_model_decode_sample_topkp", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS,
                                                                ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_generate_sample_topkp =
        h("jl_model_generate_sample_topkp", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, JAVA_FLOAT, JAVA_INT,
                                                                  JAVA_FLOAT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_decode_logprobs =
        h("jl_model_decode_logprobs", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS,
                                                            ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_generate_logprobs =
        h("jl_model_generate_logprobs", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, JAVA_FLOAT, JAVA_INT,
                                                              JAVA_FLOAT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_decode_penalized =
        h("jl_model_decode_penalized", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS,
                                                             ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_decode_constrained =
        h("jl_model_decode_constrained", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS,
                                                               ADDRESS, ADDRESS, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS,
                                                               ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_sample_multi_constrained =
        h("jl_model_sample_multi_constrained", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS,
                                                                     ADDRESS, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS,
                                                                     ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_generate_penalized =
        h("jl_model_generate_penalized", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, JAVA_FLOAT, JAVA_INT,
                                                               JAVA_FLOAT, ADDRESS, JAVA_INT, JAVA_FLOAT, JAVA_FLOAT, JAVA_FLOAT, JAVA_INT, ADDRESS,
                                                               ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_score =
        h("jl_model_score", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_decode =
        h("jl_model_decode", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_generate =
        h("jl_model_generate", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_kv_save = h("jl_model_kv_save", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle jl_model_kv_load = h("jl_model_kv_load", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS));

    private final Arena arena = Arena.ofShared();
    private final MemorySegment ctx, model;
    private final Config c;
    private final List<Long> tensorIds = new ArrayList<>();

    /**
     * Mirrors LlamaModel's constructor chain (llama/LlamaModel.java:68-115): config + weights in, a model ready for batchForward out.
     * `weights` is the same WeightLoader the reference hands to loadInputWeights / loadTransformerBlockWeights / loadOutputWeights;
     * the DistributedContext in `c.dctx()` selects this rank's rows / columns exactly as Weights.getLoadOffsets (:99-117) does.
     * `kvDType` is the KV page type: F32, BF16, or I8 for Q8_0 pages (int8 values with one f32 scale per 32 elements; tpSize 1 only,
     * and one-session decode runs the per-op graph instead of the persistent kernel).
     */
    public CudaLlamaModel(Config c, WeightLoader weights, DType workingQType, DType kvDType, int maxSessions, int tpRank, int tpSize) {
        this.c = c;
        try {
            MemorySegment out = arena.allocate(ADDRESS), info = arena.allocate(JAVA_LONG, 4);
            check((int) jl_init.invokeExact(tpRank /* one GPU per process */, out, info), MemorySegment.NULL);
            this.ctx = out.get(ADDRESS, 0);
            MemorySegment cfg = arena.allocate(CONFIG);
            cfg.set(JAVA_INT, off("context_length"), c.contextLength);
            cfg.set(JAVA_INT, off("embedding_length"), c.embeddingLength);
            cfg.set(JAVA_INT, off("hidden_length"), c.hiddenLength);
            cfg.set(JAVA_INT, off("num_heads"), c.numberOfHeads);
            cfg.set(JAVA_INT, off("num_kv_heads"), c.numberOfKeyValueHeads);
            cfg.set(JAVA_INT, off("num_layers"), c.numberOfLayers);
            cfg.set(JAVA_INT, off("vocab_size"), c.vocabularySize);
            cfg.set(JAVA_INT, off("head_size"), c.headSize);
            cfg.set(JAVA_FLOAT, off("layer_norm_eps"), c.layerNormEps);
            cfg.set(JAVA_DOUBLE, off("rope_theta"), c.ropeFreqsTheta);
            cfg.set(JAVA_DOUBLE, off("rope_scaling"), c.ropeScalingFactor == null ? 1.0 : c.ropeScalingFactor);
            cfg.set(JAVA_INT, off("working_qtype"), code(workingQType));
            cfg.set(JAVA_INT, off("kv_dtype"), code(kvDType));
            cfg.set(JAVA_INT, off("max_batch"), 256);               // jlama.max_batch_size (AbstractModel.java:57)
            cfg.set(JAVA_INT, off("max_sessions"), maxSessions);
            cfg.set(JAVA_INT, off("tp_rank"), tpRank);
            cfg.set(JAVA_INT, off("tp_size"), tpSize);
            MemorySegment mo = arena.allocate(ADDRESS);
            check((int) jl_model_create.invokeExact(ctx, cfg, mo), ctx);
            this.model = mo.get(ADDRESS, 0);

            // loadInputWeights / loadOutputWeights (LlamaModel.java:88-97,145-156)
            bind(-1, T_EMBED, weights.load("model.embed_tokens.weight"));
            bind(-1, T_OUT_NORM, weights.load("model.norm.weight"));
            if (weights.isWeightPresent("lm_head.weight")) bind(-1, T_LM_HEAD, weights.load("lm_head.weight")); // else tied to the embedding
            // loadTransformerBlockWeights (:117-143): the same names, the same row / column splits
            for (int i = c.dctx().layerStart; i < c.dctx().layerEnd; i++) {
                String b = "model.layers." + i + ".";
                bind(i, L_ATTN_NORM, weights.load(b + "input_layernorm.weight"));
                bind(i, L_Q, weights.load(b + "self_attn.q_proj.weight", c.dctx(), true, false));
                bind(i, L_K, weights.load(b + "self_attn.k_proj.weight", c.dctx(), true, false));
                bind(i, L_V, weights.load(b + "self_attn.v_proj.weight", c.dctx(), true, false));
                bind(i, L_O, weights.load(b + "self_attn.o_proj.weight", c.dctx(), false, true));
                bind(i, L_FFN_NORM, weights.load(b + "post_attention_layernorm.weight"));
                bind(i, L_GATE, weights.load(b + "mlp.gate_proj.weight", c.dctx(), true, false));
                bind(i, L_DOWN, weights.load(b + "mlp.down_proj.weight", c.dctx(), false, true));
                bind(i, L_UP, weights.load(b + "mlp.up_proj.weight", c.dctx(), true, false));
            }
            check((int) jl_model_finalize.invokeExact(model), ctx);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    private static long off(String f) { return CONFIG.byteOffset(MemoryLayout.PathElement.groupElement(f)); }
    private static int code(DType t) {
        return switch (t) { case F32 -> JL_F32; case BF16 -> JL_BF16; case Q4 -> JL_Q4; case I8 -> JL_I8;
                            default -> throw new UnsupportedOperationException(t.name()); };
    }
    private static MemorySegment scales(AbstractTensor t) {
        if (t instanceof Q4ByteBufferTensor q) return q.getBlockF().getMemorySegment();
        if (t instanceof Q8ByteBufferTensor q) return q.getBlockF().getMemorySegment();
        return MemorySegment.NULL;
    }
    private void check(int rc, MemorySegment ctxOrNull) throws Throwable {
        if (rc >= 0) return;
        String msg = ctxOrNull.equals(MemorySegment.NULL) ? "" : ((MemorySegment) jl_last_error.invokeExact(ctxOrNull)).reinterpret(1024).getString(0);
        if (rc == -4) throw new UnsupportedOperationException(msg);
        if (rc == -1) throw new IllegalArgumentException(msg);
        throw new RuntimeException("libjlama_b200: " + rc + " " + msg);
    }
    /** registerModelTensor + jl_model_set_tensor: the stored (sparse) extent of the tensor is what this rank holds. */
    private void bind(int layer, int slot, AbstractTensor t) throws Throwable {
        long id = (long) jl_register_tensor.invokeExact(ctx, code(t.dType()), (long) t.shape().sparseRowLength(),
                                                       (long) t.shape().sparseColumnLength(), t.getMemorySegment(), scales(t));
        if (id < 0) throw new OutOfMemoryError("jl_register_tensor");
        tensorIds.add(id);
        check((int) jl_model_set_tensor.invokeExact(model, layer, slot, id), ctx);
    }

    /** AbstractModel.batchForward(int[] tokens, int startPos, KvBuffer kv) (:295-312): the session index stands for the KvBuffer. */
    public void batchForward(int session, int[] tokens, int startPos) {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment tk = a.allocateFrom(JAVA_INT, tokens);
            check((int) jl_model_batch_forward.invokeExact(model, session, tk, tokens.length, startPos), ctx);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** AbstractModel.sample (:443-491) on the last forwarded row: arg-max at temperature 0, else the reference's prefix-sum rule. */
    public int sample(int session, float temperature, float uniform, float[] logitsOrNull) {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment tok = a.allocate(JAVA_INT);
            MemorySegment lg = logitsOrNull == null ? MemorySegment.NULL : a.allocate(JAVA_FLOAT, logitsOrNull.length);
            check((int) jl_model_sample.invokeExact(model, session, temperature, uniform, tok, lg), ctx);
            if (logitsOrNull != null) MemorySegment.copy(lg, JAVA_FLOAT, 0, logitsOrNull, 0, logitsOrNull.length);
            return tok.get(JAVA_INT, 0);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** forward(token, position) + sample for n concurrent sessions in one launch (the reference's batch: KvBufferCache.java:58-60). */
    public int[] decode(int[] sessions, int[] tokens, int[] positions) {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment s = a.allocateFrom(JAVA_INT, sessions), t = a.allocateFrom(JAVA_INT, tokens), p = a.allocateFrom(JAVA_INT, positions);
            MemorySegment nxt = a.allocate(JAVA_INT, tokens.length);
            check((int) jl_model_decode.invokeExact(model, tokens.length, s, t, p, nxt, MemorySegment.NULL), ctx);
            return nxt.toArray(JAVA_INT);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /**
     * decode() with per-row sampling: rows at temperature 0 take the arg-max; rows with a temperature that topK (> 0) or topP (< 1)
     * filter draw with the top-k / top-p rule (DESIGN §3.12), the others with AbstractModel.sample's rule.  uniforms[i] in [0, 1].
     */
    public int[] decode(int[] sessions, int[] tokens, int[] positions, float[] temperatures, int[] topK, float[] topP, float[] uniforms) {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment s = a.allocateFrom(JAVA_INT, sessions), t = a.allocateFrom(JAVA_INT, tokens), p = a.allocateFrom(JAVA_INT, positions);
            MemorySegment tt = a.allocateFrom(JAVA_FLOAT, temperatures), k = a.allocateFrom(JAVA_INT, topK), tp = a.allocateFrom(JAVA_FLOAT, topP);
            MemorySegment u = a.allocateFrom(JAVA_FLOAT, uniforms), nxt = a.allocate(JAVA_INT, tokens.length);
            check((int) jl_model_decode_sample_topkp.invokeExact(model, tokens.length, s, t, p, tt, k, tp, u, nxt, MemorySegment.NULL), ctx);
            return nxt.toArray(JAVA_INT);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** AbstractModel.generate with a temperature and a token filter: uniforms[i] plays the i-th nextFloat() of the loop (:576, :594). */
    public int[] generate(int session, int[] prompt, int nNew, float temperature, int topK, float topP, float[] uniforms, double[] timingsMs) {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment pr = a.allocateFrom(JAVA_INT, prompt), u = a.allocateFrom(JAVA_FLOAT, uniforms), out = a.allocate(JAVA_INT, nNew);
            MemorySegment tm = a.allocate(JAVA_DOUBLE, 2);
            check((int) jl_model_generate_sample_topkp.invokeExact(model, session, pr, prompt.length, nNew, temperature, topK, topP, u, out, tm), ctx);
            if (timingsMs != null) { timingsMs[0] = tm.getAtIndex(JAVA_DOUBLE, 0); timingsMs[1] = tm.getAtIndex(JAVA_DOUBLE, 1); }
            return out.toArray(JAVA_INT);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** Up to JL_MAX_LOGPROBS top alternatives per token (OpenAI's top_logprobs limit). */
    public static final int MAX_LOGPROBS = 20;

    /**
     * Log-probabilities of tokens (DESIGN §3.13): lp[i] is token i's, topIds[i][0..n) / topLp[i][0..n) its n most likely alternatives,
     * best first; rows without logprobs hold NaN, slots past n hold id -1 and NaN.
     */
    public record TokenLogprobs(float[] lp, int[][] topIds, float[][] topLp) {
        static TokenLogprobs of(MemorySegment lp, MemorySegment ids, MemorySegment tlp, int n) {
            int[][] ti = new int[n][];
            float[][] tl = new float[n][];
            for (int i = 0; i < n; i++) {
                ti[i] = ids.asSlice((long) i * MAX_LOGPROBS * 4, MAX_LOGPROBS * 4L).toArray(JAVA_INT);
                tl[i] = tlp.asSlice((long) i * MAX_LOGPROBS * 4, MAX_LOGPROBS * 4L).toArray(JAVA_FLOAT);
            }
            return new TokenLogprobs(lp.toArray(JAVA_FLOAT), ti, tl);
        }
    }

    /**
     * decode() with per-row sampling (as above) and log-probabilities: topN[i] = -1 (none), 0 (the chosen token's), up to 20 alternatives;
     * an OpenAI chat request's logprobs / top_logprobs.  The tokens are those of the same call without topN.  Fills `logprobs` (n rows).
     */
    public int[] decode(int[] sessions, int[] tokens, int[] positions, float[] temperatures, int[] topK, float[] topP, float[] uniforms, int[] topN,
                        TokenLogprobs[] logprobs) {
        try (Arena a = Arena.ofConfined()) {
            int n = tokens.length;
            MemorySegment s = a.allocateFrom(JAVA_INT, sessions), t = a.allocateFrom(JAVA_INT, tokens), p = a.allocateFrom(JAVA_INT, positions);
            MemorySegment tt = a.allocateFrom(JAVA_FLOAT, temperatures), k = a.allocateFrom(JAVA_INT, topK), tp = a.allocateFrom(JAVA_FLOAT, topP);
            MemorySegment u = a.allocateFrom(JAVA_FLOAT, uniforms), tn = a.allocateFrom(JAVA_INT, topN), nxt = a.allocate(JAVA_INT, n);
            MemorySegment lp = a.allocate(JAVA_FLOAT, n), ids = a.allocate(JAVA_INT, (long) n * MAX_LOGPROBS), tlp = a.allocate(JAVA_FLOAT, (long) n * MAX_LOGPROBS);
            check((int) jl_model_decode_logprobs.invokeExact(model, n, s, t, p, tt, k, tp, u, tn, nxt, lp, ids, tlp, MemorySegment.NULL), ctx);
            logprobs[0] = TokenLogprobs.of(lp, ids, tlp, n);
            return nxt.toArray(JAVA_INT);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** generate() with a token filter and topN log-probabilities for every generated token (fills logprobs[0]). */
    public int[] generate(int session, int[] prompt, int nNew, float temperature, int topK, float topP, float[] uniforms, int topN,
                          TokenLogprobs[] logprobs, double[] timingsMs) {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment pr = a.allocateFrom(JAVA_INT, prompt), u = a.allocateFrom(JAVA_FLOAT, uniforms), out = a.allocate(JAVA_INT, nNew);
            MemorySegment lp = a.allocate(JAVA_FLOAT, nNew), ids = a.allocate(JAVA_INT, (long) nNew * MAX_LOGPROBS);
            MemorySegment tlp = a.allocate(JAVA_FLOAT, (long) nNew * MAX_LOGPROBS), tm = a.allocate(JAVA_DOUBLE, 2);
            check((int) jl_model_generate_logprobs.invokeExact(model, session, pr, prompt.length, nNew, temperature, topK, topP, u, topN, out, lp, ids,
                                                               tlp, tm), ctx);
            if (timingsMs != null) { timingsMs[0] = tm.getAtIndex(JAVA_DOUBLE, 0); timingsMs[1] = tm.getAtIndex(JAVA_DOUBLE, 1); }
            logprobs[0] = TokenLogprobs.of(lp, ids, tlp, nNew);
            return out.toArray(JAVA_INT);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /**
     * Prompt scoring (an OpenAI completions request with echo and logprobs): batchForward that also returns, for each token, its
     * log-probability given everything before it in the session and topN (0..20) alternatives; entry 0 is NaN with id -1.
     */
    public TokenLogprobs score(int session, int[] tokens, int startPos, int topN) {
        try (Arena a = Arena.ofConfined()) {
            int n = tokens.length;
            MemorySegment tk = a.allocateFrom(JAVA_INT, tokens), lp = a.allocate(JAVA_FLOAT, n);
            MemorySegment ids = a.allocate(JAVA_INT, (long) n * MAX_LOGPROBS), tlp = a.allocate(JAVA_FLOAT, (long) n * MAX_LOGPROBS);
            check((int) jl_model_score.invokeExact(model, session, tk, n, startPos, topN, lp, ids, tlp), ctx);
            return TokenLogprobs.of(lp, ids, tlp, n);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** jl_penalties, member for member: nine pointers to host arrays. */
    static final StructLayout PENALTIES = MemoryLayout.structLayout(
        ADDRESS.withName("presence"), ADDRESS.withName("frequency"), ADDRESS.withName("repetition"), ADDRESS.withName("hist_off"),
        ADDRESS.withName("hist_prompt"), ADDRESS.withName("hist_ids"), ADDRESS.withName("bias_off"), ADDRESS.withName("bias_ids"),
        ADDRESS.withName("bias_vals"));

    /**
     * The penalties of one row (DESIGN §3.14): OpenAI's presence_penalty / frequency_penalty in [-2, 2], Hugging Face's repetition_penalty
     * in (0, 100] (1 = off) and OpenAI's logit_bias (biasIds[j] gets biasValues[j] in [-100, 100] added).  The history is the row's prompt
     * ids, then its generated ids (in a decode step including the token fed in).  generate() takes one without a history.
     */
    public record Penalties(float presence, float frequency, float repetition, int[] biasIds, float[] biasValues, int[] prompt, int[] generated) {
        public Penalties(float presence, float frequency, float repetition, int[] biasIds, float[] biasValues) {
            this(presence, frequency, repetition, biasIds, biasValues, new int[0], new int[0]);
        }
    }

    /** rows -> one jl_penalties in `a` (null rows are unpenalised with empty histories) */
    static MemorySegment penalties(Arena a, Penalties[] rows) {
        int n = rows.length, nh = 0, nb = 0;
        for (Penalties q : rows) if (q != null) { nh += q.prompt().length + q.generated().length; nb += q.biasIds().length; }
        MemorySegment pr = a.allocate(JAVA_FLOAT, n), fr = a.allocate(JAVA_FLOAT, n), rp = a.allocate(JAVA_FLOAT, n);
        MemorySegment hoff = a.allocate(JAVA_INT, n + 1), hp = a.allocate(JAVA_INT, n), hid = a.allocate(JAVA_INT, Math.max(nh, 1));
        MemorySegment boff = a.allocate(JAVA_INT, n + 1), bid = a.allocate(JAVA_INT, Math.max(nb, 1)), bv = a.allocate(JAVA_FLOAT, Math.max(nb, 1));
        int h = 0, b = 0;
        for (int i = 0; i < n; i++) {
            Penalties q = rows[i];
            pr.setAtIndex(JAVA_FLOAT, i, q == null ? 0f : q.presence());
            fr.setAtIndex(JAVA_FLOAT, i, q == null ? 0f : q.frequency());
            rp.setAtIndex(JAVA_FLOAT, i, q == null ? 1f : q.repetition());
            hoff.setAtIndex(JAVA_INT, i, h);
            boff.setAtIndex(JAVA_INT, i, b);
            hp.setAtIndex(JAVA_INT, i, q == null ? 0 : q.prompt().length);
            if (q == null) continue;
            for (int t : q.prompt()) hid.setAtIndex(JAVA_INT, h++, t);
            for (int t : q.generated()) hid.setAtIndex(JAVA_INT, h++, t);
            for (int j = 0; j < q.biasIds().length; j++, b++) { bid.setAtIndex(JAVA_INT, b, q.biasIds()[j]); bv.setAtIndex(JAVA_FLOAT, b, q.biasValues()[j]); }
        }
        hoff.setAtIndex(JAVA_INT, n, h);
        boff.setAtIndex(JAVA_INT, n, b);
        MemorySegment pen = a.allocate(PENALTIES);
        MemorySegment[] members = {pr, fr, rp, hoff, hp, hid, boff, bid, bv};
        for (int m = 0; m < members.length; m++) pen.setAtIndex(ADDRESS, m, members[m]);
        return pen;
    }

    /**
     * decode() with sampling, log-probabilities (topN as above) and per-row penalties (null rows unpenalised): each row is selected from
     * its processed logits; the logprobs stay those of the raw logits.  Fills `logprobs` (n rows).
     */
    public int[] decode(int[] sessions, int[] tokens, int[] positions, float[] temperatures, int[] topK, float[] topP, float[] uniforms, int[] topN,
                        Penalties[] penalties, TokenLogprobs[] logprobs) {
        try (Arena a = Arena.ofConfined()) {
            int n = tokens.length;
            MemorySegment s = a.allocateFrom(JAVA_INT, sessions), t = a.allocateFrom(JAVA_INT, tokens), p = a.allocateFrom(JAVA_INT, positions);
            MemorySegment tt = a.allocateFrom(JAVA_FLOAT, temperatures), k = a.allocateFrom(JAVA_INT, topK), tp = a.allocateFrom(JAVA_FLOAT, topP);
            MemorySegment u = a.allocateFrom(JAVA_FLOAT, uniforms), tn = a.allocateFrom(JAVA_INT, topN), nxt = a.allocate(JAVA_INT, n);
            MemorySegment lp = a.allocate(JAVA_FLOAT, n), ids = a.allocate(JAVA_INT, (long) n * MAX_LOGPROBS), tlp = a.allocate(JAVA_FLOAT, (long) n * MAX_LOGPROBS);
            MemorySegment pen = penalties(a, penalties);
            check((int) jl_model_decode_penalized.invokeExact(model, n, s, t, p, tt, k, tp, u, tn, pen, nxt, lp, ids, tlp, MemorySegment.NULL), ctx);
            logprobs[0] = TokenLogprobs.of(lp, ids, tlp, n);
            return nxt.toArray(JAVA_INT);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** the vocabulary of the model: the width of its allowed-token masks is (vocab + 31) / 32 words */
    public int vocabularySize() {
        return c.vocabularySize;
    }

    /**
     * Allowed-token masks of one call (DESIGN §3.18): a null row is unconstrained, otherwise token t is allowed where allowed[i][t].
     * Returns {allow [n_allow][words], allow_row [n]}; n_allow = the constrained rows.
     */
    static MemorySegment[] masks(Arena a, boolean[][] allowed, int vocab) {
        int words = (vocab + 31) / 32, nAllow = 0;
        for (boolean[] r : allowed) if (r != null) nAllow++;
        MemorySegment allow = a.allocate(JAVA_INT, Math.max(1, (long) nAllow * words)), rows = a.allocate(JAVA_INT, allowed.length);
        int k = 0;
        for (int i = 0; i < allowed.length; i++) {
            rows.setAtIndex(JAVA_INT, i, allowed[i] == null ? -1 : k);
            if (allowed[i] == null) continue;
            for (int t = 0; t < vocab; t++)
                if (allowed[i][t]) {
                    long w = (long) k * words + t / 32;
                    allow.setAtIndex(JAVA_INT, w, allow.getAtIndex(JAVA_INT, w) | (1 << (t % 32)));
                }
            k++;
        }
        return new MemorySegment[] {allow, rows, MemorySegment.ofArray(new int[] {nAllow})};
    }

    /**
     * decode() with penalties and allowed-token masks (a grammar engine's masks for JSON mode, a JSON schema, a regex or a choice; DESIGN
     * §3.18): each constrained row is selected from its processed logits with every token outside its allowed set at -inf, greedy rows
     * by the arg-max, sampled rows by the top-k / top-p rule.  Null mask rows are exactly what the penalties-only decode() gives them.
     */
    public int[] decode(int[] sessions, int[] tokens, int[] positions, float[] temperatures, int[] topK, float[] topP, float[] uniforms, int[] topN,
                        Penalties[] penalties, boolean[][] allowed, TokenLogprobs[] logprobs) {
        try (Arena a = Arena.ofConfined()) {
            int n = tokens.length;
            MemorySegment s = a.allocateFrom(JAVA_INT, sessions), t = a.allocateFrom(JAVA_INT, tokens), p = a.allocateFrom(JAVA_INT, positions);
            MemorySegment tt = a.allocateFrom(JAVA_FLOAT, temperatures), k = a.allocateFrom(JAVA_INT, topK), tp = a.allocateFrom(JAVA_FLOAT, topP);
            MemorySegment u = a.allocateFrom(JAVA_FLOAT, uniforms), tn = a.allocateFrom(JAVA_INT, topN), nxt = a.allocate(JAVA_INT, n);
            MemorySegment lp = a.allocate(JAVA_FLOAT, n), ids = a.allocate(JAVA_INT, (long) n * MAX_LOGPROBS), tlp = a.allocate(JAVA_FLOAT, (long) n * MAX_LOGPROBS);
            MemorySegment pen = penalties(a, penalties);
            MemorySegment[] m = masks(a, allowed, c.vocabularySize);
            int nAllow = m[2].getAtIndex(JAVA_INT, 0);
            check((int) jl_model_decode_constrained.invokeExact(model, n, s, t, p, tt, k, tp, u, tn, pen, nAllow, m[0], m[1], nxt, lp, ids, tlp,
                                                                MemorySegment.NULL), ctx);
            logprobs[0] = TokenLogprobs.of(lp, ids, tlp, n);
            return nxt.toArray(JAVA_INT);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** The first tokens of n prefilled sessions under penalties and allowed-token masks, as decode() above.  Fills `logprobs`. */
    public int[] sampleMulti(int[] sessions, float[] temperatures, int[] topK, float[] topP, float[] uniforms, int[] topN, Penalties[] penalties,
                             boolean[][] allowed, TokenLogprobs[] logprobs) {
        try (Arena a = Arena.ofConfined()) {
            int n = sessions.length;
            MemorySegment s = a.allocateFrom(JAVA_INT, sessions), tt = a.allocateFrom(JAVA_FLOAT, temperatures), k = a.allocateFrom(JAVA_INT, topK);
            MemorySegment tp = a.allocateFrom(JAVA_FLOAT, topP), u = a.allocateFrom(JAVA_FLOAT, uniforms), tn = a.allocateFrom(JAVA_INT, topN);
            MemorySegment out = a.allocate(JAVA_INT, n), lp = a.allocate(JAVA_FLOAT, n), ids = a.allocate(JAVA_INT, (long) n * MAX_LOGPROBS);
            MemorySegment tlp = a.allocate(JAVA_FLOAT, (long) n * MAX_LOGPROBS);
            MemorySegment pen = penalties(a, penalties);
            MemorySegment[] m = masks(a, allowed, c.vocabularySize);
            int nAllow = m[2].getAtIndex(JAVA_INT, 0);
            check((int) jl_model_sample_multi_constrained.invokeExact(model, n, s, tt, k, tp, u, tn, pen, nAllow, m[0], m[1], out, lp, ids, tlp,
                                                                      MemorySegment.NULL), ctx);
            logprobs[0] = TokenLogprobs.of(lp, ids, tlp, n);
            return out.toArray(JAVA_INT);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** generate() with a token filter, topN log-probabilities and the same penalties for every token (its history ignored: token k's is
     *  the prompt and the k tokens before it).  Fills logprobs[0]. */
    public int[] generate(int session, int[] prompt, int nNew, float temperature, int topK, float topP, float[] uniforms, int topN,
                          Penalties penalties, TokenLogprobs[] logprobs, double[] timingsMs) {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment pr = a.allocateFrom(JAVA_INT, prompt), u = a.allocateFrom(JAVA_FLOAT, uniforms), out = a.allocate(JAVA_INT, nNew);
            MemorySegment lp = a.allocate(JAVA_FLOAT, nNew), ids = a.allocate(JAVA_INT, (long) nNew * MAX_LOGPROBS);
            MemorySegment tlp = a.allocate(JAVA_FLOAT, (long) nNew * MAX_LOGPROBS), tm = a.allocate(JAVA_DOUBLE, 2);
            int nb = penalties.biasIds().length;
            MemorySegment bi = a.allocateFrom(JAVA_INT, penalties.biasIds()), bv = a.allocateFrom(JAVA_FLOAT, penalties.biasValues());
            check((int) jl_model_generate_penalized.invokeExact(model, session, pr, prompt.length, nNew, temperature, topK, topP, u, topN,
                                                                penalties.presence(), penalties.frequency(), penalties.repetition(), nb, bi, bv, out,
                                                                lp, ids, tlp, tm), ctx);
            if (timingsMs != null) { timingsMs[0] = tm.getAtIndex(JAVA_DOUBLE, 0); timingsMs[1] = tm.getAtIndex(JAVA_DOUBLE, 1); }
            logprobs[0] = TokenLogprobs.of(lp, ids, tlp, nNew);
            return out.toArray(JAVA_INT);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** AbstractModel.generate (:516-646) at temperature 0 over token ids; timingsMs = {prompt, generate} like Generator.Response. */
    public int[] generate(int session, int[] prompt, int nNew, double[] timingsMs) {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment pr = a.allocateFrom(JAVA_INT, prompt), out = a.allocate(JAVA_INT, nNew), tm = a.allocate(JAVA_DOUBLE, 2);
            check((int) jl_model_generate.invokeExact(model, session, pr, prompt.length, nNew, out, MemorySegment.NULL, tm), ctx);
            if (timingsMs != null) { timingsMs[0] = tm.getAtIndex(JAVA_DOUBLE, 0); timingsMs[1] = tm.getAtIndex(JAVA_DOUBLE, 1); }
            return out.toArray(JAVA_INT);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** KvBufferCache.KvBufferPage persistence (KvBufferCache.java:121-176): <dir>/<session>-L<l>C<c>.page, the reference's own files. */
    public int saveKv(int session, String workingDirectory, java.util.UUID sessionId) {
        try (Arena a = Arena.ofConfined()) {
            int n = (int) jl_model_kv_save.invokeExact(model, session, a.allocateFrom(workingDirectory), a.allocateFrom(sessionId.toString()));
            check(n, ctx);
            return n;
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }
    public int loadKv(int session, String workingDirectory, java.util.UUID sessionId) {
        try (Arena a = Arena.ofConfined()) {
            int n = (int) jl_model_kv_load.invokeExact(model, session, a.allocateFrom(workingDirectory), a.allocateFrom(sessionId.toString()));
            check(n, ctx);
            return n;
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** jl_model* for the classes of this package that take the model as an argument (CudaSessionScheduler). */
    MemorySegment handle() { return model; }

    public void resetSession(int session) {
        try { check((int) jl_model_reset_session.invokeExact(model, session), ctx); }
        catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /**
     * Each session of dst becomes what src holds for positions [0, positions): whole KV pages are shared copy-on-write, the page holding
     * positions - 1 is copied, and sampling on dst draws from src's last forwarded row (DESIGN §3.15).
     */
    public void forkSession(int src, int positions, int[] dst) {
        try (Arena a = Arena.ofConfined()) {
            check((int) jl_model_kv_fork.invokeExact(model, src, positions, dst.length, a.allocateFrom(JAVA_INT, dst)), ctx);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** {pages allocated, page-table entries}: a KV page shared by k sessions counts once in the first and k times in the second. */
    public long[] kvPageStats() {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment alloc = a.allocate(JAVA_LONG), entries = a.allocate(JAVA_LONG);
            check((int) jl_model_kv_page_stats.invokeExact(model, alloc, entries), ctx);
            return new long[] {alloc.get(JAVA_LONG, 0), entries.get(JAVA_LONG, 0)};
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /**
     * Hold the session's KV pages wholly below positions (a multiple of the page size) beyond the session's life; returns the handle
     * attachKv and releaseKv take (DESIGN §3.17).
     */
    public long retainKv(int session, int positions) {
        try {
            long h = (long) jl_model_kv_retain.invokeExact(model, session, positions);
            if (h < 0) check((int) h, ctx);
            return h;
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** The session becomes what the handle holds for [0, positions): no bytes move.  Forward at least one token before sampling. */
    public void attachKv(long handle, int positions, int session) {
        try {
            check((int) jl_model_kv_attach.invokeExact(model, handle, positions, session), ctx);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    public void releaseKv(long handle) {
        try {
            check((int) jl_model_kv_release.invokeExact(model, handle), ctx);
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    /** {handles alive, pages held by handles and by no session}. */
    public long[] kvRetained() {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment handles = a.allocate(JAVA_LONG), pages = a.allocate(JAVA_LONG);
            check((int) jl_model_kv_retained.invokeExact(model, handles, pages), ctx);
            return new long[] {handles.get(JAVA_LONG, 0), pages.get(JAVA_LONG, 0)};
        } catch (RuntimeException | Error e) { throw e; } catch (Throwable t) { throw new RuntimeException(t); }
    }

    @Override public void close() {
        try { int rc = (int) jl_model_free.invokeExact(model); } catch (Throwable ignored) { }
        arena.close();
    }
}
