"""ctypes binding of libjlama_b200.so (the C ABI in include/jlama_b200.h).

This is the Python stand-in for the Panama-FFI binding a Jlama maintainer would generate with
jextract (INTEGRATION.md).  There is no fallback: if the shared library is missing or the device is
not an sm_90 (H100) GPU, loading / jl_init fails loudly.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libjlama_b200.so")

JL_OK, JL_ERR_INVALID, JL_ERR_CUDA, JL_ERR_OOM, JL_ERR_UNSUPPORTED, JL_ERR_NCCL = 0, -1, -2, -3, -4, -5
F32, BF16, Q4, I8 = 0, 1, 2, 3
JL_MAX_DECODE_ROWS = 64  # most sessions in one jl_model_decode call
JL_MAX_LOGPROBS = 20  # most top alternatives per token of the logprob calls
MODEL_NO_GRAPH, MODEL_NO_PERSISTENT = 1, 4

T_EMBED, T_OUT_NORM, T_LM_HEAD = 0, 1, 2
L_ATTN_NORM, L_Q, L_K, L_V, L_O, L_FFN_NORM, L_GATE, L_DOWN, L_UP = range(9)


class JlamaNativeError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("jlama_b200 error %d: %s" % (code, msg))
        self.code = code


class UnsupportedOperation(JlamaNativeError):
    """UnsupportedOperationException analogue (TestOperations.java:140 relies on it)."""


class ModelConfig(C.Structure):
    _fields_ = [
        ("context_length", C.c_int), ("embedding_length", C.c_int), ("hidden_length", C.c_int),
        ("num_heads", C.c_int), ("num_kv_heads", C.c_int), ("num_layers", C.c_int), ("vocab_size", C.c_int),
        ("head_size", C.c_int), ("layer_norm_eps", C.c_float), ("rope_theta", C.c_double), ("rope_scaling", C.c_double),
        ("working_qtype", C.c_int), ("kv_dtype", C.c_int), ("max_batch", C.c_int), ("max_sessions", C.c_int),
        ("max_context", C.c_int), ("tp_rank", C.c_int), ("tp_size", C.c_int), ("prefill_tensor_core", C.c_int),
        ("flags", C.c_int), ("num_experts", C.c_int), ("experts_per_token", C.c_int), ("arch", C.c_int),
    ]


class Dctx(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "embeddingSegmentStart", "embeddingSegmentLength", "attentionSegmentStart", "attentionSegmentLength",
        "hiddenSegmentStart", "hiddenSegmentLength", "kvSegmentStart", "kvSegmentLength", "headStart", "headEnd",
        "groupHeadStart", "groupHeadEnd", "numberOfLayers", "layerStart", "layerEnd")]


class SchedStats(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("admitted", "prefill_tokens", "decode_rows", "decode_calls", "finished", "active", "queued",
                                        "spilled")]


class SchedRequestInfo(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("state", "finish_reason", "session", "start_pos", "n_prompt", "n_prefilled", "n_generated",
                                        "next_position", "spilled")] + [(n, C.c_int64) for n in ("submit_step", "first_token_step", "finish_step")] + [
        (n, C.c_double) for n in ("queue_ms", "prompt_ms", "generate_ms")]


# jl_sched_backend: the four model calls the scheduler policy is written against
SCHED_RESET_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int)
SCHED_FORWARD_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_int)
SCHED_SAMPLE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_float, C.POINTER(C.c_int32))
SCHED_DECODE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                              C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int32))


SCHED_OFFLOAD_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int64))
SCHED_RESTORE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int64)
SCHED_DISCARD_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int64)


class SchedBackend(C.Structure):
    _fields_ = [("reset_session", SCHED_RESET_FN), ("batch_forward", SCHED_FORWARD_FN), ("sample", SCHED_SAMPLE_FN),
                ("decode", SCHED_DECODE_FN), ("offload", SCHED_OFFLOAD_FN), ("restore", SCHED_RESTORE_FN), ("discard", SCHED_DISCARD_FN)]


# jl_sched_batch_backend: the batched prompt calls (jl_model_batch_forward_multi / jl_model_sample_multi)
SCHED_FORWARD_MULTI_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                     C.POINTER(C.c_int32))
SCHED_SAMPLE_MULTI_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                    C.POINTER(C.c_int32))


class SchedBatchBackend(C.Structure):
    _fields_ = [("forward_multi", SCHED_FORWARD_MULTI_FN), ("sample_multi", SCHED_SAMPLE_MULTI_FN)]


# jl_sched_topkp_backend: the calls with top-k / top-p filtered rows (jl_model_decode_sample_topkp / jl_model_sample_multi_topkp)
SCHED_DECODE_TOPKP_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                    C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                    C.POINTER(C.c_int32))
SCHED_SAMPLE_MULTI_TOPKP_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_int32),
                                          C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int32))


class SchedTopkpBackend(C.Structure):
    _fields_ = [("decode_topkp", SCHED_DECODE_TOPKP_FN), ("sample_multi_topkp", SCHED_SAMPLE_MULTI_TOPKP_FN)]


# jl_sched_logprob_backend: the calls with a logprob request (jl_model_decode_logprobs / jl_model_sample_multi_logprobs)
SCHED_DECODE_LOGPROBS_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                       C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                       C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_int32),
                                       C.POINTER(C.c_float))
SCHED_SAMPLE_MULTI_LOGPROBS_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_int32),
                                             C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                             C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_float))


class SchedLogprobBackend(C.Structure):
    _fields_ = [("decode_logprobs", SCHED_DECODE_LOGPROBS_FN), ("sample_multi_logprobs", SCHED_SAMPLE_MULTI_LOGPROBS_FN)]


class Penalties(C.Structure):
    """jl_penalties: per-row penalty arrays of the *_penalized calls (DESIGN §3.14), every member a HOST pointer"""
    _fields_ = [(n, C.c_void_p) for n in ("presence", "frequency", "repetition", "hist_off", "hist_prompt", "hist_ids", "bias_off", "bias_ids",
                                           "bias_vals")]


# jl_sched_penalty_backend: the calls with a penalised request (jl_model_decode_penalized / jl_model_sample_multi_penalized)
SCHED_DECODE_PENALIZED_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                        C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                        C.POINTER(C.c_int32), C.POINTER(Penalties), C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                        C.POINTER(C.c_int32), C.POINTER(C.c_float))
SCHED_SAMPLE_MULTI_PENALIZED_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_int32),
                                              C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(Penalties),
                                              C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_float))


class SchedPenaltyBackend(C.Structure):
    _fields_ = [("decode_penalized", SCHED_DECODE_PENALIZED_FN), ("sample_multi_penalized", SCHED_SAMPLE_MULTI_PENALIZED_FN)]


# jl_sched_constraint_backend: the calls with a constrained request (jl_model_decode_constrained / jl_model_sample_multi_constrained) and
# the vocabulary of their masks
SCHED_DECODE_CONSTRAINED_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                          C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                          C.POINTER(C.c_int32), C.POINTER(Penalties), C.c_int, C.POINTER(C.c_uint32), C.POINTER(C.c_int32),
                                          C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_float))
SCHED_SAMPLE_MULTI_CONSTRAINED_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_int32),
                                                C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(Penalties), C.c_int,
                                                C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                                C.POINTER(C.c_int32), C.POINTER(C.c_float))


class SchedConstraintBackend(C.Structure):
    _fields_ = [("decode_constrained", SCHED_DECODE_CONSTRAINED_FN), ("sample_multi_constrained", SCHED_SAMPLE_MULTI_CONSTRAINED_FN),
                ("vocab", C.c_int)]


# jl_sched_mask_fn: the mask provider of constrained requests (user, request, generated, n_generated, allow_out)
SCHED_MASK_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_uint32))


# jl_sched_fork_backend: n completions of one prompt (jl_model_kv_fork)
SCHED_FORK_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32))


class SchedForkBackend(C.Structure):
    _fields_ = [("fork", SCHED_FORK_FN)]


# jl_sched_prefix_backend: the prefix cache's retained prefixes (jl_model_kv_retain / kv_attach / kv_release / kv_retained)
SCHED_RETAIN_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int64))
SCHED_ATTACH_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int)
SCHED_RELEASE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int64)
SCHED_RETAINED_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64))


class SchedPrefixBackend(C.Structure):
    _fields_ = [("retain", SCHED_RETAIN_FN), ("attach", SCHED_ATTACH_FN), ("release", SCHED_RELEASE_FN), ("retained", SCHED_RETAINED_FN),
                ("ctx_per_page", C.c_int)]


class SchedPrefixStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("entries", "lookups", "hits", "cached_tokens", "evictions", "pages_retained_only")]


SCHED_QUEUED, SCHED_PREFILL, SCHED_DECODING, SCHED_FINISHED, SCHED_FAILED = range(5)
FINISH_NONE, FINISH_MAX_TOKENS, FINISH_STOP_TOKEN, FINISH_CANCELLED, FINISH_ERROR = range(5)
SCHED_KEEP_SESSION = 1
SCHED_CONSTRAINED = 2

# every symbol include/jlama_b200.h declares: (restype, argtypes)
_vp, _i, _i64, _f, _d = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_double
SIGNATURES = {
    "jl_init": (_i, [_i, C.POINTER(_vp), _vp]),
    "jl_shutdown": (_i, [_vp]),
    "jl_last_error": (C.c_char_p, [_vp]),
    "jl_version": (C.c_char_p, []),
    "jl_sync": (_i, [_vp]),
    "jl_kernel_launches": (_i64, [_vp]),
    "jl_debug_ktrace": (_i, [_vp, _i]),
    "jl_debug_ktrace_clear": (_i, [_vp]),
    "jl_debug_ktrace_read": (_i, [_vp, C.POINTER(C.c_uint64), _i]),
    "jl_debug_gemv_bench": (_i, [_vp, _i64, _i, _i, _i, _i, C.POINTER(_d)]),
    "jl_debug_gemm_tc_bench": (_i, [_vp, _i64, _i, _i, C.POINTER(_d)]),
    "jl_register_tensor": (_i64, [_vp, _i, _i64, _i64, _vp, _vp]),
    "jl_unregister_tensor": (_i, [_vp, _i64]),
    "jl_gemm": (_i, [_vp, _i, _vp, _vp, _i, _i, _i64, _i, _vp, _i, _i, _i, _i, _i, _i]),
    "jl_gemm_tc": (_i, [_vp, _i, _vp, _i, _i, _i64, _i, _vp, _i, _i, _i, _i, _i, _i]),
    "jl_gemm_batch": (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _vp, _i, _vp, _i, _i, _i, _i, _i, _i]),
    "jl_gemm_host": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _i, _i, _vp, _i, _i, _i, _i, _i, _i]),
    "jl_accumulate": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _i, _i, _i, _i]),
    "jl_maccumulate": (_i, [_vp, _vp, _i, _i, _vp, _i, _i, _i, _i]),
    "jl_scale": (_i, [_vp, _f, _vp, _i, _i, _i, _i]),
    "jl_saxpy": (_i, [_vp, _f, _vp, _vp, _i, _i, _i]),
    "jl_saxpy_batch": (_i, [_vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i]),
    "jl_quantize_q8": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "jl_quantize_bf16": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "jl_quantize_q4_weights": (_i, [_vp, _vp, _i64, _i64, _vp, _vp]),
    "jl_quantize_q8_weights": (_i, [_vp, _vp, _i64, _i64, _vp, _vp]),
    "jl_st_open": (_i, [C.c_char_p, C.POINTER(_vp)]),
    "jl_st_close": (_i, [_vp]),
    "jl_st_last_error": (C.c_char_p, []),
    "jl_st_count": (_i, [_vp]),
    "jl_st_find": (_i, [_vp, C.c_char_p]),
    "jl_st_info": (_i, [_vp, _i, C.POINTER(C.c_char_p), C.POINTER(_i), C.POINTER(_i), C.POINTER(_i64), C.POINTER(_i64)]),
    "jl_st_data": (_vp, [_vp, _i]),
    "jl_st_metadata": (C.c_char_p, [_vp, C.c_char_p]),
    "jl_st_majority_dtype": (_i, [_vp]),
    "jl_st_write": (_i, [C.c_char_p, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    "jl_quantize_model": (_i, [_vp, C.c_char_p, C.c_char_p, _i, C.c_char_p, C.c_char_p]),
    "jl_config_from_json": (_i, [C.c_char_p, C.POINTER(ModelConfig)]),
    "jl_model_load_safetensors": (_i, [_vp, _vp, _vp, _vp, _i, C.POINTER(_i)]),
    "jl_model_tp_layout": (_i, [_vp, C.POINTER(Dctx), C.POINTER(_i)]),
    "jl_rmsnorm": (_i, [_vp, _vp, _i, _i, _i, _vp, _f, _f, _i, _i, _i, _vp]),
    "jl_softmax": (_i, [_vp, _vp, _i, _i]),
    "jl_layernorm": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _vp, _f, _i, _i, _i, _vp]),
    "jl_activation": (_i, [_vp, _i, _vp, _i, _i, _i, _i]),
    "jl_silu_mul": (_i, [_vp, _vp, _vp, _i, _i, _i, _i]),
    "jl_precompute_freqs_cis": (_i, [_i, _i, _d, _d, _vp]),
    "jl_dctx_build": (_i, [_i] * 10 + [C.POINTER(Dctx)]),
    "jl_kv_page_geometry": (_i, [_i, _i, _i, _i, _i64, C.POINTER(_i), C.POINTER(_i)]),
    "jl_model_create": (_i, [_vp, C.POINTER(ModelConfig), C.POINTER(_vp)]),
    "jl_model_set_tensor": (_i, [_vp, _i, _i, _i64]),
    "jl_model_config_size": (_i, []),
    "jl_model_set_expert_tensor": (_i, [_vp, _i, _i, _i, _i64]),
    "jl_model_set_aux_tensor": (_i, [_vp, _i, _i, _i64]),
    "jl_model_finalize": (_i, [_vp]),
    "jl_model_free": (_i, [_vp]),
    "jl_model_reset_session": (_i, [_vp, _i]),
    "jl_model_batch_forward": (_i, [_vp, _i, _vp, _i, _i]),
    "jl_model_sample": (_i, [_vp, _i, _f, _f, _vp, _vp]),
    "jl_model_batch_forward_multi": (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    "jl_model_sample_multi": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "jl_model_decode": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "jl_model_generate": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _vp]),
    "jl_model_decode_sample": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "jl_model_generate_sample": (_i, [_vp, _i, _vp, _i, _i, _f, _vp, _vp, _vp]),
    "jl_model_decode_sample_topkp": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "jl_model_sample_multi_topkp": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "jl_model_generate_sample_topkp": (_i, [_vp, _i, _vp, _i, _i, _f, _i, _f, _vp, _vp, _vp]),
    "jl_sample_topkp": (_i, [_vp, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "jl_model_decode_logprobs": (_i, [_vp, _i] + [_vp] * 13),
    "jl_model_sample_multi_logprobs": (_i, [_vp, _i] + [_vp] * 11),
    "jl_model_generate_logprobs": (_i, [_vp, _i, _vp, _i, _i, _f, _i, _f, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "jl_model_score_multi": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "jl_model_score": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "jl_logprobs": (_i, [_vp, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "jl_model_decode_penalized": (_i, [_vp, _i] + [_vp] * 14),
    "jl_model_sample_multi_penalized": (_i, [_vp, _i] + [_vp] * 12),
    "jl_model_generate_penalized": (_i, [_vp, _i, _vp, _i, _i, _f, _i, _f, _vp, _i, _f, _f, _f, _i] + [_vp] * 7),
    "jl_apply_penalties": (_i, [_vp, _i, _i, _vp, _i64, _vp, _vp]),
    "jl_model_decode_constrained": (_i, [_vp, _i] + [_vp] * 9 + [_i] + [_vp] * 7),
    "jl_model_sample_multi_constrained": (_i, [_vp, _i] + [_vp] * 7 + [_i] + [_vp] * 7),
    "jl_select_constrained": (_i, [_vp, _i, _i, _vp, _i64] + [_vp] * 5 + [_i] + [_vp] * 3),
    "jl_moe_route": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    "jl_moe_group": (_i, [_vp, _i, _i, _i, _i] + [_vp] * 6),
    "jl_model_decode_resident": (_i, [_vp, _i, C.c_int32, _i, _i, _vp]),
    "jl_model_read_kv": (_i, [_vp, _i, _i, _i, _i, _vp]),
    "jl_model_kv_save": (_i, [_vp, _i, C.c_char_p, C.c_char_p]),
    "jl_model_kv_load": (_i, [_vp, _i, C.c_char_p, C.c_char_p]),
    "jl_model_kv_offload": (_i64, [_vp, _i]),
    "jl_model_kv_restore": (_i, [_vp, _i, _i64]),
    "jl_model_kv_discard": (_i, [_vp, _i64]),
    "jl_model_kv_pages": (_i, [_vp, _i]),
    "jl_model_kv_fork": (_i, [_vp, _i, _i, _i, _vp]),
    "jl_model_kv_page_stats": (_i, [_vp, C.POINTER(_i64), C.POINTER(_i64)]),
    "jl_model_kv_retain": (_i64, [_vp, _i, _i]),
    "jl_model_kv_attach": (_i, [_vp, _i64, _i, _i]),
    "jl_model_kv_release": (_i, [_vp, _i64]),
    "jl_model_kv_retained": (_i, [_vp, C.POINTER(_i64), C.POINTER(_i64)]),
    "jl_model_read_hidden": (_i, [_vp, _i, _vp]),
    "jl_model_debug_read": (_i, [_vp, _i, _vp, _i64]),
    "jl_model_decode_mode": (_i, [_vp, _i]),
    "jl_model_debug_trace": (_i, [_vp, _vp, _i64]),
    "jl_model_weight_bytes": (_i64, [_vp]),
    "jl_model_last_timing": (_i, [_vp, C.POINTER(_d), C.POINTER(_d)]),
    "jl_sched_create": (_i, [_vp, _i, _i, C.POINTER(_vp)]),
    "jl_sched_create_backend": (_i, [C.POINTER(SchedBackend), _vp, _i, _i, _i, _i, C.POINTER(_vp)]),
    "jl_sched_set_batch_backend": (_i, [_vp, C.POINTER(SchedBatchBackend)]),
    "jl_sched_set_topkp_backend": (_i, [_vp, C.POINTER(SchedTopkpBackend)]),
    "jl_sched_set_logprob_backend": (_i, [_vp, C.POINTER(SchedLogprobBackend)]),
    "jl_sched_set_penalty_backend": (_i, [_vp, C.POINTER(SchedPenaltyBackend)]),
    "jl_sched_set_fork_backend": (_i, [_vp, C.POINTER(SchedForkBackend)]),
    "jl_sched_set_constraint_backend": (_i, [_vp, C.POINTER(SchedConstraintBackend)]),
    "jl_sched_set_mask_provider": (_i, [_vp, _vp, _vp]),  # the provider: a SCHED_MASK_FN
    "jl_sched_set_prefix_cache": (_i, [_vp, C.POINTER(SchedPrefixBackend), _i]),
    "jl_sched_prefix_stats": (_i, [_vp, C.POINTER(SchedPrefixStats)]),
    "jl_sched_request_cached": (_i, [_vp, _i64]),
    "jl_sched_free": (_i, [_vp]),
    "jl_sched_last_error": (C.c_char_p, [_vp]),
    "jl_sched_submit": (_i64, [_vp, _vp, _i, _i, _vp, _i, _i, _i64, _f, C.c_uint64]),
    "jl_sched_submit_topkp": (_i64, [_vp, _vp, _i, _i, _vp, _i, _i, _i64, _f, _i, _f, C.c_uint64]),
    "jl_sched_submit_logprobs": (_i64, [_vp, _vp, _i, _i, _vp, _i, _i, _i64, _f, _i, _f, C.c_uint64, _i]),
    "jl_sched_submit_penalized": (_i64, [_vp, _vp, _i, _i, _vp, _i, _i, _i64, _f, _i, _f, C.c_uint64, _i, _f, _f, _f, _i, _vp, _vp]),
    "jl_sched_submit_n": (_i, [_vp, _i, _vp, _i, _i, _vp, _i, _i, _i64, _f, _i, _f, C.c_uint64, _i, _f, _f, _f, _i, _vp, _vp, _vp]),
    "jl_sched_result_logprobs": (_i, [_vp, _i64, _i, _i, _vp, _vp, _vp, C.POINTER(_i)]),
    "jl_sched_cancel": (_i, [_vp, _i64]),
    "jl_sched_step": (_i, [_vp, C.POINTER(SchedStats)]),
    "jl_sched_run": (_i, [_vp, _i, C.POINTER(SchedStats)]),
    "jl_sched_result": (_i, [_vp, _i64, _vp, _i, C.POINTER(_i), C.POINTER(_i), C.POINTER(_i)]),
    "jl_sched_request_info": (_i, [_vp, _i64, C.POINTER(SchedRequestInfo)]),
    "jl_sched_release": (_i, [_vp, _i64]),
    "jl_sched_counts": (_i, [_vp, C.POINTER(_i), C.POINTER(_i), C.POINTER(_i)]),
    "jl_comm_unique_id": (_i, [_vp, _vp]),
    "jl_comm_init": (_i, [_vp, _vp, _i, _i]),
    "jl_comm_allreduce_f32": (_i, [_vp, _vp, _i64]),
    "jl_comm_destroy": (_i, [_vp]),
}

_lib = None


def load():
    """dlopen the C-ABI library.  Raises (never falls back) when it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("%s is missing: run `python -m jlama_b200.build` (or __graft_entry__.build())" % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def ptr(a):
    """numpy array (or None) -> void*"""
    if a is None:
        return None
    return a.ctypes.data_as(C.c_void_p)


def check(ctx_handle, rc):
    if rc == JL_OK:
        return
    msg = load().jl_last_error(ctx_handle)
    msg = msg.decode() if msg else ""
    if rc == JL_ERR_UNSUPPORTED:
        raise UnsupportedOperation(rc, msg)
    raise JlamaNativeError(rc, msg)


class Context:
    """jl_ctx owner.  One per process per GPU."""

    def __init__(self, device=0):
        lib = load()
        h = C.c_void_p()
        info = (C.c_int64 * 4)()
        rc = lib.jl_init(device, C.byref(h), info)
        if rc != JL_OK:
            msg = lib.jl_last_error(None)
            raise JlamaNativeError(rc, (msg.decode() if msg else "") + " -- no CPU fallback exists")
        self.h = h
        self.lib = lib
        self.free_bytes, self.total_bytes, self.sm_count, self.cc = list(info)
        self.device = device

    def check(self, rc):
        check(self.h, rc)

    def sync(self):
        self.check(self.lib.jl_sync(self.h))

    def kernel_launches(self):
        return int(self.lib.jl_kernel_launches(self.h))

    def close(self):
        if self.h:
            self.lib.jl_shutdown(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

# jl_model_config.arch and the GPT-2 auxiliary slots (include/jlama_b200.h JL_ARCH_*, JL_AUX_*)
ARCH_LLAMA, ARCH_GPT2 = 0, 1
AUX_POS_EMBED, AUX_OUT_NORM_BIAS = 0, 1
AUX_ATTN_NORM_BIAS, AUX_Q_BIAS, AUX_K_BIAS, AUX_V_BIAS, AUX_O_BIAS, AUX_FFN_NORM_BIAS, AUX_FC_BIAS, AUX_PROJ_BIAS = range(8)
