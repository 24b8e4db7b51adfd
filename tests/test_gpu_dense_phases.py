"""The F32 / BF16 weight path (gemv_dense_kernel, jl_gemv.cu) and the GPT-2 forward pass (forward_rows_gpt2 + lm_head_rows,
jl_model.cu) pinned phase by phase against float64 references at their edges.  Per layer the GPT-2 block runs
  embed + pos_embed_add -> layernorm (ln_1) -> dense q | k | v -> + bias -> attention -> dense o -> + bias -> + residual
  -> layernorm (ln_2) -> dense c_fc -> + bias -> GELU -> dense c_proj -> + bias -> + residual
and sampling runs layernorm (ln_f) -> dense lm_head over the tied wte -> argmax_stage1 / 2.  Each case builds a one-layer GPT-2
model at the real dimensions (two more: the 2-layer gpt2-tiny and the full 12-layer gpt2-small, where only the last layer's
post-attention phases, the lm_head and layer 0's K / V page rows are checked), runs prompt passes, sample_multi calls and decode
steps, and checks every phase from the buffer that feeds it: read back with debug_read / read_kv, or exact on the host.

  x0 = wte[t] + wpe[p]                 one f32 add on the host; seen through ln_1 -> q / k / v and as o_proj's residual
  ln_1 -> q / k / v + bias             x0: LayerNorm restatement (below) -> dense bar -> one rounding for the bias add
  K / V page rows                      bit for bit the k / v rows read back (GPT-2 rotates by the identity); layer 0 of the
                                       deeper models: the dense bar from x0
  o_proj + bias + residual (debug 1)   att (debug 5) and x0: dense bar, then two f32 adds
  ln_2 (debug 12 after a prompt pass)  xb read back: LayerNorm restatement, bit for bit
  c_fc + bias -> GELU (debug 6)        ln_2 read back (restated from xb in a decode step, whose ln buffer ends at ln_f): the dense
                                       bar through GELU (|gelu'| <= 1.13), plus one ulp for the cast and the double formula's window
  c_proj + bias + residual (debug 0)   h and xb read back: dense bar, then two f32 adds
  ln_f (debug 12 after sampling)       the sampled hidden rows read back (x after decode, xb after sample_multi): bit for bit
  lm_head over wte (logits)            ln_f read back: dense bar
  arg-max token                        exact: the lowest index of the maximum, NaN never wins, an all-NaN row gives 0

Dense bar.  Each lane of gemv_dense_kernel runs a chain of ceil(K / 32) fmaf, then a 5-level xor butterfly, so against the
float64 sum the error is at most gamma(n) sum_k |a_k w_k| with n = ceil(K / 32) + 5, gamma(n) = n u / (1 - n u), u = 2^-24.  Every
f32 add after it (bias, residual) adds half an ulp of its result (2^-24 (|ref| + bar)); where the activation row is restated rather
than read back, every element whose candidates differ adds |da_k| |w_k|.

LayerNorm.  layernorm_kernel sums x and f32(x * x) in double, rounds both sums to float, then in f32: mean = sum / E, var =
sumSq / E - mean^2, inv = 1 / (float)sqrt((double)(var + eps)), out = ((x - mean) * inv) * w + b.  The restatement starts from the
exact sums (math.fsum) and must match bit for bit, NaN positions included; where an exact sum lies within length 2^-53 sum|terms|
of an f32 rounding midpoint the kernel's double sum may round either way, and every combination of the two candidates is
evaluated (ambiguous rows are counted).  Rows of mean 1e3 and spread 1e-2 cancel in var: the float formula gives a negative
variance there and NaN rows, as the reference does.

GELU.  activation_kernel evaluates 0.5 v (1 + tanh(sqrt(2 / pi) (v + 0.044715 pow(v, 3)))) in double and casts to f32.  The
restatement is the same formula in numpy float64; the result must be its f32 rounding bit for bit, except where another f32 value
lies within half an ulp plus A = 2^-47 (1 + |z|) |gelu(v)| + 2^-50 |v| of the double value (z the tanh argument; two libm's tanh
differ by an ulp near -1 and 1 + tanh cancels for negative v, so below v = -5 the double formula itself is only that good): such an
f32 value is accepted and counted.  The edges (+-0, +-1e-20, +-5, +-10, +-88, +-1e4, +-3e38, +-inf; NaN at -inf) are bit for bit.

Measured on an NVIDIA H100 80GB HBM3 (SXM, 700 W power limit, 1980 MHz max SM clock), worst err/bar per phase over every case:
  q / k / v + bias 0.025 / 0.020 / 0.021, layer-0 K / V page rows of the deeper models 0.111 / 0.080, o + bias + residual 0.080,
  fc + bias -> GELU 0.108, proj + bias + residual 0.116, lm_head 0.112; the operator GEMV F32xF32 0.263, F32xBF16 0.272,
  BF16xBF16 0.192; the Llama dense lm_head (RMSNorm prologue) 0.125 and dense o_proj + residual 0.262.  The bars are worst-case
  bounds, so these sit far below 1 while every defect of the CPU tests lands at least 13x above it.  LayerNorm (ln_2, ln_f, the operator
  rows), the K / V page rows of one-layer models, GELU and the arg-max tokens: bit for bit; ambiguous LayerNorm rows 11 (ln_1,
  restated), 2 (ln_2), 1 (ln_f), 0 in the operator rows (4 of them NaN from a negative variance); GELU operator elements accepted
  within the window 71 of 8113; 58 sampled rows resolved an exact tie or a tie of +inf.  The file takes about
  40 s on that card.

The CPU tests at the end restate jl_gemv_max_m / launch_dense_m to show that the cases reach every dense kernel variant, and show
with the same reference and bar functions that every bar rejects the defect it is there to catch by at least 4x.  Importing this
file does not load the CUDA library.
"""
import math
import zlib

import numpy as np
import pytest

from jlama_b200 import tensor as T  # numpy only
from jlama_b200.native import BF16, F32, JL_ERR_INVALID, JL_ERR_UNSUPPORTED, Q4

gpu = pytest.mark.gpu

F = np.float32
U = 2.0 ** -24          # unit roundoff of f32
SHARP = 4.0
GELU_SLOPE = 1.13       # max |gelu'(v)| of the tanh form
F32_MAX = float(np.finfo(F).max)
SMEM_LIMIT = 200 * 1024  # the dense kernels' dynamic shared-memory budget (jl_gemv_max_m, launch_dense)
ARGMAX_BLOCKS, ARGMAX_THREADS = 64, 256


# ---- references (numpy only) ---------------------------------------------------------------------------------------------
def gamma(n):
    return n * U / (1.0 - n * U)


def bf16_round(x):
    return T.bfloat16_to_float32(T.float32_to_bfloat16(np.asarray(x, dtype=F)))


def dense_ref(a, w, da=None, block=4096):
    """(ref, bar) float64 [M, N] of the dense GEMV of f32 rows a [M, K] against f32 weight rows w [N, K]; da [M, K]: the largest
    move of each activation element over its candidates (restated rows)"""
    a64 = np.asarray(a, dtype=np.float64)
    K, N = a64.shape[1], w.shape[0]
    ref, nat = np.empty((a64.shape[0], N)), np.empty((a64.shape[0], N))
    amb = np.zeros((a64.shape[0], N))
    aa = np.abs(a64)
    cols = None if da is None else np.nonzero(np.asarray(da).any(axis=0))[0]
    for r0 in range(0, N, block):
        w64 = np.asarray(w[r0:r0 + block], dtype=np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            ref[:, r0:r0 + block] = a64 @ w64.T
            nat[:, r0:r0 + block] = aa @ np.abs(w64).T
            if cols is not None and cols.size:
                amb[:, r0:r0 + block] = np.asarray(da, dtype=np.float64)[:, cols] @ np.abs(w64[:, cols]).T
    return ref, gamma(-(-K // 32) + 5) * nat + amb + 2.0 ** -140 * K


def add_f32(ref, bar, b):
    """one f32 add of b (broadcast) after a result with bar: half an ulp of the new result"""
    ref = ref + np.asarray(b, dtype=np.float64)
    return ref, bar + U * (np.abs(ref) + bar)


def err_ratio(out, ref, bar):
    """max |out - ref| / bar; NaN against NaN and equal infinities count as exact, a NaN elsewhere as infinite"""
    o = np.asarray(out, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        e = np.abs(o - ref)
    same = (np.isnan(o) & np.isnan(ref)) | (np.isinf(o) & (o == ref))
    e = np.where(same, 0.0, np.where(np.isnan(e), np.inf, e))
    r = np.where(bar > 0, e / np.where(bar > 0, bar, 1.0), np.where(e > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def same_bits(a, b):
    a, b = np.asarray(a, dtype=F), np.asarray(b, dtype=F)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def ulp_dist(a, b):
    """distance in f32 steps (NaN against NaN 0, NaN against a number huge)"""
    def key(x):
        i = np.asarray(x, dtype=F).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    a, b = np.asarray(a, dtype=F), np.asarray(b, dtype=F)
    d = np.abs(key(a) - key(b)).astype(np.float64)
    return np.where(np.isnan(a) & np.isnan(b), 0.0, np.where(np.isnan(a) | np.isnan(b), 1e30, d))


def _f32_pair(S, win):
    """the f32 values a double sum within win of the exact sum S can round to"""
    f = F(S)
    if float(f) == S or not np.isfinite(f):
        return f, f
    lo, hi = (f, np.nextafter(f, F(np.inf))) if float(f) < S else (np.nextafter(f, F(-np.inf)), f)
    return (lo, hi) if abs(S - 0.5 * (float(lo) + float(hi))) <= win else (f, f)


def ln_apply(xs, s, ss, E, eps, w, b):
    """layernorm_kernel's f32 arithmetic from the f32 sums s, ss [R]"""
    with np.errstate(all="ignore"):
        mean = (s / F(E)).astype(F)
        var = ((ss / F(E)).astype(F) - (mean * mean).astype(F)).astype(F)
        inv = (F(1) / np.sqrt((var + F(eps)).astype(F).astype(np.float64)).astype(F)).astype(F)
        y = ((xs - mean[:, None]).astype(F) * inv[:, None]).astype(F)
        return ((y * w[None, :]).astype(F) + b[None, :]).astype(F)


def ln_candidates(x, w, b, eps, E=None, offset=0, length=None, divide_by=None):
    """(cands [4, R, length] f32, ambiguous rows [R]) of LayerNorm over columns [offset, offset + length) of f32 rows x with f32
    weight / bias values w, b (indexed like the columns).  divide_by: the defect of dividing by another length than E."""
    x = np.asarray(x, dtype=F)
    length = x.shape[1] - offset if length is None else length
    E = x.shape[1] if E is None else E
    xs = x[:, offset:offset + length]
    sq = (xs * xs).astype(F)
    R = xs.shape[0]
    sums, sqs = np.empty((R, 2), dtype=F), np.empty((R, 2), dtype=F)
    for r in range(R):
        t, t2 = xs[r].astype(np.float64), sq[r].astype(np.float64)
        sums[r] = _f32_pair(math.fsum(t), length * 2.0 ** -53 * float(np.abs(t).sum()))
        sqs[r] = _f32_pair(math.fsum(t2), length * 2.0 ** -53 * float(t2.sum()))
    w = np.asarray(w, dtype=F).reshape(-1)[offset:offset + length]
    b = np.asarray(b, dtype=F).reshape(-1)[offset:offset + length]
    d = E if divide_by is None else divide_by
    c = np.stack([ln_apply(xs, sums[:, i], sqs[:, j], d, eps, w, b) for i in (0, 1) for j in (0, 1)])
    return c, (sums[:, 0] != sums[:, 1]) | (sqs[:, 0] != sqs[:, 1])


def ln_true(x, w, b, eps):
    x = np.asarray(x, dtype=np.float64)
    m = x.mean(axis=1, keepdims=True)
    v = ((x - m) ** 2).mean(axis=1, keepdims=True)
    return (x - m) / np.sqrt(v + eps) * np.asarray(w, np.float64) + np.asarray(b, np.float64)


def ln_bad_rows(out, cands):
    ok = np.zeros(out.shape[0], dtype=bool)
    for c in cands:
        ok |= same_bits(out, c).all(axis=1)
    return np.nonzero(~ok)[0]


def ln_miss_ulps(out, cands):
    """the defect's distance from the nearest candidate row, in f32 steps (max over each row, min over candidates, max over rows)"""
    return float(np.min(np.stack([ulp_dist(out, c).max(axis=1) for c in cands]), axis=0).max())


def ln_operand(x, w, b, eps):
    """(a, da): the first LayerNorm candidate of restated rows and the largest move over the others"""
    c, amb = ln_candidates(x, w, b, eps)
    a = c[0].astype(np.float64)
    with np.errstate(invalid="ignore"):
        da = np.nan_to_num(np.abs(c.astype(np.float64) - a[None]).max(axis=0), nan=0.0)
    return c[0], da, int(amb.sum())


def gelu_z(v):
    v = np.asarray(v, dtype=np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.sqrt(2.0 / 3.14159265358979323846) * (v + 0.044715 * np.power(v, 3.0))


def gelu64(v, erf=False):
    """activation_kernel's GELU in float64 (erf=True: the defect of the exact erf form)"""
    v = np.asarray(v, dtype=np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        if erf:
            from scipy.special import erf as _erf
            return 0.5 * v * (1.0 + _erf(v / np.sqrt(2.0)))
        return 0.5 * v * (1.0 + np.tanh(gelu_z(v)))


def gelu_allow(v):
    """the absolute allowance of a double GELU evaluation of v: 2^-47 (1 + |z|) of the result (pow, the argument) plus 0.5 |v| times
    2^-49 for 1 + tanh(z) (two libm's tanh differ by an ulp near +-1, where 1 + tanh cancels for negative v)"""
    v = np.asarray(v, dtype=np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        a = 2.0 ** -47 * (1.0 + np.abs(gelu_z(v))) * np.abs(gelu64(v)) + 2.0 ** -50 * np.abs(v)
    return np.where(np.isfinite(a), a, 0.0)


def gelu_check(out, x):
    """(rejected, ambiguous) element counts of GELU outputs of f32 inputs x against the double formula's f32 rounding"""
    ref = gelu64(np.asarray(x, dtype=F))
    exact = same_bits(out, ref.astype(F))
    o = np.asarray(out, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        half = 0.5 * np.abs(np.spacing(np.abs(ref).astype(F))).astype(np.float64)
        near = np.isfinite(ref) & (np.abs(o - ref) <= half + gelu_allow(x))
    return int((~(exact | near)).sum()), int((near & ~exact).sum())


def gelu_bar(ref_pre, bar_pre):
    """(ref, bar) after GELU of a pre-activation float64 reference with its bar, cast to f32"""
    g = gelu64(ref_pre)
    return g, GELU_SLOPE * bar_pre + 2.0 ** -23 * np.abs(g) + gelu_allow(ref_pre) + 2.0 ** -149


def argmax_ref(logits):
    """the lowest index of the maximum; NaN never wins; a row with no number gives 0"""
    lg = np.asarray(logits, dtype=F)
    out = np.zeros(lg.shape[0], dtype=np.int64)
    for r, row in enumerate(lg):
        ok = ~np.isnan(row)
        if ok.any():
            out[r] = int(np.nonzero(ok & (row == row[ok].max()))[0][0])
    return out


def argmax_cta(i):
    """the stage-1 CTA of argmax_stage1 that reads vocabulary index i"""
    return (i // ARGMAX_THREADS) % ARGMAX_BLOCKS


# ---- the dense launches, restated (jl_gemv_max_m / launch_dense_m) ----------------------------------------------------------
def gemv_max_m(K):
    for mm in (8, 4, 2, 1):
        if K * 4 * mm <= SMEM_LIMIT:
            return mm
    return 0


def dense_mm(M):
    return 1 if M <= 1 else 2 if M <= 2 else 4 if M <= 4 else 8


def dense_launches(M, K):
    """[(MM, dynamic shared-memory bytes, rows)] of run_gemm / gemm_locked on a dense weight"""
    ch = gemv_max_m(K)
    return [(dense_mm(min(ch, M - m0)), dense_mm(min(ch, M - m0)) * K * 4, min(ch, M - m0)) for m0 in range(0, M, ch)]


# ---- the case matrix ------------------------------------------------------------------------------------------------------
def _gcfg(E, heads, H, layers=1, vocab=50257, ctx=1024):
    return dict(E=E, heads=heads, kv_heads=heads, H=H, layers=layers, vocab=vocab, ctx=ctx, eps=1e-5)


CFGS = {
    "small": _gcfg(768, 12, 3072),
    "medium": _gcfg(1024, 16, 4096),
    "large": _gcfg(1280, 20, 5120),
    "xl": _gcfg(1600, 25, 6400),
    "tiny-2L": _gcfg(128, 4, 512, layers=2, vocab=256, ctx=64),
    "small-12L": _gcfg(768, 12, 3072, layers=12),
}
NAN_ID = 3
TIE_IDS = (17, 33000, 50000, 50256)  # one dominant row in stage-1 CTAs 0, 0, 3 and 4
INF_IDS = (20000, 50256)             # logits overflowing to +inf, in CTAs 14 and 4: the lower index sits in the later CTA
CRAFT_TOKENS = (100, 16000)          # crafted models feed tokens from here only

# steps: ("prompt", [(session, rows), ...]) one batch_forward / batch_forward_multi pass at each session's length;
# ("fill", session, rows) the same, unchecked; ("sample", sessions) one sample_multi; ("decode", sessions) one decode step
CASES = [
    dict(id="small-f32-ties", cfg="small", dtype="F32", craft="ties", sessions=9, max_batch=64,
         steps=[("prompt", [(0, 1)]), ("sample", [0]), ("prompt", [(1, 7)]), ("prompt", [(1, 9)]), ("prompt", [(2, 64)]),
                ("prompt", [(3, 8), (4, 1), (5, 2), (6, 3), (7, 4), (8, 5)]), ("sample", list(range(9))),
                ("decode", [0]), ("decode", [0, 1]), ("decode", [0, 1, 2]), ("decode", [0, 1, 2, 3, 4]), ("decode", list(range(8))),
                ("decode", list(range(9)))]),
    dict(id="medium-bf16", cfg="medium", dtype="BF16", sessions=4, max_batch=32,
         steps=[("prompt", [(0, 8)]), ("prompt", [(1, 9), (2, 7), (3, 1)]), ("sample", [0, 1, 2, 3]), ("decode", [0, 1, 2]),
                ("decode", [0, 1, 2, 3]), ("sample", [3])]),
    dict(id="large-f32-64", cfg="large", dtype="F32", sessions=65, max_batch=512,
         steps=[("fill", 0, 724), ("prompt", [(0, 300)]), ("fill", 1, 1023),
                ("prompt", [(s, 1 + s % 5) for s in range(2, 65)]), ("sample", list(range(1, 65))), ("decode", list(range(1, 65)))]),
    dict(id="xl-f32-inf", cfg="xl", dtype="F32", craft="inf", sessions=9, max_batch=16,
         steps=[("prompt", [(0, 8)]), ("prompt", [(1, 9)]), ("sample", [0, 1]), ("decode", [0, 1]),
                ("prompt", [(s, 1) for s in range(2, 9)]), ("decode", list(range(9))), ("sample", list(range(2, 9)))]),
    dict(id="tiny-2L", cfg="tiny-2L", dtype="F32", sessions=3, max_batch=16,
         steps=[("prompt", [(0, 9)]), ("sample", [0]), ("decode", [0]), ("prompt", [(1, 5), (2, 7)]), ("decode", [0, 1, 2])]),
    dict(id="small-12L", cfg="small-12L", dtype="F32", sessions=2, max_batch=16,
         steps=[("prompt", [(0, 16)]), ("sample", [0]), ("decode", [0]), ("prompt", [(1, 7)]), ("decode", [0, 1])]),
]
LM_ROWS = 16  # lm_head rows checked per call: all up to this many, else the first and last 8 (first and last chunk)

# operator API: (activation dtype, weight dtype) x K; M rows of a with a column offset against a row slice of b
OP_PAIRS = [("F32", "F32"), ("F32", "BF16"), ("BF16", "BF16")]
OP_K = (1, 31, 33, 1000, 6400, 6401)
OP_M = (1, 2, 3, 5, 8, 9, 32)
GELU_EDGES = (0.0, 1e-20, 5.0, 10.0, 88.0, 1e4, 3e38, np.inf)

# Llama models with Q4 layers and a dense tied embedding (lm_head through gemv_dense_kernel with the RMSNorm prologue), and a
# dense o_proj (the dense ADD_RESIDUAL epilogue): (embedding / o_proj dtype, norm weight dtype)
LLAMA_CASES = [("F32", "F32"), ("BF16", "BF16"), ("F32", "BF16")]
LLAMA_SAMPLE_ROWS = (1, 3, 9, 64)


def gpt2_cfg(name):
    c = dict(CFGS[name])
    c["name"] = "gpt2-" + name
    return c


def case_checkpoint(case, cfg):
    """synth checkpoint in the file layout; BF16 cases round every tensor to BF16 (the host keeps those values); crafted rows"""
    from jlama_b200 import synth
    ck = synth.make_gpt2_weights(cfg)
    if case["dtype"] == "BF16":
        ck = {k: (F32, bf16_round(v[1]), None) for k, v in ck.items()}
    craft = case.get("craft")
    if craft:
        rng = np.random.default_rng(zlib.crc32(case["id"].encode()))
        E = cfg["E"]
        b = (0.3 + 0.05 * rng.standard_normal(E)).astype(F)
        ck["ln_f.bias"] = (F32, b, None)
        wte = ck["wte.weight"][1].copy()
        wte[NAN_ID] = np.nan
        if craft == "ties":
            for i in TIE_IDS:
                wte[i] = (16 * b).astype(F)  # beats the input token's own row of the tied wte (about 0.5 E)
        else:  # sum_k ln_f_k sign(b_k) is about 0.3 E; 2 F32_MAX / 300 per element overflows the sum, never a lane's partial
            for i in INF_IDS:
                wte[i] = (np.sign(b) * F(2 * F32_MAX / 300)).astype(F)
        ck["wte.weight"] = (F32, wte, None)
    return ck


def host_weights(cfg, ck):
    g = lambda n: ck[n][1]  # noqa: E731
    hw = dict(wte=g("wte.weight"), wpe=g("wpe.weight"), lnfw=g("ln_f.weight").reshape(-1), lnfb=g("ln_f.bias").reshape(-1), layers=[])
    for i in range(cfg["layers"]):
        p = "h.%d." % i
        wq, wk, wv = [np.ascontiguousarray(t) for t in np.split(g(p + "attn.c_attn.weight").T, 3, axis=0)]
        bq, bk, bv = np.split(g(p + "attn.c_attn.bias").reshape(-1), 3)
        hw["layers"].append(dict(
            ln1w=g(p + "ln_1.weight").reshape(-1), ln1b=g(p + "ln_1.bias").reshape(-1), wq=wq, wk=wk, wv=wv, bq=bq, bk=bk, bv=bv,
            wo=np.ascontiguousarray(g(p + "attn.c_proj.weight").T), bo=g(p + "attn.c_proj.bias").reshape(-1),
            ln2w=g(p + "ln_2.weight").reshape(-1), ln2b=g(p + "ln_2.bias").reshape(-1),
            wfc=np.ascontiguousarray(g(p + "mlp.c_fc.weight").T), bfc=g(p + "mlp.c_fc.bias").reshape(-1),
            wproj=np.ascontiguousarray(g(p + "mlp.c_proj.weight").T), bproj=g(p + "mlp.c_proj.bias").reshape(-1)))
    return hw


def step_tokens(case, cfg, label, n):
    rng = np.random.default_rng(zlib.crc32(label.encode()))
    if case.get("craft"):
        return rng.integers(*CRAFT_TOKENS, n).astype(np.int32)
    t = rng.integers(0, cfg["vocab"], n).astype(np.int32)
    t[0] = cfg["vocab"] - 1  # the last wte row
    return t


def lm_rows(n):
    return np.arange(n) if n <= LM_ROWS else np.concatenate([np.arange(8), np.arange(n - 8, n)])


# ---- GPU harness ----------------------------------------------------------------------------------------------------------
WORST = {}
COUNTS = {}


def _record(phase, r):
    WORST[phase] = max(WORST.get(phase, 0.0), r)


def _count(what, n):
    COUNTS[what] = COUNTS.get(what, 0) + int(n)


def _gpt2_bf16_model(ctx, cfg, ck, **kw):
    """GPT2Model with every tensor registered as BF16 (weights, LayerNorm weights and biases, wpe): the BF16 dense kernel and the
    BF16 branches of layernorm_kernel, accumulate_kernel and pos_embed_add_kernel"""
    from jlama_b200 import native
    from jlama_b200.model import GPT2Model

    class GPT2ModelBF16(GPT2Model):
        def _load_gpt2(self, ctx, cfg, weights):
            lib, h, keep = self.lib, self.h, []

            def reg(a):
                a = np.asarray(a, dtype=F)
                raw = np.ascontiguousarray(T.float32_to_bfloat16(a.reshape(1, -1) if a.ndim == 1 else a))
                keep.append(raw)
                tid = lib.jl_register_tensor(ctx.h, BF16, raw.shape[0], raw.shape[1], native.ptr(raw), None)
                if tid < 0:
                    raise native.JlamaNativeError(-1, lib.jl_last_error(ctx.h).decode())
                self._ids.append(tid)
                return tid

            w = lambda n: weights[n][1]  # noqa: E731
            st = lambda L, slot, a: ctx.check(lib.jl_model_set_tensor(h, L, slot, reg(a)))  # noqa: E731
            sa = lambda L, slot, a: ctx.check(lib.jl_model_set_aux_tensor(h, L, slot, reg(a)))  # noqa: E731
            st(-1, native.T_EMBED, w("wte.weight")), sa(-1, native.AUX_POS_EMBED, w("wpe.weight"))
            st(-1, native.T_OUT_NORM, w("ln_f.weight")), sa(-1, native.AUX_OUT_NORM_BIAS, w("ln_f.bias"))
            for i in range(cfg["layers"]):
                p = "h.%d." % i
                st(i, native.L_ATTN_NORM, w(p + "ln_1.weight")), sa(i, native.AUX_ATTN_NORM_BIAS, w(p + "ln_1.bias"))
                for slot, a in zip((native.L_Q, native.L_K, native.L_V), np.split(w(p + "attn.c_attn.weight").T, 3, axis=0)):
                    st(i, slot, a)
                for slot, a in zip((native.AUX_Q_BIAS, native.AUX_K_BIAS, native.AUX_V_BIAS), np.split(w(p + "attn.c_attn.bias").reshape(-1), 3)):
                    sa(i, slot, a)
                st(i, native.L_O, w(p + "attn.c_proj.weight").T), sa(i, native.AUX_O_BIAS, w(p + "attn.c_proj.bias"))
                st(i, native.L_FFN_NORM, w(p + "ln_2.weight")), sa(i, native.AUX_FFN_NORM_BIAS, w(p + "ln_2.bias"))
                st(i, native.L_GATE, w(p + "mlp.c_fc.weight").T), sa(i, native.AUX_FC_BIAS, w(p + "mlp.c_fc.bias"))
                st(i, native.L_DOWN, w(p + "mlp.c_proj.weight").T), sa(i, native.AUX_PROJ_BIAS, w(p + "mlp.c_proj.bias"))
            ctx.check(lib.jl_model_finalize(h))

    return GPT2ModelBF16(ctx, cfg, ck, **kw)


def read_rows(gm, M, cfg):
    E, H = cfg["E"], cfg["H"]
    r = lambda i, n: gm.debug_read(i, M * n).reshape(M, n)  # noqa: E731
    return dict(x=r(0, E), xb=r(1, E), q=r(2, E), k=r(3, E), v=r(4, E), att=r(5, E), h=r(6, H), ln=r(12, E))


def check_rows(gm, cfg, hw, toks, pos, sess, b, kind, label):
    """every layer phase of the rows of one prompt pass or decode step; returns {phase: err/bar or count}"""
    E, L, eps = cfg["E"], cfg["layers"] - 1, cfg["eps"]
    l0, lw = hw["layers"][0], hw["layers"][L]
    res = {}

    def rec(ph, r):
        _record(ph, r)
        res[ph] = r
        assert r <= 1.0, "%s: %s err/bar %.3f" % (label, ph, r)

    x0 = (hw["wte"][toks] + hw["wpe"][pos]).astype(F)
    a, da, amb = ln_operand(x0, l0["ln1w"], l0["ln1b"], eps)
    _count("ln_1 ambiguous rows", amb)
    kp = np.stack([gm.read_kv(0, int(p), 0, session=int(s)) for p, s in zip(pos, sess)])
    vp = np.stack([gm.read_kv(0, int(p), 1, session=int(s)) for p, s in zip(pos, sess)])
    for nm, page in (("q", None), ("k", kp), ("v", vp)):
        ref, bar = add_f32(*dense_ref(a, l0["w" + nm], da), l0["b" + nm])
        if L == 0:
            rec(nm + " + bias", err_ratio(b[nm], ref, bar))
            if page is not None:
                bad = np.nonzero(~same_bits(page, b[nm]).all(axis=1))[0]
                assert bad.size == 0, "%s: %s page row of row %d is not the %s row" % (label, nm.upper(), bad[0], nm)
        elif page is not None:
            rec("%s page rows (layer 0)" % nm.upper(), err_ratio(page, ref, bar))
    if L == 0:
        ref, bar = add_f32(*add_f32(*dense_ref(b["att"], lw["wo"]), lw["bo"]), x0)
        rec("o + bias + residual", err_ratio(b["xb"], ref, bar))

    c2, amb2 = ln_candidates(b["xb"], lw["ln2w"], lw["ln2b"], eps)
    _count("ln_2 ambiguous rows", amb2.sum())
    if kind == "prompt":
        bad = ln_bad_rows(b["ln"], c2)
        assert bad.size == 0, "%s: ln_2 row %d is not the LayerNorm restatement (%.1f f32 steps off)" % (
            label, bad[0], ln_miss_ulps(b["ln"][bad[:1]], c2[:, bad[:1]]))
        res["ln_2"] = 0.0
        a, da = b["ln"], None
    else:
        a, da, _ = ln_operand(b["xb"], lw["ln2w"], lw["ln2b"], eps)
    rec("fc + bias -> GELU", err_ratio(b["h"], *gelu_bar(*add_f32(*dense_ref(a, lw["wfc"], da), lw["bfc"]))))
    ref, bar = add_f32(*add_f32(*dense_ref(b["h"], lw["wproj"]), lw["bproj"]), b["xb"])
    rec("proj + bias + residual", err_ratio(b["x"], ref, bar))
    return res


def check_head(case, cfg, hw, hidden, ln, logits, tokens, label):
    """ln_f from the hidden rows, the lm_head from ln_f, the arg-max from the logits"""
    c, amb = ln_candidates(hidden, hw["lnfw"], hw["lnfb"], cfg["eps"])
    _count("ln_f ambiguous rows", amb.sum())
    bad = ln_bad_rows(ln, c)
    assert bad.size == 0, "%s: ln_f row %d is not the LayerNorm restatement" % (label, bad[0])
    rows = lm_rows(len(hidden))
    ref, bar = dense_ref(ln[rows], hw["wte"])
    lg = logits[rows]
    craft = case.get("craft")
    if craft:
        assert np.isnan(lg[:, NAN_ID]).all(), "%s: the NaN row's logits are not NaN" % label
        ids = TIE_IDS if craft == "ties" else INF_IDS
        for i in ids[1:]:
            assert same_bits(lg[:, i], lg[:, ids[0]]).all(), "%s: identical wte rows %d and %d give different logits" % (label, ids[0], i)
        if craft == "inf":
            assert (ref[:, INF_IDS[0]] > F32_MAX).all(), "crafted rows must overflow"
            assert (lg[:, INF_IDS[0]] == np.inf).all(), "%s: overflowing logits are not +inf" % label
        keep = np.setdiff1d(np.arange(cfg["vocab"]), (NAN_ID,) + ids)
        ref, bar, lg = ref[:, keep], bar[:, keep], lg[:, keep]
    r = err_ratio(lg, ref, bar)
    _record("lm_head", r)
    assert r <= 1.0, "%s: lm_head err/bar %.3f" % (label, r)
    want = argmax_ref(logits)
    bad = np.nonzero(np.asarray(tokens) != want)[0]
    assert bad.size == 0, "%s: row %d arg-max %d, want %d" % (label, bad[0], tokens[bad[0]], want[bad[0]])
    if craft:
        expect = TIE_IDS[0] if craft == "ties" else INF_IDS[0]
        assert (want == expect).all(), "crafted rows must win"  # the ties / infinities were reached
        _count("tie rows", len(want))
    return r


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_gpt2_phases_against_float64(cuda_ctx, case):
    from jlama_b200.model import GPT2Model
    cfg = gpt2_cfg(case["cfg"])
    ck = case_checkpoint(case, cfg)
    hw = host_weights(cfg, ck)
    E = cfg["E"]
    kw = dict(max_batch=case["max_batch"], max_sessions=case["sessions"])
    gm = _gpt2_bf16_model(cuda_ctx, cfg, ck, **kw) if case["dtype"] == "BF16" else GPT2Model(cuda_ctx, cfg, ck, **kw)
    try:
        length, hidden = {}, {}
        for k, step in enumerate(case["steps"]):
            label = "%s step %d %s" % (case["id"], k, step[0])
            if step[0] == "fill":
                s, n = step[1], step[2]
                gm.batch_forward(step_tokens(case, cfg, label, n), length.get(s, 0), session=s)
                length[s] = length.get(s, 0) + n
                hidden.pop(s, None)
            elif step[0] == "prompt":
                segs = [(s, n, length.get(s, 0)) for s, n in step[1]]
                toks = [step_tokens(case, cfg, "%s %d" % (label, s), n) for s, n, _ in segs]
                if len(segs) == 1:
                    gm.batch_forward(toks[0], segs[0][2], session=segs[0][0])
                else:
                    gm.batch_forward_multi([(s, t, p) for (s, _, p), t in zip(segs, toks)])
                M = sum(n for _, n, _ in segs)
                b = read_rows(gm, M, cfg)
                pos = np.concatenate([p + np.arange(n) for _, n, p in segs])
                sess = np.concatenate([np.full(n, s) for s, n, _ in segs])
                label += " " + "+".join("%d@%d" % (n, p) for _, n, p in segs)
                res = check_rows(gm, cfg, hw, np.concatenate(toks), pos, sess, b, "prompt", label)
                r0 = 0
                for s, n, p in segs:
                    hidden[s] = b["x"][r0 + n - 1].copy()
                    length[s] = p + n
                    r0 += n
                print("%s: %s" % (label, "  ".join("%s %.3f" % kv for kv in res.items())))
            elif step[0] == "sample":
                sessions = step[1]
                tok, logits = gm.sample_multi(sessions, want_logits=True)
                n = len(sessions)
                xb, ln = gm.debug_read(1, n * E).reshape(n, E), gm.debug_read(12, n * E).reshape(n, E)
                for i, s in enumerate(sessions):  # the gathered rows are the sessions' last forwarded rows
                    if s in hidden:
                        assert same_bits(xb[i], hidden[s]).all(), "%s: row %d is not session %d's last hidden row" % (label, i, s)
                r = check_head(case, cfg, hw, xb, ln, logits, tok, "%s n=%d" % (label, n))
                print("%s n=%d: lm_head %.3f" % (label, n, r))
            else:
                sessions = np.asarray(step[1], dtype=np.int32)
                pos = np.asarray([length[s] for s in sessions], dtype=np.int32)
                toks = step_tokens(case, cfg, label, len(sessions))
                nxt, logits = gm.decode(toks, pos, sessions, want_logits=True)
                b = read_rows(gm, len(sessions), cfg)
                label += " n=%d pos %d..%d" % (len(sessions), pos.min(), pos.max())
                res = check_rows(gm, cfg, hw, toks, pos, sessions, b, "decode", label)
                res["lm_head"] = check_head(case, cfg, hw, b["x"], b["ln"], logits, nxt, label)
                for s in sessions:
                    length[int(s)] += 1
                    hidden.pop(int(s), None)
                print("%s: %s" % (label, "  ".join("%s %.3f" % kv for kv in res.items())))
    finally:
        gm.close()


@gpu
def test_debug_read_layernorm_slot(cuda_ctx):
    """slot 12 holds maxB x E floats of a GPT-2 model; Llama models refuse it"""
    from jlama_b200 import synth
    from jlama_b200.model import GPT2Model, LlamaModel
    cfg = gpt2_cfg("tiny-2L")
    gm = GPT2Model(cuda_ctx, cfg, synth.make_gpt2_weights(cfg), max_batch=16, max_sessions=2)
    try:
        gm.batch_forward(np.arange(5, dtype=np.int32), 0)
        out = np.empty(16 * cfg["E"] + 1, dtype=F)
        assert gm.lib.jl_model_debug_read(gm.h, 12, out.ctypes.data, 16 * cfg["E"]) == 0
        assert gm.lib.jl_model_debug_read(gm.h, 12, out.ctypes.data, 16 * cfg["E"] + 1) == JL_ERR_INVALID
        assert gm.lib.jl_model_debug_read(gm.h, 13, out.ctypes.data, 1) == JL_ERR_INVALID
    finally:
        gm.close()
    lcfg = synth.get_config("tiny")
    lm = LlamaModel(cuda_ctx, lcfg, synth.make_weights(lcfg, Q4, mode="direct"))
    try:
        out = np.empty(4, dtype=F)
        assert lm.lib.jl_model_debug_read(lm.h, 12, out.ctypes.data, 1) == JL_ERR_INVALID
    finally:
        lm.close()


def _op_operands(adt, wdt, K, M, seed):
    """(a tensor, a f32 values, b f32 values [N, K + 7]): a [M, K + 5] read from column 3, b rows read from column 2"""
    rng = np.random.default_rng(seed)
    av = rng.standard_normal((M, K + 5)).astype(F)
    bv = (0.5 * rng.standard_normal((96, K + 7))).astype(F)
    if adt == "BF16":
        av = bf16_round(av)
    if wdt == "BF16":
        bv = bf16_round(bv)
    a = T.BFloat16BufferTensor(T.float32_to_bfloat16(av)) if adt == "BF16" else T.FloatBufferTensor(av)
    b = T.BFloat16BufferTensor(T.float32_to_bfloat16(bv)) if wdt == "BF16" else T.FloatBufferTensor(bv)
    return a, av, b, bv


@gpu
@pytest.mark.parametrize("adt,wdt", OP_PAIRS, ids=["%sx%s" % p for p in OP_PAIRS])
def test_dense_gemv_operator_api(cuda_ops, adt, wdt):
    """batch_dot_product with dense weights (registered and host-side), column offsets and a row slice: rows 16..79 of b"""
    worst = 0.0
    for i, K in enumerate(OP_K):
        for M in OP_M:
            a, av, b, bv = _op_operands(adt, wdt, K, M, zlib.crc32(("%s %s %d %d" % (adt, wdt, K, M)).encode()))
            if (i + M) % 2:
                cuda_ops.register_model_tensor(b)
            c = T.FloatBufferTensor(np.zeros((M, 96), dtype=F))
            try:
                cuda_ops.batch_dot_product(c, a, b, 3, 2, K, 0, 16, 64)
            finally:
                cuda_ops.unregister_model_tensor(b)
            ref, bar = dense_ref(av[:, 3:3 + K], bv[16:80, 2:2 + K])
            r = err_ratio(c.data[:, 16:80], ref, bar)
            assert r <= 1.0, (adt, wdt, K, M, r)
            assert not c.data[:, :16].any() and not c.data[:, 80:].any(), (adt, wdt, K, M)
            worst = max(worst, r)
    _record("operator GEMV %sx%s" % (adt, wdt), worst)
    print("%sx%s: worst err/bar %.3f" % (adt, wdt, worst))


def _ln_rows(E, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((12, E)).astype(F)
    x[0] = (1e3 + 1e-2 * rng.standard_normal(E)).astype(F)  # cancellation: var may come out negative -> NaN
    x[1] = (-1e3 + 1e-2 * rng.standard_normal(E)).astype(F)
    x[2] = F(7.25)                                           # constant: var 0 -> 1 / sqrt(eps)
    x[3] = 0.0
    x[4] *= F(1e4)
    x[5] *= F(1e-4)
    x[6] += F(50)
    return x


@gpu
@pytest.mark.parametrize("wdt", ["F32", "BF16"])
def test_layernorm_operator_api_edges(cuda_ops, wdt):
    E = 1600
    rng = np.random.default_rng(21)
    x = _ln_rows(E, 22)
    w = (1 + 0.1 * rng.standard_normal((1, E))).astype(F)
    b = (0.05 * rng.standard_normal((1, E))).astype(F)
    if wdt == "BF16":
        w, b = bf16_round(w), bf16_round(b)
        wt, bt = T.BFloat16BufferTensor(T.float32_to_bfloat16(w)), T.BFloat16BufferTensor(T.float32_to_bfloat16(b))
    else:
        wt, bt = T.FloatBufferTensor(w), T.FloatBufferTensor(b)
    nan_rows, amb = 0, 0
    for E_, off, length in ((E, 0, E), (E, 64, 1000), (768, 0, 768)):
        out = cuda_ops.layernorm(T.FloatBufferTensor(x), wt, bt, 1e-5, embedding_length=E_, offset=off, length=length).data
        c, a = ln_candidates(x, w, b, 1e-5, E=E_, offset=off, length=length)
        got = out[:, off:off + length]
        bad = ln_bad_rows(got, c)
        assert bad.size == 0, (wdt, E_, off, length, bad, ln_miss_ulps(got[bad], c[:, bad]))
        assert not out[:, :off].any() and not out[:, off + length:].any()
        assert np.isfinite(got[2]).all() and np.isfinite(got[3]).all()  # var 0: 1 / sqrt(eps)
        nan_rows += int(np.isnan(got).all(axis=1).sum())
        amb += int(a.sum())
        if length == E_:  # for information: the distance from the true LayerNorm of the ordinary rows
            d = np.abs(got[4:].astype(np.float64) - ln_true(x[4:, off:off + length], w[0, off:off + length], b[0, off:off + length], 1e-5)).max()
            print("%s E=%d [%d, %d): float64 distance of the ordinary rows %.2e" % (wdt, E_, off, off + length, d))
    _count("LayerNorm op NaN rows", nan_rows)
    _count("LayerNorm op ambiguous rows", amb)
    print("%s: NaN rows (negative variance) %d, ambiguous rows %d" % (wdt, nan_rows, amb))


@gpu
def test_gelu_operator_api_edges(cuda_ops):
    edges = np.array([s * v for v in GELU_EDGES for s in (1.0, -1.0)], dtype=F)
    rng = np.random.default_rng(23)
    sweep = np.concatenate([np.linspace(-12, 12, 4097), 3 * rng.standard_normal(4000)]).astype(F)
    x = np.concatenate([edges, sweep]).reshape(1, -1)
    pad = np.full((1, 7), 1.5, dtype=F)
    t = T.FloatBufferTensor(np.concatenate([pad, x, pad], axis=1))
    cuda_ops.activation("gelu", t, 7, x.shape[1])
    out = t.data[0, 7:7 + x.shape[1]]
    assert (t.data[0, :7] == 1.5).all() and (t.data[0, -7:] == 1.5).all()
    n = len(edges)
    assert same_bits(out[:n], gelu64(edges).astype(F)).all(), list(zip(edges, out[:n], gelu64(edges).astype(F)))
    assert np.isnan(out[n - 1]) and out[n - 2] == np.inf  # -inf -> 0.5 (-inf) (1 + -1) = NaN; +inf -> +inf
    bad, amb = gelu_check(out, x[0])
    _count("GELU op ambiguous", amb)
    print("GELU: %d rejected, %d accepted within the window" % (bad, amb))
    assert bad == 0


@gpu
@pytest.mark.parametrize("emb,norm", LLAMA_CASES, ids=["emb-%s-norm-%s" % c for c in LLAMA_CASES])
def test_llama_dense_head_and_o_proj(cuda_ctx, emb, norm):
    """Q4 layers, a dense tied embedding (the lm_head through the PRO_RMSNORM_F32 prologue) and a dense o_proj (EPI_ADD_RESIDUAL)"""
    from jlama_b200 import synth
    from jlama_b200.model import LlamaModel
    from test_gpu_decode_gemm import norm_apply, rms_rsf
    edt = F32 if emb == "F32" else BF16
    cfg = synth.get_config("tiny", layers=1, tied=True)
    E = cfg["E"]
    w = synth.make_weights(cfg, Q4, mode="direct", embed_dtype=edt)
    w["model.layers.0.self_attn.o_proj.weight"] = synth.make_tensor(5, E, E, edt, "quantize")
    f32 = lambda t: T.bfloat16_to_float32(t[1]) if t[0] == BF16 else np.asarray(t[1], dtype=F)  # noqa: E731
    if norm == "BF16":
        for k in list(w):
            if k.endswith("norm.weight"):
                w[k] = (BF16, T.float32_to_bfloat16(w[k][1]), None)
    S = max(LLAMA_SAMPLE_ROWS)
    gm = LlamaModel(cuda_ctx, cfg, w, max_batch=256, max_sessions=S)
    try:
        segs = [(s, np.random.default_rng(s).integers(0, cfg["vocab"], 1 + s % 3).astype(np.int32), 0) for s in range(S)]
        gm.batch_forward_multi(segs)
        M = sum(len(t) for _, t, _ in segs)
        att, xb, x = (gm.debug_read(i, M * E).reshape(M, E) for i in (5, 1, 0))
        toks = np.concatenate([t for _, t, _ in segs])
        emb_w = f32(w["model.embed_tokens.weight"])
        ref, bar = add_f32(*dense_ref(att, f32(w["model.layers.0.self_attn.o_proj.weight"])), emb_w[toks])
        r = err_ratio(xb, ref, bar)
        _record("Llama dense o_proj + residual", r)
        assert r <= 1.0, r
        last = np.cumsum([len(t) for _, t, _ in segs]) - 1
        wn, eps = f32(w["model.norm.weight"]).reshape(-1), cfg["eps"]
        for n in LLAMA_SAMPLE_ROWS:
            tok, logits = gm.sample_multi(list(range(n)), want_logits=True)
            h = gm.debug_read(1, n * E).reshape(n, E)
            assert same_bits(h, x[last[:n]]).all()
            rsf = rms_rsf(h, eps)
            a = norm_apply(h, wn, rsf).astype(F)
            da = np.zeros(a.shape)
            for r2 in (np.nextafter(rsf, F(0)), np.nextafter(rsf, F(np.inf))):
                da = np.maximum(da, np.abs(norm_apply(h, wn, r2.astype(F)).astype(F).astype(np.float64) - a))
            ref, bar = dense_ref(a, emb_w, da)
            r = err_ratio(logits, ref, bar)
            _record("Llama dense lm_head (RMSNorm prologue)", r)
            assert r <= 1.0, (n, r)
            assert (tok == argmax_ref(logits)).all(), n
            print("emb %s norm %s n=%d: lm_head err/bar %.3f" % (emb, norm, n, r))
    finally:
        gm.close()


@gpu
def test_finalize_refuses_dense_gate_up_and_dense_experts(cuda_ctx):
    """SiLU * up runs fused into the gate/up GEMV for quantised weights only: F32 / BF16 gate/up or experts are refused where the
    checkpoint is bound, naming the layer and slot"""
    from jlama_b200 import native, synth
    from jlama_b200.model import LlamaModel
    cfg = synth.get_config("tiny")
    for wdt in (F32, BF16):
        with pytest.raises(native.JlamaNativeError) as ei:
            LlamaModel(cuda_ctx, cfg, synth.make_weights(cfg, wdt))
        assert ei.value.code == JL_ERR_UNSUPPORTED and "layer 0 slot 6 (gate)" in str(ei.value), str(ei.value)
    w = synth.make_weights(cfg, Q4, mode="direct")
    for nm in ("gate_proj", "up_proj"):
        w["model.layers.1.mlp.%s.weight" % nm] = synth.make_tensor(3, cfg["H"], cfg["E"], F32, "quantize")
    with pytest.raises(native.JlamaNativeError) as ei:
        LlamaModel(cuda_ctx, cfg, w)
    assert ei.value.code == JL_ERR_UNSUPPORTED and "layer 1 slot 6 (gate)" in str(ei.value), str(ei.value)
    mcfg = synth.get_config("tiny-mixtral")
    with pytest.raises(native.JlamaNativeError) as ei:
        LlamaModel(cuda_ctx, mcfg, synth.make_weights(mcfg, F32))
    assert ei.value.code == JL_ERR_UNSUPPORTED and "layer 0 expert 0 weight 0 (w1)" in str(ei.value), str(ei.value)
    w = synth.make_weights(mcfg, Q4, mode="direct")
    w["model.layers.1.block_sparse_moe.experts.5.w3.weight"] = synth.make_tensor(4, mcfg["H"], mcfg["E"], BF16, "quantize")
    with pytest.raises(native.JlamaNativeError) as ei:
        LlamaModel(cuda_ctx, mcfg, w)
    assert ei.value.code == JL_ERR_UNSUPPORTED and "layer 1 expert 5 weight 2 (w3)" in str(ei.value), str(ei.value)


@gpu
def test_zz_report():
    """the worst err/bar per phase and the ambiguity counts over the cases that ran"""
    for k in sorted(WORST):
        print("dense phase %-34s: worst err/bar %.3f" % (k, WORST[k]))
    for k in sorted(COUNTS):
        print("count %-38s: %d" % (k, COUNTS[k]))


# ---- the case matrix, checked on the CPU ----------------------------------------------------------------------------------
def _case_gemvs(case):
    """((M, K) of every dense GEMV the case's steps launch, the positions its prompt passes and decode steps reach); checks that
    every step is one valid call"""
    cfg = CFGS[case["cfg"]]
    E, H = cfg["E"], cfg["H"]
    out, length, reached = [], {}, {"prompt": set(), "decode": set()}
    for step in case["steps"]:
        if step[0] in ("fill", "prompt"):
            segs = [(step[1], step[2])] if step[0] == "fill" else step[1]
            M = sum(n for _, n in segs)  # a fill may be longer: batch_forward cuts it into max_batch-row passes, unchecked
            assert (M <= case["max_batch"] or step[0] == "fill") and len({s for s, _ in segs}) == len(segs), case["id"]
            for s, n in segs:
                assert s < case["sessions"]
                if step[0] == "prompt":
                    reached["prompt"] |= set(range(length.get(s, 0), length.get(s, 0) + n))
                length[s] = length.get(s, 0) + n
                assert length[s] <= cfg["ctx"]
            if step[0] == "fill":
                continue
        elif step[0] == "sample":
            M = len(step[1])
            assert all(length.get(s, 0) > 0 for s in step[1]) and len(set(step[1])) == M
            out.append((M, E))
            continue
        else:
            M = len(step[1])
            assert M <= 64 and len(set(step[1])) == M
            for s in step[1]:  # a decode step continues a forwarded session: every position below it holds K / V rows
                assert 0 < length.get(s, 0) < cfg["ctx"], (case["id"], s)
                reached["decode"].add(length[s])
                length[s] += 1
            out.append((M, E))
        out += [(M, E), (M, E), (M, E), (M, H)]  # q | k | v, o, c_fc, c_proj
    return out, reached


def test_case_matrix_reaches_every_dense_variant():
    seen = set()
    for case in CASES:
        cfg = CFGS[case["cfg"]]
        assert cfg["E"] % cfg["heads"] == 0
        gemvs, reached = _case_gemvs(case)
        seen.add(("wdt", case["dtype"]))
        seen.add(("prologue", "PRO_F32"))
        seen.add(("epilogue", "STORE"))
        for M, K in gemvs:
            ls = dense_launches(M, K)
            seen |= {("MM", mm) for mm, _, _ in ls}
            seen |= {("dead rows", mm) for mm, _, r in ls if r < mm}
            if len(ls) > 1:
                seen.add("chunked M > 8" if gemv_max_m(K) == 8 else "chunked below 8")
            if any(s == SMEM_LIMIT for _, s, _ in ls):
                seen.add("204800 bytes")
        if 1023 in reached["prompt"] and cfg["ctx"] == 1024:
            seen.add("position 1023")
        if cfg["ctx"] - 1 in reached["decode"] and cfg["ctx"] == 1024:
            seen.add("decode at the last position")
        craft = case.get("craft")
        if craft:
            ids = TIE_IDS if craft == "ties" else INF_IDS
            assert all(i >= CRAFT_TOKENS[1] or i < CRAFT_TOKENS[0] for i in ids + (NAN_ID,))  # never fed as input
            assert max(ids) == cfg["vocab"] - 1 and cfg["vocab"] % 2 == 1
            if len({argmax_cta(i) for i in ids}) > 1:
                seen.add(("ties across stage-1 CTAs", craft))
            if craft == "inf" and argmax_cta(ids[0]) > argmax_cta(ids[1]):
                seen.add("the lowest tied index in a later CTA")
        if cfg["H"] == 6400:
            seen.add("K = 6400")
    # the operator cases
    for adt, wdt in OP_PAIRS:
        seen.add(("wdt", wdt))
        seen.add(("prologue", "PRO_BF16_GLOBAL" if adt == "BF16" else "PRO_F32"))
        for K in OP_K:
            for M in OP_M:
                ls = dense_launches(M, K)
                if K == 6401 and gemv_max_m(K) == 4 and len(ls) > 1:
                    seen.add("4-row chunks at K = 6401")
    for emb, _ in LLAMA_CASES:
        seen |= {("wdt", emb), ("prologue", "PRO_RMSNORM_F32"), ("epilogue", "ADD_RESIDUAL")}
        seen |= {("MM", dense_mm(min(8, n))) for n in LLAMA_SAMPLE_ROWS}
    want = [("MM", 1), ("MM", 2), ("MM", 4), ("MM", 8), ("dead rows", 4), ("dead rows", 8), "chunked M > 8", "204800 bytes",
            "4-row chunks at K = 6401", ("wdt", "F32"), ("wdt", "BF16"), ("prologue", "PRO_F32"), ("prologue", "PRO_RMSNORM_F32"),
            ("prologue", "PRO_BF16_GLOBAL"), ("epilogue", "STORE"), ("epilogue", "ADD_RESIDUAL"), ("ties across stage-1 CTAs", "ties"),
            ("ties across stage-1 CTAs", "inf"), "the lowest tied index in a later CTA", "position 1023", "decode at the last position",
            "K = 6400"]
    missing = [x for x in want if x not in seen]
    assert not missing, missing
    # K = 6400 fills the budget with 8 rows exactly; one more column drops to 4-row chunks
    assert gemv_max_m(6400) == 8 and 8 * 6400 * 4 == SMEM_LIMIT and gemv_max_m(6401) == 4
    # prompt passes of 1, 7, 8, 9, 64 and 300 rows, decode steps of 1, 2, 3, 5, 8, 9 and 64 sessions, sample_multi of 1..64 rows
    prompts = {sum(n for _, n in st[1]) for c in CASES for st in c["steps"] if st[0] == "prompt"}
    multi = any(len(st[1]) > 1 for c in CASES for st in c["steps"] if st[0] == "prompt")
    decodes = {len(st[1]) for c in CASES for st in c["steps"] if st[0] == "decode"}
    samples = {len(st[1]) for c in CASES for st in c["steps"] if st[0] == "sample"}
    assert {1, 7, 8, 9, 64, 300} <= prompts and multi, prompts
    assert {1, 2, 3, 5, 8, 9, 64} <= decodes, decodes
    assert 1 in samples and 64 in samples and any(8 < n < 64 for n in samples), samples
    assert {c["cfg"] for c in CASES} == set(CFGS) and {CFGS[c]["heads"] for c in ("xl",)} == {25}
    assert {c["dtype"] for c in CASES} == {"F32", "BF16"}


# ---- sharpness of the bars (CPU) --------------------------------------------------------------------------------------------
def _ratio(r, what):
    print("%s: err/bar %.1f" % (what, r))
    assert r >= SHARP, (what, r)


def _gemv_case(M=16, K=768, N=256, seed=1):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((M, K)).astype(F), (0.02 * rng.standard_normal((N, K))).astype(F)


def _f32_gemv(a, w):
    """an f32 evaluation in the kernel's shape: 32 lane chains of fmaf (rounded per step) and a butterfly"""
    M, K = a.shape
    acc = np.zeros((32, M, w.shape[0]), dtype=F)
    for k0 in range(0, K, 32):
        for lane in range(min(32, K - k0)):
            k = k0 + lane
            acc[lane] = (acc[lane].astype(np.float64) + np.outer(a[:, k], w[:, k]).astype(np.float64)).astype(F)
    while acc.shape[0] > 1:
        h = acc.shape[0] // 2
        acc = (acc[:h] + acc[h:]).astype(F)
    return acc[0]


def test_dense_bar_accepts_the_kernels_order():
    for K in (31, 33, 768):
        a, w = _gemv_case(M=4, K=K, N=64, seed=K)
        ref, bar = dense_ref(a, w)
        assert err_ratio(_f32_gemv(a, w), ref, bar) <= 0.5, K


def test_bar_rejects_a_dropped_last_k_element():
    for K in (33, 768, 6400):
        a, w = _gemv_case(K=K, seed=2)
        ref, bar = dense_ref(a, w)
        _ratio(err_ratio(dense_ref(a[:, :-1], w[:, :-1])[0], ref, bar), "last K element dropped, K=%d" % K)


def test_bar_rejects_the_k_bias_on_v():
    cfg = gpt2_cfg("small")
    rng = np.random.default_rng(3)
    a = rng.standard_normal((8, cfg["E"])).astype(F)
    wv = (0.02 * rng.standard_normal((cfg["E"], cfg["E"]))).astype(F)
    bk, bv = (0.01 * rng.standard_normal((2, cfg["E"]))).astype(F)
    ref, bar = add_f32(*dense_ref(a, wv), bv)
    _ratio(err_ratio(add_f32(*dense_ref(a, wv), bk)[0], ref, bar), "k bias added to v")


def test_bar_rejects_the_next_wpe_row():
    """o_proj + bias + residual of x0 = wte[t] + wpe[p] against wpe[p + 1]"""
    rng = np.random.default_rng(4)
    E = 768
    wte, wpe = (0.5 * rng.standard_normal((64, E))).astype(F), (0.1 * rng.standard_normal((1024, E))).astype(F)
    att, wo = rng.standard_normal((8, E)).astype(F), (0.004 * rng.standard_normal((E, E))).astype(F)
    toks, pos = np.arange(8), np.array([0, 1, 2, 500, 1000, 1021, 1022, 5])
    x0 = (wte[toks] + wpe[pos]).astype(F)
    ref, bar = add_f32(*dense_ref(att, wo), x0)
    _ratio(err_ratio(add_f32(*dense_ref(att, wo), (wte[toks] + wpe[pos + 1]).astype(F))[0], ref, bar), "wpe[p + 1]")


def test_bar_rejects_layernorm_defects():
    """bit for bit: the defect's output lies at least 4 f32 steps from every candidate"""
    E = 768
    x = _ln_rows(E, 5)[4:]
    rng = np.random.default_rng(6)
    w, b = (1 + 0.1 * rng.standard_normal(E)).astype(F), (0.05 * rng.standard_normal(E)).astype(F)
    c, _ = ln_candidates(x, w, b, 1e-5)
    assert ln_bad_rows(c[0], c).size == 0
    _ratio(ln_miss_ulps(ln_candidates(x, w, b, 0.0)[0][0], c), "eps dropped from LayerNorm")
    c2, _ = ln_candidates(x, w, b, 1e-5, E=E, offset=0, length=700)
    _ratio(ln_miss_ulps(ln_candidates(x, w, b, 1e-5, E=E, offset=0, length=700, divide_by=700)[0][0], c2),
           "LayerNorm dividing by length instead of E")


def test_bar_rejects_erf_gelu():
    rng = np.random.default_rng(7)
    a, wfc = rng.standard_normal((16, 768)).astype(F), (0.02 * rng.standard_normal((512, 768))).astype(F)
    ref, bar = add_f32(*dense_ref(a, wfc), (0.01 * rng.standard_normal(512)).astype(F))
    g, gb = gelu_bar(ref, bar)
    _ratio(err_ratio(gelu64(ref, erf=True), g, gb), "erf GELU instead of tanh GELU (through the fc bar)")
    x = np.linspace(-4, 4, 2001).astype(F)
    bad, _ = gelu_check(gelu64(x, erf=True).astype(F), x)
    print("erf GELU: %d of %d elements rejected bit for bit" % (bad, x.size))
    assert 4 * bad >= x.size
    assert gelu_check(gelu64(x).astype(F), x)[0] == 0


def test_bar_rejects_a_chunk_reading_the_previous_chunks_rows():
    a, w = _gemv_case(M=16, K=768, seed=8)
    ref, bar = dense_ref(a, w)
    out = ref.copy()
    out[8:] = ref[:8]
    _ratio(err_ratio(out, ref, bar), "dense chunk 2 from chunk 1's activation rows")
    out = ref.copy()
    out[8] = ref[7]  # only the first row of the chunk
    _ratio(err_ratio(out, ref, bar), "dense chunk 2's first row from the row before it")


def test_bar_rejects_a_skipped_last_lm_head_row():
    rng = np.random.default_rng(9)
    a, wte = rng.standard_normal((4, 256)).astype(F), (0.5 * rng.standard_normal((1000, 256))).astype(F)
    ref, bar = dense_ref(a, wte)
    for what, fill in (("left zero", 0.0), ("stale from another row", ref[::-1, -1])):
        out = ref.copy()
        out[:, -1] = fill
        _ratio(err_ratio(out, ref, bar), "lm_head's last row skipped, output %s" % what)


def _argmax_higher(logits):
    lg = np.asarray(logits, dtype=F)
    out = np.zeros(lg.shape[0], dtype=np.int64)
    for r, row in enumerate(lg):
        ok = ~np.isnan(row)
        if ok.any():
            out[r] = int(np.nonzero(ok & (row == row[ok].max()))[0][-1])
    return out


def test_argmax_rule_and_the_higher_index_defect():
    lg = np.zeros((5, 50257), dtype=F)
    for i in TIE_IDS:
        lg[0, i] = 9.0
    lg[1, list(INF_IDS)] = np.inf
    lg[1, NAN_ID] = np.nan
    lg[2] = np.nan
    lg[3] = -np.inf
    lg[4, :] = np.nan
    lg[4, 7] = -np.inf
    assert argmax_ref(lg).tolist() == [TIE_IDS[0], INF_IDS[0], 0, 0, 7]
    bad = _argmax_higher(lg)
    assert (bad[:2] != argmax_ref(lg)[:2]).all()  # every tie row rejected by the exact check
    print("tie to the higher index: %d of 2 tie rows rejected" % int((bad[:2] != argmax_ref(lg)[:2]).sum()))
