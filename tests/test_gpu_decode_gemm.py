"""The decode GEMV and GEMM kernels pinned against exact integer references at their edges.  Five kernels serve the weight
matrices of a decode step:

  pd            the GEMV phases, lm_head and arg-max of the persistent kernel (pdecode_kernel, jl_pdecode.cu / jl_gemv_body.cuh):
                one session per step, the default
  gemv_decode   gemv_decode_kernel (jl_gemv.cu), LONG (split rows) or short, RMSNorm + Q8 or Q8 prologue: Q4 weights at one row in
                the per-op graph
  generic       gemv_kernel (jl_gemv.cu), MM 1 / 2 / 4 / 8 rows, Q8 or F32 activations: Q8_0 weights at one row, the F32 lm_head at
                1..8 rows, and every shape the fast kernels refuse
  gemm8         gemm8_kernel (jl_gemm8.cu), 8 or 16 warps, k-split 1..16: 2..8-row steps and 8-row prefill chunks
  gemm64        gemm64_quant_kernel + gemm64_kernel (jl_gemm64.cu), NT 2 / 4 / 6 / 8, k-split, and FA (the lm_head's F32 activations
                as three BF16 planes): 9..64-row steps

Every case runs a decode step of n sessions on one-layer models with synth "direct" weights (every nibble pattern, scales of
mixed sign) and reads back q / k / v, att, xb, h, x (debug_read) and the logits.  Each phase is checked from the buffer that
feeds it: QKV from the embedding row (dequantised on the host), o_proj from att (residual: the embedding row), gate/up from xb,
down from h (residual: xb), the final norm + lm_head from x.  A 3-layer model checks the last layer's gate/up, down and lm_head.

References (numpy).  The activations are restated in float32 with one rounding per operation, as every kernel writes them:
rsf = f32(1 / sqrt(sum f64(x * x) / E + eps)), y = f32(f32(0 + w) * f32(rsf * x)), then per 32-block mx = max|y|,
d = f32(mx / 127), id = f32(127 / mx) (0 at mx = 0), q = trunc(f32(f32(y * id) + 0.5)).  The kernels form the double sum in
different orders (and divide by E or multiply by 1/E), so q is also recomputed with rsf moved by +-1 ulp; every element whose q
moves is ambiguous and adds one int8 step |d * s_w * w_q| to its outputs' bar (the count is printed; it is 0 almost everywhere).
  Q8 x Q4 / Q8 x Q8_0:  ref = sum_b d_b * s_b * isum_b with isum the exact integer block sum (Q4: (nibble - 8) * q), over
                        row blocks of exact float32 block products; nat = sum_b |d_b * s_b * isum_b|;
                        |out - ref| <= TAU * nat + ambiguity (+ 2^-23 |out| after a residual add).
  SiLU * up:            ref = silu(g_ref) * u_ref; bar |silu'(g)| |u| e_g + |silu(g)| e_u + 2^-22 |h| from the gate / up bars
                        (+ 2^-126 (1 + |u|) where silu(g) underflows, at g below about -87).
  F32 lm_head:          ref = sum_b s_b * sum_k y_k * q_k with y restated in f32; |out - ref| <= TAU_F * sum |y_k * q_k * s_b|.

Measured on an NVIDIA H100 80GB HBM3 (SXM, 700 W power limit, 1980 MHz max SM clock) over every case below, as
max |out - ref| / nat with the ambiguity and the residual rounding taken off (the uncrafted cases stay at or below 2.5e-7):
  pd 5.0e-7, gemv_decode 1.5e-7, generic 1.7e-7 (F32 lm_head 5.6e-7), gemm8 6.0e-7, gemm64 1.2e-6 (FA 5.8e-7).
TAU = 2^-17 = 7.6e-6 leaves 6.2x headroom over the worst of the Q8 paths (gemm64's gate/up on the crafted 8B operands) and
TAU_F = 2^-18 = 3.8e-6 6.5x over the F32 lm_head paths; both stay no looser than the tensor-core GEMM's 2^-16.
The worst err/bar per kernel is pd 0.42, gemv_decode 0.39, generic 0.37 (F32 lm_head 0.15), gemm8 0.47, gemm64 0.49 (FA 0.15).
Every value above 0.25 is an o_proj or down_proj output whose residual is far larger than the product (the crafted 1e4 embedding
rows, the small models' down projections): there the add's final rounding, at most half an ulp against the one-ulp allowance, is
most of the error.
Ambiguous elements: at most 2 per phase.  The whole file takes about 75 s on that card.

Arg-max.  Every decode step's next token must be the lowest index of the maximum of its logits.  A crafted Q4 lm_head (all rows
zero but a row r at 1, 15 and 40 and its exact negation -r, nibbles 1..15 mirrored, at vocab - 1, 16 and 41) ties the maximum on
purpose, across the strip boundary 15 / 16 and inside one warp's rows: the copies must be bit-identical, -r must be exactly -r, and
the other rows exactly 0.  An all-zero lm_head must give token 0 on every route (pd's packed cross-CTA compare, argmax_stage1/2).
Determinism.  The same step run twice (n = 1 pd, n = 8 and 64 with k-splits) must give bit-identical buffers.
Untouched rows.  After a 64-row step, a 9-row step (gemm64 pads it to 16 rows) must leave rows 9..63 of every buffer unchanged.

Host selection.  host_rule() restates which kernel runs each phase and with what parameters (run_gemm, jl_launch_gemv, launch_q,
jl_gemm8_supported / g8_warps / g8_ksplit, jl_gemm64_supported / g64_nt / g64_ksplit / g64_fa, jl_pdecode_supported and
pd_smem_bytes); test_case_matrix_reaches_every_kernel_variant checks, on the CPU, that the cases reach every variant.  On the GPU
each step recomputes the labels for the card's SM count and asserts decode_mode().  JL_G8_WARPS / JL_G8_KSPLIT are read once per
process and are never set here.

The CPU tests at the end show, with the same reference functions, that the bars reject each defect they are there to catch by at
least 4x.  FA's lo plane (the last 8 bits of a 24-bit significand, 2^-17 of |y|) cannot be seen: its contribution to a logit is
far below TAU_F * sum |y q s|.  Importing this file does not load the CUDA library.
"""
import functools
import zlib

import numpy as np
import pytest

from jlama_b200 import tensor as T  # numpy only
from jlama_b200.native import I8, MODEL_NO_GRAPH, MODEL_NO_PERSISTENT, Q4

gpu = pytest.mark.gpu

TAU = 2.0 ** -17
TAU_F = 2.0 ** -18
SHARP = 4.0
ULP_RES = 2.0 ** -23   # the rounding of the residual add (one ulp)
ULP_SILU = 2.0 ** -22  # silu rounded to f32, then the product
TINY = 2.0 ** -126     # below the smallest normal f32 a flushed or subnormal silu(g) * u may differ by this much (times 1 + |u|)
H100_SMS = 132  # the labels below are computed for an H100 SXM; the GPU run recomputes them for the card it has
MAX_CONTEXT = 64

# ---- references (numpy only) ---------------------------------------------------------------------------------------------
F = np.float32


def unpack_weights(wdt, data, scales):
    """(values int8 [N, K], scales f32 [N, K/32]) of a Q4 (nibble - 8; byte i of a block: element i low, i + 16 high) or Q8_0
    tensor"""
    if wdt == Q4:
        N, half = data.shape
        b = data.reshape(N, half // 16, 16)
        v = np.concatenate([b & 0x0F, b >> 4], axis=2).reshape(N, half * 2).astype(np.int8) - np.int8(8)
        return v, np.asarray(scales, dtype=F)
    return np.asarray(data, dtype=np.int8), np.asarray(scales, dtype=F)


def dequant_rows(wq, s, rows):
    """f32(value * scale) of the given rows: the embedding kernels' dequantisation"""
    v = wq[rows].astype(F)
    return (v * np.repeat(s[rows], 32, axis=1)).astype(F)


def rms_rsf(x, eps):
    """f32(1 / sqrt(sum f64(f32(x * x)) / E + eps)) per row"""
    ss = (x * x).astype(np.float64).sum(axis=1)
    return (1.0 / np.sqrt(ss / x.shape[1] + np.float64(F(eps)))).astype(F)


def norm_apply(x, w, rsf):
    return (F(0) + np.asarray(w, dtype=F))[None, :] * (rsf[:, None] * x)


def quant_q8(y, round_nearest=False):
    """(q int32 [M, K], d f32 [M, K/32]): d = f32(mx / 127), q = trunc(f32(f32(y * f32(127 / mx)) + 0.5)); round_nearest: the
    defect of rounding y * id to nearest instead"""
    M, K = y.shape
    yb = y.reshape(M, K // 32, 32)
    mx = np.abs(yb).max(axis=2)
    d = (mx / F(127)).astype(F)
    idv = np.where(mx != 0, F(127) / np.where(mx != 0, mx, F(1)), F(0)).astype(F)
    p = (yb * idv[:, :, None]).astype(F)
    q = np.rint(p) if round_nearest else np.trunc((p + F(0.5)).astype(F))
    return q.reshape(M, K).astype(np.int32), d


def restate_act(x, norm_w=None, eps=1e-5, round_nearest=False):
    """Q8 activations of f32 rows x (RMSNorm'd first when norm_w is given): (q, d, dq) with dq [M, K] the largest move of q under
    rsf +- 1 ulp (0 where unambiguous)"""
    x = np.asarray(x, dtype=F)
    if norm_w is None:
        q, d = quant_q8(x, round_nearest)
        return q, d, np.zeros(q.shape, dtype=np.int32)
    rsf = rms_rsf(x, eps)
    q, d = quant_q8(norm_apply(x, norm_w, rsf), round_nearest)
    dq = np.zeros(q.shape, dtype=np.int32)
    for r2 in (np.nextafter(rsf, F(0)), np.nextafter(rsf, F(np.inf))):
        q2, _ = quant_q8(norm_apply(x, norm_w, r2.astype(F)), round_nearest)
        dq = np.maximum(dq, np.abs(q2 - q))
    return q, d, dq


def restate_f32(x, norm_w, eps):
    x = np.asarray(x, dtype=F)
    return norm_apply(x, norm_w, rms_rsf(x, eps)).astype(F)


def _row_step(nb, M, K):
    return int(max(16, min((1 << 24) // max(1, nb * M), (1 << 22) // K)))


def int_gemm_ref(q, d, wq, s, dq=None):
    """(ref, nat, amb) [M, N] float64 of Q8 activations (q, d) against (wq, s): exact integer block sums from float32 block
    products (|isum| <= 32 * 127 * 128 < 2^24) over row blocks of the weights"""
    M, K = q.shape
    N, nb = wq.shape[0], K // 32
    A = q.reshape(M, nb, 32).transpose(1, 0, 2).astype(F)
    d64 = d.T.astype(np.float64)[:, :, None]
    ref, nat = np.empty((M, N)), np.empty((M, N))
    step = _row_step(nb, M, K)
    for r0 in range(0, N, step):
        W = wq[r0:r0 + step].reshape(-1, nb, 32).transpose(1, 2, 0).astype(F)
        t = np.matmul(A, W).astype(np.float64) * d64 * s[r0:r0 + step].T.astype(np.float64)[:, None, :]
        ref[:, r0:r0 + step] = t.sum(axis=0)
        nat[:, r0:r0 + step] = np.abs(t).sum(axis=0)
    amb = np.zeros((M, N))
    if dq is not None and dq.any():
        cols = np.nonzero(dq.any(axis=0))[0]
        a = dq[:, cols] * np.abs(d[:, cols // 32].astype(np.float64))
        amb = a @ np.abs(wq[:, cols].astype(np.float64) * s[:, cols // 32].astype(np.float64)).T
    return ref, nat, amb


def f32_gemm_ref(y, wq, s):
    """(ref, nat) [M, N] float64 of f32 activations y against (wq, s): sum_b s_b * sum_k y_k q_k, nat = sum |y_k q_k s_b|"""
    M, K = y.shape
    N, nb = wq.shape[0], K // 32
    Y = y.reshape(M, nb, 32).transpose(1, 0, 2).astype(np.float64)
    ref, nat = np.empty((M, N)), np.empty((M, N))
    ay = np.abs(y.astype(np.float64))
    step = _row_step(nb, M, K)
    for r0 in range(0, N, step):
        wv = wq[r0:r0 + step].astype(np.float64)
        sv = s[r0:r0 + step].astype(np.float64)
        W = wv.reshape(-1, nb, 32).transpose(1, 2, 0)
        ref[:, r0:r0 + step] = (np.matmul(Y, W) * sv.T[:, None, :]).sum(axis=0)
        nat[:, r0:r0 + step] = ay @ np.abs(wv * np.repeat(sv, 32, axis=1)).T
    return ref, nat


def sigmoid(g):
    return 1.0 / (1.0 + np.exp(-g))


def silu(g):
    return g * sigmoid(g)


def dsilu(g):
    sg = sigmoid(g)
    return sg * (1.0 + g * (1.0 - sg))


def err_bar(out, ref, bar):
    """max over elements of |out - ref| / bar (a zero bar demands an exact result)"""
    e = np.abs(np.asarray(out, dtype=np.float64) - ref)
    r = np.where(bar > 0, e / np.where(bar > 0, bar, 1.0), np.where(e > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def level_of(out, ref, nat, extra):
    """max of (|out - ref| - extra) / nat where nat > 0: the measured error in units of the natural scale"""
    e = np.maximum(np.abs(np.asarray(out, dtype=np.float64) - ref) - extra, 0.0)
    live = nat > 0
    return float((e[live] / nat[live]).max()) if live.any() else 0.0


def check_int_phase(out, x_in, wq, s, norm_w=None, eps=1e-5, residual=None):
    """one Q8 x (Q4 | Q8_0) phase with a store or residual epilogue: (err/bar, level, ambiguous count)"""
    q, d, dq = restate_act(x_in, norm_w, eps)
    ref, nat, amb = int_gemm_ref(q, d, wq, s, dq)
    extra = amb
    if residual is not None:
        ref = ref + residual.astype(np.float64)
        extra = amb + ULP_RES * np.abs(ref)
    return err_bar(out, ref, TAU * nat + extra), level_of(out, ref, nat, extra), int((dq > 0).sum())


def check_silu_phase(h, x_in, wg, sg, wu, su, norm_w, eps):
    q, d, dq = restate_act(x_in, norm_w, eps)
    g, ng, ag = int_gemm_ref(q, d, wg, sg, dq)
    u, nu, au = int_gemm_ref(q, d, wu, su, dq)
    ref = silu(g) * u
    eg, eu = TAU * ng + ag, TAU * nu + au
    a, b = np.abs(dsilu(g)) * np.abs(u), np.abs(silu(g))
    floor = ULP_SILU * np.abs(ref) + TINY * (1.0 + np.abs(u))
    extra = a * ag + b * au + floor
    bar = a * eg + b * eu + floor
    return err_bar(h, ref, bar), level_of(h, ref, a * ng + b * nu, extra), int((dq > 0).sum())


def check_f32_phase(out, x_in, wq, s, norm_w, eps):
    y = restate_f32(x_in, norm_w, eps)
    ref, nat = f32_gemm_ref(y, wq, s)
    return err_bar(out, ref, TAU_F * nat), level_of(out, ref, nat, 0.0), 0


# ---- the host's selection rule, restated ------------------------------------------------------------------------------------
GEMV_MAX_M, MAX_ROWS, MAX_SPLITS = 8, 64, 32
SMEM_GEMV = 200 * 1024
G8_SMEM_LIMIT = G64_SMEM_LIMIT = 227 * 1024
PD_NT, PD_MAX_TP, MG_MAX_GROUP, FA_MAX_POS, FA_HPASS = 512, 8, 8, 1024, 4
NORMQ, F32Q, NORMF, = "normq", "f32q", "normf32"


def phases(cfg):
    """phase -> (K, segment rows, prologue, epilogue) of forward_rows / lm_head_rows"""
    E, H = cfg["E"], cfg["H"]
    kv = cfg["kv_heads"] * (E // cfg["heads"])
    return {"qkv": (E, [E, kv, kv], NORMQ, "store"), "o": (E, [E], F32Q, "residual"), "gu": (E, [H, H], NORMQ, "silu"),
            "down": (H, [E], F32Q, "residual"), "lm": (E, [cfg["vocab"]], NORMF, "store")}


def total_rows(seg, epi):
    return seg[0] if epi == "silu" else sum(seg)


def gemv_max_m(pro, K):
    smem1 = (K // 32) * 40 if pro in (NORMQ, F32Q) else K * 4
    return next((mm for mm in (8, 4, 2, 1) if smem1 * mm <= SMEM_GEMV), 0)


def g8_stages(K, nwarp):
    act = 8 * (K + 16) + 8 * (K // 32 + 1) * 8 + 2 * nwarp * 2 * 128 * 4
    if act + 2048 >= G8_SMEM_LIMIT:
        return 0
    return min((G8_SMEM_LIMIT - 2048 - act) // (nwarp * 3072), 6)


def gemm8_supported(wd, pro, epi, M, K, seg):
    bpc = 8 if wd == Q4 else 4
    if not 2 <= M <= 8 or pro not in (NORMQ, F32Q) or (K // 32) % bpc:
        return False
    if epi == "silu" and len(seg) != 2:
        return False
    if epi != "silu" and any(r % 16 for r in seg[:-1]):
        return False
    return g8_stages(K, 8) >= 2


def g8_warps(K):
    return 16 if g8_stages(K, 16) >= 3 else 8


def g8_ksplit(wd, K, rows, sm, nwarp):
    nch = (K // 32) // (8 if wd == Q4 else 4)
    strips = -(-rows // 16)
    want = 1
    while want < nwarp and strips * want < sm * nwarp:
        want <<= 1
    return next((s for s in (16, 8, 4, 2) if s <= want and nch % s == 0), 1)


def g64_nt(M):
    return 2 if M <= 16 else (4 if M <= 32 else (6 if M <= 48 else 8))


def g64_stages(wd, epi, nt, fa):
    bpc = 8 if wd == Q4 else 4
    nw = 2 if epi == "silu" else 1
    stage = 8 * nw * 3072 + (0 if fa else nt * 8 * (bpc * 32 + 16) + bpc * nt * 8 * 8)
    return min((G64_SMEM_LIMIT - 1024) // stage, 6)


def gemm64_supported(wd, pro, epi, M, K, seg):
    fa = pro == NORMF
    if not GEMV_MAX_M < M <= MAX_ROWS:
        return False
    if fa and (epi != "store" or len(seg) != 1):
        return False
    if (K // 32) % (8 if wd == Q4 else 4):
        return False
    if epi == "silu" and len(seg) != 2:
        return False
    if epi != "silu" and any(r % 16 for r in seg[:-1]):
        return False
    return g64_stages(wd, epi, g64_nt(M), fa) >= 2


def g64_ksplit(wd, K, rows, sm):
    groups = -(-(-(-rows // 16)) // 8)
    nch = (K // 32) // (8 if wd == Q4 else 4)
    ks = 1
    while ks < 8 and groups * ks * 2 <= sm and nch % (ks * 2) == 0:
        ks *= 2
    return ks


def launch_gemv(wd, pro, epi, M, K, seg, sm):
    """jl_launch_gemv of M <= 8 rows"""
    rows = total_rows(seg, epi)
    if gemm8_supported(wd, pro, epi, M, K, seg):
        nw = g8_warps(K)
        return dict(kernel="gemm8", wd=wd, epi=epi, M=M, warps=nw, ks=g8_ksplit(wd, K, rows, sm, nw))
    mm = 1 if M <= 1 else (2 if M <= 2 else (4 if M <= 4 else 8))
    nt = 640 if epi == "silu" else 512
    if wd == Q4 and pro != NORMF and mm == 1 and (pro == F32Q or K <= 16 * nt):
        return dict(kernel="gemv_decode", wd=wd, epi=epi, M=1, long=-(-(K // 32) // 128) > 1, pro=pro)
    return dict(kernel="generic", wd=wd, epi=epi, M=M, mm=mm, act="F32" if pro == NORMF else "Q8")


def run_gemm(wd, pro, epi, M, K, seg, sm, wide):
    """the launches of run_gemm for M rows"""
    if wide and M > GEMV_MAX_M and gemm64_supported(wd, pro, epi, M, K, seg):
        rows = total_rows(seg, epi)
        return [dict(kernel="gemm64", wd=wd, epi=epi, M=M, nt=g64_nt(M), ks=g64_ksplit(wd, K, rows, sm), fa=pro == NORMF)]
    chunk = gemv_max_m(pro, K)
    assert chunk >= 1
    return [launch_gemv(wd, pro, epi, min(chunk, M - m0), K, seg, sm) for m0 in range(0, M, chunk)]


def pd_smem_bytes(cfg, G):
    E, H = cfg["E"], cfg["H"]
    hs = E // cfg["heads"]
    kv = cfg["kv_heads"] * hs
    kmax, rmax = max(E, H, E), max(E, H, E + 2 * kv)
    acts = max(((kmax // 32) * 40 + 15) // 16 * 16 + (-(-rmax // G) + 2) * 2 * (PD_NT // 32) * 4 + 64, E * 4)
    att = (MG_MAX_GROUP * hs + 2 * hs + FA_MAX_POS * MG_MAX_GROUP + 2 * (PD_NT // 32) * MG_MAX_GROUP + (PD_NT // 32) * FA_HPASS * hs) * 4 + 64
    m = max(acts, att + 1024, (-(-E // G) + 2) * PD_MAX_TP * 4)
    return (m + 1023) // 1024 * 1024


def pd_eligible(cfg, flags, sm, max_context=MAX_CONTEXT):
    """use_pd: jl_model_finalize's checks (one quantised dtype, Q8 activations) and jl_pdecode_supported"""
    E, H, heads, kvh = cfg["E"], cfg["H"], cfg["heads"], cfg["kv_heads"]
    hs, group = E // heads, heads // kvh
    if flags & (MODEL_NO_PERSISTENT | MODEL_NO_GRAPH) or hs not in (32, 64, 128) or heads % kvh or group > MG_MAX_GROUP:
        return False
    if E % 32 or H % 32 or E > 16 * PD_NT or kvh > sm or group & (group - 1):
        return False
    if pd_smem_bytes(cfg, sm) > SMEM_GEMV:
        return False
    cap = min(sm // kvh, MAX_SPLITS)
    return cap >= 1 and -(-max_context // cap) <= FA_MAX_POS - 32


def host_rule(cfg, n, flags, sm, wd, prefill=False):
    """phase -> [launch dicts] of one decode step of n sessions (or a prefill pass of n rows)"""
    if not prefill and n == 1 and pd_eligible(cfg, flags, sm):
        return {ph: [dict(kernel="pd", wd=wd, epi=epi, M=1)] for ph, (_, _, _, epi) in phases(cfg).items()}
    out = {}
    for ph, (K, seg, pro, epi) in phases(cfg).items():
        if prefill and ph == "lm":
            continue
        out[ph] = run_gemm(wd, pro, epi, n, K, seg, sm, wide=not prefill)
    return out


def label(ln):
    wd = "Q4" if ln["wd"] == Q4 else "Q8_0"
    k = ln["kernel"]
    if k == "gemm8":
        return "gemm8 %s %s M%d w%d ks%d" % (wd, ln["epi"], ln["M"], ln["warps"], ln["ks"])
    if k == "gemm64":
        return "gemm64 %s %s%s nt%d ks%d" % (wd, "FA " if ln["fa"] else "", ln["epi"], ln["nt"], ln["ks"])
    if k == "gemv_decode":
        return "gemv_decode %s %s %s %s" % (wd, ln["epi"], "LONG" if ln["long"] else "short", ln["pro"])
    if k == "generic":
        return "generic %s %s MM%d %s" % (wd, ln["epi"], ln["mm"], ln["act"])
    return "pd %s %s" % (wd, ln["epi"])


def family(launches):
    """the kernel a phase's measured level is recorded under"""
    ks = sorted({ln["kernel"] + (" FA" if ln.get("fa") else "") + (" F32" if ln.get("act") == "F32" else "") for ln in launches})
    return "+".join(ks)


# ---- the case matrix ------------------------------------------------------------------------------------------------------
def _cfg(E, H, heads, kv_heads, vocab, layers=1):
    return dict(E=E, H=H, heads=heads, kv_heads=kv_heads, vocab=vocab, layers=layers)


CFGS = {
    # one Llama-3-8B layer; vocab 2050 leaves a partial 16-row strip
    "8b": _cfg(4096, 14336, 32, 8, 2050),
    # K = E = 8192 = 16 * 512: the RMSNorm prologue's limit in launch_decode and jl_pdecode_supported
    "e8192": _cfg(8192, 2048, 64, 8, 512),
    # QKV LONG at 1.25 chunks; H 2080 = 65 blocks divides by neither 8 nor 4: down_proj falls back to the generic kernel
    "e5120": _cfg(5120, 2080, 40, 8, 512),
    "small": _cfg(256, 512, 8, 4, 512),
    "small-3L": _cfg(256, 512, 8, 4, 512, layers=3),
    # 5 and 11 blocks: every phase of a 2..64-row step on the generic kernel (Q8 and F32 activations, all three epilogues)
    "odd": _cfg(160, 352, 5, 5, 300),
}

ALL = ["pd", "perop", 2, 8, 9, 17, 64]
CASES = [
    dict(id="8b-Q4", cfg="8b", wd=Q4, steps=ALL),
    dict(id="8b-Q8_0", cfg="8b", wd=I8, steps=ALL),
    dict(id="8b-Q4-crafted", cfg="8b", wd=Q4, craft=True, steps=[8, 64]),
    dict(id="e8192-Q4", cfg="e8192", wd=Q4, steps=["pd", "perop", 33]),
    dict(id="e5120-Q4", cfg="e5120", wd=Q4, steps=["pd", "perop", 3, 12, 48]),
    dict(id="e5120-Q8_0", cfg="e5120", wd=I8, steps=["pd", "perop", 3, 12, 48]),
    dict(id="small-Q4", cfg="small", wd=Q4, steps=["pd", 2, 9, 16, 64]),
    dict(id="small-Q8_0", cfg="small", wd=I8, steps=["pd", 2, 9, 16, 64]),
    dict(id="small-3L-Q4", cfg="small-3L", wd=Q4, steps=["pd", 2, 9, 64]),
    dict(id="small-Q4-crafted", cfg="small", wd=Q4, craft=True, steps=["pd", "perop", 2, 9, 64]),
    dict(id="small-Q8_0-crafted", cfg="small", wd=I8, craft=True, steps=["pd", "perop", 2, 9, 64]),
    dict(id="odd-Q4", cfg="odd", wd=Q4, steps=["pd", "perop", 3, 12]),
    dict(id="odd-Q8_0", cfg="odd", wd=I8, steps=["pd", "perop", 3, 12]),
]
PREFILL = dict(id="small-Q4-prefill-11", cfg="small", wd=Q4, rows=11)


def step_n(step):
    return 1 if step in ("pd", "perop") else step


def step_flags(step):
    return MODEL_NO_PERSISTENT if step == "perop" else 0


def case_labels(case, sm=H100_SMS):
    cfg = CFGS[case["cfg"]]
    return [(step, host_rule(cfg, step_n(step), step_flags(step), sm, case["wd"])) for step in case["steps"]]


# ---- weights ----------------------------------------------------------------------------------------------------------------
def llama_cfg(name):
    from jlama_b200 import synth
    c = CFGS[name]
    return synth.get_config("tiny", E=c["E"], H=c["H"], heads=c["heads"], kv_heads=c["kv_heads"], layers=c["layers"], vocab=c["vocab"],
                            ctx=256)


def craft_tensor(wd, t):
    """zero weight scales (row 3, and block 2 of every row), rows of the extreme codes (nibbles 0 / 15, Q8_0 -128 / 127)"""
    dt, data, scales = t
    data, scales = data.copy(), scales.copy()
    scales[3] = 0
    scales[:, 2] = 0
    if wd == Q4:
        data[1], data[2] = 0x00, 0xFF
    else:
        data[1], data[2] = -128, 127
    return (dt, data, scales)


def craft_norm(t):
    """a zeroed 32-block (activation scale 0) and a block whose one large element quantises the rest to 0"""
    dt, w, s = t
    w = w.copy()
    w[:, 32:64] = 0
    w[:, 5 * 32 + 7] = 5000.0
    return (dt, w, s)


@functools.lru_cache(maxsize=None)
def weights(name, wd, craft=False, lm=None):
    """synth direct weights; craft: the crafted operands; lm: 'tied' / 'zero' crafted Q4 lm_head (arg-max)"""
    from jlama_b200 import synth
    w = synth.make_weights(llama_cfg(name), wdtype=wd, mode="direct")
    if craft:
        for k in list(w):
            if k.endswith("norm.weight"):
                w[k] = craft_norm(w[k])
            elif k == "model.embed_tokens.weight":
                dt, data, s = w[k]
                w[k] = (dt, data, (s * F(1e4)).astype(F))  # large residuals
            else:
                w[k] = craft_tensor(wd, w[k])
    if lm is not None:
        assert wd == Q4
        dt, data, s = w["lm_head.weight"]
        V = data.shape[0]
        data = np.full_like(data, 0x88)
        if lm == "tied":
            rng = np.random.default_rng(7)
            lo, hi = rng.integers(1, 16, (2, data.shape[1]))
            pos, neg = (lo | (hi << 4)).astype(np.uint8), ((16 - lo) | ((16 - hi) << 4)).astype(np.uint8)
            for r in TIE_POS:
                data[r] = pos
            for r in TIE_NEG(V):
                data[r] = neg
            s = np.tile(s[7], (V, 1))
        w["lm_head.weight"] = (dt, data, s)
    return w


TIE_POS = (1, 15, 40)


def TIE_NEG(V):
    return (V - 1, 16, 41)


class Ref:
    """host copies of one model's weights as (values, scales)"""

    def __init__(self, name, wd, w):
        self.cfg = llama_cfg(name)
        self.eps = self.cfg["eps"]
        self.t = {k: unpack_weights(*v[:1], v[1], v[2]) if v[0] in (Q4, I8) else v[1] for k, v in w.items()}

    def layer(self, L, name):
        return self.t["model.layers.%d.%s" % (L, name)]

    def norm(self, key):
        return np.asarray(self.t[key], dtype=F).reshape(-1)


# ---- GPU harness ----------------------------------------------------------------------------------------------------------
def make_model(ctx, name, wd, flags=0, craft=False, lm=None, sessions=MAX_ROWS):
    from jlama_b200.model import LlamaModel
    w = weights(name, wd, craft, lm)
    return LlamaModel(ctx, llama_cfg(name), w, max_sessions=sessions, max_context=MAX_CONTEXT, flags=flags), w


def read_bufs(gm, n):
    c = gm.cfg
    E, H = c["E"], c["H"]
    kv = c["kv_heads"] * (E // c["heads"])
    return dict(x=gm.debug_read(0, n * E).reshape(n, E), xb=gm.debug_read(1, n * E).reshape(n, E),
                q=gm.debug_read(2, n * E).reshape(n, E), k=gm.debug_read(3, n * kv).reshape(n, kv),
                v=gm.debug_read(4, n * kv).reshape(n, kv), att=gm.debug_read(5, n * E).reshape(n, E),
                h=gm.debug_read(6, n * H).reshape(n, H), logits=gm.debug_read(7, n * c["vocab"]).reshape(n, c["vocab"]))


WORST = {}


def _record(kernel, err, lvl):
    w, l = WORST.get(kernel, (0.0, 0.0))
    WORST[kernel] = (max(w, err), max(l, lvl))


def check_phases(ref, tokens, b, logits, rule, label_, layers=1, prefill=False):
    """every phase of the last layer from the buffers that feed it; returns [(phase, kernel, err/bar, level, ambiguous)]"""
    L = layers - 1
    eps = ref.eps
    res = []

    def rec(ph, r):
        kern = family(rule[ph])
        _record(kern, r[0], r[1])
        assert r[0] <= 1.0, "%s %s (%s): err/bar %.3f, level %.2e" % (label_, ph, "; ".join(label(x) for x in rule[ph]), r[0], r[1])
        res.append((ph, kern, r[0], r[1], r[2]))

    if layers == 1:
        wq_e, s_e = ref.t["model.embed_tokens.weight"]
        x0 = dequant_rows(wq_e, s_e, np.asarray(tokens))
        (wq, sq), (wk, sk), (wv, sv) = ref.layer(L, "self_attn.q_proj.weight"), ref.layer(L, "self_attn.k_proj.weight"), \
            ref.layer(L, "self_attn.v_proj.weight")
        W = np.concatenate([wq, wk, wv]) if not prefill else np.concatenate([wk, wv])
        S = np.concatenate([sq, sk, sv]) if not prefill else np.concatenate([sk, sv])
        out = np.concatenate([b["q"], b["k"], b["v"]], axis=1) if not prefill else np.concatenate([b["k"], b["v"]], axis=1)
        rec("qkv", check_int_phase(out, x0, W, S, ref.norm("model.layers.%d.input_layernorm.weight" % L), eps))
        wo, so = ref.layer(L, "self_attn.o_proj.weight")
        rec("o", check_int_phase(b["xb"], b["att"], wo, so, residual=x0))
    (wg, sg), (wu, su) = ref.layer(L, "mlp.gate_proj.weight"), ref.layer(L, "mlp.up_proj.weight")
    rec("gu", check_silu_phase(b["h"], b["xb"], wg, sg, wu, su, ref.norm("model.layers.%d.post_attention_layernorm.weight" % L), eps))
    wd_, sd = ref.layer(L, "mlp.down_proj.weight")
    rec("down", check_int_phase(b["x"], b["h"], wd_, sd, residual=b["xb"]))
    if logits is not None:
        wl, sl = ref.t["lm_head.weight"]
        rec("lm", check_f32_phase(logits, b["x"], wl, sl, ref.norm("model.norm.weight"), eps))
    return res


def assert_argmax(nxt, logits, label_):
    want = np.argmax(logits, axis=1)
    assert np.array_equal(np.asarray(nxt), want), "%s: next tokens %s, lowest index of the maximum %s" % (label_, list(nxt[:8]), list(want[:8]))


def decode_step(gm, n, rng, vocab, tokens=None):
    """one step of sessions 0 .. n - 1, all at position 0: every session's KV pages below its position exist (a 1024-wide KV row
    puts one position in a page), and the attention is not what this file checks"""
    toks = rng.integers(0, vocab, n).astype(np.int32) if tokens is None else tokens
    nxt, logits = gm.decode(toks, np.zeros(n, dtype=np.int32), sessions=np.arange(n, dtype=np.int32), want_logits=True)
    return toks, nxt, logits


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_decode_gemm_against_exact_references(cuda_ctx, case):
    sm = cuda_ctx.sm_count
    cfg = CFGS[case["cfg"]]
    rng = np.random.default_rng(zlib.crc32(case["id"].encode()))
    models = {}
    try:
        ref = None
        for step in case["steps"]:
            flags = step_flags(step)
            if flags not in models:
                models[flags] = make_model(cuda_ctx, case["cfg"], case["wd"], flags, case.get("craft", False))
            gm, w = models[flags]
            ref = ref or Ref(case["cfg"], case["wd"], w)
            n = step_n(step)
            rule = host_rule(cfg, n, flags, sm, case["wd"])
            pd = rule["qkv"][0]["kernel"] == "pd"
            assert gm.decode_mode(n) == (3 if pd else 1), (case["id"], step)
            toks, nxt, logits = decode_step(gm, n, rng, cfg["vocab"])
            lab = "%s step %s (n=%d)" % (case["id"], step, n)
            assert_argmax(nxt, logits, lab)
            res = check_phases(ref, toks, read_bufs(gm, n), logits, rule, lab, cfg["layers"])
            for ph, kern, e, lv, amb in res:
                print("%s %-4s %-26s err/bar %.3f level %.2e ambiguous %d  [%s]" % (lab, ph, kern, e, lv, amb,
                                                                                    "; ".join(label(x) for x in rule[ph])))
    finally:
        for gm, _ in models.values():
            gm.close()


@gpu
def test_prefill_chunks_against_exact_references(cuda_ctx):
    """an 11-row exact prefill pass: gemm8 at 8 rows, then at 3 (q is rotated in place by the attention, so k / v stand for QKV)"""
    sm = cuda_ctx.sm_count
    c = PREFILL
    cfg = CFGS[c["cfg"]]
    rule = host_rule(cfg, c["rows"], 0, sm, c["wd"], prefill=True)
    assert [[ln["kernel"] + str(ln["M"]) for ln in rule[ph]] for ph in ("qkv", "o", "gu", "down")] == [["gemm88", "gemm83"]] * 4
    gm, w = make_model(cuda_ctx, c["cfg"], c["wd"])
    try:
        ref = Ref(c["cfg"], c["wd"], w)
        toks = np.random.default_rng(11).integers(0, cfg["vocab"], c["rows"]).astype(np.int32)
        gm.batch_forward(toks, 0, session=0)
        res = check_phases(ref, toks, read_bufs(gm, c["rows"]), None, rule, c["id"], prefill=True)
        for ph, kern, e, lv, amb in res:
            print("%s %-4s %-10s err/bar %.3f level %.2e ambiguous %d" % (c["id"], ph, kern, e, lv, amb))
    finally:
        gm.close()


@gpu
@pytest.mark.parametrize("lm", ["tied", "zero"])
def test_argmax_ties_and_zero_lm_head(cuda_ctx, lm):
    """the crafted lm_heads on every route: pd, the per-op arg-max after the generic F32 lm_head (1 and 2 rows) and after
    gemm64's FA (9 and 64 rows)"""
    sm = cuda_ctx.sm_count
    cfg = CFGS["small"]
    V = cfg["vocab"]
    rng = np.random.default_rng(5)
    for flags, steps in ((0, ["pd", 2, 9, 64]), (MODEL_NO_PERSISTENT, ["perop"])):
        gm, w = make_model(cuda_ctx, "small", Q4, flags, lm=lm)
        try:
            ref = Ref("small", Q4, w)
            for step in steps:
                n = step_n(step)
                rule = host_rule(cfg, n, flags, sm, Q4)
                assert gm.decode_mode(n) == (3 if step == "pd" else 1)
                toks, nxt, logits = decode_step(gm, n, rng, V)
                lab = "%s lm_head, step %s [%s]" % (lm, step, label(rule["lm"][0]))
                assert_argmax(nxt, logits, lab)
                check_phases(ref, toks, read_bufs(gm, n), logits, rule, lab)
                others = np.setdiff1d(np.arange(V), TIE_POS + TIE_NEG(V))
                assert not np.any(logits[:, others]), lab
                if lm == "zero":
                    assert not np.any(logits) and not np.any(nxt), lab
                    continue
                pos, neg = logits[:, list(TIE_POS)], logits[:, list(TIE_NEG(V))]
                assert np.array_equal(pos.view(np.uint32), np.repeat(pos[:, :1], 3, axis=1).view(np.uint32)), lab
                assert np.array_equal(neg, -pos), lab
                print("%s: row values %s, tokens %s" % (lab, pos[:4, 0].tolist(), nxt[:4].tolist()))
        finally:
            gm.close()


@gpu
def test_determinism_and_untouched_rows(cuda_ctx):
    """the same step twice gives the same bits (pd, and k-split > 1 at 8 and 64 rows); a 9-row step after a 64-row step leaves
    rows 9..63 of every buffer unchanged"""
    sm = cuda_ctx.sm_count
    cfg = CFGS["8b"]
    rng = np.random.default_rng(3)
    gm, _ = make_model(cuda_ctx, "8b", Q4)
    try:
        for n in (1, 8, 64):
            rule = host_rule(cfg, n, 0, sm, Q4)
            if n > 1:
                assert any(ln.get("ks", 1) > 1 for ph in rule.values() for ln in ph), n
            toks, nxt, logits = decode_step(gm, n, rng, cfg["vocab"])
            first = read_bufs(gm, n)
            _, nxt2, logits2 = decode_step(gm, n, rng, cfg["vocab"], tokens=toks)
            again = read_bufs(gm, n)
            assert np.array_equal(nxt, nxt2) and np.array_equal(logits.view(np.uint32), logits2.view(np.uint32)), n
            for k in first:
                assert np.array_equal(first[k].view(np.uint32), again[k].view(np.uint32)), (n, k)
        decode_step(gm, 64, rng, cfg["vocab"])
        before = read_bufs(gm, 64)
        assert host_rule(cfg, 9, 0, sm, Q4)["qkv"][0]["nt"] == 2
        decode_step(gm, 9, rng, cfg["vocab"])
        after = read_bufs(gm, 64)
        for k in before:
            assert np.array_equal(before[k][9:].view(np.uint32), after[k][9:].view(np.uint32)), "rows 9..63 of %s changed" % k
            assert not np.array_equal(before[k][:9].view(np.uint32), after[k][:9].view(np.uint32)), k
    finally:
        gm.close()


@gpu
def test_zz_report():
    """the worst err/bar and level per kernel over the cases that ran"""
    for k in sorted(WORST):
        print("decode gemm %-28s: worst level %.2e, err/bar %.3f" % (k, WORST[k][1], WORST[k][0]))


# ---- the case matrix, checked on the CPU ----------------------------------------------------------------------------------
def _all_launches(sm=H100_SMS):
    for case in CASES:
        for step, rule in case_labels(case, sm):
            for ph, lns in rule.items():
                for ln in lns:
                    yield case, step, ph, ln
    c = PREFILL
    for ph, lns in host_rule(CFGS[c["cfg"]], c["rows"], 0, sm, c["wd"], prefill=True).items():
        for ln in lns:
            yield c, "prefill", ph, ln


def test_case_matrix_reaches_every_kernel_variant():
    seen = set()
    for case, step, ph, ln in _all_launches():
        k, wd, epi = ln["kernel"], ln["wd"], ln["epi"]
        seen.add((k, wd, epi))
        if k == "gemv_decode":
            seen.add(("gemv_decode", "LONG" if ln["long"] else "short"))
            seen.add(("gemv_decode", ln["pro"]))
        elif k == "gemm8":
            seen.add(("gemm8", "warps", ln["warps"]))
            seen.add(("gemm8", "ks", min(ln["ks"], 2)))
        elif k == "gemm64":
            seen.add(("gemm64", "nt", ln["nt"]))
            seen.add(("gemm64", "ks", min(ln["ks"], 2)))
            if ln["fa"]:
                seen.add(("gemm64", "FA", wd, ln["ks"] > 1))
        elif k == "generic":
            seen.add(("generic", "MM", ln["mm"]))
            seen.add(("generic", ln["act"], wd))
            if step_n(step) >= 2 and ln["act"] == "Q8":
                seen.add(("generic", "inside an n >= 2 step", wd))
        if case["cfg"] == "e8192" and k == "pd":
            seen.add(("pd", "E 8192"))
    missing = []
    for wd in (Q4, I8):
        for epi in ("store", "residual", "silu"):
            for k in ("pd", "gemm8", "gemm64", "generic"):
                missing += [] if (k, wd, epi) in seen else [(k, wd, epi)]
        missing += [x for x in (("generic", "F32", wd), ("generic", "Q8", wd), ("generic", "inside an n >= 2 step", wd),
                                ("gemm64", "FA", wd, True)) if x not in seen]
    for epi in ("store", "residual", "silu"):
        missing += [] if ("gemv_decode", Q4, epi) in seen else [("gemv_decode", epi)]
    want = [("gemv_decode", "LONG"), ("gemv_decode", "short"), ("gemv_decode", NORMQ), ("gemv_decode", F32Q),
            ("gemm8", "warps", 8), ("gemm8", "warps", 16), ("gemm8", "ks", 1), ("gemm8", "ks", 2),
            ("gemm64", "nt", 2), ("gemm64", "nt", 4), ("gemm64", "nt", 6), ("gemm64", "nt", 8), ("gemm64", "ks", 1), ("gemm64", "ks", 2),
            ("generic", "MM", 1), ("generic", "MM", 2), ("generic", "MM", 4), ("generic", "MM", 8), ("pd", "E 8192")]
    missing += [x for x in want if x not in seen]
    assert not missing, missing


def test_host_rule_edges():
    """the restated rule at its boundaries (132 SMs)"""
    c8 = CFGS["8b"]
    r = host_rule(c8, 1, MODEL_NO_PERSISTENT, H100_SMS, Q4)
    assert [label(r[p][0]) for p in ("qkv", "down", "lm")] == [
        "gemv_decode Q4 store short normq", "gemv_decode Q4 residual LONG f32q", "generic Q4 store MM1 F32"]
    r = host_rule(c8, 8, 0, H100_SMS, Q4)
    assert [(x[0]["warps"], x[0]["ks"]) for x in (r["qkv"], r["o"], r["gu"], r["down"])] == [(16, 8), (16, 16), (16, 4), (8, 8)]
    r = host_rule(c8, 64, 0, H100_SMS, Q4)
    assert [(x[0]["nt"], x[0]["ks"]) for x in (r["qkv"], r["o"], r["gu"], r["down"], r["lm"])] == [(8, 2), (8, 4), (8, 1), (8, 4), (8, 4)]
    assert r["lm"][0]["fa"]
    # E 8192: exactly at the prologue's 16 * 512 limit, and inside pd's shared memory
    assert pd_eligible(CFGS["e8192"], 0, H100_SMS) and pd_smem_bytes(CFGS["e8192"], H100_SMS) <= SMEM_GEMV
    assert not pd_eligible(dict(CFGS["e8192"], E=8192 + 32 * 8, heads=66), 0, H100_SMS)
    # 40 / 8 heads: a group of 5 has no persistent kernel; H 2080 sends down_proj to the generic kernel inside gemm8 / gemm64 steps
    assert not pd_eligible(CFGS["e5120"], 0, H100_SMS)
    r = host_rule(CFGS["e5120"], 12, 0, H100_SMS, Q4)
    assert [label(x) for x in r["down"]] == ["generic Q4 residual MM8 Q8", "generic Q4 residual MM4 Q8"]
    assert r["qkv"][0]["kernel"] == "gemm64" and r["gu"][0]["kernel"] == "gemm64"
    assert [g64_nt(m) for m in (9, 16, 17, 32, 33, 48, 49, 64)] == [2, 2, 4, 4, 6, 6, 8, 8]
    assert gemv_max_m(NORMF, 8192) == 4 and gemv_max_m(F32Q, 14336) == 8


def test_reference_quantiser_matches_the_host_quantiser():
    """quant_q8 equals tensor.quantize_q8_activations (the reference back-end's quantiser) bit for bit, zero blocks included"""
    rng = np.random.default_rng(1)
    x = (rng.standard_normal((3, 256)) * np.exp(rng.uniform(-8, 8, (3, 1)))).astype(F)
    x[1, 64:96] = 0
    q, d = quant_q8(x)
    qh, dh = T.quantize_q8_activations(x)
    assert np.array_equal(qh.astype(np.int32), q)
    assert np.array_equal(dh.view(np.uint32), d.view(np.uint32))


# ---- sharpness of the bars (CPU) --------------------------------------------------------------------------------------------
def _problem(wd=Q4, M=4, K=4096, N=96, seed=2):
    """Q8 activations of random rows and synth-direct weights"""
    from jlama_b200 import synth
    t = synth.make_tensor(seed, N, K, wd, "direct")
    wq, s = unpack_weights(wd, t[1], t[2])
    x = np.random.default_rng(seed).standard_normal((M, K)).astype(F)
    q, d, _ = restate_act(x)
    return x, q, d, wq, s


def _ratio(out, ref, bar, what):
    r = err_bar(out, ref, bar)
    print("%s: err/bar %.1f" % (what, r))
    assert r >= SHARP, (what, r)


def test_bar_accepts_f32_accumulation():
    """acc = f32(acc + f32(f32(d * s) * isum)) block by block, and a k-split of 8 partial sums added in order, stay within the bar"""
    for wd, K in ((Q4, 14336), (I8, 4096)):
        x, q, d, wq, s = _problem(wd, M=2, K=K, N=64)
        ref, nat, _ = int_gemm_ref(q, d, wq, s)
        nb = K // 32
        A = q.reshape(2, nb, 32).astype(np.int64)
        W = wq.reshape(64, nb, 32).astype(np.int64)
        isum = np.einsum("mbk,nbk->bmn", A, W).astype(F)
        parts = []
        for blocks in np.array_split(np.arange(nb), 8):
            acc = np.zeros((2, 64), dtype=F)
            for b in blocks:
                acc = (acc + (d[:, b][:, None] * s[:, b][None, :]).astype(F) * isum[b]).astype(F)
            parts.append(acc)
        out = parts[0]
        for p_ in parts[1:]:
            out = (out + p_).astype(F)
        assert err_bar(out, ref, TAU * nat) <= 0.25


def test_bar_rejects_a_dropped_or_doubled_block():
    x, q, d, wq, s = _problem()
    ref, nat, _ = int_gemm_ref(q, d, wq, s)
    for f in (0, 2):
        q2 = q.copy()
        q2[:, 37 * 32:38 * 32] *= f
        _ratio(int_gemm_ref(q2, d, wq, s)[0], ref, TAU * nat, "block %s" % ("dropped" if f == 0 else "doubled"))


def test_bar_rejects_a_dropped_ksplit_share():
    x, q, d, wq, s = _problem(K=14336)
    ref, nat, _ = int_gemm_ref(q, d, wq, s)
    q2 = q.copy()
    q2[:, 3 * 14336 // 8:4 * 14336 // 8] = 0
    _ratio(int_gemm_ref(q2, d, wq, s)[0], ref, TAU * nat, "k-split share dropped")


def test_bar_rejects_a_neighbouring_rows_weight_scale():
    for wd in (Q4, I8):
        x, q, d, wq, s = _problem(wd)
        ref, nat, _ = int_gemm_ref(q, d, wq, s)
        s2 = s.copy()
        s2[10, 9] = s[11, 9]
        _ratio(int_gemm_ref(q, d, wq, s2)[0], ref, TAU * nat, "one weight scale from the neighbouring row")


def test_bar_rejects_another_sessions_activation_scale():
    """gemm64 keeps the activation scales as [K/32][mpad]: a wrong index reads another session's scale of the same block"""
    x, q, d, wq, s = _problem(M=16)
    ref, nat, _ = int_gemm_ref(q, d, wq, s)
    d2 = d.copy()
    d2[5, 20] = d[6, 20]
    _ratio(int_gemm_ref(q, d2, wq, s)[0], ref, TAU * nat, "activation scale of another session")


def test_bar_rejects_swapped_nibble_halves():
    x, q, d, wq, s = _problem()
    ref, nat, _ = int_gemm_ref(q, d, wq, s)
    w2 = wq.reshape(wq.shape[0], -1, 2, 16)[:, :, ::-1].reshape(wq.shape)
    _ratio(int_gemm_ref(q, d, w2, s)[0], ref, TAU * nat, "Q4 nibble halves swapped")


def test_bar_rejects_a_missing_offset():
    x, q, d, wq, s = _problem()
    ref, nat, _ = int_gemm_ref(q, d, wq, s)
    w2 = wq.copy()
    w2[:, 64:96] += 8
    _ratio(int_gemm_ref(q, d, w2, s)[0], ref, TAU * nat, "-8 offset missing on one block")


def test_bar_rejects_round_to_nearest_quantisation():
    x, q, d, wq, s = _problem()
    w = np.random.default_rng(4).uniform(0.5, 1.5, x.shape[1]).astype(F)
    q, d, dq = restate_act(x, w)
    ref, nat, amb = int_gemm_ref(q, d, wq, s, dq)
    q2, d2, _ = restate_act(x, w, round_nearest=True)
    _ratio(int_gemm_ref(q2, d2, wq, s)[0], ref, TAU * nat + amb, "quantiser rounding to nearest")


def test_bar_rejects_a_missing_or_doubled_residual():
    x, q, d, wq, s = _problem()
    ref, nat, _ = int_gemm_ref(q, d, wq, s)
    res = np.random.default_rng(5).standard_normal(ref.shape).astype(F)
    full = ref + res
    bar = TAU * nat + ULP_RES * np.abs(full)
    _ratio(ref, full, bar, "residual missing")
    _ratio(ref + 2 * res, full, bar, "residual doubled")


def test_bar_rejects_silu_on_up():
    x, q, d, wq, s = _problem(N=128)
    g, ng, _ = int_gemm_ref(q, d, wq[:64], s[:64])
    u, nu, _ = int_gemm_ref(q, d, wq[64:], s[64:])
    ref = silu(g) * u
    bar = np.abs(dsilu(g)) * np.abs(u) * TAU * ng + np.abs(silu(g)) * TAU * nu + ULP_SILU * np.abs(ref)
    _ratio(silu(u) * g, ref, bar, "SiLU applied to up")


def test_bar_rejects_a_row_written_to_the_neighbouring_session():
    x, q, d, wq, s = _problem(M=9)
    ref, nat, _ = int_gemm_ref(q, d, wq, s)
    out = ref.copy()
    out[8] = ref[7]
    _ratio(out, ref, TAU * nat, "row 7 written to session 8")


def _planes(y):
    hi = T.bfloat16_to_float32(T.float32_to_bfloat16(y))
    r1 = (y - hi).astype(F)
    mid = T.bfloat16_to_float32(T.float32_to_bfloat16(r1))
    lo = T.bfloat16_to_float32(T.float32_to_bfloat16((r1 - mid).astype(F)))
    return hi, mid, lo


def test_bar_rejects_a_dropped_fa_plane():
    """FA splits each f32 activation into hi + mid + lo BF16 planes (exact).  A dropped mid plane is rejected; the lo plane sits
    below the bar (its ratio is printed)"""
    for wd in (Q4, I8):
        x, q, d, wq, s = _problem(wd, M=16, N=64)
        y = restate_f32(x, np.ones(x.shape[1], dtype=F), 1e-5)
        hi, mid, lo = _planes(y)
        assert np.array_equal(((hi + mid).astype(F) + lo).astype(F), y)
        ref, nat = f32_gemm_ref(y, wq, s)
        _ratio(f32_gemm_ref((hi + lo).astype(F), wq, s)[0], ref, TAU_F * nat, "FA mid plane dropped")
        r = err_bar(f32_gemm_ref((hi + mid).astype(F), wq, s)[0], ref, TAU_F * nat)
        print("FA lo plane dropped: err/bar %.3f (not visible)" % r)
