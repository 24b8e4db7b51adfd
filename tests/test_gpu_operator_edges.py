"""The operator-level API (the host-buffer entry points of jl_runtime.cu) and the temperature draw pinned against exact references
at their edges.  Every reference is a numpy restatement of the operator's own arithmetic; importing this file does not load the CUDA
library.

Quantised jl_gemm (gemm_locked -> gemv_kernel, prologues PRO_F32 / PRO_BF16_GLOBAL / PRO_Q8_GLOBAL), F32, BF16 and I8 activations
x Q4 and Q8_0 weights, M 1..32 (MM 1 / 2 / 4 / 8 with dead rows, and the row-chunk loop), K from 32 to 51200 (both sides of the
4096-element register chunk, F32 at MM 8 filling exactly 200 KiB at 6400, F32 at MM 1 at 51200), every activation column offset and
odd row strides, weight column / row offsets, result offsets, N 1..129, and crafted operands (zero rows, nibbles 0 and 15 only,
scales of mixed sign from 1e-30 to 1e30):
  I8 activations:   ref = sum_b d_b * s_b * isum_b with isum the exact integer block sum, nat = sum_b |d_b s_b isum_b|;
                    |out - ref| <= TAU * nat.
  F32 / BF16:       ref = the float64 product of the (BF16-widened) activations and the dequantised weights, nat = sum |a w s|;
                    |out - ref| <= TAU_F * nat.
  TAU = 2^-17 and TAU_F = 2^-18 are test_gpu_decode_gemm.py's bars for the same kernel.  Columns of the result outside the written
  slice keep their values, a call with an unaligned column offset or row stride gives the same bits as the packed copy of the same
  operands, and every refusal of gemm_locked (k, weight offset or I8 activation offset not a multiple of 32, an I8 row stride that is
  not whole blocks, K beyond the shared memory at one row) returns its code and writes nothing.
accumulate / maccumulate / scale: bit for bit, one rounding per element (Q4: f32((nibble - 8) * scale) first), b of 1 or a_rows
  rows, Q4 offsets that are not whole blocks, lengths past the 1024 x 256 grid; elements outside [offset, offset + length) unchanged;
  I8 b refused (accumulate_kernel has no I8 branch).
saxpy / saxpy_batch: bit for bit against y = fma(x_r, alpha_r, y) row by row in row order (fma restated exactly: the double
  product is exact, the double sum is rounded to odd, then to float).  The reference differs here on purpose: Panama fuses only up
  to loopBound(limit) and takes y + a * x in its tails, and its batched form leaves the tail elements of each 4-row group to the
  one-row tails (PanamaTensorOperations.java:2659-2698).  This project fuses every element of every row (DESIGN.md §6).
Quantisers: bit for bit against tensor.py's restatements of the reference quantisers at their edges (zero blocks, single non-zero,
  exact x * id + 0.5 ties on both signs, subnormal blocks, RNE ties, NaN payloads, values rounding to inf, +-max ties, the
  Float.MIN_VALUE path, the clamp at 15 and the int8 wraps, grid-stride wraps).  NaN and inf in the Q8 activation quantiser follow
  the kernel (DESIGN.md §6): a NaN element quantises to 0 and does not enter its block's maximum; a block holding +-inf gets scale inf
  and all-zero values.
rmsnorm: rsf = f32(1 / sqrt(sum f64(f32(x * x)) / E + eps)) over the slice, divided by E; out = f32(f32(adj + w) * f32(rsf * x)),
  each row equal to the restatement at rsf or rsf +- 1 ulp (the double sums are formed in another order); zeros outside the slice.
layernorm: the float sums (double sums rounded once) within their own rounding uncertainty: each row must equal the restatement for
  one of sum, sumSq in {f32(s - t), f32(s), f32(s + t)}, t = n * 2^-52 * sum |term|.
activation (SiLU, GELU-tanh, TANH), silu_mul: the double expression rounded once to float; the output must lie in
  [f32(y - t), f32(y + t)] (one value unless y is within t of a float midpoint) with t a few double ulps of the expression (for GELU, of its 1 + tanh term, which cancels for
  large negative inputs), and equal f32(y) bit for bit (sign of zero included) where t = 0.
softmax: restated in the kernel's order (1024 threads striding, the warp butterfly, the 32 warp sums in sequence; the pre-offset
  elements divided as well, VectorMath.java:87): every output bit-exact.  Separately, against the reference's sequential float sum,
  |out - out_seq| <= (length + 64) 2^-23 |out|.
Temperature draw (softmax_sample_kernel through jl_select_constrained with no filter, penalty or mask): restated exactly (256
  threads striding, the warp butterfly, the 8 warp sums in sequence, acc += e_i / t on one thread, vocab - 1 when u is never
  reached): every token equal.  Against oracle.sample_temperature (the reference's sequential sums) tokens are equal except where u
  lies within (vocab + 64) 2^-23 of a step of the float64 CDF between the two tokens (the count is printed).  decode_sample at n = 1
  (persistent kernel) and n = 3 picks what the restatement picks from the logits it hands back.

Measured on an NVIDIA H100 80GB HBM3 (SXM, 700 W power limit, 1980 MHz max SM clock): worst err/bar over the gemm cases
F32 x Q4 0.019, F32 x Q8_0 0.045, BF16 x Q4 0.029, BF16 x Q8_0 0.010, I8 x Q4 0.020, I8 x Q8_0 0.018 (test_zz_report prints them).
accumulate, maccumulate, scale, saxpy, the four quantisers, softmax and the draw: exact, with no exponential at a float midpoint
in any softmax or draw row; rmsnorm, layernorm, activation and silu_mul within their windows; softmax's worst distance to the
sequential sum 0.037 of its bound.  The whole file takes about 11 s on that card.

The CPU tests at the end check that the case matrix reaches every variant (MM 1 / 2 / 4 / 8, the chunk loop, every grid-stride wrap,
every refusal) and that each bar rejects its target defect by at least 4x (exact checks: that the defect changes the output).
"""
import ctypes as C
import fractions
import zlib

import numpy as np
import pytest

from jlama_b200 import tensor as T  # numpy only
from jlama_b200.native import BF16, F32, I8, JL_ERR_INVALID, JL_ERR_UNSUPPORTED, JL_OK, Q4, ptr

gpu = pytest.mark.gpu

TAU = 2.0 ** -17   # I8 activations (test_gpu_decode_gemm.py)
TAU_F = 2.0 ** -18  # F32 / BF16 activations (test_gpu_decode_gemm.py)
SHARP = 4.0
H100_SMS = 132
SMEM_GEMV = 200 * 1024
F = np.float32
f64 = np.float64

# ---- exact float helpers (numpy only) --------------------------------------------------------------------------------------


def bits(x):
    return np.ascontiguousarray(x, dtype=F).view(np.uint32)


def same_bits(a, b):
    """bit-equal, any NaN equal to any NaN"""
    a, b = np.asarray(a, dtype=F), np.asarray(b, dtype=F)
    return (bits(a) == bits(b)) | (np.isnan(a) & np.isnan(b))


def fma_f32(a, b, c):
    """f32(a * b + c) rounded once: the double product is exact, the double sum is rounded to odd, then to float (53 >= 2 * 24 + 2)"""
    p = np.asarray(a, dtype=f64) * np.asarray(b, dtype=f64)
    c = np.asarray(c, dtype=f64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)  # TwoSum: p + c = s + e exactly
        even = (s.view(np.uint64) & np.uint64(1)) == 0
        fix = (e != 0) & even & np.isfinite(s)
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(F)


def interval_ok(out, y, t):
    """out within [f32(y - t), f32(y + t)] (each end rounded to nearest: one value unless y is within t of a float midpoint);
    bit-exact f32(y) (sign of zero included) where t == 0; NaN matches NaN"""
    out = np.asarray(out, dtype=F)
    y = np.asarray(y, dtype=f64)
    with np.errstate(invalid="ignore", over="ignore"):
        lo, hi = (y - t).astype(F), (y + t).astype(F)
        inside = (out >= lo) & (out <= hi) & (t > 0)
    return inside | same_bits(out, y.astype(F))


# ---- quantised jl_gemm: references and the host rule -----------------------------------------------------------------------


def unpack_q4(data):
    N, half = data.shape
    b = data.reshape(N, half // 16, 16)
    return (np.concatenate([b & 0x0F, b >> 4], axis=2).reshape(N, half * 2).astype(np.int16) - 8).astype(np.int8)


def pack_q4(nib):
    N, K = nib.shape
    b = nib.reshape(N, K // 32, 32).astype(np.uint8)
    return (b[:, :, :16] | (b[:, :, 16:] << 4)).reshape(N, K // 2).astype(np.uint8)


def f32_gemm_ref(a, wq, s):
    """(ref, nat) [M, N] float64: sum_k a_k * w_k * s_b(k) and sum |a_k w_k s_b(k)|"""
    ws = wq.astype(f64) * np.repeat(s.astype(f64), 32, axis=1)
    a64 = a.astype(f64)
    return a64 @ ws.T, np.abs(a64) @ np.abs(ws).T


def int_gemm_ref(q, d, wq, s):
    """(ref, nat) [M, N] float64 of Q8 activations (q, d) against (wq, s): exact integer block sums"""
    M, K = q.shape
    N, nb = wq.shape[0], K // 32
    A = q.reshape(M, nb, 32).transpose(1, 0, 2).astype(f64)
    W = wq.reshape(N, nb, 32).transpose(1, 2, 0).astype(f64)
    isum = np.matmul(A, W)  # [nb, M, N], exact (|isum| < 2^22)
    t = isum * d.T.astype(f64)[:, :, None] * s.T.astype(f64)[:, None, :]
    return t.sum(axis=0), np.abs(t).sum(axis=0)


def err_bar(out, ref, bar):
    e = np.abs(np.asarray(out, dtype=f64) - ref)
    r = np.where(bar > 0, e / np.where(bar > 0, bar, 1.0), np.where(e > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def gemv_max_m(act, K):
    """jl_gemv_max_m for quantised weights: Q8 staging is 40 bytes per block and row, F32 staging (F32 and BF16) 4 bytes per element"""
    smem1 = (K // 32) * 40 if act == "I8" else K * 4
    return next((mm for mm in (8, 4, 2, 1) if smem1 * mm <= SMEM_GEMV), 0)


def gemm_rule(c):
    """gemm_locked restated: ("refuse", code) or the MM of each launch of the row-chunk loop"""
    act, K, M = c["act"], c["K"], c["M"]
    if K % 32 or c["boff"] % 32 or (act == "I8" and c["aoff"] % 32):
        return ("refuse", JL_ERR_INVALID)
    if act == "I8" and c["lda"] % 32:
        return ("refuse", JL_ERR_INVALID)
    chunk = gemv_max_m(act, K)
    if chunk < 1:
        return ("refuse", JL_ERR_UNSUPPORTED)
    mms = []
    for m0 in range(0, M, chunk):
        mc = min(chunk, M - m0)
        mms.append(next(mm for mm in (1, 2, 4, 8) if mc <= mm))
    return mms


def _case(act, wd, M, K, N, aoff=0, lda=None, boff=0, n0=0, roff=0, craft=False):
    if lda is None:
        lda = aoff + K
    return dict(act=act, wd=wd, M=M, K=K, N=N, aoff=aoff, lda=lda, boff=boff, n0=n0, roff=roff, craft=craft)


ACTS = ("F32", "BF16", "I8")
WDS = (Q4, I8)
KS = ((32, 3), (4064, 2), (4096, 2), (4128, 2), (6400, 8), (6432, 8), (8192, 4), (14336, 3), (51200, 2))


def gemm_cases(act, wd):
    cs = [_case(act, wd, M, 1024, 17, boff=32, n0=2) for M in (1, 2, 3, 4, 5, 8, 9, 32)]
    cs += [_case(act, wd, M, K, 17 if K < 14336 else 7) for K, M in KS]
    offs = (0, 1, 2, 3, 4, 7, 8, 32, 512) if act != "I8" else (0, 32, 512)
    for aoff in offs:
        extra = 5 if act != "I8" else 64  # odd row strides for F32 / BF16, whole blocks for I8
        cs.append(_case(act, wd, 3, 256, 16, aoff=aoff, lda=aoff + 256 + extra, boff=64, n0=5, roff=2))
    if act != "I8":
        cs.append(_case(act, wd, 9, 512, 16, aoff=3, lda=1027, boff=32, n0=1))  # odd lda across a chunk loop at MM 8 + MM 1
    cs += [_case(act, wd, 4, 512, N, boff=32, n0=3, roff=-3) for N in (1, 7, 16, 17, 129)]
    cs.append(_case(act, wd, 9, 1024, 33, boff=0, n0=4, roff=1, craft=True))
    cs.append(_case(act, wd, 2, 4096, 16, craft=True))
    return cs


REFUSALS = [
    _case("F32", Q4, 2, 48, 8),                        # k % 32
    _case("F32", Q4, 2, 64, 8, boff=16),               # weight column offset % 32
    _case("I8", Q4, 2, 64, 8, aoff=16, lda=128),       # I8 activation offset % 32
    _case("I8", I8, 2, 64, 8, lda=80),                 # I8 row stride not whole blocks
    _case("F32", Q4, 1, 51232, 8),                     # F32 staging beyond the shared memory at one row
    _case("BF16", I8, 1, 51232, 8),
]


def gemm_operands(c, seed):
    """(a [M, lda] in its dtype, a_scales or None, the f32 / int values of the used slice, wdata, wscales, wq [N_w, K_w] ints)"""
    rng = np.random.default_rng(seed)
    M, K, lda, aoff = c["M"], c["K"], c["lda"], c["aoff"]
    Kw = (c["boff"] + K + 64 + 31) // 32 * 32
    Nw = c["n0"] + c["N"] + 3
    if c["craft"]:
        nib = np.where(rng.random((Nw, Kw)) < 0.5, 0, 15)
        sgn = np.where(rng.random((Nw, Kw // 32)) < 0.5, -1.0, 1.0)
        s = (sgn * 10.0 ** rng.uniform(-30, 30, (Nw, Kw // 32))).astype(F)
    else:
        nib = rng.integers(0, 16, (Nw, Kw))
        s = (rng.uniform(0.5, 2.0, (Nw, Kw // 32)) * np.where(rng.random((Nw, Kw // 32)) < 0.5, -1, 1) / 64).astype(F)
    if c["wd"] == Q4:
        wdata = pack_q4(nib)
        wq = unpack_q4(wdata)
    else:
        wq = rng.integers(-128, 128, (Nw, Kw)).astype(np.int8)
        if c["craft"]:
            wq = np.where(nib == 0, -128, 127).astype(np.int8)
        wdata = wq
    a_scales = None
    if c["act"] == "I8":
        a = rng.integers(-127, 128, (M, lda)).astype(np.int8)
        a_scales = (rng.uniform(0.5, 2.0, (M, lda // 32)) / 128).astype(F)
        if c["craft"]:
            a[0] = 0
            a_scales[0] = 0
        vals = a[:, aoff:aoff + K]
    else:
        x = rng.standard_normal((M, lda)).astype(F)
        if c["craft"]:
            x[0] = 0
        if c["act"] == "BF16":
            a = T.float32_to_bfloat16(x)
            vals = T.bfloat16_to_float32(a)[:, aoff:aoff + K]
        else:
            a = x
            vals = x[:, aoff:aoff + K]
    return a, a_scales, vals, wdata, s, wq


ADT = {"F32": F32, "BF16": BF16, "I8": I8}
SENTINEL = F(-7.25)


def run_gemm(ctx, c, a, a_scales, b_id, ldc):
    r = np.full((c["M"], ldc), SENTINEL, dtype=F)
    rc = ctx.lib.jl_gemm(ctx.h, ADT[c["act"]], ptr(np.ascontiguousarray(a)), ptr(a_scales), c["aoff"], c["lda"], b_id, c["boff"],
                         ptr(r), c["roff"], c["M"], c["n0"], c["N"], c["K"], ldc)
    return rc, r


def register(ctx, wd, wdata, s):
    cols = wdata.shape[1] * (2 if wd == Q4 else 1)
    tid = ctx.lib.jl_register_tensor(ctx.h, wd, wdata.shape[0], cols, ptr(np.ascontiguousarray(wdata)), ptr(np.ascontiguousarray(s)))
    assert tid >= 0
    return tid


WORST = {}


@gpu
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("wd", WDS, ids=["Q4", "Q8_0"])
def test_gemm_against_exact_references(cuda_ctx, act, wd):
    ctx = cuda_ctx
    wname = "Q4" if wd == Q4 else "Q8_0"
    for i, c in enumerate(gemm_cases(act, wd)):
        rule = gemm_rule(c)
        assert rule[0] != "refuse", c
        a, a_scales, vals, wdata, s, wq = gemm_operands(c, zlib.crc32(repr(sorted(c.items())).encode()) + i)
        b_id = register(ctx, wd, wdata, s)
        try:
            c0 = c["n0"] - c["roff"]
            ldc = c0 + c["N"] + 3
            rc, r = run_gemm(ctx, c, a, a_scales, b_id, ldc)
            assert rc == JL_OK, (c, ctx.lib.jl_last_error(ctx.h))
            rows = slice(c["n0"], c["n0"] + c["N"])
            cols = slice(c["boff"], c["boff"] + c["K"])
            wsl, ssl = wq[rows, cols], s[rows, c["boff"] // 32:(c["boff"] + c["K"]) // 32]
            if act == "I8":
                d = a_scales[:, c["aoff"] // 32:(c["aoff"] + c["K"]) // 32]
                ref, nat = int_gemm_ref(vals.astype(np.int32), d, wsl, ssl)
                bar = TAU * nat
            else:
                ref, nat = f32_gemm_ref(vals, wsl, ssl)
                bar = TAU_F * nat
            out = r[:, c0:c0 + c["N"]]
            e = err_bar(out, ref, bar)
            key = "%s x %s" % (act, wname)
            WORST[key] = max(WORST.get(key, 0.0), e)
            label = "%s M%d K%d N%d aoff %d lda %d boff %d n0 %d roff %d%s launches MM %s" % (
                key, c["M"], c["K"], c["N"], c["aoff"], c["lda"], c["boff"], c["n0"], c["roff"], " crafted" if c["craft"] else "", rule)
            print("%s: err/bar %.3f" % (label, e))
            assert e <= 1.0, label
            outside = np.ones(r.shape, dtype=bool)
            outside[:, c0:c0 + c["N"]] = False
            assert np.all(bits(r[outside]) == bits(SENTINEL)), label + ": columns outside the slice written"
            if c["craft"]:
                assert not np.any(out[0]), label + ": zero activation row"
            if c["aoff"] or c["lda"] != c["aoff"] + c["K"]:
                # the same operands packed at column 0 with lda = K: the same bits
                cp = dict(c, aoff=0, lda=c["K"])
                ap = np.ascontiguousarray(a[:, c["aoff"]:c["aoff"] + c["K"]])
                sp = None if a_scales is None else np.ascontiguousarray(a_scales[:, c["aoff"] // 32:(c["aoff"] + c["K"]) // 32])
                rc2, r2 = run_gemm(ctx, cp, ap, sp, b_id, ldc)
                assert rc2 == JL_OK
                assert np.array_equal(bits(r2), bits(r)), label + ": unaligned call differs from the packed copy"
        finally:
            ctx.lib.jl_unregister_tensor(ctx.h, b_id)


@gpu
def test_gemm_refusals_write_nothing(cuda_ctx):
    ctx = cuda_ctx
    for i, c in enumerate(REFUSALS):
        rule = gemm_rule(c)
        assert rule[0] == "refuse", c
        a, a_scales, vals, wdata, s, wq = gemm_operands(c, 900 + i)
        b_id = register(ctx, c["wd"], wdata, s)
        try:
            ldc = c["N"] + 2
            rc, r = run_gemm(ctx, c, a, a_scales, b_id, ldc)
            assert rc == rule[1], (c, rc)
            assert np.all(bits(r) == bits(SENTINEL)), c
        finally:
            ctx.lib.jl_unregister_tensor(ctx.h, b_id)


@gpu
def test_zz_report():
    for k in sorted(WORST):
        print("jl_gemm %-12s worst err/bar %.3f" % (k, WORST[k]))


# ---- accumulate / maccumulate / scale ----------------------------------------------------------------------------------------


def q4_row_values(data, scales, ldb):
    """f32((nibble - 8) * scale) of every element of Q4 rows [rows, ldb]"""
    v = unpack_q4(data).astype(F)
    return (v * np.repeat(scales, 32, axis=1)).astype(F)


def accumulate_ref(a, b_vals, b_rows, offset, length, offset_ignored=False):
    out = a.copy()
    sl = slice(offset, offset + length)
    src = b_vals[:, 0:length] if offset_ignored else b_vals[:, sl]
    out[:, sl] = (a[:, sl] + (src if b_rows > 1 else np.broadcast_to(src[:1], a[:, sl].shape))).astype(F)
    return out


ACC_CASES = [  # (a_rows, b_rows, lda, ldb, offset, length)
    (3, 1, 1024, 1024, 0, 1024),
    (3, 3, 1024, 1056, 7, 1000),
    (2, 2, 300064, 300064, 40, 300000),  # past the 1024 x 256 grid
    (1, 1, 96, 96, 33, 31),
]


@gpu
@pytest.mark.parametrize("bdt", ["F32", "BF16", "Q4"])
def test_accumulate_bit_exact(cuda_ctx, bdt):
    ctx = cuda_ctx
    rng = np.random.default_rng(21)
    for a_rows, b_rows, lda, ldb, off, ln in ACC_CASES:
        a = rng.standard_normal((a_rows, lda)).astype(F)
        if bdt == "F32":
            b = rng.standard_normal((b_rows, ldb)).astype(F)
            bv, scales, dt = b, None, F32
        elif bdt == "BF16":
            b = T.float32_to_bfloat16(rng.standard_normal((b_rows, ldb)))
            bv, scales, dt = T.bfloat16_to_float32(b), None, BF16
        else:
            b = pack_q4(rng.integers(0, 16, (b_rows, ldb)))
            scales = rng.uniform(-2, 2, (b_rows, ldb // 32)).astype(F)
            bv, dt = q4_row_values(b, scales, ldb), Q4
        want = accumulate_ref(a, bv, b_rows, off, ln)
        got = a.copy()
        rc = ctx.lib.jl_accumulate(ctx.h, ptr(got), a_rows, lda, dt, ptr(b), ptr(scales), b_rows, ldb, off, ln)
        assert rc == JL_OK
        assert np.array_equal(bits(got), bits(want)), (bdt, a_rows, b_rows, off, ln)
    # I8 b is refused: the kernel would read it as Q4
    a = np.zeros((1, 64), dtype=F)
    q = np.ones((1, 64), dtype=np.int8)
    s = np.ones((1, 2), dtype=F)
    assert ctx.lib.jl_accumulate(ctx.h, ptr(a), 1, 64, I8, ptr(q), ptr(s), 1, 64, 0, 64) == JL_ERR_UNSUPPORTED
    assert not np.any(a)


@gpu
def test_maccumulate_and_scale_bit_exact(cuda_ctx):
    ctx = cuda_ctx
    rng = np.random.default_rng(22)
    for a_rows, b_rows, lda, ldb, off, ln in ACC_CASES:
        a = rng.standard_normal((a_rows, lda)).astype(F)
        b = rng.standard_normal((b_rows, ldb)).astype(F)
        want = a.copy()
        sl = slice(off, off + ln)
        want[:, sl] = (a[:, sl] * (b[:, sl] if b_rows > 1 else b[:1, sl])).astype(F)
        got = a.copy()
        assert ctx.lib.jl_maccumulate(ctx.h, ptr(got), a_rows, lda, ptr(b), b_rows, ldb, off, ln) == JL_OK
        assert np.array_equal(bits(got), bits(want)), ("maccumulate", a_rows, b_rows, off, ln)
        f = F(-1.0 / 3.0)
        want = a.copy()
        want[:, sl] = (a[:, sl] * f).astype(F)
        got = a.copy()
        assert ctx.lib.jl_scale(ctx.h, C.c_float(f), ptr(got), a_rows, lda, off, ln) == JL_OK
        assert np.array_equal(bits(got), bits(want)), ("scale", a_rows, off, ln)


# ---- saxpy ---------------------------------------------------------------------------------------------------------------


def saxpy_ref(alpha, x, y, xoff, yoff, limit, aoff, xrow, batch, fused=True):
    out = y.copy()
    acc = y[yoff:yoff + limit].copy()
    for r in range(batch):
        xv, al = x[xrow + r, xoff:xoff + limit], alpha[aoff + r]
        acc = fma_f32(xv, al, acc) if fused else (acc + (xv * al).astype(F)).astype(F)
    out[yoff:yoff + limit] = acc
    return out


@gpu
def test_saxpy_bit_exact(cuda_ctx):
    ctx = cuda_ctx
    rng = np.random.default_rng(23)
    for batch in range(1, 10):
        for limit, xoff, yoff, aoff, xrow in ((1001, 3, 5, 2, 1), (64, 0, 0, 0, 0), (257, 17, 1, 4, 3)):
            ldx = xoff + limit + 7
            x = rng.standard_normal((xrow + batch + 1, ldx)).astype(F)
            alpha = rng.standard_normal(aoff + batch + 2).astype(F)
            y = rng.standard_normal(yoff + limit + 4).astype(F)
            want = saxpy_ref(alpha, x, y, xoff, yoff, limit, aoff, xrow, batch)
            got = y.copy()
            rc = ctx.lib.jl_saxpy_batch(ctx.h, ptr(alpha), ptr(x), ldx, ptr(got), xoff, yoff, limit, aoff, xrow, batch)
            assert rc == JL_OK
            assert np.array_equal(bits(got), bits(want)), (batch, limit, xoff, yoff, aoff, xrow)
    # the scalar form: one fused row
    x = rng.standard_normal(40).astype(F)
    y = rng.standard_normal(50).astype(F)
    al = F(0.3)
    want = y.copy()
    want[9:9 + 31] = fma_f32(x[5:36], al, y[9:40])
    got = y.copy()
    assert ctx.lib.jl_saxpy(ctx.h, C.c_float(al), ptr(x), ptr(got), 5, 9, 31) == JL_OK
    assert np.array_equal(bits(got), bits(want))


# ---- quantisers -----------------------------------------------------------------------------------------------------------


def q8_act_ref(x, offset, length, ldx):
    """the Q8 activation quantiser as the kernel computes it: fmaxf maximum (a NaN element does not enter it), d = f32(mx / 127),
    id = f32(127 / mx) (0 at mx == 0), q = (int8)(int)f32(f32(x * id) + 0.5) with (int) saturating and NaN -> 0"""
    rows = x.shape[0]
    q = np.zeros((rows, ldx), dtype=np.int8)
    s = np.zeros((rows, ldx // 32), dtype=F)
    b = x[:, offset:offset + length].reshape(rows, length // 32, 32)
    ab = np.abs(b)
    allnan = np.isnan(ab).all(axis=2)
    mx = np.where(allnan, F(np.nan), np.nanmax(np.where(np.isnan(ab), F(-1), ab), axis=2)).astype(F)
    with np.errstate(all="ignore"):
        d = (mx / F(127)).astype(F)
        idv = np.where(mx != 0, F(127) / mx, F(0)).astype(F)
        f = ((b * idv[..., None]).astype(F) + F(0.5)).astype(F)
        t = np.where(np.isnan(f), 0.0, np.clip(np.trunc(f.astype(f64)), -2147483648.0, 2147483647.0)).astype(np.int64)
    q[:, offset:offset + length] = ((t + 128) % 256 - 128).reshape(rows, length).astype(np.int8)
    s[:, offset // 32:(offset + length) // 32] = d
    return q, s


def q8_act_rows():
    """crafted rows of 32-element blocks"""
    blocks = []
    z = np.zeros(32, dtype=F)
    blocks.append(z)                                    # all zero
    one = z.copy()
    one[17] = -3.5
    blocks.append(one)                                  # a single non-zero
    tie = np.array([127, 2.5, -2.5, 0.5, -0.5, 1.5, -1.5, 126.5, -126.5] + [0] * 23, dtype=F)
    blocks.append(tie)                                  # id = 1: exact x * id + 0.5 ties on both signs
    blocks.append((np.arange(32, dtype=F) - 16) * F(1e-44))  # subnormal block: id overflows to inf
    blocks.append(np.linspace(-1e-37, 1e-37, 32).astype(F))
    inf = np.linspace(-1, 1, 32).astype(F)
    inf[3] = np.inf
    blocks.append(inf)
    ninf = inf.copy()
    ninf[3] = -np.inf
    blocks.append(ninf)
    nan = np.linspace(-1, 1, 32).astype(F)
    nan[5] = np.nan
    blocks.append(nan)                                  # a NaN element
    blocks.append(np.full(32, np.nan, dtype=F))         # all NaN
    rng = np.random.default_rng(31)
    blocks.append((rng.standard_normal(32) * 1e30).astype(F))
    return np.concatenate(blocks)


@gpu
def test_quantize_q8_activations_bit_exact(cuda_ctx):
    ctx = cuda_ctx
    crafted = q8_act_rows()
    nb = crafted.size // 32
    ldx = crafted.size + 64
    x = np.zeros((2, ldx), dtype=F)
    x[0, 32:32 + crafted.size] = crafted
    x[1, 32:32 + crafted.size] = crafted[::-1]
    cases = [(x, 32, crafted.size)]
    rng = np.random.default_rng(32)
    big = (rng.standard_normal((4, 81920 + 64)) * 3).astype(F)  # 10240 blocks: past sm_count * 8 CTAs of 8 warps
    cases.append((big, 64, 81920))
    for xx, off, ln in cases:
        rows, ld = xx.shape
        q = np.full((rows, ld), 99, dtype=np.int8)
        s = np.full((rows, ld // 32), 99, dtype=F)
        assert ctx.lib.jl_quantize_q8(ctx.h, ptr(xx), rows, ld, off, ln, ptr(q), ptr(s)) == JL_OK
        qr, sr = q8_act_ref(xx, off, ln, ld)
        assert np.array_equal(q, qr), np.argwhere(q != qr)[:8]
        assert np.all(same_bits(s, sr)), np.argwhere(~same_bits(s, sr))[:8]
    assert rows * ln // 32 > cuda_ctx.sm_count * 8 * 8
    # finite blocks: equal to the host mirror of the reference quantiser
    fin = np.nan_to_num(x, nan=0.0, posinf=0.0, neginf=0.0)  # the host mirror keeps the reference's NaN-propagating maximum
    qh, sh = T.quantize_q8_activations(fin, 32, crafted.size)
    qr, sr = q8_act_ref(fin, 32, crafted.size, ldx)
    assert np.array_equal(qh, qr) and np.array_equal(bits(sh), bits(sr))
    print("Q8 activations: %d crafted blocks and %d blocks past the grid, bit-exact" % (nb, 4 * 81920 // 32))


def bf16_edge_values():
    v = []
    for m in (0x00000, 0x10000):  # even and odd bf16 mantissa below
        v += [0x3F800000 | m | 0x8000, 0xBF800000 | m | 0x8000, 0x3F800000 | m | 0x8001, 0x3F800000 | m | 0x7FFF]  # ties and neighbours
    v += [0x7FC00000, 0x7F800001, 0xFFC12345, 0x7FFFFFFF, 0xFF800000, 0x7F800000]  # NaN payloads, +-inf
    v += [0x7F7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0xFF7FFFFF]  # values rounding up to inf, a tie that does
    v += [0x00000001, 0x00008000, 0x00018000, 0x007FFFFF, 0x80008001, 0x00000000, 0x80000000]  # subnormals and zeros
    return np.array(v, dtype=np.uint32).view(F)


@gpu
def test_quantize_bf16_bit_exact(cuda_ctx):
    ctx = cuda_ctx
    edges = bf16_edge_values()
    rng = np.random.default_rng(33)
    ld = 300000 + 40
    x = rng.standard_normal((2, ld)).astype(F)
    x[:, 40:40 + edges.size] = edges
    off, ln = 40, 300000  # past the 1024 x 256 grid
    out = np.full((2, ld), 0xABCD, dtype=np.uint16)
    assert ctx.lib.jl_quantize_bf16(ctx.h, ptr(x), 2, ld, off, ln, ptr(out)) == JL_OK
    want = np.zeros((2, ld), dtype=np.uint16)
    want[:, off:off + ln] = T.float32_to_bfloat16(x[:, off:off + ln])
    assert np.array_equal(out, want), np.argwhere(out != want)[:8]


def weight_edge_rows(cols):
    """rows of 32-blocks: +-max ties (the first index keeps its sign), all-zero blocks, nibble boundaries, subnormal blocks"""
    rng = np.random.default_rng(34)
    x = (rng.standard_normal((8, cols)) * 2).astype(F)
    b = x.reshape(8, cols // 32, 32)
    b[0, 0] = 0                                        # all zero: the Float.MIN_VALUE path
    b[0, 1, :] = 0
    b[0, 1, 4], b[0, 1, 9] = -3.0, 3.0                 # +-max tie, negative first
    b[0, 2, :] = 0
    b[0, 2, 4], b[0, 2, 9] = 3.0, -3.0                 # +-max tie, positive first
    b[1, 0] = np.linspace(-8, 8, 32).astype(F)          # nibble boundaries and the clamp at 15
    b[1, 1] = (np.arange(32, dtype=F) - 16) * F(0.5)
    b[1, 2] = np.linspace(-1, 1, 32).astype(F) * F(8.0 / 7.5)
    b[2, 0] = (np.arange(32, dtype=F) - 16) * F(1e-44)  # subnormal: the inverse scale overflows, (int) saturates, (byte) wraps
    b[2, 1] = np.linspace(-3e-39, 3e-39, 32).astype(F)
    b[2, 2] = F(1.4e-45)
    return x


@gpu
@pytest.mark.parametrize("kind", ["Q4", "Q8_0"])
def test_quantize_weights_bit_exact(cuda_ctx, kind):
    ctx = cuda_ctx
    for rows, cols in ((8, 128), (40, 16384)):  # 40 x 512 blocks: past sm_count * 16 CTAs of 8 warps
        x = weight_edge_rows(cols) if rows == 8 else np.random.default_rng(35).uniform(-5, 5, (rows, cols)).astype(F)
        s = np.zeros((rows, cols // 32), dtype=F)
        if kind == "Q4":
            q = np.zeros((rows, cols // 2), dtype=np.uint8)
            assert ctx.lib.jl_quantize_q4_weights(ctx.h, ptr(x), rows, cols, ptr(q), ptr(s)) == JL_OK
            qr, sr = T.quantize_q4(x)
        else:
            q = np.zeros((rows, cols), dtype=np.int8)
            assert ctx.lib.jl_quantize_q8_weights(ctx.h, ptr(x), rows, cols, ptr(q), ptr(s)) == JL_OK
            qr, sr = T.quantize_q8_weights(x)
        assert np.array_equal(q, qr), (kind, rows, np.argwhere(q != qr)[:8])
        assert np.all(same_bits(s, sr)), (kind, rows)
    assert 40 * 16384 // 32 > cuda_ctx.sm_count * 16 * 8


# ---- rmsnorm / layernorm ----------------------------------------------------------------------------------------------------


def rms_ref(x, w, adj, eps, E, offset, length, div=None):
    """(out for rsf, out for rsf - 1 ulp, out for rsf + 1 ulp); div: the divisor (E; the defect divides by length)"""
    sl = slice(offset, offset + length)
    with np.errstate(over="ignore", invalid="ignore"):
        ss = (x[:, sl] * x[:, sl]).astype(f64).sum(axis=1)
        rsf = (1.0 / np.sqrt(ss / (E if div is None else div) + f64(F(eps)))).astype(F)
        outs = []
        for r in (rsf, np.nextafter(rsf, F(0)), np.nextafter(rsf, F(np.inf))):
            o = np.zeros_like(x)
            o[:, sl] = ((F(adj) + w[sl])[None, :] * (r[:, None] * x[:, sl]).astype(F)).astype(F)
            outs.append(o)
    return outs


def rows_match_one(out, cands):
    ok = np.zeros(out.shape[0], dtype=bool)
    for c in cands:
        ok |= np.all(same_bits(out, c), axis=1)
    return ok


@gpu
@pytest.mark.parametrize("wdt", ["F32", "BF16"])
def test_rmsnorm_window_rule(cuda_ctx, wdt):
    ctx = cuda_ctx
    rng = np.random.default_rng(41)
    for E, ldx, off, ln, adj in ((4096, 4096, 0, 4096, 0.0), (4096, 4096, 0, 4096, 1.0), (1000, 1040, 24, 600, 1.0), (256, 300, 3, 250, 0.0)):
        x = (rng.standard_normal((5, ldx)) * 3).astype(F)
        x[1] = 0                                          # zero row
        x[2, off:off + 4] = F(3e19)                       # squares overflow: rsf = 0
        wf = rng.uniform(-2, 2, off + ln).astype(F)
        if wdt == "BF16":
            wraw = T.float32_to_bfloat16(wf)
            wv, dt = T.bfloat16_to_float32(wraw), BF16
        else:
            wraw, wv, dt = wf, wf, F32
        out = np.full_like(x, 5.0)
        rc = ctx.lib.jl_rmsnorm(ctx.h, ptr(x), x.shape[0], ldx, dt, ptr(wraw), C.c_float(adj), C.c_float(1e-5), E, off, ln, ptr(out))
        assert rc == JL_OK
        cands = rms_ref(x, wv, adj, 1e-5, E, off, ln)
        ok = rows_match_one(out, cands)
        assert ok.all(), (wdt, E, off, ln, adj, np.nonzero(~ok)[0])


def ln_ref_cands(x, w, b, eps, E, offset, length):
    """the candidate outputs of each row: sum and sumSq each rounded from s - t, s, s + t"""
    sl = slice(offset, offset + length)
    xs = x[:, sl].astype(f64)
    sq = (x[:, sl] * x[:, sl]).astype(F).astype(f64)
    s, ss = xs.sum(axis=1), sq.sum(axis=1)
    ts = length * 2.0 ** -52 * np.abs(xs).sum(axis=1)
    tss = length * 2.0 ** -52 * sq.sum(axis=1)
    outs = []
    for s32 in ((s - ts).astype(F), s.astype(F), (s + ts).astype(F)):
        for ss32 in ((ss - tss).astype(F), ss.astype(F), (ss + tss).astype(F)):
            mean = (s32 / F(E)).astype(F)
            var = ((ss32 / F(E)).astype(F) - (mean * mean).astype(F)).astype(F)
            inv = (F(1) / np.sqrt((var + F(eps)).astype(F).astype(f64)).astype(F)).astype(F)
            o = np.zeros_like(x)
            o[:, sl] = ((((x[:, sl] - mean[:, None]).astype(F) * inv[:, None]).astype(F) * w[None, sl]).astype(F) + b[None, sl]).astype(F)
            outs.append(o)
    return outs


@gpu
def test_layernorm_two_candidate_rule(cuda_ctx):
    ctx = cuda_ctx
    rng = np.random.default_rng(42)
    for E, ldx, off, ln in ((768, 768, 0, 768), (768, 800, 16, 700)):
        x = rng.standard_normal((4, ldx)).astype(F)
        x[1] = F(0.1)                                     # constant rows: the variance is the rounding of E[x^2] - mean^2
        x[2] = F(-3.0)
        w = rng.uniform(-2, 2, off + ln).astype(F)
        b = rng.uniform(-1, 1, off + ln).astype(F)
        out = np.full_like(x, 5.0)
        rc = ctx.lib.jl_layernorm(ctx.h, ptr(x), 4, ldx, F32, ptr(w), F32, ptr(b), C.c_float(1e-5), E, off, ln, ptr(out))
        assert rc == JL_OK
        cands = ln_ref_cands(x, w, b, 1e-5, E, off, ln)
        inside = out[:, off:off + ln]
        ok = rows_match_one(inside, [c[:, off:off + ln] for c in cands])
        assert ok.all(), (E, off, ln, np.nonzero(~ok)[0])
        assert np.all(out[:, :off] == 5.0) and np.all(out[:, off + ln:] == 5.0)


# ---- activation / silu_mul ----------------------------------------------------------------------------------------------------


def act_ref(kind, v):
    """(y, t): the kernel's double expression and its rounding allowance"""
    v = np.asarray(v, dtype=F).astype(f64)
    with np.errstate(all="ignore"):
        if kind == 0:
            y = v * (1.0 / (1.0 + np.exp(-v)))
            t = np.abs(y) * 2.0 ** -48
        elif kind == 1:
            z = np.sqrt(2.0 / 3.14159265358979323846) * (v + 0.044715 * np.power(v, 3.0))
            y = 0.5 * v * (1.0 + np.tanh(z))
            t = np.abs(y) * 2.0 ** -48 + np.abs(0.5 * v) * 2.0 ** -50  # 1 + tanh(z) cancels for large negative v
        else:
            y = np.tanh(v)
            t = np.abs(y) * 2.0 ** -48
    t = np.where(np.isfinite(t), t, 0.0)
    return y, t


def act_inputs():
    rng = np.random.default_rng(51)
    v = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-45, -1e-45, 3.4e38, -3.4e38, 1e13, -1e13, 1e30, -1e30]
    v += list(np.linspace(-104, -88, 97))           # SiLU into the subnormals
    v += list(np.linspace(-12, 12, 481))
    v += list(rng.standard_normal(400) * 4)
    return np.array(v, dtype=F)


@gpu
@pytest.mark.parametrize("kind", [0, 1, 2], ids=["silu", "gelu", "tanh"])
def test_activation_rounding_rule(cuda_ctx, kind):
    ctx = cuda_ctx
    v = act_inputs()
    n = v.size
    ld, off = n + 9, 4
    x = np.full((3, ld), 7.5, dtype=F)
    for r in range(3):
        x[r, off:off + n] = np.roll(v, 37 * r)
    got = x.copy()
    assert ctx.lib.jl_activation(ctx.h, kind, ptr(got), 3, ld, off, n) == JL_OK
    y, t = act_ref(kind, x[:, off:off + n])
    ok = interval_ok(got[:, off:off + n], y, t)
    assert ok.all(), [(float(a), float(b)) for a, b in zip(x[:, off:off + n][~ok][:6], got[:, off:off + n][~ok][:6])]
    assert np.all(got[:, :off] == 7.5) and np.all(got[:, off + n:] == 7.5)
    # the grid-stride wrap: rows * length past sm_count * 8 CTAs of 256 threads
    rows, ln = 3, 100003
    big = np.random.default_rng(52).standard_normal((rows, ln + 2)).astype(F) * 6
    got = big.copy()
    assert ctx.lib.jl_activation(ctx.h, kind, ptr(got), rows, ln + 2, 1, ln) == JL_OK
    assert rows * ln > cuda_ctx.sm_count * 8 * 256
    y, t = act_ref(kind, big[:, 1:1 + ln])
    assert interval_ok(got[:, 1:1 + ln], y, t).all()
    assert np.array_equal(bits(got[:, 0]), bits(big[:, 0])) and np.array_equal(bits(got[:, -1]), bits(big[:, -1]))


@gpu
def test_silu_mul_rounding_rule(cuda_ctx):
    ctx = cuda_ctx
    v = act_inputs()
    n, ld, off = v.size, v.size + 5, 2
    g = np.full((2, ld), 3.0, dtype=F)
    g[0, off:off + n], g[1, off:off + n] = v, v[::-1]
    u = np.random.default_rng(53).standard_normal((2, ld)).astype(F)
    got = g.copy()
    assert ctx.lib.jl_silu_mul(ctx.h, ptr(got), ptr(u), 2, ld, off, n) == JL_OK
    y, t = act_ref(0, g[:, off:off + n])
    with np.errstate(invalid="ignore", over="ignore"):
        lo, hi = (y - t).astype(F), (y + t).astype(F)
        uu = u[:, off:off + n]
        p1, p2 = (lo * uu).astype(F), (hi * uu).astype(F)
        o = got[:, off:off + n]
        ok = ((o >= np.minimum(p1, p2)) & (o <= np.maximum(p1, p2)) & (t > 0)) | same_bits(o, (y.astype(F) * uu).astype(F))
    assert ok.all(), np.argwhere(~ok)[:6]
    assert np.all(got[:, :off] == 3.0) and np.all(got[:, off + n:] == 3.0)


# ---- softmax ---------------------------------------------------------------------------------------------------------------------


def butterfly(v):
    """warp_sum over the last axis (32 lanes): lane l += lane l ^ o for o = 16 .. 1; every lane ends with lane 0's value"""
    v = v.astype(F).copy()
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., idx ^ o]).astype(F)
    return v[..., 0]


def block_sum(e, threads, sequential=False):
    """the kernels' float sum of e: `threads` threads striding, the warp butterfly, the warp sums in sequence from 0"""
    if sequential:
        return np.cumsum(e.astype(F), dtype=F)[-1] if e.size else F(0)
    n = e.size
    pad = -(-n // threads) * threads
    ee = np.zeros(pad, dtype=F)
    ee[:n] = e
    per = np.zeros(threads, dtype=F)
    for j in range(pad // threads):
        per = (per + ee[j * threads:(j + 1) * threads]).astype(F)
    w = butterfly(per.reshape(threads // 32, 32))
    t = F(0)
    for s in w:
        t = F(t + s)
    return t


def exp_f32(y64):
    """(f32(exp(y)), alternative rounding where exp(y) is within a few double ulps of a float midpoint)"""
    with np.errstate(all="ignore"):
        e = np.exp(y64)
        tol = e * 2.0 ** -48
        lo, hi = (e - tol).astype(F), (e + tol).astype(F)
    main = e.astype(F)
    alt = np.where(lo != main, lo, hi).astype(F)
    return main, alt


def softmax_ref(x, offset, length, sequential=False, from_offset=False):
    """(candidate outputs [2, n], e ambiguity count): the kernel's arithmetic in its order"""
    x = np.asarray(x, dtype=F)
    sl = slice(offset, offset + length)
    mx = x[sl].max()
    main, alt = exp_f32((x[sl] - mx).astype(F).astype(f64))
    outs = []
    for e in (main, alt):
        s = block_sum(e, 1024, sequential)
        o = x.copy()
        o[sl] = e
        start = offset if from_offset else 0
        o[start:offset + length] = (o[start:offset + length] / s).astype(F)
        outs.append(o)
    return outs, int((main != alt).sum())


def softmax_rows():
    rng = np.random.default_rng(61)
    rows = []
    for n in (1, 31, 1024, 1025, 3000, 128256):
        rows.append((0, (rng.standard_normal(n) * 4).astype(F)))
    r = (rng.standard_normal(3000) * 2).astype(F)
    r[::7] = -np.inf
    rows.append((0, r))                                       # -inf entries
    rows.append((0, np.full(1025, 2.5, dtype=F)))             # all equal
    d = np.zeros(2000, dtype=F)
    d[1234] = 90.0
    rows.append((0, d))                                       # one dominant entry
    for off in (1, 37, 1024):
        rows.append((off, np.concatenate([(rng.standard_normal(off) * 5).astype(F), (rng.standard_normal(1500) * 3).astype(F)])))
    return rows


@gpu
def test_softmax_bit_exact_in_kernel_order(cuda_ctx):
    ctx = cuda_ctx
    worst = 0.0
    for off, row in softmax_rows():
        ln = row.size - off
        got = row.copy()
        assert ctx.lib.jl_softmax(ctx.h, ptr(got), off, ln) == JL_OK
        cands, amb = softmax_ref(row, off, ln)
        ok = same_bits(got, cands[0]) | same_bits(got, cands[1])
        assert ok.all(), (off, ln, np.nonzero(~ok)[0][:8], amb)
        seq, _ = softmax_ref(row, off, ln, sequential=True)
        fin = np.isfinite(seq[0]) & (seq[0] != 0)
        rel = np.abs(got[fin].astype(f64) - seq[0][fin]) / np.abs(seq[0][fin].astype(f64))
        bound = (ln + 64) * 2.0 ** -23
        r = float(rel.max() / bound) if rel.size else 0.0
        worst = max(worst, r)
        assert r <= 1.0, (off, ln, r)
        print("softmax offset %d length %d: exact (ambiguous e %d), distance to the sequential sum %.3f of its bound" % (off, ln, amb, r))
    print("softmax: worst distance to the sequential sum %.3f of the bound" % worst)


# ---- the temperature draw --------------------------------------------------------------------------------------------------------


def draw_ref(logits, temp, u, off_by_one=False, sequential=False, e_override=None):
    """softmax_sample_kernel restated: e_i = f32(exp((f64 l_i - f64 m) / f64 T)), t = the 256-thread sum, acc += f32(e_i / t) in
    index order, the first i with acc >= u, else vocab - 1"""
    l = np.asarray(logits, dtype=F)
    mx = l.max()
    if e_override is None:
        with np.errstate(all="ignore"):
            e = np.exp((l.astype(f64) - f64(mx)) / f64(F(temp))).astype(F)
    else:
        e = e_override
    t = block_sum(e, 256, sequential)
    acc = np.cumsum((e / t).astype(F), dtype=F)
    hit = np.nonzero(acc >= F(u))[0]
    if hit.size == 0:
        return len(l) - 1, acc
    i = int(hit[0])
    return (i + 1 if off_by_one and i + 1 < len(l) else i), acc


def draw_candidates(logits, temp, u):
    """the restated token, and the token with the exponentials that sit at a float midpoint rounded the other way"""
    l = np.asarray(logits, dtype=F)
    with np.errstate(all="ignore"):
        main, alt = exp_f32((l.astype(f64) - f64(l.max())) / f64(F(temp)))
    a, acc = draw_ref(l, temp, u, e_override=main)
    if (main == alt).all():
        return {a}, acc
    return {a, draw_ref(l, temp, u, e_override=alt)[0]}, acc


def draw_rows(V, rng):
    rows = [(rng.standard_normal(V) * 3).astype(F)]
    r = (rng.standard_normal(V) * 2).astype(F)
    r[rng.random(V) < 0.3] = -np.inf
    r[V // 2] = r[np.isfinite(r)].max()                      # a tie of the maximum
    r[0] = r[V // 2]
    rows.append(r)
    single = np.full(V, -np.inf, dtype=F)
    single[(V * 2) // 3] = 1.5
    rows.append(single)                                      # one finite entry
    return rows


TEMPS = (1e-3, 0.05, 0.7, 1.0, 3.0, 100.0)
VOCABS = (8, 255, 256, 257, 32000, 128256)


def draw_uniforms(acc, rng):
    us = [F(0), F(1), np.nextafter(F(1), F(0)), F(rng.random())]
    steps = np.nonzero(np.diff(np.concatenate([[F(0)], acc])) > 0)[0]
    for j in list(steps[:2]) + list(steps[-2:]) + list(rng.choice(steps, min(2, steps.size), replace=False)):
        a = acc[j]
        us += [a, np.nextafter(a, F(0)), np.nextafter(a, F(1))]
    return [F(min(max(x, F(0)), F(1))) for x in us]


def select_host(ctx, rows, temps, us):
    rows = np.ascontiguousarray(rows, dtype=F)
    n, V = rows.shape
    t = np.ascontiguousarray(temps, dtype=F)
    u = np.ascontiguousarray(us, dtype=F)
    out = np.full(n, -5, dtype=np.int32)
    rc = ctx.lib.jl_select_constrained(ctx.h, n, V, ptr(rows), V, ptr(t), None, None, ptr(u), None, 0, None, None, ptr(out))
    return rc, out


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_temperature_draw_exact(cuda_ctx, oracle, V):
    ctx = cuda_ctx
    rng = np.random.default_rng(V + 7)
    rows, temps, us, want = [], [], [], []
    for row in draw_rows(V, rng):
        for temp in TEMPS:
            _, acc = draw_ref(row, temp, 0.5)
            for u in draw_uniforms(acc, rng):
                cand, _ = draw_candidates(row, temp, u)
                rows.append(row), temps.append(temp), us.append(u), want.append(cand)
    rc, out = select_host(ctx, np.stack(rows), temps, us)
    assert rc == JL_OK
    bad = [(i, temps[i], float(us[i]), int(out[i]), sorted(want[i])) for i in range(len(rows)) if int(out[i]) not in want[i]]
    assert not bad, bad[:6]
    amb = sum(len(w) > 1 for w in want)
    # against the reference's sequential sums: equal unless u sits within the bound of a float64 CDF step between the two tokens
    near, bound = 0, (V + 64) * 2.0 ** -23
    for i in range(len(rows)):
        o = oracle.sample_temperature(rows[i], temps[i], us[i])
        if o == int(out[i]):
            continue
        l = rows[i].astype(f64)
        with np.errstate(all="ignore"):
            e = np.exp((l - l.max()) / f64(F(temps[i])))
        cdf = np.cumsum(e) / e.sum()
        lo, hi = sorted((o, int(out[i])))
        gap = np.abs(cdf[max(lo - 1, 0):hi + 1] - f64(us[i])).min()
        assert gap <= bound, (V, temps[i], float(us[i]), o, int(out[i]), gap)
        near += 1
    print("temperature draw V=%d: %d rows exact (%d with a midpoint exponential); %d differ from the sequential reference, all "
          "within %.1e of a CDF step" % (V, len(rows), amb, near, bound))


@gpu
@pytest.mark.parametrize("n", [1, 3])
def test_decode_sample_picks_the_restated_token(cuda_ctx, n):
    from jlama_b200 import synth
    from jlama_b200.model import LlamaModel
    cfg = synth.get_config("tiny")
    m = LlamaModel(cuda_ctx, cfg, synth.make_weights(cfg), max_sessions=4, max_context=64)
    try:
        if n == 1:
            assert m.decode_mode(1) == 3
        rng = np.random.default_rng(70 + n)
        sess = np.arange(n, dtype=np.int32)
        toks = rng.integers(0, cfg["vocab"], n).astype(np.int32)
        temps = np.array([0.7, 1.0, 3.0][:n], dtype=F)
        us = rng.random(n).astype(F)
        nxt, lg = m.decode(toks, np.zeros(n, dtype=np.int32), sessions=sess, want_logits=True, temperatures=temps, uniforms=us)
        for i in range(n):
            cand, _ = draw_candidates(lg[i], temps[i], us[i])
            assert int(nxt[i]) in cand, (n, i, int(nxt[i]), cand)
    finally:
        m.close()


# ---- the case matrix and the sharpness of the bars (CPU) ------------------------------------------------------------------------


def test_case_matrix_reaches_every_variant():
    seen = set()
    for act in ACTS:
        staging = "Q8" if act == "I8" else "F32"
        for wd in WDS:
            for c in gemm_cases(act, wd):
                mms = gemm_rule(c)
                assert mms[0] != "refuse", c
                for mm in mms:
                    seen.add((act, wd, "MM", mm))
                if len(mms) > 1:
                    seen.add((act, wd, "chunk loop"))
                if c["K"] == 6400 and act != "I8":
                    assert gemv_max_m(act, 6400) == 8 and 8 * 6400 * 4 == SMEM_GEMV
                    seen.add((act, wd, "MM 8 at 200 KiB"))
                if c["K"] == 51200 and act != "I8":
                    assert gemv_max_m(act, 51200) == 1
                    seen.add((act, wd, "MM 1 at 200 KiB"))
                nblk = c["K"] // 32
                seen.add((act, wd, "chunks", min(-(-nblk // 128), 2), nblk % 128 == 0))
                if c["aoff"] % 4 or (c["lda"] % 4 and c["M"] > 1):
                    seen.add((staging, wd, "unaligned"))
            seen.add((staging, "refusal", "none"))
    missing = []
    for act in ACTS:
        for wd in WDS:
            missing += [x for x in [(act, wd, "MM", mm) for mm in (1, 2, 4, 8)] + [(act, wd, "chunk loop")] if x not in seen]
            missing += [x for x in [(act, wd, "chunks", 1, True), (act, wd, "chunks", 1, False), (act, wd, "chunks", 2, False),
                                    (act, wd, "chunks", 2, True)] if x not in seen]
            if act != "I8":
                missing += [x for x in [(act, wd, "MM 8 at 200 KiB"), (act, wd, "MM 1 at 200 KiB"), ("F32", wd, "unaligned")] if x not in seen]
    assert not missing, missing
    codes = [gemm_rule(c) for c in REFUSALS]
    assert all(r[0] == "refuse" for r in codes)
    assert sorted({r[1] for r in codes}) == sorted({JL_ERR_INVALID, JL_ERR_UNSUPPORTED})
    assert gemv_max_m("F32", 51232) == 0 and gemv_max_m("I8", 51232) >= 1
    # the grid-stride wraps the GPU tests reach (they assert these for the card they run on as well)
    assert 2 * 300000 > 0 and 300000 > 1024 * 256                  # accumulate / maccumulate / scale / bf16
    assert 4 * 81920 // 32 > H100_SMS * 8 * 8                      # quantize_q8
    assert 40 * 16384 // 32 > H100_SMS * 16 * 8                    # quantize_q4 / q8 weights
    assert 3 * 100003 > H100_SMS * 8 * 256                         # activation


def test_fma_restatement_is_exact():
    """fma_f32 against exact rational arithmetic, near-midpoint sums included"""
    rng = np.random.default_rng(81)
    a = rng.standard_normal(3000).astype(F)
    b = rng.standard_normal(3000).astype(F)
    c = (-(a.astype(f64) * b.astype(f64))).astype(F)  # heavy cancellation
    c[::2] = rng.standard_normal(1500).astype(F)
    c[1::4] = (c[1::4] + np.ldexp(F(1), -30)).astype(F)
    got = fma_f32(a, b, c)
    for i in range(0, 3000, 7):
        ex = fractions.Fraction(float(a[i])) * fractions.Fraction(float(b[i])) + fractions.Fraction(float(c[i]))
        f = F(float(ex))
        cands = [np.nextafter(f, F(-np.inf)), f, np.nextafter(f, F(np.inf))]
        dist = [abs(fractions.Fraction(float(x)) - ex) for x in cands]
        best = min(dist)
        ok = [x for x, dd in zip(cands, dist) if dd == best]
        want = ok[0] if len(ok) == 1 else [x for x in ok if not (bits(x) & 1)][0]
        assert bits(got[i]) == bits(want), (i, a[i], b[i], c[i])


def _ratio(out, ref, bar, what):
    r = err_bar(out, ref, bar)
    print("%s: err/bar %.1f" % (what, r))
    assert r >= SHARP, (what, r)


def test_bar_rejects_a_dropped_k_element():
    for act in ("F32", "I8"):
        for K in (4096, 14336, 51200):
            c = _case(act, Q4, 2, K, 17)
            a, a_scales, vals, wdata, s, wq = gemm_operands(c, 5)
            w, sl = wq[:17, :K], s[:17, :K // 32]
            v2 = vals.copy()
            v2[:, K - 1] = 0  # the last element of the row never loaded
            if act == "I8":
                ref, nat = int_gemm_ref(vals.astype(np.int32), a_scales[:, :K // 32], w, sl)
                bad, _ = int_gemm_ref(v2.astype(np.int32), a_scales[:, :K // 32], w, sl)
                _ratio(bad, ref, TAU * nat, "%s K %d: last K element dropped" % (act, K))
            else:
                ref, nat = f32_gemm_ref(vals, w, sl)
                bad, _ = f32_gemm_ref(v2, w, sl)
                _ratio(bad, ref, TAU_F * nat, "%s K %d: last K element dropped" % (act, K))


def test_bar_accepts_f32_accumulation():
    """the kernel's own order (f32 fma chains per block, per-lane block sums, the butterfly) stays well within the F32 bar"""
    c = _case("F32", Q4, 2, 14336, 8)
    a, _, vals, wdata, s, wq = gemm_operands(c, 6)
    w, sl = wq[:8, :14336], s[:8, :448]
    ref, nat = f32_gemm_ref(vals, w, sl)
    nb = 448
    part = np.zeros((2, 8, nb), dtype=F)
    A, W = vals.reshape(2, nb, 32), w.reshape(8, nb, 32).astype(F)
    for k in range(32):
        part = fma_f32(A[:, None, :, k], W[None, :, :, k], part)
    lanes = np.zeros((2, 8, 32), dtype=F)
    for bi in range(nb):
        lanes[:, :, bi % 32] = fma_f32(sl[None, :, bi], part[:, :, bi], lanes[:, :, bi % 32])
    out = butterfly(lanes)
    assert err_bar(out, ref, TAU_F * nat) <= 0.25


def test_exact_checks_reject_their_defects():
    rng = np.random.default_rng(91)
    # accumulate: the offset ignored in the Q4 path
    b = pack_q4(rng.integers(0, 16, (1, 1056)))
    sc = rng.uniform(-2, 2, (1, 33)).astype(F)
    bv = q4_row_values(b, sc, 1056)
    a = rng.standard_normal((2, 1056)).astype(F)
    good, bad = accumulate_ref(a, bv, 1, 7, 1000), accumulate_ref(a, bv, 1, 7, 1000, offset_ignored=True)
    assert (~same_bits(good, bad)).sum() > 100
    # saxpy unfused
    x = rng.standard_normal((5, 300)).astype(F)
    al = rng.standard_normal(5).astype(F)
    y = rng.standard_normal(300).astype(F)
    n_unfused = (~same_bits(saxpy_ref(al, x, y, 0, 0, 300, 0, 0, 5), saxpy_ref(al, x, y, 0, 0, 300, 0, 0, 5, fused=False))).sum()
    assert n_unfused > 10, n_unfused
    # BF16 ties rounded to the odd neighbour
    e = bf16_edge_values()
    tie = (bits(e) & 0xFFFF) == 0x8000
    rne = T.float32_to_bfloat16(e)
    odd_tie = np.where(tie & np.isfinite(e), ((bits(e) >> 16) | 1).astype(np.uint16), rne)
    assert (rne != odd_tie).sum() >= 2
    # softmax normalising only from the offset
    for off, row in softmax_rows():
        if off:
            good, _ = softmax_ref(row, off, row.size - off)
            bad, _ = softmax_ref(row, off, row.size - off, from_offset=True)
            assert (~same_bits(good[0], bad[0])).sum() == off
    # softmax with the sum in sequential order instead of the kernel's
    diff = 0
    for off, row in softmax_rows():
        if row.size >= 1025:
            good, _ = softmax_ref(row, off, row.size - off)
            bad, _ = softmax_ref(row, off, row.size - off, sequential=True)
            diff += int((~same_bits(good[0], bad[0])).sum() > 0)
    assert diff >= 2, diff
    # rmsnorm dividing by length instead of E
    x = rng.standard_normal((2, 1040)).astype(F)
    w = rng.uniform(-2, 2, 1040).astype(F)
    good = rms_ref(x, w, 1.0, 1e-5, 1000, 24, 600)
    bad = rms_ref(x, w, 1.0, 1e-5, 1000, 24, 600, div=600)[0]
    assert not rows_match_one(bad, good).any()
    rel = np.abs(bad[:, 24:624] - good[0][:, 24:624]).max() / np.abs(good[0][:, 24:624]).max()
    assert rel > 0.1, rel


def test_draw_restatement_rejects_its_defects():
    """the prefix off by one, and the sum in sequential order, change the token on the crafted uniforms"""
    rng = np.random.default_rng(92)
    off1 = seq = total = 0
    for V in (255, 257, 32000):
        for row in draw_rows(V, rng)[:2]:
            for temp in (0.7, 3.0):
                _, acc = draw_ref(row, temp, 0.5)
                for u in draw_uniforms(acc, rng):
                    want, _ = draw_ref(row, temp, u)
                    total += 1
                    off1 += draw_ref(row, temp, u, off_by_one=True)[0] != want
                    seq += draw_ref(row, temp, u, sequential=True)[0] != want
    print("draw defects over %d rows: off by one %d, sequential sum %d" % (total, off1, seq))
    assert off1 >= total // 2 and seq >= 1


def test_rounding_windows_admit_one_value_almost_everywhere():
    """the two-candidate rules stay bit-exact away from float midpoints: a second candidate is rare"""
    rng = np.random.default_rng(94)
    v = (rng.standard_normal(100000) * 4).astype(F)
    main, alt = exp_f32(v.astype(f64))
    assert (main != alt).sum() <= 5, (main != alt).sum()
    for kind in (0, 1, 2):
        w = v[v > -4] if kind == 1 else v  # GELU below -4: 1 + tanh cancels, the double value itself is uncertain in float bits
        y, t = act_ref(kind, w)
        two = (y - t).astype(F) != (y + t).astype(F)
        assert two.sum() <= 5, (kind, two.sum())
        assert not interval_ok(np.nextafter(y.astype(F), F(np.inf)), y, t)[~two].any()


def test_q8_activation_restatement_matches_the_host_mirror_on_finite_rows():
    rng = np.random.default_rng(93)
    x = (rng.standard_normal((3, 256)) * np.exp(rng.uniform(-8, 8, (3, 1)))).astype(F)
    x[1, 64:96] = 0
    q, s = q8_act_ref(x, 32, 192, 256)
    qh, sh = T.quantize_q8_activations(x, 32, 192)
    assert np.array_equal(q, qh) and np.array_equal(bits(s), bits(sh))
