"""The tensor-core kernels pinned against float64 references at their edges: the wgmma prefill GEMM (jl_gemm_tc.cu) called
through jl_gemm_tc, the tiled prefill attention (jl_attn_prefill.cu) checked as a kernel inside one-layer models, and the
2..8-row int8 decode GEMM (jl_gemm8.cu) at the Llama-3-8B layer shapes.

wgmma GEMM.  The reference is the float64 product of the same BF16-rounded operands: bf16(a) and bf16(f32((nibble - 8) * scale))
(Q4) or bf16(f32(q * scale)) (Q8_0), exactly what the producer warps write into the weight tile.  Those products are exact in
f32, so what is left is the tensor core's f32 accumulation.  The bar is per element and relative to the element's own scale:
|c - ref| <= GEMM_TAU * sum_k |a_k w_k|.  Measured on an H100 80GB HBM3 (SXM, 700 W power limit): max |c - ref| / sum_k |a_k w_k|
is 1.1e-6 over every case below, reached at K = 14336 (9.6e-7 at N = 256, 1.1e-6 at N = 4096); GEMM_TAU = 2**-16 = 1.5e-5
leaves about 14x headroom.

Prefill attention.  The emulated reference follows the kernel's rounding points: q, K and V rounded to BF16, 64-key tiles in
order with an online max per tile, e = exp(s - running max) with P = bf16(e) for P.V while the row sum takes the unrounded e,
everything else in float64.  Bar: |o - ref| <= 2**-12 * max|V| per element (max|V| of the query head's KV head).  Measured on
the same H100: 1.0e-4 of max|V| at most (2.4x below the bar), from single elements of P that land on the other side of a BF16
rounding boundary because the kernel's scores are f32 sums; 1e-7 where none does.  The plain float64 softmax of the unrounded
q, K, V must agree within 2**-7 * max|V|; measured 3.0e-3 at most.

gemm8.  Integer Q8 x Q4 / Q8 x Q8_0 arithmetic with the clean / flip bars of test_gpu_layer8b.py: a step-row is clean
(<= 1e-5 of the row maximum) or carries single flipped int8 activations (<= 5e-3), at most a third of the step-rows flip, and
K/V rows stay within 2e-5 (see the test for the oracle's Q8_0 arithmetic).

The CPU tests at the end show, with the same reference functions, that every bar rejects the defects it is there to catch.
Importing this file does not load the CUDA library.
"""
import os

import numpy as np
import pytest

from jlama_b200 import tensor as T  # numpy only
from jlama_b200.native import BF16, F32, I8, JL_ERR_INVALID, JL_ERR_UNSUPPORTED, Q4

gpu = pytest.mark.gpu

GEMM_TAU = 2.0 ** -16
ATTN_EMUL_BAR = 2.0 ** -12  # of max|V|
ATTN_F64_BAR = 2.0 ** -7    # of max|V|
SHARP = 4.0                 # a defect must exceed its bar by this factor
SENTINEL = np.float32(-1234.5)
WDT = {"Q4": Q4, "Q8_0": I8}


# ---- references (numpy only) ---------------------------------------------------------------------------------------------
def bf16(x):
    """round-to-nearest-even to BF16, returned as float32"""
    return T.bfloat16_to_float32(T.float32_to_bfloat16(np.asarray(x, dtype=np.float32)))


def dequant_bf16(wdt, q, s, swap_nibbles=False):
    """weight rows as the producer warps write them into the tile: f32(q' * scale) rounded once to BF16, q' = nibble - 8 (Q4,
    element j = low nibble of byte j, element j + 16 = its high nibble) or the int8 (Q8_0); float64"""
    rows = q.shape[0]
    if wdt == Q4:
        b = q.reshape(rows, -1, 16)
        lo = (b & 0x0F).astype(np.float32) - np.float32(8)
        hi = (b >> 4).astype(np.float32) - np.float32(8)
        if swap_nibbles:
            lo, hi = hi, lo
        v = np.concatenate([lo, hi], axis=2) * s[..., None]
    else:
        v = q.astype(np.float32).reshape(rows, -1, 32) * s[..., None]
    return bf16(v.astype(np.float32).reshape(rows, -1)).astype(np.float64)


def gemm_ref(a16, w16):
    """float64 product of the BF16-rounded operands, and the natural scale sum_k |a_k w_k| of every element"""
    return a16 @ w16.T, np.abs(a16) @ np.abs(w16).T


def gemm_err(c, ref, nat, tau=GEMM_TAU):
    """(max of |c - ref| / (tau * nat), max of |c - ref| / nat); an element whose natural scale is 0 must be exactly 0"""
    err = np.abs(np.asarray(c, dtype=np.float64) - ref)
    if np.any(err[nat == 0] > 0):
        return np.inf, np.inf
    live = nat > 0
    if not live.any():
        return 0.0, 0.0
    rel = float((err[live] / nat[live]).max())
    return rel / tau, rel


def gemm_err_blocked(c, a16, wdt, q, s, tau=GEMM_TAU, block=2048):
    """gemm_err over weight-row blocks (the 8B shapes would need GBs of float64 weights at once)"""
    worst, level = 0.0, 0.0
    for r0 in range(0, q.shape[0], block):
        ref, nat = gemm_ref(a16, dequant_bf16(wdt, q[r0:r0 + block], s[r0:r0 + block]))
        w, l = gemm_err(c[:, r0:r0 + ref.shape[1]], ref, nat, tau)
        worst, level = max(worst, w), max(level, l)
    return worst, level


def attn_emulated(q, k, v, pos0, group, scale, causal_shift=0, head_map=None, skip_rescale_tile=None, ambiguity=False):
    """Prefill attention of rows at positions pos0 .. pos0 + R - 1 with the kernel's rounding points.  q [R, Hq, hs], k / v
    [P, Hkv, hs] (positions 0 .. P - 1) as float32; returns [R, Hq, hs] float64.  The keyword arguments mutate the computation
    (the sharpness tests): the causal limit moved, query heads mapped to other KV heads, the rescale skipped on one tile.
    ambiguity: also return the allowance [R, Hq, hs] for elements of P whose BF16 rounding the kernel's f32 scores can move: e
    within 2^-20 scale sum|q k| + 2^-23 (|s| + |max|) + 2^-21 (relative) of a BF16 midpoint adds one BF16 step * |V| / l."""
    R, Hq, hs = q.shape
    P = k.shape[0]
    kv_of = np.arange(Hq) // group if head_map is None else np.asarray(head_map)
    qb = bf16(q).astype(np.float64)
    kb = bf16(k).astype(np.float64)[:, kv_of]
    vb = bf16(v).astype(np.float64)[:, kv_of]
    lim = np.clip(pos0 + np.arange(R) + causal_shift, 0, P - 1)  # last key each row sees
    m = np.full((R, Hq), -np.inf)
    l = np.zeros((R, Hq))
    o = np.zeros((R, Hq, hs))
    amb = np.zeros((R, Hq, hs))
    with np.errstate(invalid="ignore", over="ignore"):
        for tile, t0 in enumerate(range(0, int(lim.max()) + 1, 64)):
            kt, vt = kb[t0:t0 + 64], vb[t0:t0 + 64]
            s = np.einsum("rhd,khd->rhk", qb, kt) * scale
            vis = (t0 + np.arange(kt.shape[0]))[None, :] <= lim[:, None]
            s = np.where(vis[:, None, :], s, -np.inf)
            mx = np.maximum(m, s.max(axis=-1))
            al = np.exp(m - mx)
            if tile == skip_rescale_tile:
                al = np.ones_like(al)
            e = np.exp(s - mx[..., None])
            l = l * al + e.sum(axis=-1)
            o = o * al[..., None] + np.einsum("rhk,khd->rhd", bf16(e).astype(np.float64), vt)
            if ambiguity:
                lo = T.bfloat16_to_float32((e.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)).astype(np.float64)
                step = np.ldexp(1.0, np.frexp(lo)[1] - 8)  # the BF16 step above lo
                nat = np.einsum("rhd,khd->rhk", np.abs(qb), np.abs(kt)) * scale
                win = 2.0 ** -20 * nat + 2.0 ** -23 * (np.abs(s) + np.abs(mx)[..., None]) + 2.0 ** -21
                near = vis[:, None, :] & (np.abs(e - (lo + 0.5 * step)) <= win * e)
                amb = amb * al[..., None] + np.einsum("rhk,khd->rhd", np.where(near, step, 0.0), np.abs(vt))
            m = mx
    if ambiguity:
        return o / l[..., None], amb / l[..., None]
    return o / l[..., None]


def attn_f64(q, k, v, pos0, group, scale):
    """plain float64 causal softmax attention of the unrounded q, K, V"""
    R, Hq, hs = q.shape
    kv_of = np.arange(Hq) // group
    k64, v64 = k.astype(np.float64)[:, kv_of], v.astype(np.float64)[:, kv_of]
    s = np.einsum("rhd,khd->rhk", q.astype(np.float64), k64) * scale
    vis = np.arange(k.shape[0])[None, :] <= (pos0 + np.arange(R))[:, None]
    s = np.where(vis[:, None, :], s, -np.inf)
    p = np.exp(s - s.max(axis=-1, keepdims=True))
    return np.einsum("rhk,khd->rhd", p, v64) / p.sum(axis=-1)[..., None]


def attn_err(o, ref, v, group):
    """max of |o - ref| / max|V of the query head's KV head|"""
    vmax = np.abs(v).max(axis=(0, 2))[np.arange(o.shape[1]) // group]
    return float((np.abs(np.asarray(o, dtype=np.float64) - ref) / vmax[None, :, None]).max())


# ---- weights ---------------------------------------------------------------------------------------------------------------
def make_weights(wdt, rows, cols, seed, kind="random"):
    """raw (q, scales) of a Q4 / Q8_0 tensor.  kind "extreme": whole blocks of nibbles 0 and 15 (int8 -128 / -127 / 127),
    zero-scale blocks, zero rows, negative scales and scales spread over 1e-6 .. 1e2 in one row, between random rows."""
    rng = np.random.default_rng(seed)
    nb = cols // 32
    sign = np.where(rng.random((rows, nb)) < 0.5, -1.0, 1.0)
    if wdt == Q4:
        q = rng.integers(0, 256, (rows, cols // 2), dtype=np.uint8)
        s = ((0.5 + rng.random((rows, nb))) * 0.01 * sign).astype(np.float32)
    else:
        q = rng.integers(-128, 128, (rows, cols), dtype=np.int8)
        s = ((0.5 + rng.random((rows, nb))) * 0.001 * sign).astype(np.float32)
    if kind == "extreme":
        qb = q.reshape(rows, nb, -1)
        if wdt == Q4:
            qb[0:16, 0::2] = 0x00   # nibbles 0: -8 * scale
            qb[0:16, 1::2] = 0xFF   # nibbles 15: 7 * scale
        else:
            qb[0:16, 0::3] = -128
            qb[0:16, 1::3] = -127
            qb[0:16, 2::3] = 127
        s[16:32, ::3] = 0.0                                                       # zero-scale blocks
        s[32:40] = 0.0                                                            # whole rows: the result must be exactly 0
        s[40:56] = (np.logspace(-6, 2, nb)[None, :] * sign[40:56]).astype(np.float32)  # 1e-6 .. 1e2 in one row
        s[56:72] = -np.abs(s[56:72])                                              # negative scales only
        s[72:88] = -np.abs(s[72:88]) * 100.0
        if wdt == Q4:
            qb[40:48, ::2] = 0xFF
        else:
            qb[40:48, ::2] = 127
    return q, s


def _report(label, worst, level):
    print("%s: err/bar %.3f  max|c - ref|/sum|a w| %.2e" % (label, worst, level))


# ---- wgmma GEMM through jl_gemm_tc --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tc_weights(cuda_ctx):
    """registered weight tensors, made once per (dtype, shape, kind, seed)"""
    from jlama_b200.native import ptr
    reg = {}

    def get(wdt, rows, cols, seed=0, kind="random"):
        key = (wdt, rows, cols, seed, kind)
        if key not in reg:
            q, s = make_weights(wdt, rows, cols, seed, kind)
            tid = cuda_ctx.lib.jl_register_tensor(cuda_ctx.h, wdt, rows, cols, ptr(q), ptr(s))
            assert tid >= 0, cuda_ctx.lib.jl_last_error(cuda_ctx.h)
            reg[key] = (tid, q, s)
        return reg[key]
    yield get
    for tid, _, _ in reg.values():
        cuda_ctx.lib.jl_unregister_tensor(cuda_ctx.h, tid)


def _activations(rng, t, lda, adt):
    """host activations (F32 or BF16 raw) and their BF16-rounded float64 values"""
    a = rng.standard_normal((t, lda)).astype(np.float32)
    if adt == "BF16":
        raw = T.float32_to_bfloat16(a)
        return raw, BF16, T.bfloat16_to_float32(raw).astype(np.float64)
    return a, F32, bf16(a).astype(np.float64)


def _gemm_tc(ctx, a_host, a_dtype, a_col_off, tid, b_col_off, n0, n, k, ldc, roffset, expect=0):
    """one jl_gemm_tc call into a sentinel-filled [T, ldc] result; returns the result"""
    from jlama_b200.native import ptr
    t, lda = a_host.shape
    out = np.full((t, ldc), SENTINEL, dtype=np.float32)
    rc = ctx.lib.jl_gemm_tc(ctx.h, a_dtype, ptr(a_host), a_col_off, lda, tid, b_col_off, ptr(out), roffset, t, n0, n, k, ldc)
    if expect == 0:
        ctx.check(rc)
    return rc, out


def _full_gemm(cuda_ctx, tc_weights, wdt, adt, t, n, k, seed):
    tid, q, s = tc_weights(WDT[wdt], n, k)
    a_host, a_dt, a16 = _activations(np.random.default_rng(seed), t, k, adt)
    _, c = _gemm_tc(cuda_ctx, a_host, a_dt, 0, tid, 0, 0, n, k, n, 0)
    return gemm_err_blocked(c, a16, WDT[wdt], q, s)


@gpu
@pytest.mark.parametrize("adt", ["F32", "BF16"])
@pytest.mark.parametrize("wdt", ["Q4", "Q8_0"])
@pytest.mark.parametrize("K", [64, 128, 192, 256, 320, 4096, 14336])
def test_gemm_tc_reduction_lengths(cuda_ctx, tc_weights, wdt, adt, K):
    """nk = K / 64 = 1..5 stages around the 3-deep register prefetch and the 4-stage ring, and the two 8B reduction lengths"""
    worst, level = _full_gemm(cuda_ctx, tc_weights, wdt, adt, 129, 256, K, K)
    _report("K=%d %s x %s" % (K, adt, wdt), worst, level)
    assert worst <= 1.0


@gpu
@pytest.mark.parametrize("adt", ["F32", "BF16"])
@pytest.mark.parametrize("wdt", ["Q4", "Q8_0"])
@pytest.mark.parametrize("T_", [16, 17, 127, 128, 129, 255, 256, 300])
def test_gemm_tc_token_tiles(cuda_ctx, tc_weights, wdt, adt, T_):
    """a ragged first token tile, exact tiles, and ragged later tiles (rows past T zero-filled by the TMA)"""
    worst, level = _full_gemm(cuda_ctx, tc_weights, wdt, adt, T_, 256, 320, T_)
    _report("T=%d %s x %s" % (T_, adt, wdt), worst, level)
    assert worst <= 1.0


@gpu
@pytest.mark.parametrize("adt", ["F32", "BF16"])
@pytest.mark.parametrize("wdt", ["Q4", "Q8_0"])
@pytest.mark.parametrize("N,K", [(4096, 4096), (1024, 4096), (14336, 4096), (4096, 14336)])
def test_gemm_tc_llama3_8b_projections(cuda_ctx, tc_weights, wdt, adt, N, K):
    """q/o_proj, k/v_proj, gate/up_proj and down_proj of Llama-3-8B on a 256-token prefill chunk"""
    worst, level = _full_gemm(cuda_ctx, tc_weights, wdt, adt, 256, N, K, N + K)
    _report("N=%d K=%d %s x %s" % (N, K, adt, wdt), worst, level)
    assert worst <= 1.0


@gpu
@pytest.mark.parametrize("adt", ["F32", "BF16"])
@pytest.mark.parametrize("wdt", ["Q4", "Q8_0"])
def test_gemm_tc_slices(cuda_ctx, cuda_ops, tc_weights, wdt, adt):
    """weight row slices n0 / n, weight column offsets with K < cols, activation column offsets with lda > a_col_off + K, and a
    result slice inside wider rows: the columns outside the written slice stay untouched.  With Q8_0 weights every n0 > 0 call
    reads rows n0 .. n0 + n - 1 at the Q8_0 row pitch (cols bytes), not at the Q4 one (cols / 2)."""
    N, cols, t, lda = 512, 640, 130, 600
    w = WDT[wdt]
    tid, q, s = tc_weights(w, N, cols, seed=7)
    a_host, a_dt, a16 = _activations(np.random.default_rng(11), t, lda, adt)
    worst_all, level_all = 0.0, 0.0
    for n0 in (0, 128, N - 128):
        for n in sorted({128, N - n0}):
            for a_off, b_off, k in ((0, 0, 512), (8, 64, 512), (64, 128, 512), (8, 0, 448)):
                ldc, c0 = n + 96, 40
                _, out = _gemm_tc(cuda_ctx, a_host, a_dt, a_off, tid, b_off, n0, n, k, ldc, n0 - c0)
                w16 = dequant_bf16(w, q[n0:n0 + n], s[n0:n0 + n])[:, b_off:b_off + k]
                ref, nat = gemm_ref(a16[:, a_off:a_off + k], w16)
                worst, level = gemm_err(out[:, c0:c0 + n], ref, nat)
                worst_all, level_all = max(worst_all, worst), max(level_all, level)
                label = "n0=%d n=%d a_col_off=%d b_col_off=%d K=%d %s x %s" % (n0, n, a_off, b_off, k, adt, wdt)
                assert worst <= 1.0, label
                outside = np.concatenate([out[:, :c0], out[:, c0 + n:]], axis=1)
                assert np.all(outside == SENTINEL), label + ": columns outside the slice were written"
    _report("slices %s x %s" % (adt, wdt), worst_all, level_all)
    # the same row slice through CudaTensorOperations.batch_dot_product_tensor_core
    bt = T.Q4ByteBufferTensor(q, s) if w == Q4 else T.Q8ByteBufferTensor(q, s)
    cuda_ops.register_model_tensor(bt)
    try:
        at = T.FloatBufferTensor(a_host) if adt == "F32" else T.BFloat16BufferTensor(a_host)
        c = T.FloatBufferTensor(np.zeros((t, N), dtype=np.float32))
        cuda_ops.batch_dot_product_tensor_core(c, at, bt, 64, 128, 512, 0, 256, 128)
        ref, nat = gemm_ref(a16[:, 64:576], dequant_bf16(w, q[256:384], s[256:384])[:, 128:640])
        assert gemm_err(c.data[:, 256:384], ref, nat)[0] <= 1.0
        assert not c.data[:, :256].any() and not c.data[:, 384:].any()
    finally:
        cuda_ops.unregister_model_tensor(bt)


@gpu
@pytest.mark.parametrize("adt", ["F32", "BF16"])
@pytest.mark.parametrize("wdt", ["Q4", "Q8_0"])
def test_gemm_tc_weight_and_activation_extremes(cuda_ctx, tc_weights, wdt, adt):
    """extreme weight blocks (make_weights kind "extreme"); activation rows of zeros, of 1e3 and of 1e-3"""
    N, K, t = 256, 512, 144
    tid, q, s = tc_weights(WDT[wdt], N, K, seed=3, kind="extreme")
    rng = np.random.default_rng(5)
    a = rng.standard_normal((t, K)).astype(np.float32)
    a[0] = 0.0
    a[1] *= 1e3
    a[2] *= 1e-3
    a[3, ::2] = 0.0
    if adt == "BF16":
        a_host, a_dt = T.float32_to_bfloat16(a), BF16
        a16 = T.bfloat16_to_float32(a_host).astype(np.float64)
    else:
        a_host, a_dt, a16 = a, F32, bf16(a).astype(np.float64)
    _, c = _gemm_tc(cuda_ctx, a_host, a_dt, 0, tid, 0, 0, N, K, N, 0)
    worst, level = gemm_err_blocked(c, a16, WDT[wdt], q, s)
    _report("extremes %s x %s" % (adt, wdt), worst, level)
    assert worst <= 1.0
    assert not c[0].any() and not c[:, 32:40].any()  # zero activations / zero-scale rows give exact zeros


@gpu
def test_gemm_tc_refusals(cuda_ctx, tc_weights):
    """shapes and offsets the kernel cannot take are refused on the host, before any launch of the GEMM, and write nothing"""
    rng = np.random.default_rng(2)
    for wdt in (Q4, I8):
        tid, _, _ = tc_weights(wdt, 256, 128, seed=1)
        a = rng.standard_normal((32, 128)).astype(np.float32)
        cases = {  # (a_col_off, lda, b_col_off, n0, n, k): all in range, only misaligned
            "K % 64": (0, 128, 0, 0, 128, 96),
            "n % 128": (0, 128, 0, 0, 64, 64),
            "n0 % 128": (0, 128, 0, 64, 128, 64),
            "b_col_off % 64": (0, 128, 32, 0, 128, 64),
            "a_col_off % 8": (4, 128, 0, 0, 128, 64),
        }
        for label, (a_off, lda, b_off, n0, n, k) in cases.items():
            launches = cuda_ctx.kernel_launches()
            rc, out = _gemm_tc(cuda_ctx, np.ascontiguousarray(a[:, :lda]), F32, a_off, tid, b_off, n0, n, k, 256, 0, expect=None)
            assert rc in (JL_ERR_UNSUPPORTED, JL_ERR_INVALID), (label, rc)
            assert np.all(out == SENTINEL), label
            assert cuda_ctx.kernel_launches() - launches <= 1, label  # at most the F32 -> BF16 conversion of the activations
        q8 = np.zeros((32, 128), dtype=np.int8)
        rc, out = _gemm_tc(cuda_ctx, q8, I8, 0, tid, 0, 0, 128, 64, 256, 0, expect=None)
        assert rc == JL_ERR_UNSUPPORTED and np.all(out == SENTINEL), "I8 activations"
        odd = np.ascontiguousarray(a[:, :100])
        rc, out = _gemm_tc(cuda_ctx, odd, F32, 0, tid, 0, 0, 128, 64, 256, 0, expect=None)
        assert rc in (JL_ERR_UNSUPPORTED, JL_ERR_INVALID) and np.all(out == SENTINEL), "lda % 8"


# ---- tiled prefill attention inside one-layer models --------------------------------------------------------------------
ATTN_CONFIGS = {
    "hs64-g1": dict(E=512, heads=8, kv_heads=8),
    "hs64-g2": dict(E=512, heads=8, kv_heads=4),
    "hs64-g4": dict(E=512, heads=8, kv_heads=2),
    "hs64-g8": dict(E=1024, heads=16, kv_heads=2),
    # 8 layers of 1024-wide KV rows: 128 (F32) / 256 (BF16) positions and 8 layers per KV page, so the tile loads go through
    # the kernel's page look-ahead and the layer offset inside a page; every other config gets one position per page
    "hs128-g1": dict(E=1024, heads=8, kv_heads=8, layers=8),
    "hs128-g2": dict(E=1024, heads=8, kv_heads=4),
    "hs128-g4": dict(E=1024, heads=8, kv_heads=2),
    "hs128-g8": dict(E=1024, heads=8, kv_heads=1),
}
# prompt chunks per max_batch: every chunk takes the tensor-core path (>= 16 rows); pos0 > 0, ragged last 16-row blocks
CHUNKS = {16: [16] * 5, 48: [48, 37, 48, 17], 256: [44, 256]}


@gpu
@pytest.mark.parametrize("max_batch", [16, 48, 256])
@pytest.mark.parametrize("kvdt", ["F32", "BF16"])
@pytest.mark.parametrize("name", list(ATTN_CONFIGS))
def test_prefill_attention_kernel_against_float64(cuda_ctx, name, kvdt, max_batch):
    from jlama_b200 import native, synth
    from jlama_b200.model import LlamaModel
    over = dict(layers=1, H=1024, vocab=512)
    over.update(ATTN_CONFIGS[name])
    cfg = synth.get_config("small", **over)
    hs, Hq, Hkv = cfg["E"] // cfg["heads"], cfg["heads"], cfg["kv_heads"]
    group, L = Hq // Hkv, cfg["layers"] - 1
    scale = float(np.float32(1.0 / np.sqrt(hs)))
    gm = LlamaModel(cuda_ctx, cfg, synth.make_weights(cfg), prefill_tensor_core=1, max_batch=max_batch, kv_dtype=getattr(native, kvdt))
    chunks = CHUNKS[max_batch]
    prompt = synth.random_prompt(cfg, sum(chunks), seed=100 + list(ATTN_CONFIGS).index(name))
    k = np.zeros((len(prompt), Hkv, hs), dtype=np.float32)
    v = np.zeros_like(k)
    worst, worst64 = 0.0, 0.0
    saved = os.environ.get("JL_PA_WARPS")
    try:
        gm.reset_session(0)
        a = 0
        for rows in chunks:
            b = a + rows
            outs = {}
            for warps in ("4", "8"):  # both CTA shapes (group 8 always runs the 8-warp one)
                os.environ["JL_PA_WARPS"] = warps
                gm.batch_forward(prompt[a:b], a)
                q = gm.debug_read(2, rows * Hq * hs).reshape(rows, Hq, hs)
                outs[warps] = gm.debug_read(5, rows * Hq * hs).reshape(rows, Hq, hs)
            for pos in range(a, b):
                k[pos] = gm.read_kv(L, pos, 0).reshape(Hkv, hs)
                v[pos] = gm.read_kv(L, pos, 1).reshape(Hkv, hs)
            emul = attn_emulated(q, k[:b], v[:b], a, group, scale)
            exact = attn_f64(q, k[:b], v[:b], a, group, scale)
            for warps, o in outs.items():
                e, e64 = attn_err(o, emul, v[:b], group), attn_err(o, exact, v[:b], group)
                assert e <= ATTN_EMUL_BAR and e64 <= ATTN_F64_BAR, (name, kvdt, a, b, warps, e, e64)
                worst, worst64 = max(worst, e), max(worst64, e64)
            a = b
    finally:
        if saved is None:
            os.environ.pop("JL_PA_WARPS", None)
        else:
            os.environ["JL_PA_WARPS"] = saved
        gm.close()
    print("prefill attention %s %s KV max_batch %d: err/max|V| %.2e (emulated, bar %.1e), %.2e (float64, bar %.1e)" % (
        name, kvdt, max_batch, worst, ATTN_EMUL_BAR, worst64, ATTN_F64_BAR))


# ---- gemm8 at the Llama-3-8B layer shapes ---------------------------------------------------------------------------------
DIMS_8B = dict(ctx=512, E=4096, H=14336, heads=32, kv_heads=8, layers=1, vocab=2048, eps=1e-5, rope_theta=500000.0)
G8_PROMPTS = [2, 3, 4, 5, 3, 2, 5, 4]  # prompt length of session s: the rows of a decode step sit at different positions
G8_STEPS = 8


def _layer8b_weights(oracle, wdt):
    """checkpoint of a one-layer model with the 8B layer dimensions and the seeds of layer 0 of the 8B checkpoint"""
    from jlama_b200 import synth
    cfg = synth.get_config("llama-3-8b", **DIMS_8B)
    cfg["name"] = "llama-3-8b-layer0"
    big = synth.get_config("llama-3-8b")
    w = {name: synth.make_one(big, name, rows, cols, kind, wdt, "quantize", q4_fn=oracle.quantize_q4)
         for name, rows, cols, kind in synth.tensor_specs(cfg)}
    return cfg, w


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max())


def _clean_or_flip(errs, what):
    errs = sorted(errs)
    flips = [e for e in errs if e > 1e-5]
    print("%s: %d of %d step-rows flip, worst %.2e, median %.2e" % (what, len(flips), len(errs), errs[-1], errs[len(errs) // 2]))
    assert errs[-1] <= 5e-3, (what, errs)
    assert 3 * len(flips) <= len(errs), (what, errs)


@pytest.fixture(scope="module")
def layer8b(cuda_ctx, oracle):
    """per weight dtype: the GPU model (8 sessions), the oracle's teacher-forced run of every session alone, and the same run on
    the GPU's M = 1 decode path"""
    from jlama_b200 import synth
    from jlama_b200.model import LlamaModel
    runs = {}

    def get(wdt):
        if wdt in runs:
            return runs[wdt]
        cfg, w = _layer8b_weights(oracle, wdt)
        om = oracle.OracleLlama(cfg, w, act_q8=True)
        gm = LlamaModel(cuda_ctx, cfg, w, max_context=64, max_sessions=8)
        E = cfg["E"]
        solo, alone = [], []
        for s, plen in enumerate(G8_PROMPTS):
            prompt = synth.random_prompt(cfg, plen, seed=700 + s)
            om.reset()
            tok, _ = om.sample(om.batch_forward(prompt, 0))
            steps = []
            for j in range(G8_STEPS):
                pos = plen + j
                oh = om.batch_forward([tok], pos)
                nxt, ol = om.sample(oh)
                steps.append(dict(tok=tok, pos=pos, hidden=oh, logits=ol, k=om.kv_row(0, pos, 0), v=om.kv_row(0, pos, 1)))
                tok = nxt
            solo.append((prompt, steps))
            gm.reset_session(s)
            gm.batch_forward(prompt, 0, session=s)
            mine = []
            for st in steps:
                _, lg = gm.decode([st["tok"]], [st["pos"]], sessions=[s], want_logits=True)
                mine.append(dict(hidden=gm.debug_read(0, E), logits=lg[0].copy(), k=gm.read_kv(0, st["pos"], 0, session=s),
                                 v=gm.read_kv(0, st["pos"], 1, session=s)))
            alone.append(mine)
        om.close()
        runs[wdt] = (cfg, gm, solo, alone)
        return runs[wdt]
    yield get
    for _, gm, _, _ in runs.values():
        gm.close()


@gpu
@pytest.mark.parametrize("n", [2, 3, 5, 8])
@pytest.mark.parametrize("wdt", ["Q4", "Q8_0"])
def test_gemm8_decode_rows_at_8b_layer_shapes(layer8b, wdt, n):
    """n sessions decoded together, teacher-forced: QKV with the fused RMSNorm prologue, o_proj with the residual epilogue,
    gate/up with SiLU, down_proj at K = 14336 and the k-split reduction, all on gemm8.

    Every row is held to the clean / flip bars against the same session decoded alone on the M = 1 path.  Against the oracle
    the same bars hold for Q4 weights, where the oracle runs the same Q8 x Q4 block arithmetic.  For Q8_0 weights the oracle
    takes F32 activations (the reference quantises activations only for Q4 weights, LlamaModel.java:176-184) while the GPU
    quantises them to Q8, so there the oracle bounds a different arithmetic: 5e-2 of the row maximum for hidden rows, logits
    and K/V (measured on an H100 at these shapes: 1.5e-2 hidden / logits, 2.0e-2 K/V)."""
    cfg, gm, solo, alone = layer8b(WDT[wdt])
    E = cfg["E"]
    assert gm.decode_mode(n) == 1
    for s in range(n):
        gm.reset_session(s)
        gm.batch_forward(solo[s][0], 0, session=s)
    vs_oracle, vs_alone, kv_oracle, kv_alone = [], [], 0.0, 0.0
    for j in range(G8_STEPS):
        steps = [solo[s][1][j] for s in range(n)]
        _, lg = gm.decode([st["tok"] for st in steps], [st["pos"] for st in steps], sessions=list(range(n)), want_logits=True)
        hid = gm.debug_read(0, n * E).reshape(n, E)
        for s, st in enumerate(steps):
            mine = alone[s][j]
            vs_oracle.append(max(_rel(hid[s], st["hidden"]), _rel(lg[s], st["logits"])))
            vs_alone.append(max(_rel(hid[s], mine["hidden"]), _rel(lg[s], mine["logits"])))
            for which, key in ((0, "k"), (1, "v")):
                row = gm.read_kv(0, st["pos"], which, session=s)
                kv_oracle, kv_alone = max(kv_oracle, _rel(row, st[key])), max(kv_alone, _rel(row, mine[key]))
    print("gemm8 %s n=%d: K/V %.2e vs oracle, %.2e vs M=1" % (wdt, n, kv_oracle, kv_alone))
    _clean_or_flip(vs_alone, "gemm8 %s n=%d vs M=1" % (wdt, n))
    assert kv_alone <= 2e-5
    if wdt == "Q4":
        _clean_or_flip(vs_oracle, "gemm8 %s n=%d vs oracle" % (wdt, n))
        assert kv_oracle <= 2e-5
    else:
        print("gemm8 %s n=%d vs oracle (F32 activations): worst %.2e" % (wdt, n, max(vs_oracle)))
        assert max(vs_oracle) <= 5e-2 and kv_oracle <= 5e-2


# ---- sharpness of the bars (CPU) ------------------------------------------------------------------------------------------
def _gemm_case(wdt, seed=0):
    rng = np.random.default_rng(seed)
    q, s = make_weights(wdt, 256, 1088, seed)
    a16 = bf16(rng.standard_normal((48, 1152)).astype(np.float32)).astype(np.float64)
    return q, s, a16


@pytest.mark.parametrize("wdt", ["Q4", "Q8_0"])
def test_gemm_bar_accepts_f32_accumulation(wdt):
    """the bar is not tighter than an f32 accumulation of the same operands"""
    q, s, a16 = _gemm_case(WDT[wdt])
    w16 = dequant_bf16(WDT[wdt], q, s)[:, :1024]
    ref, nat = gemm_ref(a16[:, :1024], w16)
    c32 = a16[:, :1024].astype(np.float32) @ w16.T.astype(np.float32)
    assert gemm_err(c32, ref, nat)[0] <= 1.0


@pytest.mark.parametrize("wdt", ["Q4", "Q8_0"])
def test_gemm_bar_rejects_defects(wdt):
    w = WDT[wdt]
    q, s, a16 = _gemm_case(w)
    K, a_off, b_off, n0, n = 1024, 64, 64, 128, 128
    a = a16[:, a_off:a_off + K]
    w16 = dequant_bf16(w, q, s)[:, b_off:b_off + K]
    ref, nat = gemm_ref(a, w16)
    defects = {}
    s2 = s.copy()
    s2[5, b_off // 32 + 7] = 0.0  # one weight block dropped
    defects["block dropped"] = a @ dequant_bf16(w, q, s2)[:, b_off:b_off + K].T
    w2 = w16.copy()  # two 16-byte (8-element) chunks of one row swapped, as a swizzle slip would
    w2[9, 3 * 64 + 16:3 * 64 + 24], w2[9, 3 * 64 + 24:3 * 64 + 32] = w16[9, 3 * 64 + 24:3 * 64 + 32], w16[9, 3 * 64 + 16:3 * 64 + 24]
    defects["16-byte chunks swapped"] = a @ w2.T
    defects["a_col_off ignored"] = a16[:, :K] @ w16.T
    if w == Q4:
        defects["nibbles exchanged"] = a @ dequant_bf16(w, q, s, swap_nibbles=True)[:, b_off:b_off + K].T
    for label, c in defects.items():
        assert gemm_err(c, ref, nat)[0] >= SHARP, label
    if w == I8:
        # rows n0 .. n0 + n - 1 of a Q8_0 tensor read at the Q4 row pitch (cols / 2 bytes), scales at the right rows
        cols = q.shape[1]
        wrong = q.reshape(-1)[n0 * cols // 2:n0 * cols // 2 + n * cols].reshape(n, cols)
        ref, nat = gemm_ref(a, dequant_bf16(w, q[n0:n0 + n], s[n0:n0 + n])[:, b_off:b_off + K])
        c = a @ dequant_bf16(w, wrong, s[n0:n0 + n])[:, b_off:b_off + K].T
        assert gemm_err(c, ref, nat)[0] >= SHARP, "Q4 row pitch on Q8_0 weights"


def _attn_case():
    rng = np.random.default_rng(3)
    R, pos0, Hq, Hkv, hs = 100, 40, 8, 2, 64
    q = (2.0 * rng.standard_normal((R, Hq, hs))).astype(np.float32)
    k = rng.standard_normal((pos0 + R, Hkv, hs)).astype(np.float32)
    v = rng.standard_normal((pos0 + R, Hkv, hs)).astype(np.float32)
    return q, k, v, pos0, Hq // Hkv, float(np.float32(1 / 8))


def test_attention_bars_accept_the_exact_softmax():
    q, k, v, pos0, group, scale = _attn_case()
    ref = attn_emulated(q, k, v, pos0, group, scale)
    assert attn_err(attn_f64(q, k, v, pos0, group, scale), ref, v, group) <= ATTN_F64_BAR
    assert attn_err(ref, attn_f64(q, k, v, pos0, group, scale), v, group) <= ATTN_F64_BAR


def test_attention_bar_rejects_defects():
    q, k, v, pos0, group, scale = _attn_case()
    ref = attn_emulated(q, k, v, pos0, group, scale)
    Hq, Hkv = q.shape[1], k.shape[1]
    defects = {
        "causal limit + 1": attn_emulated(q, k, v, pos0, group, scale, causal_shift=1),
        "causal limit - 1": attn_emulated(q, k, v, pos0, group, scale, causal_shift=-1),
        "wrong KV head": attn_emulated(q, k, v, pos0, group, scale, head_map=(np.arange(Hq) // group + 1) % Hkv),
        "rescale skipped on tile 1": attn_emulated(q, k, v, pos0, group, scale, skip_rescale_tile=1),
    }
    for label, o in defects.items():
        assert attn_err(o, ref, v, group) >= SHARP * ATTN_EMUL_BAR, label
