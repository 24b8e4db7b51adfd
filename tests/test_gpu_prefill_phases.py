"""The tensor-core prefill pass (forward_rows_tc, jl_model.cu) pinned phase by phase against float64 references at its edges.
Every prompt chunk of 16 rows or more of a model built with prefill_tensor_core = 1 takes this pass: per layer
  rmsnorm_bf16 -> gemm_tc q / k / v -> rope_kv_append -> prefill attention -> quantize_bf16 -> gemm_tc o (+ residual x)
  -> rmsnorm_bf16 -> gemm_tc gate / up -> silu_mul_bf16 -> gemm_tc down (+ residual xb)
after the embedding lookup.  Each case builds a one-layer model (two of them 2 or 3 layers, where only the last layer's attention
phases, gate / up, SiLU * up and down are checked), runs one pass with batch_forward or batch_forward_multi, and reads back x, xb,
q, k, v, att, h (gate), up (debug_read 10), the BF16 operand buffer (11: down_proj's input) and the pass's KV page rows.  Every
phase is checked from the buffer that feeds it, which is exact on the host:

  embed + attn RMSNorm -> BF16 -> k, v   from the token ids: the host-dequantised embedding rows x0 (also o_proj's residual)
  q after RoPE (in place)                 the float64 q reference rotated in float64 with the table index quirk
                                          (pair pos * hs / 2 + kvh_global * hs + j, kvh_global = h / group)
  K / V page rows                         bit for bit: rope_f32(k) and v read back, rounded RNE for BF16 pages
  attention                               q read back and the page rows: attn_emulated / attn_f64 of test_gpu_tc_kernels.py
  o_proj + residual                       x0 + f64(bf16(att) . bf16(Wo))
  FFN RMSNorm -> BF16 -> gate, up         xb read back
  SiLU * up -> BF16                       h and up read back: bit for bit (below)
  down + residual                         xb + f64(abf . bf16(Wd)), abf read back exactly

GEMM reference.  The operand is restated in float32 with one rounding per operation as rmsnorm_bf16_kernel writes it,
rsf = f32(1 / sqrt(sum f64(f32(x * x)) / E + eps)), y = f32(f32(0 + w) * f32(rsf * x)), a = bf16_rne(y), and multiplied in
float64 with bf16(f32(q * scale)) of the weights (what gemm_tc's producer warps write).  The kernel forms the double sum in
another order, so the operand is also restated with rsf moved by +-1 ulp: every element whose BF16 rounding moves is ambiguous
and adds one BF16 step * |w| to its outputs' bar.  Bar: |out - ref| <= TAU * sum_k |a_k w_k| + ambiguity (+ one ulp of the
output where a residual is added).  q after RoPE: the rotated bars |c| e0 + |s| e1 plus 2 ulp of |q0 c| + |q1 s|.

SiLU * up.  silu_mul_bf16_kernel computes f32(g / (1 + __expf(-g))) * u with the fast intrinsics; the reference is
bf16_rne(p), p = silu64(g) * u in float64.  The result must be that BF16 value bit for bit, except where p lies within
W(g) = 2^-18 + 1.2 |g| sigmoid(-g) 2^-23 relative of a BF16 rounding midpoint (__expf's error grows with |g|, 2 + 1.17 |g| ulp);
there either neighbour is accepted.  Where g < -87 the denominator reaches 2^126 and __fdividef returns 0 by its definition (true
|silu(g)| < 1e-35): 0 is accepted there too.  Both counts are printed.

Attention.  The bars of test_gpu_tc_kernels.py: 2^-12 of max|V| against the emulated reference, 2^-7 against plain float64.
At the Llama-3-8B shapes (hs 128, scores of tens) an element of P that lies near a BF16 midpoint rounds either way under the
kernel's f32 scores, and single such flips reached 0.93 of the plain 2^-12 bar; so the emulated bar adds, like the GEMM bar,
an allowance of one BF16 step * |V| / l for every element of P within 2^-20 scale sum|q k| + 2^-23 (|s| + |max|) + 2^-21
(relative) of a midpoint (attn_emulated(ambiguity=True)).

Measured on an NVIDIA H100 80GB HBM3 (SXM, 700 W power limit, 1980 MHz max SM clock) over every case below, as the worst
err/bar and the worst level (|out - ref| less the ambiguity and residual-rounding allowances, over sum_k |a_k w_k|):
  k 0.039 / 6.0e-7, v 0.037 / 5.6e-7, q after RoPE 0.039 / 5.7e-7, o_proj + residual 0.491 / 6.5e-7,
  gate 0.045 / 6.9e-7, up 0.046 / 7.0e-7, down + residual 0.466 / 3.1e-6 (the crafted case's SiLU outputs in the hundreds;
  1.6e-6 in the 8B passes, at most 4e-7 elsewhere).
TAU = 2^-16 = 1.5e-5 leaves 4.9x headroom over the worst level and equals test_gpu_tc_kernels.py's GEMM bar (2^-17 would leave
2.4x).  The err/bar values near 0.5 are o_proj / down outputs whose residual (the crafted 1e4 rows) is far larger than the
product: there the add's final rounding, at most half an ulp against the one-ulp allowance, is most of the error.
Attention: worst err/bar 0.48 (0.93 without the allowance) with 3.6e-7 of max|V| outside the allowance; 4.0e-3 of max|V|
against plain float64 (err/bar 0.51).  K / V page rows: bit for bit everywhere.  SiLU * up: no element outside the accepted
set; near-midpoint elements at most 7877 per pass (of 384 x 14336, the 2048-row pass), __fdividef zeros 120 (the crafted case,
whose gate outputs reach below -88 and above 88).
Ambiguous operand elements (rsf +- 1 ulp): at most 27 per pass for q / k / v and 41 for gate / up (the 8B passes); attention
outputs with a nonzero allowance: 1138816 of 1572864 in the 2048-row pass.  The file takes about 100 s on that card.

Routing.  Every checked pass must go through forward_rows_tc: its launches are 1 embed + 13 per layer (two RMSNorms, seven GEMMs,
RoPE / KV append, attention, the BF16 conversion of att, SiLU * up) + 1 copy of the last rows.  The exact path launches more.

The CPU tests at the end show, with the same reference and bar functions, that every bar rejects the defect it is there to catch
by at least 4x (the exact SiLU * up bar: at least a quarter of the elements leave the accepted set).  Importing this file does
not load the CUDA library.
"""
import os
import zlib

import numpy as np
import pytest

from jlama_b200 import tensor as T  # numpy only
from jlama_b200.native import BF16, F32, I8, JL_ERR_INVALID, Q4
from test_gpu_decode_attention import rope_rotate
from test_gpu_decode_gemm import norm_apply, rms_rsf
from test_gpu_tc_kernels import ATTN_EMUL_BAR, ATTN_F64_BAR, attn_emulated, attn_err, attn_f64, bf16, dequant_bf16

gpu = pytest.mark.gpu

TAU = 2.0 ** -16
SHARP = 4.0
ULP = 2.0 ** -23        # one ulp of an f32 result, relative
SILU_WIN = 2.0 ** -18   # SiLU * up: the window around a BF16 midpoint where either neighbour is accepted (plus the __expf term)
SILU_ZERO_G = -87.0     # below this gate value __fdividef may return 0
LAUNCHES_PER_LAYER = 13
H100_SMS = 132
F = np.float32


# ---- references (numpy only) ---------------------------------------------------------------------------------------------
def bf16_bits(x):
    return T.float32_to_bfloat16(np.asarray(x, dtype=F))


def bf16_trunc(x):
    """the defect: BF16 by truncation instead of RNE"""
    b = (np.asarray(x, dtype=F).view(np.uint32) >> 16).astype(np.uint32) << 16
    return b.view(F)


def norm_weight_f32(w):
    """norm weights (F32 or BF16 raw) as the kernel reads them"""
    w = np.asarray(w).reshape(-1)
    return T.bfloat16_to_float32(w) if w.dtype == np.uint16 else w.astype(F)


def operand(x, w, eps, rounding=bf16):
    """(a float64 [R, K], da float64 [R, K]): the BF16 operand rmsnorm_bf16_kernel writes for f32 rows x and norm weights w (f32
    values), and the largest move of each element under rsf +- 1 ulp (0 where unambiguous)"""
    x = np.asarray(x, dtype=F)
    r = rms_rsf(x, eps)
    a = rounding(norm_apply(x, w, r).astype(F)).astype(np.float64)
    da = np.zeros_like(a)
    for r2 in (np.nextafter(r, F(0)), np.nextafter(r, F(np.inf))):
        da = np.maximum(da, np.abs(rounding(norm_apply(x, w, r2.astype(F)).astype(F)).astype(np.float64) - a))
    return a, da


def _row_block(K):
    return max(128, (1 << 24) // K)


def gemm_ref(a, da, t, residual=None, tau=TAU):
    """(ref, bar, nat, extra) float64 [R, N] of BF16 operands a [R, K] (ambiguity da) against the raw weights t = (wdt, q, s),
    blocked over weight rows.  bar = tau * nat + extra, extra = ambiguity (+ one ulp of |ref| after a residual add)."""
    wdt, q, s = t
    R, N = a.shape[0], q.shape[0]
    ref, nat, amb = np.empty((R, N)), np.empty((R, N)), np.zeros((R, N))
    cols = np.nonzero(da.any(axis=0))[0]
    aa = np.abs(a)
    step = _row_block(a.shape[1])
    for r0 in range(0, N, step):
        w16 = dequant_bf16(wdt, q[r0:r0 + step], s[r0:r0 + step])
        ref[:, r0:r0 + step] = a @ w16.T
        nat[:, r0:r0 + step] = aa @ np.abs(w16).T
        if cols.size:
            amb[:, r0:r0 + step] = da[:, cols] @ np.abs(w16[:, cols]).T
    extra = amb
    if residual is not None:
        ref = ref + np.asarray(residual, dtype=np.float64)
        extra = amb + ULP * np.abs(ref)
    return ref, tau * nat + extra, nat, extra


def err_level(out, ref, bar, nat, extra):
    """(max |out - ref| / bar, max (|out - ref| - extra) / nat): a zero bar demands an exact result, NaN counts as infinite"""
    e = np.abs(np.asarray(out, dtype=np.float64) - ref)
    e = np.where(np.isnan(e), np.inf, e)
    r = np.where(bar > 0, e / np.where(bar > 0, bar, 1.0), np.where(e > 0, np.inf, 0.0))
    live = nat > 0
    lv = np.maximum(e - extra, 0.0)[live] / nat[live]
    return (float(r.max()) if r.size else 0.0), (float(lv.max()) if lv.size else 0.0)


def rope_pairs(table, pos, kv_of, hs, shift=0):
    """(c, s) float64 [R, H, hs / 2]: the table pairs each row's heads read (pos * hs / 2 + kv_of[h] * hs + j + shift)"""
    tab = np.asarray(table, dtype=F).reshape(-1, 2)
    hp = hs // 2
    idx = np.asarray(pos)[:, None, None] * hp + np.asarray(kv_of)[None, :, None] * hs + np.arange(hp)[None, None, :] + shift
    return tab[idx, 0].astype(np.float64), tab[idx, 1].astype(np.float64)


def rotate_ref(ref, bar, nat, extra, table, pos, kv_of, hs, shift=0, sign=1.0):
    """RoPE of the float64 q reference [R, Hq * hs] and its bars: (ref, bar, nat, extra) of the rotated rows.  shift / sign
    mutate the rotation (the sharpness tests): pair index moved, sine sign flipped."""
    R, Hq = ref.shape[0], len(kv_of)
    hp = hs // 2
    c, s = rope_pairs(table, pos, kv_of, hs, shift)
    s = s * sign
    parts = [x.reshape(R, Hq, hs) for x in (ref, bar, nat, extra)]
    (q0, q1), (b0, b1), (n0, n1), (x0, x1) = [(p[..., :hp], p[..., hp:]) for p in parts]
    ac, as_ = np.abs(c), np.abs(s)
    r0, r1 = q0 * c - q1 * s, q0 * s + q1 * c
    u0, u1 = 2 * ULP * (np.abs(q0 * c) + np.abs(q1 * s)), 2 * ULP * (np.abs(q0 * s) + np.abs(q1 * c))
    out = []
    for a0, a1 in ((r0, r1), (ac * b0 + as_ * b1 + u0, as_ * b0 + ac * b1 + u1), (ac * n0 + as_ * n1, as_ * n0 + ac * n1),
                   (ac * x0 + as_ * x1 + u0, as_ * x0 + ac * x1 + u1)):
        out.append(np.concatenate([a0, a1], axis=2).reshape(R, Hq * hs))
    return tuple(out)


def silu64(g):
    g = np.asarray(g, dtype=np.float64)
    with np.errstate(over="ignore"):
        return g / (1.0 + np.exp(-g))


def _zero(bits):
    return np.where((bits & 0x7FFF) == 0, 0, bits).astype(np.uint16)


def silu_check(out_bits, g, u):
    """SiLU * up against bf16_rne(silu64(g) * u): (rejected, ambiguous, zero-by-__fdividef) element counts"""
    g, u = np.asarray(g, dtype=F), np.asarray(u, dtype=F)
    p = silu64(g) * u.astype(np.float64)
    f = p.astype(F)
    ref = _zero(bf16_bits(f))
    lo = (f.view(np.uint32) >> 16).astype(np.uint16)       # the BF16 value toward zero
    hi = (lo + 1).astype(np.uint16)                          # and the one away from zero
    lo64, hi64 = T.bfloat16_to_float32(lo).astype(np.float64), T.bfloat16_to_float32(hi).astype(np.float64)
    with np.errstate(over="ignore"):
        win = SILU_WIN + 1.2 * np.abs(g.astype(np.float64)) / (1.0 + np.exp(g.astype(np.float64))) * ULP
    near = np.abs(p - 0.5 * (lo64 + hi64)) <= win * np.abs(p) + 2.0 ** -148
    out = _zero(np.asarray(out_bits, dtype=np.uint16))
    ok = out == ref
    ok |= near & ((out == _zero(lo)) | (out == _zero(hi)))
    zero_g = g < SILU_ZERO_G
    ok |= zero_g & (out == 0)
    return int((~ok).sum()), int((near & (ref != 0)).sum()), int((zero_g & (out == 0) & (ref != 0)).sum())


def attn_check(o, ref, amb, v, group):
    """(err/bar, level, ambiguous outputs) of attention rows: |o - ref| <= ATTN_EMUL_BAR * max|V| + amb per element (max|V| of
    the query head's KV head); level = max (|o - ref| - amb) / max|V|"""
    vmax = np.abs(v).max(axis=(0, 2))[np.arange(o.shape[1]) // group][None, :, None]
    e = np.abs(np.asarray(o, dtype=np.float64) - ref)
    e = np.where(np.isnan(e), np.inf, e)
    return float((e / (ATTN_EMUL_BAR * vmax + amb)).max()), float((np.maximum(e - amb, 0.0) / vmax).max()), int((amb > 0).sum())


def kv_page_rows(k, v, table, pos, hkv, hs, kvdt):
    """the raw K / V page rows rope_kv_append_kernel writes for k / v rows [R, kv_len] at positions pos"""
    kr = np.stack([rope_rotate(k[i].reshape(hkv, hs), table, int(pos[i]), np.arange(hkv)).reshape(-1) for i in range(len(pos))])
    if kvdt == F32:
        return kr.view(np.uint32), np.asarray(v, dtype=F).view(np.uint32)
    return bf16_bits(kr), bf16_bits(v)


# ---- the case matrix ------------------------------------------------------------------------------------------------------
def _cfg(E, H, heads, kv_heads, layers=1, ctx=1024, vocab=512, theta=10000.0):
    return dict(E=E, H=H, heads=heads, kv_heads=kv_heads, layers=layers, ctx=ctx, vocab=vocab, rope_theta=theta)


CFGS = {
    "g4-hs64": _cfg(512, 1536, 8, 2),
    "g1-hs64": _cfg(512, 1024, 8, 8),
    "g8-hs64": _cfg(1024, 1024, 16, 2),
    "g1-hs128-2L": _cfg(1024, 1024, 8, 8, layers=2),
    "g4-hs128": _cfg(1024, 2048, 8, 2),
    "g8-hs128-3L": _cfg(1024, 1024, 8, 1, layers=3),
    "8b": _cfg(4096, 14336, 32, 8, ctx=2048, vocab=2048, theta=500000.0),
}

# passes: each a list of segments (session, rows, pos0); every pass is checked.  norm: F32 / BF16 norm weights with zero and
# negative entries; craft: the F32 embedding with crafted rows, a gate projection reaching |g| > 88 and exactly-zero up rows
CASES = [
    dict(id="g4-hs64-Q4", cfg="g4-hs64", wd="Q4", kv="F32", norm="F32", max_batch=256,
         passes=[[(0, 16, 0)], [(0, 17, 16)], [(0, 127, 33)], [(0, 128, 160)], [(0, 129, 288)]]),
    dict(id="g4-hs128-Q8_0-bf16", cfg="g4-hs128", wd="Q8_0", kv="BF16", norm="BF16", max_batch=300,
         passes=[[(0, 255, 0)], [(0, 256, 255)], [(0, 300, 511)]]),
    dict(id="g1-hs64-Q4-crafted", cfg="g1-hs64", wd="Q4", kv="F32", norm="F32", craft=True, max_batch=512,
         passes=[[(0, 300, 0)], [(0, 16, 300)]]),
    dict(id="g8-hs64-Q8_0", cfg="g8-hs64", wd="Q8_0", kv="F32", norm="F32", max_batch=256,
         passes=[[(0, 128, 0)], [(0, 255, 128)]]),
    dict(id="g1-hs128-2L-Q4-bf16", cfg="g1-hs128-2L", wd="Q4", kv="BF16", norm="BF16", max_batch=256,
         passes=[[(0, 129, 0)], [(0, 127, 129)]]),
    dict(id="g8-hs128-3L-Q8_0", cfg="g8-hs128-3L", wd="Q8_0", kv="BF16", norm="F32", max_batch=256,
         passes=[[(0, 256, 0)], [(0, 17, 256)]]),
    # several sessions in one pass (block-table attention, rows of three sessions in one GEMM tile), after a lone pass of session 2
    dict(id="g4-hs64-Q4-multi", cfg="g4-hs64", wd="Q4", kv="F32", norm="F32", max_batch=512, sessions=4,
         passes=[[(2, 60, 0)], [(0, 127, 0), (1, 17, 0), (2, 129, 60)], [(3, 33, 0), (0, 48, 127), (1, 200, 17)]]),
    # the bench's regime: 16 token tiles per GEMM, K = 14336, the 8-warp attention CTA chosen by the row count, 2048 positions
    dict(id="8b-Q4-2048", cfg="8b", wd="Q4", kv="F32", norm="F32", max_batch=2048, passes=[[(0, 2048, 0)]]),
    dict(id="8b-Q8_0-300", cfg="8b", wd="Q8_0", kv="F32", norm="F32", max_batch=300, passes=[[(0, 300, 0)]]),
]
PASS_SIZES = (16, 17, 127, 128, 129, 255, 256, 300)
CHECK_ALL_ROWS = 384  # larger passes: the first and last 128-row token tiles and a seeded sample of 128 other rows


def pa_warps(rows, cfg, sm):
    """pa_warps (jl_attn_prefill.cu) without JL_PA_WARPS: 8 warps for group 8, or when rows * kv_heads >= 64 * SMs"""
    return 8 if cfg["heads"] // cfg["kv_heads"] == 8 or rows * cfg["kv_heads"] >= 64 * sm else 4


def pass_label(case, segs, sm=H100_SMS):
    cfg = CFGS[case["cfg"]]
    M = sum(r for _, r, _ in segs)
    return "%s %s M=%d tiles=%d warps=%d" % (case["id"], "+".join("%d@%d" % (r, p) for _, r, p in segs), M, -(-M // 128),
                                             pa_warps(M, cfg, sm))


def checked_rows(M, seed):
    if M <= CHECK_ALL_ROWS:
        return np.arange(M)
    last = (M - 1) // 128 * 128
    mid = np.random.default_rng(seed).choice(np.arange(128, last), 128, replace=False)
    return np.unique(np.concatenate([np.arange(128), mid, np.arange(last, M)]))


# ---- weights ----------------------------------------------------------------------------------------------------------------
def llama_cfg(name):
    from jlama_b200 import synth
    c = CFGS[name]
    return synth.get_config("tiny", **c)


def craft_norm(w):
    w = w.copy()
    w[:, ::7] = 0.0
    w[:, 3::5] *= -1.0
    return w


def case_weights(case):
    """synth direct weights (every nibble pattern, scales of mixed sign), norm weights with zero and negative entries, and the
    crafted operands"""
    from jlama_b200 import synth
    cfg = llama_cfg(case["cfg"])
    wd = Q4 if case["wd"] == "Q4" else I8
    w = synth.make_weights(cfg, wd, mode="direct")
    rng = np.random.default_rng(zlib.crc32(case["id"].encode()))
    for k in list(w):
        if k.endswith("norm.weight"):
            v = craft_norm(w[k][1])
            w[k] = (BF16, T.float32_to_bfloat16(v), None) if case["norm"] == "BF16" else (F32, v, None)
    if case.get("craft"):
        E, V = cfg["E"], cfg["vocab"]
        emb = rng.standard_normal((V, E)).astype(F)
        emb[0] = 0.0           # eps-dominated norm, exact-zero operand
        emb[1] *= F(1e4)
        emb[2] *= F(1e-4)
        w["model.embed_tokens.weight"] = (F32, emb, None)
        L = cfg["layers"] - 1
        gk, uk = "model.layers.%d.mlp.gate_proj.weight" % L, "model.layers.%d.mlp.up_proj.weight" % L
        dt, q, s = w[gk]
        s = s.copy()
        s[:64] = np.sign(s[:64]) * np.logspace(-2, 0.5, 64, dtype=F)[:, None]  # gate rows reaching |g| in the hundreds
        w[gk] = (dt, q, s.astype(F))
        dt, q, s = w[uk]
        s = s.copy()
        s[64:80] = 0.0  # up rows that are exactly zero
        w[uk] = (dt, q, s)
    return cfg, w


def pass_tokens(case, segs, vocab):
    rng = np.random.default_rng(zlib.crc32(("%s %s" % (case["id"], segs)).encode()))
    out = []
    for _, rows, _ in segs:
        t = rng.integers(0, vocab, rows).astype(np.int32)
        if case.get("craft"):
            t[::37], t[5::41], t[9::43] = 0, 1, 2
        out.append(t)
    return out


def embed_rows(t, tokens):
    wdt, q, s = t
    if wdt == F32:
        return q[tokens].astype(F)
    if wdt == Q4:
        b = q[tokens].reshape(len(tokens), -1, 16)
        v = np.concatenate([b & 0x0F, b >> 4], axis=2).reshape(len(tokens), -1).astype(F) - F(8)
    else:
        v = q[tokens].astype(F)
    return (v * np.repeat(s[tokens], 32, axis=1)).astype(F)


# ---- GPU harness ----------------------------------------------------------------------------------------------------------
WORST = {}


def _record(phase, err, lvl):
    w, l = WORST.get(phase, (0.0, 0.0))
    WORST[phase] = (max(w, err), max(l, lvl))


def read_pass(gm, M, cfg):
    E, H = cfg["E"], cfg["H"]
    kv = cfg["kv_heads"] * (E // cfg["heads"])
    return dict(x=gm.debug_read(0, M * E).reshape(M, E), xb=gm.debug_read(1, M * E).reshape(M, E),
                q=gm.debug_read(2, M * E).reshape(M, E), k=gm.debug_read(3, M * kv).reshape(M, kv),
                v=gm.debug_read(4, M * kv).reshape(M, kv), att=gm.debug_read(5, M * E).reshape(M, E),
                h=gm.debug_read(6, M * H).reshape(M, H), up=gm.debug_read(10, M * H).reshape(M, H),
                abf=gm.debug_read(11, M * H // 2).view(np.uint16).reshape(M, H))


def _runs(idx):
    """consecutive runs [(start, stop)] of sorted indices"""
    cuts = np.nonzero(np.diff(idx) != 1)[0] + 1
    return [(int(r[0]), int(r[-1]) + 1) for r in np.split(idx, cuts)]


def check_pass(gm, case, cfg, w, table, segs, tokens, b, label):
    """every phase of the pass from the buffers that feed it; returns {phase: (err/bar, level, ambiguous)}"""
    E, H, Hq, Hkv = cfg["E"], cfg["H"], cfg["heads"], cfg["kv_heads"]
    hs, group, L, eps = E // Hq, Hq // Hkv, cfg["layers"] - 1, cfg["eps"]
    kvdt = F32 if case["kv"] == "F32" else BF16
    M = sum(r for _, r, _ in segs)
    sess = np.concatenate([np.full(r, s) for s, r, _ in segs])
    pos = np.concatenate([p + np.arange(r) for _, r, p in segs])
    toks = np.concatenate(tokens)
    sel = checked_rows(M, zlib.crc32(label.encode()))
    lw = lambda n: w["model.layers.%d.%s" % (L, n)]  # noqa: E731
    res = {}

    def rec(ph, r, amb=0):
        _record(ph, r[0], r[1])
        assert r[0] <= 1.0, "%s: %s err/bar %.3f, level %.2e" % (label, ph, r[0], r[1])
        res[ph] = (r[0], r[1], amb)

    # K / V page rows: rope_f32(k) and v of every row of the pass, bit for bit
    kp = np.stack([gm.read_kv(L, int(pos[i]), 0, session=int(sess[i])) for i in range(M)])
    vp = np.stack([gm.read_kv(L, int(pos[i]), 1, session=int(sess[i])) for i in range(M)])
    want_k, want_v = kv_page_rows(b["k"], b["v"], table, pos, Hkv, hs, kvdt)
    got_k, got_v = (kp.view(np.uint32), vp.view(np.uint32)) if kvdt == F32 else (bf16_bits(kp), bf16_bits(vp))
    for nm, g_, e_ in (("K", got_k, want_k), ("V", got_v, want_v)):
        bad = np.nonzero((g_ != e_).any(axis=1))[0]
        assert bad.size == 0, "%s: %s page row of row %d (session %d, position %d) is not the appended row" % (
            label, nm, bad[0], sess[bad[0]], pos[bad[0]])
    res["kv"] = (0.0, 0.0, 0)

    if L == 0:
        x0 = embed_rows(w["model.embed_tokens.weight"], toks[sel])
        a, da = operand(x0, norm_weight_f32(lw("input_layernorm.weight")[1]), eps)
        amb = int((da > 0).sum())
        for nm, key in (("k", "self_attn.k_proj.weight"), ("v", "self_attn.v_proj.weight")):
            ref, bar, nat, extra = gemm_ref(a, da, lw(key))
            rec(nm, err_level(b[nm][sel], ref, bar, nat, extra), amb)
        ref, bar, nat, extra = gemm_ref(a, da, lw("self_attn.q_proj.weight"))
        rot = rotate_ref(ref, bar, nat, extra, table, pos[sel], np.arange(Hq) // group, hs)
        rec("q+rope", err_level(b["q"][sel], *rot), amb)

    # attention: per segment, runs of checked rows against the session's page rows
    worst, level, n_amb, worst64 = 0.0, 0.0, 0, 0.0
    scale = float(F(1.0 / np.sqrt(hs)))
    q3 = b["q"].reshape(M, Hq, hs)
    row0 = 0
    for s, rows, p0 in segs:
        mine = sel[(sel >= row0) & (sel < row0 + rows)]
        P = p0 + rows
        K = np.stack([gm.read_kv(L, p, 0, session=s) for p in range(P)]).reshape(P, Hkv, hs)
        V = np.stack([gm.read_kv(L, p, 1, session=s) for p in range(P)]).reshape(P, Hkv, hs)
        for r0, r1 in _runs(mine):
            pa = p0 + r0 - row0
            o = b["att"][r0:r1].reshape(r1 - r0, Hq, hs)
            Kr, Vr = K[:pa + r1 - r0], V[:pa + r1 - r0]
            e, lv, n = attn_check(o, *attn_emulated(q3[r0:r1], Kr, Vr, pa, group, scale, ambiguity=True), Vr, group)
            e64 = attn_err(o, attn_f64(q3[r0:r1], Kr, Vr, pa, group, scale), Vr, group)
            assert e <= 1.0 and e64 <= ATTN_F64_BAR, "%s: attention rows %d..%d (session %d): err/bar %.3f, %.2e of max|V| (float64)" % (
                label, r0, r1 - 1, s, e, e64)
            worst, level, n_amb, worst64 = max(worst, e), max(level, lv), n_amb + n, max(worst64, e64)
        row0 += rows
    _record("attention (emulated)", worst, level)
    _record("attention (float64)", worst64 / ATTN_F64_BAR, worst64)
    res["attn"] = (worst, level, n_amb)

    if L == 0:
        a_o = bf16(b["att"][sel]).astype(np.float64)
        ref, bar, nat, extra = gemm_ref(a_o, np.zeros_like(a_o), lw("self_attn.o_proj.weight"), residual=x0)
        rec("o+res", err_level(b["xb"][sel], ref, bar, nat, extra))

    a, da = operand(b["xb"][sel], norm_weight_f32(lw("post_attention_layernorm.weight")[1]), eps)
    amb = int((da > 0).sum())
    for nm, key in (("h", "mlp.gate_proj.weight"), ("up", "mlp.up_proj.weight")):
        ref, bar, nat, extra = gemm_ref(a, da, lw(key))
        rec("gate" if nm == "h" else "up", err_level(b[nm][sel], ref, bar, nat, extra), amb)

    bad, near, zeros = silu_check(b["abf"][sel], b["h"][sel], b["up"][sel])
    assert bad == 0, "%s: SiLU * up: %d elements are not bf16_rne(silu(g) * u)" % (label, bad)
    res["silu"] = (0.0, 0.0, near)
    res["silu zero"] = (0.0, 0.0, zeros)

    a_d = T.bfloat16_to_float32(b["abf"][sel]).astype(np.float64)
    ref, bar, nat, extra = gemm_ref(a_d, np.zeros_like(a_d), lw("mlp.down_proj.weight"), residual=b["xb"][sel])
    rec("down+res", err_level(b["x"][sel], ref, bar, nat, extra))
    return res


def rope_table(lib, cfg):
    hs = cfg["E"] // cfg["heads"]
    positions = cfg["ctx"] + 2 * cfg["kv_heads"]
    table = np.empty(positions * hs, dtype=F)
    assert lib.jl_precompute_freqs_cis(hs, positions, cfg["rope_theta"], cfg.get("rope_scale", 1.0), table.ctypes.data) == 0
    return table


@pytest.fixture
def no_pa_override():
    """the attention CTA shape chosen by the row count, as in production"""
    saved = os.environ.pop("JL_PA_WARPS", None)
    yield
    if saved is not None:
        os.environ["JL_PA_WARPS"] = saved


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_prefill_phases_against_float64(cuda_ctx, no_pa_override, case):
    from jlama_b200.model import LlamaModel
    sm = cuda_ctx.sm_count
    cfg, w = case_weights(case)
    kvdt = F32 if case["kv"] == "F32" else BF16
    gm = LlamaModel(cuda_ctx, cfg, w, kv_dtype=kvdt, max_batch=case["max_batch"], max_sessions=case.get("sessions", 1),
                    prefill_tensor_core=1)
    try:
        table = rope_table(cuda_ctx.lib, cfg)
        for s in range(case.get("sessions", 1)):
            gm.reset_session(s)
        for segs in case["passes"]:
            tokens = pass_tokens(case, segs, cfg["vocab"])
            M = sum(r for _, r, _ in segs)
            label = pass_label(case, segs, sm)
            c0 = cuda_ctx.kernel_launches()
            if len(segs) == 1:
                gm.batch_forward(tokens[0], segs[0][2], session=segs[0][0])
            else:
                gm.batch_forward_multi([(s, t, p) for (s, _, p), t in zip(segs, tokens)])
            launches = cuda_ctx.kernel_launches() - c0
            assert launches == 2 + LAUNCHES_PER_LAYER * cfg["layers"], "%s: %d launches: not one tensor-core pass" % (label, launches)
            b = read_pass(gm, M, cfg)
            if case.get("craft"):
                assert b["h"].min() < -88 and b["h"].max() > 88, (label, b["h"].min(), b["h"].max())
                assert not b["up"][:, 64:80].any() and not (b["abf"][:, 64:80] & 0x7FFF).any()
            res = check_pass(gm, case, cfg, w, table, segs, tokens, b, label)
            print("%s: %s" % (label, "  ".join("%s %.3f/%.1e/%d" % (ph, e, lv, amb) for ph, (e, lv, amb) in res.items())))
    finally:
        gm.close()


@gpu
def test_debug_read_sources_of_tensor_core_models(cuda_ctx):
    """up (10) and the BF16 operand buffer (11) exist only in tensor-core prefill models; elsewhere they are refused"""
    from jlama_b200 import synth
    from jlama_b200.model import LlamaModel
    cfg = llama_cfg("g4-hs64")
    w = synth.make_weights(cfg, Q4, mode="direct")
    H = cfg["H"]
    for ptc in (0, 1):
        gm = LlamaModel(cuda_ctx, cfg, w, max_batch=32, prefill_tensor_core=ptc)
        try:
            gm.batch_forward(synth.random_prompt(cfg, 20), 0)
            out = np.full(4, 7.0, dtype=F)
            for which, n in ((10, 32 * H), (11, 32 * H // 2)):
                rc = gm.lib.jl_model_debug_read(gm.h, which, out.ctypes.data, 1)
                assert rc == (0 if ptc else JL_ERR_INVALID), (ptc, which, rc)
                if ptc:
                    assert gm.lib.jl_model_debug_read(gm.h, which, out.ctypes.data, n + 1) == JL_ERR_INVALID, which
            assert gm.lib.jl_model_debug_read(gm.h, 12, out.ctypes.data, 1) == JL_ERR_INVALID
        finally:
            gm.close()


@gpu
def test_zz_report():
    """the worst err/bar and level per phase over the cases that ran"""
    for k in sorted(WORST):
        print("prefill phase %-22s: worst err/bar %.3f, level %.2e" % (k, WORST[k][0], WORST[k][1]))


# ---- the case matrix, checked on the CPU ----------------------------------------------------------------------------------
def test_case_matrix_reaches_every_edge():
    seen = set()
    for case in CASES:
        cfg = CFGS[case["cfg"]]
        hs, group = cfg["E"] // cfg["heads"], cfg["heads"] // cfg["kv_heads"]
        # tc_ok (jl_model_finalize): every GEMM dimension a multiple of 128
        kv = cfg["kv_heads"] * hs
        assert all(d % 128 == 0 for d in (cfg["E"], cfg["H"], kv)), case["id"]
        seen |= {("wd", case["wd"]), ("kv", case["kv"]), ("norm", case["norm"]), ("hs", hs), ("group", group),
                 ("layers>1", cfg["layers"] > 1)}
        if case.get("craft"):
            seen.add("crafted activations")
        for segs in case["passes"]:
            M = sum(r for _, r, _ in segs)
            assert M <= case["max_batch"] and all(r >= 16 for _, r, _ in segs), (case["id"], segs)  # one tensor-core pass
            assert len({s for s, _, _ in segs}) == len(segs)
            for _, r, p in segs:
                assert p + r <= cfg["ctx"]
                seen.add(("rows", r, p > 0))
            if len(segs) >= 3 and len({r for _, r, _ in segs}) == len(segs) and len({p for _, _, p in segs}) > 1:
                seen.add("3+ segments of different lengths and positions")
            seen.add(("warps", pa_warps(M, cfg, H100_SMS)))
            if case["cfg"] == "8b":
                seen.add(("8b", case["wd"], M, pa_warps(M, cfg, H100_SMS)))
    want = [("rows", r, p) for r in PASS_SIZES for p in (False, True)]
    want += [("wd", "Q4"), ("wd", "Q8_0"), ("kv", "F32"), ("kv", "BF16"), ("norm", "F32"), ("norm", "BF16"), ("hs", 64), ("hs", 128),
             ("group", 1), ("group", 4), ("group", 8), ("layers>1", True), "crafted activations",
             "3+ segments of different lengths and positions", ("warps", 4), ("warps", 8),
             ("8b", "Q4", 2048, 8), ("8b", "Q8_0", 300, 4)]
    missing = [x for x in want if x not in seen]
    assert not missing, missing
    # the 2048-row pass takes the 8-warp CTA from its row count alone (group 4), and checks 384 rows
    assert CFGS["8b"]["heads"] // CFGS["8b"]["kv_heads"] == 4 and pa_warps(2048, CFGS["8b"], H100_SMS) == 8
    rows = checked_rows(2048, 1)
    assert len(rows) == 384 and rows[127] == 127 and rows[-128] == 1920 and rows[-1] == 2047


def test_checked_rows_cover_first_and_last_tiles():
    for M in (300, 384, 385, 2048, 1000):
        r = checked_rows(M, 5)
        assert set(range(min(M, 128))) <= set(r.tolist()) and set(range((M - 1) // 128 * 128, M)) <= set(r.tolist())
        assert np.array_equal(r, np.unique(r)) and (M <= CHECK_ALL_ROWS) == (len(r) == M)


# ---- sharpness of the bars (CPU) --------------------------------------------------------------------------------------------
def _weights(wdt, N, K, seed):
    from jlama_b200 import synth
    t = synth.make_tensor(seed, N, K, wdt, "direct")
    return t


def _ratio(r, what):
    print("%s: err/bar %.1f" % (what, r))
    assert r >= SHARP, (what, r)


def _norm_case(M=64, K=512, seed=1):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((M, K)).astype(F)
    x[0] = 0.0
    x[1] *= F(1e-4)
    x[2] *= F(1e4)
    w = craft_norm((1.0 + 0.1 * rng.standard_normal((1, K))).astype(F)).reshape(-1)
    return x, w


@pytest.mark.parametrize("wd", ["Q4", "Q8_0"])
def test_bar_accepts_f32_accumulation(wd):
    """an f32 accumulation of the same operands, in 64-wide K blocks, stays within the bar"""
    x, w = _norm_case(K=4096)
    t = _weights(Q4 if wd == "Q4" else I8, 128, 4096, 3)
    a, da = operand(x, w, 1e-5)
    ref, bar, nat, extra = gemm_ref(a, da, t)
    w16 = dequant_bf16(t[0], t[1], t[2]).astype(F)
    acc = np.zeros((x.shape[0], 128), dtype=F)
    for k0 in range(0, 4096, 64):
        acc = (acc + a[:, k0:k0 + 64].astype(F) @ w16[:, k0:k0 + 64].T).astype(F)
    assert err_level(acc, ref, bar, nat, extra)[0] <= 0.25


def test_bar_rejects_a_truncated_norm_operand():
    x, w = _norm_case()
    t = _weights(Q4, 128, 512, 4)
    a, da = operand(x, w, 1e-5)
    ref, bar, nat, extra = gemm_ref(a, da, t)
    at, _ = operand(x, w, 1e-5, rounding=bf16_trunc)
    _ratio(err_level(gemm_ref(at, np.zeros_like(at), t)[0], ref, bar, nat, extra)[0], "norm operand truncated to BF16")


def test_bar_rejects_bf16_norm_weights_read_as_f32():
    x, w = _norm_case()
    t = _weights(I8, 128, 512, 5)
    wb = T.float32_to_bfloat16(w)
    a, da = operand(x, norm_weight_f32(wb), 1e-5)
    ref, bar, nat, extra = gemm_ref(a, da, t)
    as_f32 = np.concatenate([wb.view(F), np.zeros(len(w) // 2, dtype=F)])  # pairs of BF16 read as one f32, then past the end
    aw, _ = operand(x, as_f32, 1e-5)
    _ratio(err_level(gemm_ref(aw, np.zeros_like(aw), t)[0], ref, bar, nat, extra)[0], "BF16 norm weights read as F32")


def test_bar_rejects_a_dropped_eps():
    """visible on the zero row (NaN) and on the 1e-4 row (eps-dominated: rsf moves by 30x)"""
    x, w = _norm_case()
    t = _weights(Q4, 128, 512, 6)
    a, da = operand(x, w, 1e-5)
    ref, bar, nat, extra = gemm_ref(a, da, t)
    with np.errstate(divide="ignore", invalid="ignore"):
        a0, _ = operand(x, w, 0.0)  # the zero row becomes NaN
    out = gemm_ref(a0, np.zeros_like(a0), t)[0]
    _ratio(err_level(out, ref, bar, nat, extra)[0], "eps dropped")
    _ratio(err_level(out[1:2], ref[1:2], bar[1:2], nat[1:2], extra[1:2])[0], "eps dropped, the 1e-4 row")


def test_bar_rejects_residual_defects():
    rng = np.random.default_rng(7)
    t = _weights(Q4, 128, 512, 7)
    a = bf16(rng.standard_normal((64, 512))).astype(np.float64)
    res = rng.standard_normal((64, 128)).astype(F)
    ref, bar, nat, extra = gemm_ref(a, np.zeros_like(a), t, residual=res)
    plain = gemm_ref(a, np.zeros_like(a), t)[0]
    for what, out in (("residual missing", plain), ("residual added twice", plain + 2 * res),
                      ("residual from row r + 1", plain + np.roll(res, -1, axis=0)),
                      ("residual from row r - 1", plain + np.roll(res, 1, axis=0))):
        _ratio(err_level(out, ref, bar, nat, extra)[0], what)


def test_bar_rejects_a_dropped_last_k_block():
    rng = np.random.default_rng(8)
    for K in (512, 14336):
        t = _weights(Q4, 128, K, 8)
        a = bf16(rng.standard_normal((16, K))).astype(np.float64)
        ref, bar, nat, extra = gemm_ref(a, np.zeros_like(a), t)
        a2 = a.copy()
        a2[:, -64:] = 0.0
        _ratio(err_level(gemm_ref(a2, np.zeros_like(a2), t)[0], ref, bar, nat, extra)[0], "last 64-wide K block dropped, K=%d" % K)


def test_bar_rejects_tile_2_from_tile_1_operands():
    rng = np.random.default_rng(9)
    t = _weights(I8, 128, 512, 9)
    a = bf16(rng.standard_normal((256, 512))).astype(np.float64)
    ref, bar, nat, extra = gemm_ref(a, np.zeros_like(a), t)
    out = ref.copy()
    out[128:] = ref[:128]
    _ratio(err_level(out, ref, bar, nat, extra)[0], "token tile 2 from tile 1's operands")


def _rope_case():
    """q reference rows at positions 1..64 with a float32 RoPE table of theta 10000 (hs 64, 8 heads over 2 KV heads)"""
    hs, Hq, group, P = 64, 8, 4, 64
    j = np.arange(hs // 2)
    freqs = 1.0 / 10000.0 ** (2.0 * j / hs)
    ang = np.arange(P + 2 * 2 + 1)[:, None] * freqs[None, :]
    table = np.stack([np.cos(ang), np.sin(ang)], axis=2).astype(F).reshape(-1)
    rng = np.random.default_rng(10)
    t = _weights(Q4, Hq * hs, 512, 10)
    a = bf16(rng.standard_normal((P, 512))).astype(np.float64)
    return table, np.arange(1, P + 1), np.arange(Hq) // group, hs, a, t


def test_bar_rejects_rope_defects():
    table, pos, kv_of, hs, a, t = _rope_case()
    base = gemm_ref(a, np.zeros_like(a), t)
    ref, bar, nat, extra = rotate_ref(*base, table, pos, kv_of, hs)
    assert err_level(ref.astype(F), ref, bar, nat, extra)[0] <= 0.25  # the f32 store of the rotated value
    for what, kw in (("RoPE pair index + 1", dict(shift=1)), ("RoPE pair index - 1", dict(shift=-1)),
                     ("RoPE sine sign flipped", dict(sign=-1.0))):
        _ratio(err_level(rotate_ref(*base, table, pos, kv_of, hs, **kw)[0], ref, bar, nat, extra)[0], what)


def test_rope_reference_matches_the_f32_page_rotation():
    """the float64 rotation of a float32 row is within 2 ulp of rope_rotate's float32 one (the page rows' reference)"""
    table, pos, kv_of, hs, a, t = _rope_case()
    x = np.random.default_rng(11).standard_normal((len(pos), 2 * hs)).astype(F)
    z = np.zeros(x.shape)
    ref, bar, nat, extra = rotate_ref(x.astype(np.float64), z, np.abs(x.astype(np.float64)), z, table, pos, np.arange(2), hs)
    f32 = np.stack([rope_rotate(x[i].reshape(2, hs), table, int(pos[i]), np.arange(2)).reshape(-1) for i in range(len(pos))])
    assert err_level(f32, ref, bar, nat, extra)[0] <= 1.0


def _silu_case(seed=12):
    rng = np.random.default_rng(seed)
    g = (rng.standard_normal((64, 512)) * np.logspace(-1, 2.2, 512)[None, :]).astype(F)  # |g| up to a few hundred
    u = rng.standard_normal((64, 512)).astype(F)
    u[:, 7] = 0.0
    return g, u


def _silu_f32(g, u):
    """the kernel's arithmetic with the correctly rounded exponential and division, in float32"""
    with np.errstate(over="ignore"):
        d = (F(1) + np.exp(-g.astype(F))).astype(F)
    return ((g / d).astype(F) * u).astype(F)


def test_silu_bar_accepts_f32_arithmetic():
    g, u = _silu_case()
    bad, near, zeros = silu_check(bf16_bits(_silu_f32(g, u)), g, u)
    print("f32 SiLU * up: %d rejected, %d ambiguous, %d zero" % (bad, near, zeros))
    assert bad == 0
    # __fdividef's 0 below g = -87 is accepted there and only there
    out = bf16_bits(_silu_f32(g, u))
    out[g < SILU_ZERO_G] = 0
    assert silu_check(out, g, u)[0] == 0
    out2 = bf16_bits(_silu_f32(g, u))
    mid = (g > -80) & (g < -5) & (u != 0)
    out2[mid] = 0
    assert silu_check(out2, g, u)[0] == int(mid.sum())


def test_silu_bar_rejects_defects():
    g, u = _silu_case()
    n = g.size
    f = _silu_f32(g, u)
    for what, out in (("SiLU * up truncated to BF16", (bf16_trunc(f).view(np.uint32) >> 16).astype(np.uint16)),
                      ("gate and up swapped", bf16_bits(_silu_f32(u, g)))):
        bad = silu_check(out, g, u)[0]
        print("%s: %d of %d elements rejected" % (what, bad, n))
        assert 4 * bad >= n, what


def test_attention_bar_with_ambiguity_rejects_defects():
    """at Llama-3-8B-like magnitudes (hs 128, scores of tens), where many elements of P are ambiguous, the bar with its
    allowance still rejects the defects test_gpu_tc_kernels.py shows for the plain emulated bar"""
    rng = np.random.default_rng(13)
    R, pos0, Hq, Hkv, hs = 96, 160, 8, 2, 128
    q = (4.0 * rng.standard_normal((R, Hq, hs))).astype(F)
    k = (2.0 * rng.standard_normal((pos0 + R, Hkv, hs))).astype(F)
    v = rng.standard_normal((pos0 + R, Hkv, hs)).astype(F)
    group, scale = Hq // Hkv, float(F(1 / np.sqrt(hs)))
    ref, amb = attn_emulated(q, k, v, pos0, group, scale, ambiguity=True)
    print("ambiguous outputs: %d of %d, worst allowance %.2e of max|V|" % ((amb > 0).sum(), amb.size, amb.max()))
    assert attn_check(ref, ref, amb, v, group)[0] == 0.0
    defects = {
        "causal limit + 1": attn_emulated(q, k, v, pos0, group, scale, causal_shift=1),
        "causal limit - 1": attn_emulated(q, k, v, pos0, group, scale, causal_shift=-1),
        "wrong KV head": attn_emulated(q, k, v, pos0, group, scale, head_map=(np.arange(Hq) // group + 1) % Hkv),
        "rescale skipped on tile 1": attn_emulated(q, k, v, pos0, group, scale, skip_rescale_tile=1),
    }
    for what, o in defects.items():
        _ratio(attn_check(o, ref, amb, v, group)[0], what)
