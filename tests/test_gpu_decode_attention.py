"""The decode attention kernels pinned against float64 references at their edges.  Four implementations serve a decode step:

  pd     the flat task inside the persistent kernel (jl_attn_flat.cuh via pd_attention, jl_pdecode.cu): one session per step
  flat   the flat task as its own launch (flat_decode_attention_kernel, jl_attention.cu): 2..16 rows (or more at the 32-split cap)
  tiled  the tiled online-softmax task (fused_decode_attention_kernel -> attention_task, jl_attn_task.cuh), merged by the last CTA
  perop  rope_kv_append + paged_attention + attention_merge (jl_attention.cu): exact prefill, and tensor-core prefill where the
         tensor-core attention does not apply (head size 32, groups that are not powers of two)

Every case runs one-layer models (or checks the last layer of an 8-layer one), places K/V rows in the session's pages with kv_load
(random rows everywhere, so any read past the causal limit or of a stale row shows), runs a step, and reads back q / k / v / the
attention output (debug_read) and the pages (kv_save).

Append.  The stored K row of the new position must equal the raw k rotated in float32 with one rounding per operation (the pair
at index pos * hs / 2 + kv_head * hs + j of the table, for q and k alike), the stored V row the raw v, both RNE-rounded to BF16 with
BF16 KV.  Every other row of the checked layer's pages must be unchanged.  Both are compared bit for bit.

Output.  The reference is softmax(scale * q.K[0..pos]) . V in float64 of the rotated q and of K / V as read back from the pages.
Per element: |o - ref| <= ATTN_TAU * max|V| * max(1, max|s|), with max|V| over the visible rows of the query head's KV head and
max|s| the largest |score| of the head: f32 scores carry an error proportional to their size, which the crafted +-80 scores make
visible.  A row at position 0 must return its own V row exactly (the one-element softmax is 1, and 1 * v / 1 rounds to v).

Measured on an NVIDIA H100 80GB HBM3 (SXM, 700 W power limit, 1980 MHz max SM clock) over every case below, as
|o - ref| / (max|V| * max(1, max|s|)), and in brackets as plain |o - ref| / max|V|:
  pd 8.7e-8 (1.1e-6), flat 1.2e-7 (1.5e-6), tiled 6.8e-8 (2.0e-6), perop 1.1e-7 (8.0e-6, at the crafted +-80 scores).
ATTN_TAU = 2**-20 = 9.5e-7 leaves 8x headroom over the worst of them (err/bar 0.09 pd, 0.12 flat, 0.07 tiled, 0.11 perop).
The whole file takes about 100 s on that card.

Host selection.  host_rule() restates how the library picks the variant and the split count (run_decode's split buckets,
attention()'s bound, flat_decode_ok, fill_pd, pick_splits); every case is labelled with its variant and split count, and
test_case_matrix_covers_the_edges checks the labels, on the CPU, against the edges this file is meant to reach.  On the GPU each
decode case also asserts decode_mode().  JL_ATTN_FLAT is read once per process, so the flat variant is always on here.

GQA groups 5 and 7 (10 and 14 query heads over 2 KV heads) finalize and run on the tiled and per-op paths like 3 and 6.

The CPU tests at the end show, with the same reference functions, that the bar rejects each defect it is there to catch by at
least 4x.  Importing this file does not load the CUDA library.
"""
import ctypes as C
import os
import tempfile
import zlib

import numpy as np
import pytest

from jlama_b200 import tensor as T  # numpy only
from jlama_b200.native import F32, MODEL_NO_GRAPH, MODEL_NO_PERSISTENT

gpu = pytest.mark.gpu

ATTN_TAU = 2.0 ** -20
SHARP = 4.0
MAX_SPLITS = 32
SPLIT_BUCKETS = (1, 2, 3, 4, 6, 8, 12, 16, 24, 32)
FA_MAX_POS = 1024
PAGE_BYTES = 1 << 23
H100_SMS = 132  # the labels below are computed for an H100 SXM; the GPU run recomputes them for the card it has


# ---- references (numpy only) ---------------------------------------------------------------------------------------------
def rope_rotate(x, table, pos, kv_of):
    """x [heads, hs] rotated with the pairs at index pos * hs / 2 + kv_of[h] * hs + j of `table` (flat [.., 2] float32):
    x0 * c - x1 * s and x0 * s + x1 * c in float32, one rounding per operation"""
    hs = x.shape[1]
    hp = hs // 2
    tab = np.asarray(table, dtype=np.float32).reshape(-1, 2)
    idx = pos * hp + np.asarray(kv_of)[:, None] * hs + np.arange(hp)[None, :]
    c, s = tab[idx, 0], tab[idx, 1]
    x0, x1 = np.asarray(x[:, :hp], dtype=np.float32), np.asarray(x[:, hp:], dtype=np.float32)
    return np.concatenate([x0 * c - x1 * s, x0 * s + x1 * c], axis=1).astype(np.float32)


def attn_ref(q, K, V, group, scale, head_map=None, weight=None):
    """one row: q [Hq, hs] (rotated), K / V [n, Hkv, hs] (the positions the row sees).  softmax(scale * q.K^T) . V in float64;
    returns (out [Hq, hs], scores [Hq, n]).  head_map / weight mutate the computation (the sharpness tests): query heads mapped
    to other KV heads, per-position multiplicities (0 drops a position, 2 counts it twice)."""
    Hq = q.shape[0]
    kv_of = np.arange(Hq) // group if head_map is None else np.asarray(head_map)
    k64, v64 = K.astype(np.float64)[:, kv_of], V.astype(np.float64)[:, kv_of]
    s = np.einsum("hd,nhd->hn", q.astype(np.float64), k64) * scale
    p = np.exp(s - s.max(axis=1, keepdims=True))
    if weight is not None:
        p = p * np.asarray(weight, dtype=np.float64)[None, :]
    return np.einsum("hn,nhd->hd", p, v64) / p.sum(axis=1)[:, None], s


def attn_tiled(q, K, V, group, scale, tile, skip_rescale_tile=None):
    """online softmax over `tile`-position tiles in float64; skip_rescale_tile: that tile leaves the running sums unscaled"""
    Hq = q.shape[0]
    kv_of = np.arange(Hq) // group
    k64, v64 = K.astype(np.float64)[:, kv_of], V.astype(np.float64)[:, kv_of]
    m = np.full(Hq, -np.inf)
    l = np.zeros(Hq)
    o = np.zeros(q.shape)
    for j, t0 in enumerate(range(0, K.shape[0], tile)):
        s = np.einsum("hd,nhd->hn", q.astype(np.float64), k64[t0:t0 + tile]) * scale
        mx = np.maximum(m, s.max(axis=1))
        corr = np.ones(Hq) if j == skip_rescale_tile else np.exp(m - mx)
        e = np.exp(s - mx[:, None])
        l = l * corr + e.sum(axis=1)
        o = o * corr[:, None] + np.einsum("hn,nhd->hd", e, v64[t0:t0 + tile])
        m = mx
    return o / l[:, None]


def attn_err(o, ref, s, V, group):
    """(max over elements of |o - ref| / (ATTN_TAU * max|V| * max(1, max|s|)), max of |o - ref| / max|V|); max|V| over the
    visible rows of the query head's KV head, max|s| over the head's scores"""
    Hq = ref.shape[0]
    vmax = np.abs(V.astype(np.float64)).max(axis=(0, 2))[np.arange(Hq) // group]
    vmax = np.where(vmax > 0, vmax, np.finfo(np.float64).tiny)
    smax = np.maximum(1.0, np.abs(s).max(axis=1))
    d = np.abs(np.asarray(o, dtype=np.float64) - ref)
    return float((d / (vmax * smax)[:, None]).max() / ATTN_TAU), float((d / vmax[:, None]).max())


def split_ranges(n, splits, align):
    """[t0, t1) of every split of an n-position context, as the kernels cut it (per split rounded up to `align` positions)"""
    per = -(-(-(-n // splits)) // align) * align
    return [(s * per, min(n, s * per + per)) for s in range(splits)]


# ---- the host's selection rule, restated ------------------------------------------------------------------------------------
def kv_page_geometry(layers, context_length, kv_len, esz, max_bytes=PAGE_BYTES):
    """jl_kv_page_geometry: (layers per page, context positions per page)"""
    s = 2 * esz * kv_len
    opt_l, opt_c, best = 1, 1, 0
    for x in range(layers, 0, -1):
        y = max_bytes // (x * s)
        if 1 <= y <= context_length:
            if x * y > best:
                opt_l, opt_c, best = x, y, x * y
            if x * y < best:
                break
    return opt_l, opt_c


def pd_cap(kv_heads, sm):
    return min(sm // kv_heads, MAX_SPLITS)


def pd_eligible(cfg, flags, max_context, sm):
    """persistent decode (use_pd): Llama, Q8 activations, one quantised weight dtype, power-of-two group, head size 32/64/128,
    and at most 992 positions per split at the reserved context (jl_model_finalize)"""
    hs, group = cfg["E"] // cfg["heads"], cfg["heads"] // cfg["kv_heads"]
    if cfg.get("gpt2") or flags & (MODEL_NO_PERSISTENT | MODEL_NO_GRAPH) or group & (group - 1) or hs not in (32, 64, 128):
        return False
    cap = pd_cap(cfg["kv_heads"], sm)
    return -(-max_context // cap) <= FA_MAX_POS - 32


def pd_splits(pos, kv_heads, sm):
    """fill_pd (token 0 of a launch) and the kernel's recompute (later tokens): one split per 64 positions up to the cap"""
    return max(1, min(-(-(pos + 1) // 64), pd_cap(kv_heads, sm)))


def decode_bucket(n, max_pos):
    """run_decode: one split per 64 positions (per 64 * n with n rows), bucketed"""
    s = -(-(max_pos + 1) // 64)
    if n > 1:
        s = -(-s // n)
    return min(next((b for b in SPLIT_BUCKETS if b >= s), MAX_SPLITS), MAX_SPLITS)


def pick_splits(max_pos, rows, kv_heads, sm):
    want = -(-(max_pos + 1) // 128)
    fill = max(1, (sm * 2) // max(1, kv_heads * rows))
    s = max(1, min(want, fill, MAX_SPLITS))
    b = 1
    while b < s:
        b <<= 1
    return min(b, MAX_SPLITS)


def tc_prefill_ok(cfg):
    """tensor-core prefill GEMMs (tc_ok) for Q4 weights on one rank"""
    E, hs = cfg["E"], cfg["E"] // cfg["heads"]
    return not cfg.get("gpt2") and all(v % 128 == 0 for v in (E, cfg["H"], E, cfg["kv_heads"] * hs))


def host_rule(case, rows, sm):
    """(variant, splits) the library picks for one step of `case` (rows: [(session, position)] of a decode step, [(session,
    pos0, count)] of a prefill pass)"""
    cfg = CFGS[case["cfg"]]
    hs, Hkv = cfg["E"] // cfg["heads"], cfg["kv_heads"]
    group = cfg["heads"] // Hkv
    mc = max_context_of(case, sm)
    if case["kind"] == "prefill":
        n = sum(r for _, _, r in rows)
        max_pos = max(p + r - 1 for _, p, r in rows)
        if case.get("ptc") and tc_prefill_ok(cfg) and len(rows) == 1 and n >= 16:
            assert hs not in (64, 128) or group & (group - 1), "the tensor-core attention would take this pass"
        return "perop", pick_splits(max_pos, n, Hkv, sm)
    n = len(rows)
    max_pos = max(p for _, p in rows)
    if n == 1 and pd_eligible(cfg, case.get("flags", 0), mc, sm):
        return "pd", pd_splits(max_pos, Hkv, sm)
    splits = decode_bucket(n, max_pos)
    bound = mc - 1 if splits >= MAX_SPLITS else splits * 64 * n - 1
    per = -(-(-(-(bound + 1) // splits)) // 32) * 32
    if n >= 2 and not group & (group - 1) and hs in (64, 128) and per <= FA_MAX_POS:
        return "flat", splits
    return "tiled", splits


# ---- the case matrix ------------------------------------------------------------------------------------------------------
def _llama(E, heads, kv_heads, layers=1):
    return dict(E=E, heads=heads, kv_heads=kv_heads, layers=layers, H=256, vocab=256, ctx=32768)


CFGS = {
    "hs32-g1": _llama(256, 8, 8),
    "hs32-g2": _llama(256, 8, 4),
    "hs32-g3": _llama(384, 12, 4),
    "hs32-g4": _llama(256, 8, 2),
    "hs32-g6": _llama(384, 12, 2),
    "hs32-g8": _llama(256, 8, 1),
    "hs64-g1": _llama(512, 8, 8),
    "hs64-g2": _llama(512, 8, 4),
    "hs64-g3": _llama(768, 12, 4),
    "hs64-g4": _llama(512, 8, 2),
    "hs64-g5": _llama(640, 10, 2),
    "hs64-g6": _llama(768, 12, 2),
    "hs64-g7": _llama(896, 14, 2),
    "hs64-g8": _llama(512, 8, 1),
    "hs128-g2": _llama(1024, 8, 4),
    "hs128-g4": _llama(1024, 8, 2),
    "hs128-g8": _llama(1024, 8, 1),
    # 8 layers of 1024-wide KV rows: 8 layers and 128 (F32) / 256 (BF16) positions per page, so the checked layer 7 sits at an
    # offset inside its page and page boundaries fall inside the attended context
    "hs128-g1-8L": _llama(1024, 8, 8, layers=8),
    # GPT-2: identity RoPE, multi-head, head size 32, one position per page
    "gpt2-hs32": dict(E=128, heads=4, kv_heads=4, layers=1, H=512, vocab=256, ctx=1024, gpt2=True),
}

TILE_EDGES = [0, 1, 31, 32, 33, 63, 64, 65]


def _spread(n, top, seed):
    """n distinct sessions at different positions in [0, top], the first at top"""
    rng = np.random.default_rng(seed)
    pos = [top] + sorted(rng.choice(top, n - 1, replace=False).tolist(), reverse=True)
    return [(s, int(p)) for s, p in enumerate(pos)]


def _singles(positions, session=0):
    return [[(session, p)] for p in positions]


CASES = [
    # ---- pd: one session per step through the persistent kernel ----
    dict(id="pd-hs32-g1-F32-tiles", cfg="hs32-g1", kind="decode", variant="pd", steps=_singles(TILE_EDGES + [127, 128, 129])),
    dict(id="pd-hs32-g8-BF16-cap-page-per-row", cfg="hs32-g8", kvdt="BF16", kind="decode", variant="pd",
         steps=_singles([0, 1, 65, 1983, 1984, 2047, 2048, 2049])),
    dict(id="pd-hs64-g2-F32-buckets", cfg="hs64-g2", kind="decode", variant="pd", steps=_singles([0, 63, 64, 65, 1023, 1024, 1025, 2049])),
    dict(id="pd-hs64-g4-BF16-tiles-cap", cfg="hs64-g4", kvdt="BF16", kind="decode", variant="pd", steps=_singles(TILE_EDGES + [4000])),
    dict(id="pd-hs128-g4-F32-cap", cfg="hs128-g4", kind="decode", variant="pd", steps=_singles([0, 31, 32, 33, 2047, 2048, 2049, 6000])),
    dict(id="pd-hs128-g8-BF16", cfg="hs128-g8", kvdt="BF16", kind="decode", variant="pd", steps=_singles([0, 65, 3000])),
    dict(id="pd-hs128-g2-F32", cfg="hs128-g2", kind="decode", variant="pd", steps=_singles([1, 500])),
    dict(id="pd-hs64-g8-F32", cfg="hs64-g8", kind="decode", variant="pd", steps=_singles([0, 129, 2500])),
    # max_context = 992 * cap: the last position puts 992 positions in every split
    dict(id="pd-hs32-g1-F32-992-per-split", cfg="hs32-g1", kind="decode", variant="pd", max_context="pd992", steps="pd992-last"),
    dict(id="pd-hs128-g1-8L-F32-page-boundary", cfg="hs128-g1-8L", kind="decode", variant="pd", max_context=2048,
         steps=_singles([126, 127, 128, 129, 255, 256, 257])),
    dict(id="pd-hs128-g1-8L-BF16-page-boundary", cfg="hs128-g1-8L", kvdt="BF16", kind="decode", variant="pd", max_context=2048,
         steps=_singles([255, 256, 257])),
    dict(id="pd-hs64-g4-F32-rewind", cfg="hs64-g4", kind="decode", variant="pd", init={0: 600}, steps=_singles([100, 333])),
    dict(id="pd-hs64-g4-F32-resident-crossing-64", cfg="hs64-g4", kind="resident", variant="pd", steps=[(0, 60, 16)]),
    dict(id="pd-hs32-g2-BF16-resident-crossing-128", cfg="hs32-g2", kvdt="BF16", kind="resident", variant="pd", steps=[(0, 120, 16)]),
    # ---- flat: 2..16 rows (or 17+ at the 32-split cap) as its own launch ----
    dict(id="flat-hs64-g1-F32-tiles", cfg="hs64-g1", kind="decode", variant="flat",
         steps=[[(0, 0), (1, 31)], [(0, 32), (1, 33), (2, 1)], [(0, 63), (1, 64)], [(0, 65), (1, 0), (2, 64)]]),
    dict(id="flat-hs64-g2-BF16-3-8-rows", cfg="hs64-g2", kvdt="BF16", kind="decode", variant="flat",
         steps=[_spread(3, 127, 1), _spread(8, 129, 2), _spread(8, 1000, 3)]),
    dict(id="flat-hs128-g4-F32-16-rows", cfg="hs128-g4", kind="decode", variant="flat", steps=[_spread(16, 1100, 4), _spread(16, 65, 5)]),
    dict(id="flat-hs128-g8-BF16-empty-splits", cfg="hs128-g8", kvdt="BF16", kind="decode", variant="flat",
         steps=[[(0, 1000), (1, 3), (2, 0), (3, 200)]]),
    dict(id="flat-hs64-g8-F32", cfg="hs64-g8", kind="decode", variant="flat", steps=[[(0, 127), (1, 128)], [(0, 255), (1, 3)]]),
    dict(id="flat-hs128-g2-F32", cfg="hs128-g2", kind="decode", variant="flat", steps=[[(0, 383), (1, 384), (2, 385)]]),
    # the 32-split cap with max_context 32768: 1024 positions per split
    dict(id="flat-hs64-g4-F32-1024-per-split", cfg="hs64-g4", kind="decode", variant="flat", max_context=32768,
         steps=[[(0, 32767), (1, 5)]]),
    dict(id="flat-hs64-g4-BF16-1024-per-split", cfg="hs64-g4", kvdt="BF16", kind="decode", variant="flat", max_context=32768,
         steps=[[(0, 32766), (1, 0)]]),
    dict(id="flat-hs64-g4-F32-17-rows-at-cap", cfg="hs64-g4", kind="decode", variant="flat", max_context=32768,
         steps=[[(0, 30000)] + [(s, 3 * s) for s in range(1, 17)]]),
    dict(id="flat-hs128-g1-8L-F32-page-boundary", cfg="hs128-g1-8L", kind="decode", variant="flat", max_context=2048,
         steps=[[(0, 127), (1, 128), (2, 129)], [(0, 255), (1, 256), (2, 0)]]),
    dict(id="flat-hs128-g1-8L-BF16-page-boundary", cfg="hs128-g1-8L", kvdt="BF16", kind="decode", variant="flat", max_context=2048,
         steps=[[(0, 255), (1, 256), (2, 257)]]),
    # session 1 forked from session 0 at 300 positions: context pages 0 and 1 shared, page 2 copied
    dict(id="flat-hs128-g1-8L-F32-fork", cfg="hs128-g1-8L", kind="decode", variant="flat", max_context=2048, fork=(0, 1, 300),
         steps=[[(1, 300), (2, 40), (0, 299)], [(1, 301), (0, 302)]]),
    dict(id="flat-hs64-g4-F32-rewind", cfg="hs64-g4", kind="decode", variant="flat", init={0: 600, 1: 50},
         steps=[[(0, 100), (1, 5)]]),
    # ---- tiled ----
    dict(id="tiled-hs64-g4-F32-1-row-tiles-buckets", cfg="hs64-g4", kind="decode", variant="tiled", flags=MODEL_NO_PERSISTENT,
         max_context=16384, steps=_singles(TILE_EDGES + [191, 192, 193, 1599, 8191, 8192, 8193])),
    dict(id="tiled-hs128-g2-BF16-1-row-eager", cfg="hs128-g2", kvdt="BF16", kind="decode", variant="tiled",
         flags=MODEL_NO_PERSISTENT | MODEL_NO_GRAPH, steps=_singles([0, 64, 383, 384, 385, 3000])),
    dict(id="tiled-hs32-g1-F32", cfg="hs32-g1", kind="decode", variant="tiled", steps=[_spread(2, 65, 6), _spread(3, 700, 7)]),
    dict(id="tiled-hs32-g2-BF16", cfg="hs32-g2", kind="decode", variant="tiled", steps=[[(0, 0), (1, 33)], _spread(3, 129, 8)]),
    dict(id="tiled-hs32-g4-F32-cap", cfg="hs32-g4", kind="decode", variant="tiled", steps=[[(0, 6200), (1, 0), (2, 64)]]),
    dict(id="tiled-hs32-g8-BF16", cfg="hs32-g8", kind="decode", variant="tiled", steps=[_spread(2, 300, 9)]),
    dict(id="tiled-hs32-g3-F32", cfg="hs32-g3", kind="decode", variant="tiled", steps=_singles([0, 33, 64, 65, 700]) + [_spread(3, 130, 10)]),
    dict(id="tiled-hs32-g6-BF16", cfg="hs32-g6", kind="decode", variant="tiled", steps=_singles([0, 31, 2100]) + [_spread(3, 64, 11)]),
    dict(id="tiled-hs64-g3-F32", cfg="hs64-g3", kind="decode", variant="tiled", steps=_singles([0, 1, 32, 63, 64, 1000]) + [_spread(4, 400, 12)]),
    dict(id="tiled-hs64-g6-BF16", cfg="hs64-g6", kind="decode", variant="tiled", steps=_singles([0, 65, 2049]) + [_spread(3, 1500, 13)]),
    dict(id="tiled-hs64-g5-F32", cfg="hs64-g5", kind="decode", variant="tiled", steps=_singles([0, 33, 500]) + [_spread(2, 64, 14)]),
    dict(id="tiled-hs64-g7-BF16", cfg="hs64-g7", kind="decode", variant="tiled", steps=_singles([0, 32, 700]) + [_spread(3, 128, 15)]),
    dict(id="tiled-hs128-g8-F32-1-row", cfg="hs128-g8", kind="decode", variant="tiled", flags=MODEL_NO_PERSISTENT, steps=_singles([0, 33, 2000])),
    dict(id="tiled-hs64-g2-F32-17-rows", cfg="hs64-g2", kind="decode", variant="tiled", steps=[_spread(17, 2000, 16), _spread(17, 64, 17)]),
    dict(id="tiled-hs64-g4-BF16-64-rows", cfg="hs64-g4", kvdt="BF16", kind="decode", variant="tiled", steps=[_spread(64, 3000, 18)]),
    dict(id="tiled-gpt2-hs32-F32-page-per-row", cfg="gpt2-hs32", kind="decode", variant="tiled", max_context=1024,
         steps=_singles([0, 1, 31, 32, 33, 63, 64, 65, 500, 1023]) + [_spread(3, 700, 19)]),
    dict(id="tiled-gpt2-hs32-BF16", cfg="gpt2-hs32", kvdt="BF16", kind="decode", variant="tiled", max_context=1024,
         steps=[_spread(2, 129, 20)]),
    # ---- perop: rope_kv_append + paged_attention (+ merge) ----
    dict(id="perop-hs64-g4-F32-rows-cap", cfg="hs64-g4", kind="prefill", variant="perop",
         steps=[[(0, 0, 1), (1, 127, 1), (2, 128, 1), (3, 4000, 1)]]),
    dict(id="perop-hs64-g2-BF16-128-boundaries", cfg="hs64-g2", kvdt="BF16", kind="prefill", variant="perop",
         steps=[[(0, p, 1)] for p in (0, 1, 63, 64, 65, 127, 128, 255, 256, 257, 383, 384, 4095, 4096)]),
    dict(id="perop-hs64-g4-F32-chunks", cfg="hs64-g4", kind="prefill", variant="perop", steps=[[(0, 0, 70)], [(0, 60, 5)], [(1, 120, 140)]]),
    dict(id="perop-hs32-g1-F32-tc-prefill", cfg="hs32-g1", kind="prefill", variant="perop", ptc=1, steps=[[(0, 100, 20)], [(0, 0, 1)]]),
    dict(id="perop-hs32-g3-BF16-tc-prefill", cfg="hs32-g3", kvdt="BF16", kind="prefill", variant="perop", ptc=1, steps=[[(0, 30, 40)]]),
    dict(id="perop-hs64-g3-F32-tc-prefill", cfg="hs64-g3", kind="prefill", variant="perop", ptc=1, steps=[[(0, 60, 20)], [(0, 1000, 16)]]),
    dict(id="perop-hs64-g6-BF16-tc-prefill", cfg="hs64-g6", kvdt="BF16", kind="prefill", variant="perop", ptc=1, steps=[[(0, 200, 17)]]),
    dict(id="perop-hs32-g6-F32", cfg="hs32-g6", kind="prefill", variant="perop", steps=[[(0, 0, 1), (1, 65, 1), (2, 5000, 1)]]),
    dict(id="perop-hs64-g5-BF16", cfg="hs64-g5", kind="prefill", variant="perop", steps=[[(0, 0, 3), (1, 129, 2)]]),
    dict(id="perop-hs64-g7-F32", cfg="hs64-g7", kind="prefill", variant="perop", steps=[[(0, 250, 10)]]),
    dict(id="perop-hs128-g8-F32", cfg="hs128-g8", kind="prefill", variant="perop", steps=[[(0, 0, 1), (1, 3000, 1)]]),
    dict(id="perop-hs32-g8-BF16", cfg="hs32-g8", kind="prefill", variant="perop", steps=[[(0, 900, 4)]]),
    dict(id="perop-hs128-g1-8L-F32-page-boundary", cfg="hs128-g1-8L", kind="prefill", variant="perop", max_context=2048,
         steps=[[(0, 127, 1), (1, 128, 1), (2, 129, 1)], [(0, 250, 10)]]),
    dict(id="perop-gpt2-hs32-F32", cfg="gpt2-hs32", kind="prefill", variant="perop", max_context=1024,
         steps=[[(0, 0, 40)], [(0, 500, 1), (1, 0, 1)]]),
]

# crafted K rows (one-layer models): the kinds and where they run
CRAFT_KINDS = ["late-max", "first-max", "uniform", "underflow", "range80"]
CRAFT_CASES = {
    "pd": dict(cfg="hs64-g4", kind="decode", variant="pd", rows=[(0, 700)]),
    "flat": dict(cfg="hs64-g4", kind="decode", variant="flat", rows=[(0, 700), (1, 300)]),
    "tiled": dict(cfg="hs64-g4", kind="decode", variant="tiled", flags=MODEL_NO_PERSISTENT, rows=[(0, 700)]),
    "tiled-g6": dict(cfg="hs64-g6", kind="decode", variant="tiled", rows=[(0, 700), (1, 300)]),
    "perop": dict(cfg="hs64-g4", kind="prefill", variant="perop", rows=[(0, 700, 1), (1, 300, 1)]),
}


def max_context_of(case, sm):
    mc = case.get("max_context", 8192)
    if mc == "pd992":
        return (FA_MAX_POS - 32) * pd_cap(CFGS[case["cfg"]]["kv_heads"], sm)
    return mc


def steps_of(case, sm):
    if case["steps"] == "pd992-last":
        return [[(0, max_context_of(case, sm) - 1)]]
    return case["steps"]


def step_rows(case, step):
    """[(session, position)] of every row of a step, in the order of the step's activation rows"""
    if case["kind"] == "prefill":
        return [(s, p0 + r) for s, p0, cnt in step for r in range(cnt)]
    if case["kind"] == "resident":
        s, p0, cnt = step
        return [(s, p0 + r) for r in range(cnt)]
    return list(step)


def case_label(case, sm=H100_SMS):
    cfg = CFGS[case["cfg"]]
    labels = []
    for step in steps_of(case, sm):
        if case["kind"] == "resident":
            s, p0, cnt = step
            a, b = pd_splits(p0, cfg["kv_heads"], sm), pd_splits(p0 + cnt - 1, cfg["kv_heads"], sm)
            labels.append("pd splits %d->%d pos %d..%d" % (a, b, p0, p0 + cnt - 1))
            continue
        v, s = host_rule(case, step, sm)
        labels.append("%s splits %d rows %d" % (v, s, len(step_rows(case, step))))
    return "; ".join(labels)


# ---- GPU harness ----------------------------------------------------------------------------------------------------------
class Harness:
    """one model of a case: its page geometry, RoPE table, and what every page of the checked layer must hold"""

    def __init__(self, cuda_ctx, case, cfg_name=None, kvdt=None, flags=None, max_context=None, max_sessions=None):
        from jlama_b200 import native, synth
        from jlama_b200.model import GPT2Model, LlamaModel
        self.ctx, self.lib = cuda_ctx, cuda_ctx.lib
        spec = CFGS[cfg_name or case["cfg"]]
        self.spec = spec
        self.kvdt = getattr(native, kvdt or case.get("kvdt", "F32"))
        flags = case.get("flags", 0) if flags is None else flags
        self.max_context = max_context or max_context_of(case, cuda_ctx.sm_count)
        self.hs = spec["E"] // spec["heads"]
        self.Hq, self.Hkv = spec["heads"], spec["kv_heads"]
        self.group, self.L = self.Hq // self.Hkv, spec["layers"] - 1
        self.kv_len, self.attn_seg = self.Hkv * self.hs, spec["E"]
        self.scale = float(np.float32(1.0 / np.sqrt(self.hs)))
        if spec.get("gpt2"):
            cfg = synth.get_gpt2_config("gpt2-tiny")
            cfg.update(E=spec["E"], heads=spec["heads"], kv_heads=spec["heads"], layers=spec["layers"], H=spec["H"], vocab=spec["vocab"],
                       ctx=spec["ctx"])
            self.gm = GPT2Model(cuda_ctx, cfg, synth.make_gpt2_weights(cfg), kv_dtype=self.kvdt, max_sessions=max_sessions,
                                max_context=self.max_context, flags=flags)
            self.table = np.tile(np.array([1.0, 0.0], dtype=np.float32), (cfg["ctx"] + 2 * self.Hkv) * self.hs // 2)
        else:
            cfg = synth.get_config("tiny", E=spec["E"], H=spec["H"], heads=spec["heads"], kv_heads=spec["kv_heads"], layers=spec["layers"],
                                   vocab=spec["vocab"], ctx=spec["ctx"])
            self.gm = LlamaModel(cuda_ctx, cfg, synth.make_weights(cfg, mode="direct"), kv_dtype=self.kvdt, max_sessions=max_sessions,
                                 max_context=self.max_context, flags=flags, prefill_tensor_core=case.get("ptc", 0))
            positions = cfg["ctx"] + 2 * self.Hkv
            self.table = np.empty(positions * self.hs, dtype=np.float32)
            assert self.lib.jl_precompute_freqs_cis(self.hs, positions, cfg["rope_theta"], cfg.get("rope_scale", 1.0),
                                                    self.table.ctypes.data_as(C.c_void_p)) == 0
        self.cfg = cfg
        self.esz = 4 if self.kvdt == F32 else 2
        lpp, cpp = C.c_int(), C.c_int()
        assert self.lib.jl_kv_page_geometry(cfg["layers"], cfg["ctx"], self.kv_len, self.esz, PAGE_BYTES, C.byref(lpp), C.byref(cpp)) == 0
        assert (lpp.value, cpp.value) == kv_page_geometry(cfg["layers"], cfg["ctx"], self.kv_len, self.esz)
        assert lpp.value == cfg["layers"], "one layer page: every page file holds all layers"
        self.lpp, self.cpp = lpp.value, cpp.value
        self.shape = (self.lpp, 2, self.cpp, self.kv_len)
        self.raw = np.uint32 if self.kvdt == F32 else np.uint16
        self.expect = {}  # session -> [page raw arrays, by context page]
        self.rng = np.random.default_rng(zlib.crc32(case["id"].encode()))
        self.tmp = tempfile.TemporaryDirectory()

    def close(self):
        self.gm.close()
        self.tmp.cleanup()

    # -- raw page values
    def to_raw(self, x):
        x = np.asarray(x, dtype=np.float32)
        return x.view(np.uint32) if self.kvdt == F32 else T.float32_to_bfloat16(x)

    def to_f32(self, raw):
        return raw.view(np.float32) if self.kvdt == F32 else T.bfloat16_to_float32(raw)

    def k_sigma(self):
        """K rows of scores with a spread of about 3 for queries of the synthetic weights (|q| ~ 0.02 sqrt(E) per element)"""
        return 3.0 / (0.02 * np.sqrt(self.spec["E"]))

    def random_page(self):
        x = self.rng.standard_normal(self.shape, dtype=np.float32)
        x[:, 0] *= np.float32(self.k_sigma())
        return self.to_raw(x)

    def craft(self, session, upto):
        """random K / V in every row of the pages holding positions 0 .. upto (all layers), loaded with kv_load"""
        self.gm.reset_session(session)
        pages = min(upto + 1 + 2 * self.cpp, self.max_context) // self.cpp  # and a few rows past the last position
        self.expect[session] = [self.random_page() for _ in range(max(pages, upto // self.cpp + 1))]
        self.load(session)

    def load(self, session):
        d = tempfile.mkdtemp(dir=self.tmp.name)
        for cp, page in enumerate(self.expect[session]):
            page.tofile(os.path.join(d, "s-L0C%d.page" % cp))
        self.gm.reset_session(session)
        assert self.gm.kv_load(d, "s", session=session) == len(self.expect[session])
        for f in os.listdir(d):
            os.remove(os.path.join(d, f))

    def read_pages(self, session, n_pages=None):
        """the session's first n_pages (default: as many as expected) as kv_save writes them (through its page table, shared
        pages included)"""
        d = tempfile.mkdtemp(dir=self.tmp.name)
        self.gm.kv_save(d, "s", session=session)
        pages = []
        for cp in range(len(self.expect[session]) if n_pages is None else n_pages):
            f = os.path.join(d, "s-L0C%d.page" % cp)
            pages.append(np.fromfile(f, dtype=self.raw).reshape(self.shape))
            os.remove(f)
        return pages

    def snapshot(self, session, upto):
        self.expect[session] = self.read_pages(session, upto // self.cpp + 1)

    def layer_rows(self, pages, which):
        """[positions, kv_len] float32 of the checked layer"""
        rl = self.L % self.lpp
        return self.to_f32(np.concatenate([p[rl, which] for p in pages], axis=0))

    def append_expected(self, session, pos, k_raw, v_raw):
        """the rows an append of (k, v) at pos must leave in the checked layer"""
        pages = self.expect[session]
        while len(pages) <= pos // self.cpp:
            pages.append(np.zeros(self.shape, dtype=self.raw))  # a page allocated by the step starts zeroed
        k_rot = rope_rotate(k_raw.reshape(self.Hkv, self.hs), self.table, pos, np.arange(self.Hkv)).reshape(-1)
        cp, rc, rl = pos // self.cpp, pos % self.cpp, self.L % self.lpp
        pages[cp][rl, 0, rc] = self.to_raw(k_rot)
        pages[cp][rl, 1, rc] = self.to_raw(v_raw)

    def fork(self, src, dst, positions):
        self.gm.kv_fork(src, [dst], positions)
        pages = [p.copy() for p in self.expect[src][:-(-positions // self.cpp)]]
        part = positions % self.cpp
        if part:
            pages[-1][:, :, part:] = 0  # the copied partial page keeps the rows below the fork point
        self.expect[dst] = pages

    def step(self, kind, step, tokens):
        if kind == "decode":
            self.gm.decode(tokens, [p for _, p in step], sessions=[s for s, _ in step])
        else:
            segs, off = [], 0
            for s, p0, cnt in step:
                segs.append((s, tokens[off:off + cnt], p0))
                off += cnt
            self.gm.batch_forward_multi(segs)

    def read_step(self, M):
        return (self.gm.debug_read(2, M * self.attn_seg).reshape(M, self.Hq, self.hs),
                self.gm.debug_read(3, M * self.kv_len).reshape(M, self.kv_len),
                self.gm.debug_read(4, M * self.kv_len).reshape(M, self.kv_len),
                self.gm.debug_read(5, M * self.attn_seg).reshape(M, self.Hq, self.hs))

    def check_pages(self, sessions, label):
        """every page row of the checked layer as expected, bit for bit; returns {session: (K, V)} float32 [positions, kv_len]"""
        out = {}
        rl = self.L % self.lpp
        for s in sessions:
            got = self.read_pages(s)
            for cp, (g, e) in enumerate(zip(got, self.expect[s])):
                if not np.array_equal(g[rl], e[rl]):
                    which, rc = np.argwhere((g[rl] != e[rl]).any(axis=-1))[0]
                    raise AssertionError("%s: session %d %s row of position %d differs from the expected page content" % (
                        label, s, "KV"[which], cp * self.cpp + rc))
            out[s] = (self.layer_rows(got, 0), self.layer_rows(got, 1))
        return out

    def check_outputs(self, rows, q_rot, att, kv, label, variant):
        worst, level = 0.0, 0.0
        kv_of = np.arange(self.Hq) // self.group
        for i, (s, pos) in enumerate(rows):
            K = kv[s][0][:pos + 1].reshape(pos + 1, self.Hkv, self.hs)
            V = kv[s][1][:pos + 1].reshape(pos + 1, self.Hkv, self.hs)
            ref, sc = attn_ref(q_rot[i], K, V, self.group, self.scale)
            e, lv = attn_err(att[i], ref, sc, V, self.group)
            assert e <= 1.0, "%s: row %d (session %d, position %d): err/bar %.3f, |o - ref|/max|V| %.2e" % (label, i, s, pos, e, lv)
            if pos == 0:
                assert np.array_equal(att[i], V[0][kv_of]), "%s: row %d at position 0 does not return its V row" % (label, i)
            worst, level = max(worst, e), max(level, lv)
        _record(variant, worst, level)
        return worst, level


WORST = {}


def _record(variant, worst, level):
    w, l = WORST.get(variant, (0.0, 0.0))
    WORST[variant] = (max(w, worst), max(l, level))


def _run_rows_step(h, case, step, tokens, variant, label):
    """one decode step or prefill pass: the append and the output of every row"""
    rows = step_rows(case, step)
    M = len(rows)
    h.step(case["kind"], step, tokens)
    q, k, v, att = h.read_step(M)
    if case["kind"] == "decode":
        q_rot = [rope_rotate(q[i], h.table, p, np.arange(h.Hq) // h.group) for i, (_, p) in enumerate(rows)]
    else:
        q_rot = list(q)  # rope_kv_append rotated q in place
    for i, (s, p) in enumerate(rows):
        h.append_expected(s, p, k[i], v[i])
    kv = h.check_pages(sorted({s for s, _ in rows}), label)
    return h.check_outputs(rows, q_rot, att, kv, label, variant)


def _max_rows(case, sm):
    """session -> the largest position any step of the case reaches"""
    top = {}
    for step in steps_of(case, sm):
        rows = step_rows(case, step)
        for s, p in rows:
            top[s] = max(top.get(s, 0), p)
    return top


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_decode_attention_against_float64(cuda_ctx, case):
    sm = cuda_ctx.sm_count
    top = _max_rows(case, sm)
    n_sess = max(top) + 2  # + a scratch session for the probes of the resident case
    h = Harness(cuda_ctx, case, max_sessions=n_sess)
    try:
        fork = case.get("fork")
        for s, upto in sorted(top.items()):
            if fork and s == fork[1]:
                continue
            if s in case.get("init", {}):
                n = case["init"][s]
                h.gm.reset_session(s)
                h.gm.batch_forward(h.rng.integers(0, h.cfg["vocab"], n), 0, session=s)  # real rows: a rewind reads past them
                h.snapshot(s, max(upto, n - 1))
            else:
                h.craft(s, upto)
        if fork:
            h.fork(*fork)
        worst, level = 0.0, 0.0
        for i, step in enumerate(steps_of(case, sm)):
            label = "%s step %d" % (case["id"], i)
            if case["kind"] == "resident":
                w, l = _resident_step(h, step, label)
                variant = "pd"
            else:
                variant, splits = host_rule(case, step, sm)
                assert variant == case["variant"], (label, variant)
                if case["kind"] == "decode":
                    n = len(step)
                    graph = not case.get("flags", 0) & MODEL_NO_GRAPH
                    assert h.gm.decode_mode(n) == (3 if variant == "pd" else (1 if graph else 0)), label
                tokens = h.rng.integers(0, h.cfg["vocab"], len(step_rows(case, step)))
                w, l = _run_rows_step(h, case, step, tokens, variant, label)
                label += " (%s, %d splits, positions %s)" % (variant, splits, [p for _, p in step_rows(case, step)][:8])
            print("%s: err/bar %.3f  |o - ref|/max|V| %.2e" % (label, w, l))
            worst, level = max(worst, w), max(level, l)
    finally:
        h.close()
    print("%s [%s]: worst err/bar %.3f, |o - ref|/max|V| %.2e" % (case["id"], case_label(case, sm), worst, level))


def _resident_step(h, step, label):
    """decode_resident of cnt tokens from p0: every appended row and the last token's output; the raw k / v of each fed token come
    from a one-token probe on the scratch session (for a one-layer model they depend on the token only)"""
    s, p0, cnt = step
    scratch = h.gm.max_sessions - 1
    assert h.gm.decode_mode(1) == 3
    first = int(h.rng.integers(0, h.cfg["vocab"]))
    out = h.gm.decode_resident(first, p0, cnt, session=s)
    q, k, v, att = h.read_step(1)
    fed = [first] + [int(t) for t in out[:-1]]
    probes = {}
    for t in sorted(set(fed)):
        h.gm.reset_session(scratch)
        h.gm.decode([t], [0], sessions=[scratch])
        _, pk, pv, _ = h.read_step(1)
        probes[t] = (pk[0].copy(), pv[0].copy())
    assert np.array_equal(probes[fed[-1]][0], k[0]) and np.array_equal(probes[fed[-1]][1], v[0]), label
    for i, t in enumerate(fed):
        h.append_expected(s, p0 + i, *probes[t])
    kv = h.check_pages([s], label)
    pos = p0 + cnt - 1
    q_rot = [rope_rotate(q[0], h.table, pos, np.arange(h.Hq) // h.group)]
    return h.check_outputs([(s, pos)], q_rot, att, kv, label, "pd")


def _craft_scores(kind, n, rng):
    """target scores of positions 0 .. n - 1 (the rows before the appended one)"""
    t = rng.standard_normal(n)
    if kind == "late-max":
        t[n - 8:] += 15.0  # the maximum in the last tile, after small early tiles: the running max moves late
    elif kind == "first-max":
        t[:8] += 15.0
    elif kind == "underflow":
        t[:32] += 60.0     # split 0 holds the maximum; the middle splits sit ~120 below it: exp underflows to 0 in f32
        t[32:] -= 60.0
    elif kind == "range80":
        t = rng.uniform(-80.0, 80.0, n)
    return t


@gpu
@pytest.mark.parametrize("kind", CRAFT_KINDS)
@pytest.mark.parametrize("where", list(CRAFT_CASES))
def test_decode_attention_crafted_scores(cuda_ctx, where, kind):
    """K rows placed so that every query head of a KV head sees chosen scores: the maximum in the last or the first tile,
    identical keys (a uniform softmax), splits whose merge factor underflows to 0, scores over +-80.  The step runs once on random
    rows to learn q (which depends on the token only), then again on the crafted rows."""
    sm = cuda_ctx.sm_count
    spec = dict(CRAFT_CASES[where])
    rows_spec = spec.pop("rows")
    case = dict(spec, id="crafted-%s-%s" % (where, kind), steps=[rows_spec])
    variant, splits = host_rule(case, rows_spec, sm)
    assert variant == spec["variant"]
    rows = step_rows(case, rows_spec)
    h = Harness(cuda_ctx, case, max_sessions=len(rows) + 1)
    try:
        for s, p in rows:
            h.craft(s, p)
        tokens = h.rng.integers(0, h.cfg["vocab"], len(rows))
        h.step(case["kind"], rows_spec, tokens)
        q = h.read_step(len(rows))[0]
        rl = h.L % h.lpp
        for i, (s, p) in enumerate(rows):
            qr = rope_rotate(q[i], h.table, p, np.arange(h.Hq) // h.group) if case["kind"] == "decode" else q[i]
            tgt = _craft_scores(kind, p, h.rng)
            shared = h.rng.standard_normal(h.hs) * h.k_sigma()
            for kvh in range(h.Hkv):
                Qg = qr[kvh * h.group:(kvh + 1) * h.group].astype(np.float64)
                if kind == "uniform":
                    krows = np.tile(shared, (p, 1))
                else:  # min-norm K rows with Qg . k = target / scale for every head of the group, plus noise outside Qg's span
                    noise = h.rng.standard_normal((p, h.hs)) * 0.1
                    pinv = np.linalg.pinv(Qg)
                    krows = noise - noise @ Qg.T @ pinv.T + np.outer(tgt / h.scale, pinv @ np.ones(h.group))
                for t in range(p):
                    cp, rc = t // h.cpp, t % h.cpp
                    raw = h.expect[s][cp][rl, 0, rc].copy()
                    raw[kvh * h.hs:(kvh + 1) * h.hs] = h.to_raw(krows[t].astype(np.float32))
                    h.expect[s][cp][rl, 0, rc] = raw
            h.load(s)
        w, l = _run_rows_step(h, case, rows_spec, tokens, variant, case["id"])
        print("%s (%s, %d splits): err/bar %.3f  |o - ref|/max|V| %.2e" % (case["id"], variant, splits, w, l))
    finally:
        h.close()


@gpu
def test_zz_report():
    """the worst err/bar and |o - ref| / max|V| per variant over the cases that ran"""
    for v in ("pd", "flat", "tiled", "perop"):
        if v in WORST:
            print("decode attention %-5s: worst err/bar %.3f, |o - ref|/max|V| %.2e (bar %.1e of max|V| * max(1, max|s|))" % (
                v, WORST[v][0], WORST[v][1], ATTN_TAU))


# ---- the case matrix, checked on the CPU ----------------------------------------------------------------------------------
def test_case_labels_match_the_host_rule():
    """every case's declared variant is what the host picks for each of its steps (on a 132-SM H100)"""
    for case in CASES:
        for step in steps_of(case, H100_SMS):
            if case["kind"] == "resident":
                assert pd_eligible(CFGS[case["cfg"]], case.get("flags", 0), max_context_of(case, H100_SMS), H100_SMS)
                continue
            assert host_rule(case, step, H100_SMS)[0] == case["variant"], (case["id"], step)
            rows = step_rows(case, step)
            assert len({s for s, _ in rows}) == len(rows) or case["kind"] == "prefill", case["id"]
    for where, c in CRAFT_CASES.items():
        assert host_rule(dict(c, id=where), c["rows"], H100_SMS)[0] == c["variant"], where


def test_case_matrix_covers_the_edges():
    seen = dict(variant=set(), hs=set(), group=set(), kvdt=set(), caps=set(), per_split=0, page_boundary=False, layer_offset=False,
                crossing=False, rewind=False, fork=False, positions={v: set() for v in ("pd", "flat", "tiled", "perop")})
    batch = set()
    for case in CASES:
        cfg = CFGS[case["cfg"]]
        hs, group = cfg["E"] // cfg["heads"], cfg["heads"] // cfg["kv_heads"]
        kvdt = case.get("kvdt", "F32")
        v = case["variant"]
        seen["variant"].add(v)
        seen["hs"].add(hs)
        seen["group"].add((v, group))
        seen["kvdt"].add((v, kvdt))
        lpp, cpp = kv_page_geometry(cfg["layers"], cfg["ctx"], cfg["kv_heads"] * hs, 4 if kvdt == "F32" else 2)
        seen["layer_offset"] |= (cfg["layers"] - 1) % lpp > 0
        seen["rewind"] |= bool(case.get("init"))
        seen["fork"] |= bool(case.get("fork"))
        for step in steps_of(case, H100_SMS):
            if case["kind"] == "resident":
                s, p0, cnt = step
                seen["crossing"] |= pd_splits(p0, cfg["kv_heads"], H100_SMS) != pd_splits(p0 + cnt - 1, cfg["kv_heads"], H100_SMS)
                continue
            rows = step_rows(case, step)
            _, splits = host_rule(case, step, H100_SMS)
            if splits == MAX_SPLITS:
                seen["caps"].add(v)
            if case["kind"] == "decode":
                batch.add(len(rows))
                assert len(rows) == 1 or len({p for _, p in rows}) == len(rows), (case["id"], "rows at different positions")
            for _, p in rows:
                seen["positions"][v].add(p)
                if p % cpp in (cpp - 1, 0, 1) and p >= cpp - 1 and cpp > 1:
                    seen["page_boundary"] = True
                if v in ("flat", "pd"):
                    per = split_ranges(p + 1, splits, 32)[0][1]
                    seen["per_split"] = max(seen["per_split"], per)
    assert seen["variant"] == {"pd", "flat", "tiled", "perop"}
    assert seen["hs"] == {32, 64, 128}
    for g in (1, 2, 4, 8):
        assert any(gg == g for _, gg in seen["group"]), g
    for g in (3, 5, 6, 7):
        assert ("tiled", g) in seen["group"] and ("perop", g) in seen["group"], g
    for v in ("pd", "flat", "tiled", "perop"):
        assert {(v, "F32"), (v, "BF16")} <= seen["kvdt"], v
        assert {0, 1, 64}.issubset(seen["positions"][v]), v
    for v in ("pd", "tiled"):
        assert set(TILE_EDGES) <= seen["positions"][v], v
    assert seen["caps"] == {"pd", "flat", "tiled", "perop"}
    assert seen["per_split"] > 1000
    assert seen["page_boundary"] and seen["layer_offset"] and seen["crossing"] and seen["rewind"] and seen["fork"]
    assert {2, 3, 8, 16, 17, 64} <= batch
    assert any(CFGS[c["cfg"]].get("gpt2") for c in CASES)


def test_host_rule_edges():
    """the restated rule at its boundaries: 64-position decode buckets, 128-position pick_splits steps, the 32-split cap"""
    assert [decode_bucket(1, p) for p in (63, 64, 191, 192, 1535, 1536, 1599)] == [1, 2, 3, 4, 24, 32, 32]
    assert [pick_splits(p, 1, 2, H100_SMS) for p in (127, 128, 255, 256, 3968, 5000)] == [1, 2, 2, 4, 32, 32]
    assert pd_splits(2047, 2, H100_SMS) == 32 and pd_splits(2048, 2, H100_SMS) == 32 and pd_splits(2047, 8, H100_SMS) == 16
    c = dict(cfg="hs64-g4", kind="decode", max_context=32768)
    assert host_rule(c, [(0, 32767), (1, 0)], H100_SMS) == ("flat", 32)
    assert host_rule(c, [(0, 2400)] + [(s, s) for s in range(1, 17)], H100_SMS)[0] == "tiled"
    assert host_rule(dict(c, max_context=4096), [(0, 60), (1, 1)], H100_SMS) == ("flat", 1)
    assert host_rule(dict(c, max_context=4096), [(0, 60)], H100_SMS) == ("pd", 1)
    assert split_ranges(32768, 32, 32)[-1] == (31744, 32768)


# ---- sharpness of the bar (CPU) ---------------------------------------------------------------------------------------------
def _sharp_case(n=300, Hq=8, Hkv=2, hs=64, hot=None, seed=3):
    """q / K / V of one row at position n - 1; `hot`: positions whose scores (every head) sit 10 above the rest"""
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((Hq, hs)).astype(np.float32)
    K = (rng.standard_normal((n + 1, Hkv, hs)) * 0.25).astype(np.float32)  # row n: a stale row past the causal limit
    V = rng.standard_normal((n + 1, Hkv, hs)).astype(np.float32)
    scale = float(np.float32(1 / np.sqrt(hs)))
    group = Hq // Hkv
    for t in hot or ():
        for kvh in range(Hkv):
            Qg = q[kvh * group:(kvh + 1) * group].astype(np.float64)
            K[t, kvh] = (np.linalg.pinv(Qg) @ np.full(group, 10.0 / scale)).astype(np.float32)
    return q, K, V, group, scale


def _rejects(o, q, K, V, group, scale, what):
    ref, s = attn_ref(q, K, V, group, scale)
    e, _ = attn_err(o, ref, s, V, group)
    assert e >= SHARP, (what, e)


def test_bar_accepts_f32_arithmetic():
    """float32 scores, exponentials and accumulation (what the kernels do) stay within the bar, at ordinary and +-80 scores"""
    for n, spread in ((1000, 1.0), (4000, 1.0), (700, 80.0)):
        q, K, V, group, scale = _sharp_case(n=n)
        K = (K * spread).astype(np.float32)
        ref, s = attn_ref(q, K[:n], V[:n], group, scale)
        kv_of = np.arange(q.shape[0]) // group
        s32 = (np.einsum("hd,nhd->hn", q, K[:n][:, kv_of]).astype(np.float32) * np.float32(scale)).astype(np.float32)
        e = np.exp((s32 - s32.max(axis=1, keepdims=True)).astype(np.float64)).astype(np.float32)
        o = np.zeros(q.shape, dtype=np.float32)
        for t in range(n):  # position by position in f32, as the P.V loops accumulate
            o = (o + e[:, t:t + 1] * V[t][kv_of]).astype(np.float32)
        o = o / e.sum(axis=1, dtype=np.float32)[:, None]
        err, lvl = attn_err(o, ref, s, V[:n], group)
        assert err <= 0.25, (n, spread, err, lvl, np.abs(s).max())


def test_bar_rejects_a_moved_causal_limit():
    n = 300
    q, K, V, group, scale = _sharp_case(n=n, hot=[n])  # the row past the limit would dominate
    o, _ = attn_ref(q, K[:n + 1], V[:n + 1], group, scale)
    _rejects(o, q, K[:n], V[:n], group, scale, "causal limit + 1")
    q, K, V, group, scale = _sharp_case(n=n, hot=[n - 1])  # the current position carries the maximum
    o, _ = attn_ref(q, K[:n - 1], V[:n - 1], group, scale)
    _rejects(o, q, K[:n], V[:n], group, scale, "causal limit - 1")


def test_bar_rejects_a_stale_current_row():
    n = 300
    q, K, V, group, scale = _sharp_case(n=n, hot=[n - 1])
    Ks, Vs = K.copy(), V.copy()
    rng = np.random.default_rng(9)
    Ks[n - 1] = (rng.standard_normal(K[n - 1].shape) * 0.25).astype(np.float32)  # the page's old content
    Vs[n - 1] = rng.standard_normal(V[n - 1].shape).astype(np.float32)
    o, _ = attn_ref(q, Ks[:n], Vs[:n], group, scale)
    _rejects(o, q, K[:n], V[:n], group, scale, "stale current row")


def test_bar_rejects_the_wrong_kv_head():
    n = 300
    q, K, V, group, scale = _sharp_case(n=n, hot=[17])
    Hq, Hkv = q.shape[0], K.shape[1]
    o, _ = attn_ref(q, K[:n], V[:n], group, scale, head_map=(np.arange(Hq) // group + 1) % Hkv)
    _rejects(o, q, K[:n], V[:n], group, scale, "wrong KV head")


@pytest.mark.parametrize("align,splits", [(32, 8), (64, 4)])
def test_bar_rejects_a_dropped_or_doubled_split(align, splits):
    n = 700
    ranges = split_ranges(n, splits, align)
    t0, t1 = ranges[2]
    q, K, V, group, scale = _sharp_case(n=n, hot=[t0 + 5])  # the dropped split holds the maximum
    for label, f in (("dropped", 0.0), ("doubled", 2.0)):
        w = np.ones(n)
        w[t0:t1] = f
        o, _ = attn_ref(q, K[:n], V[:n], group, scale, weight=w)
        _rejects(o, q, K[:n], V[:n], group, scale, "split %s" % label)
    q, K, V, group, scale = _sharp_case(n=n)  # natural data: a doubled split still shows
    w = np.ones(n)
    w[t0:t1] = 2.0
    o, _ = attn_ref(q, K[:n], V[:n], group, scale, weight=w)
    _rejects(o, q, K[:n], V[:n], group, scale, "split doubled, natural data")


@pytest.mark.parametrize("tile", [32, 64])
def test_bar_rejects_a_skipped_rescale(tile):
    n = 300
    q, K, V, group, scale = _sharp_case(n=n, hot=[3 * tile + 2])  # the running maximum moves in tile 3
    o = attn_tiled(q, K[:n], V[:n], group, scale, tile, skip_rescale_tile=3)
    _rejects(o, q, K[:n], V[:n], group, scale, "rescale skipped")
    assert attn_err(attn_tiled(q, K[:n], V[:n], group, scale, tile), *attn_ref(q, K[:n], V[:n], group, scale), V[:n], group)[0] < 1e-3


def test_bar_rejects_rope_indexed_by_the_query_head():
    n, pos = 300, 299
    rng = np.random.default_rng(4)
    hs, Hq, Hkv = 64, 8, 2
    table = np.stack([np.cos(np.arange((pos + 2 * Hq + 4) * hs // 2) * 0.37),
                      np.sin(np.arange((pos + 2 * Hq + 4) * hs // 2) * 0.37)], axis=1).astype(np.float32)
    raw = rng.standard_normal((Hq, hs)).astype(np.float32)
    q, K, V, group, scale = _sharp_case(n=n, Hq=Hq, Hkv=Hkv, hs=hs)
    q_ok = rope_rotate(raw, table, pos, np.arange(Hq) // group)
    q_bad = rope_rotate(raw, table, pos, np.arange(Hq))
    K = (K * 16).astype(np.float32)  # scores of a few units, so that the rotation matters
    o, _ = attn_ref(q_bad, K[:n], V[:n], group, scale)
    _rejects(o, q_ok, K[:n], V[:n], group, scale, "RoPE by query head")


def test_bar_rejects_a_row_from_the_neighbouring_page():
    n, cpp = 300, 128
    for p in (cpp - 1, cpp, 2 * cpp):  # the last row of a page, the first of the next
        q, K, V, group, scale = _sharp_case(n=n, hot=[p])
        Kb, Vb = K.copy(), V.copy()
        other = p + cpp if p % cpp == cpp - 1 else p - cpp  # same offset, neighbouring page
        Kb[p], Vb[p] = K[other], V[other]
        o, _ = attn_ref(q, Kb[:n], Vb[:n], group, scale)
        _rejects(o, q, K[:n], V[:n], group, scale, "row %d from the neighbouring page" % p)


def test_rope_reference_is_one_rounding_per_operation():
    """the float32 rotation equals a float64 evaluation rounded after every operation, and GPT-2's identity table is exact"""
    rng = np.random.default_rng(6)
    x = rng.standard_normal((4, 32)).astype(np.float32)
    tab = rng.standard_normal((200 * 16, 2)).astype(np.float32)
    got = rope_rotate(x, tab, 7, np.array([0, 0, 1, 1]))
    idx = 7 * 16 + np.array([0, 0, 1, 1])[:, None] * 32 + np.arange(16)
    c, s = tab[idx, 0].astype(np.float64), tab[idx, 1].astype(np.float64)
    f = lambda v: np.float32(v).astype(np.float64)  # noqa: E731
    x0, x1 = x[:, :16].astype(np.float64), x[:, 16:].astype(np.float64)
    want = np.concatenate([f(f(x0 * c) - f(x1 * s)), f(f(x0 * s) + f(x1 * c))], axis=1).astype(np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    ident = np.tile(np.array([1.0, 0.0], dtype=np.float32), 200 * 16)
    assert np.array_equal(rope_rotate(x, ident, 7, np.array([0, 1, 2, 3])).view(np.uint32), x.view(np.uint32))
