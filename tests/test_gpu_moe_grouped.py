"""The grouped mixture-of-experts path (forward_rows at M >= 2, DESIGN §3.8): the rows of a step or prompt pass grouped by expert on
the device (moe_group_kernel, jl_elementwise.cu) and every selected expert streamed once per launch for all of its rows (gemm64's
grouped mode, jl_gemm64.cu).

Group kernel, bit for bit through jl_moe_group on crafted selections against a numpy stable counting sort (np.argsort, kind
"stable", of the flattened [M][k] selections): counts, offsets, the pair list and the tile table, at 1..64 experts, k 1..8,
M 2..2048, with every row on one expert (tiles cut past R rows), empty experts, uniform and random selections.

Phases inside models.  Each phase of the last layer's block is checked from the buffer that feeds it with the restatements and
bars of test_gpu_moe.py (router probabilities and selections from xb, SiLU * up from xb through the selected experts' w1 / w3,
x = d_0 + d_1 + ... + xb from the h rows), on tiny-mixtral, small-mixtral and a one-layer model at Mixtral-8x7B's E / H, Q4 and
Q8_0 experts, decode steps of 2..64 rows and prompt passes of 16..300 rows; the zero router sends every row to experts 0..k-1
and leaves the others empty.

Companions: a row's bits do not depend on the rows that share its step, so a session's logits equal its twin's in another step
with other companions routed elsewhere, at another row.  Graphs: replayed steps whose selections differ equal MODEL_NO_GRAPH steps
bit for bit.  Launches: one decode step launches as many kernels at 16 as at 64 rows.  End to end: 16 concurrent small-mixtral
sessions through the scheduler against the oracle, under the near-tie rule of test_gpu_batched_decode.py.

Importing this file does not load the CUDA library.
"""
import zlib

import numpy as np
import pytest

from jlama_b200.native import I8, JL_ERR_INVALID, MODEL_NO_GRAPH, Q4
from test_gpu_batched_decode import _check_against_oracle
from test_gpu_moe import (MoeRef, case_weights, check_gate_up, check_probs, check_selection, check_sum, decode_step, down_refs,
                          read_bufs, rkey, router_ref)

gpu = pytest.mark.gpu


# ---- the group kernel, restated (numpy only) --------------------------------------------------------------------------------
def tile_bound(pairs, ne, R):
    return (pairs + ne * (R - 1)) // R


def group_ref(sel, ne, R):
    """(counts, offsets, pairs, tiles [n][4]) of selections sel [M][k]: a stable counting sort of the pairs row * k + slot"""
    flat = np.asarray(sel, dtype=np.int64).reshape(-1)
    pairs = np.argsort(flat, kind="stable").astype(np.int32)
    counts = np.bincount(flat, minlength=ne).astype(np.int32)
    offsets = (np.cumsum(counts) - counts).astype(np.int32)
    tiles = [(e, offsets[e] + f, min(R, counts[e] - f), 0) for e in range(ne) for f in range(0, counts[e], R)]
    return counts, offsets, pairs, np.array(tiles, dtype=np.int32).reshape(-1, 4)


def selections(kind, M, ne, k, rng):
    """[M][k] int32, k distinct experts per row as the router gives"""
    if kind == "one":  # every row's slot 0 on one expert
        e0 = int(rng.integers(0, ne))
        return ((e0 + np.arange(k)[None, :] + np.zeros((M, 1), dtype=np.int64)) % ne).astype(np.int32)
    if kind == "empty":  # experts 0..k-1 only
        return np.tile(np.arange(k, dtype=np.int32), (M, 1))
    if kind == "uniform":
        return ((np.arange(M)[:, None] + np.arange(k)[None, :]) % ne).astype(np.int32)
    return np.argsort(rng.random((M, ne)), axis=1)[:, :k].astype(np.int32)


def moe_group(ctx, sel, ne, R):
    sel = np.ascontiguousarray(sel, dtype=np.int32)
    M, k = sel.shape
    counts, offsets = np.full(ne, -1, dtype=np.int32), np.full(ne, -1, dtype=np.int32)
    pairs = np.full(M * k, -1, dtype=np.int32)
    tiles = np.full((tile_bound(M * k, ne, R), 4), -1, dtype=np.int32)
    nt = np.zeros(1, dtype=np.int32)
    ctx.check(ctx.lib.jl_moe_group(ctx.h, M, ne, k, R, sel.ctypes.data, counts.ctypes.data, offsets.ctypes.data, pairs.ctypes.data,
                                   tiles.ctypes.data, nt.ctypes.data))
    return counts, offsets, pairs, tiles[:int(nt[0])]


GROUP_NE, GROUP_K, GROUP_M, GROUP_R = [1, 4, 8, 33, 64], [1, 2, 8], [2, 9, 64, 300, 2048], [16, 48, 64]
KINDS = ["one", "empty", "uniform", "random"]


@gpu
def test_group_kernel_bit_for_bit(cuda_ctx):
    rng = np.random.default_rng(41)
    calls = 0
    for ne in GROUP_NE:
        for k in [k for k in GROUP_K if k <= ne]:
            for M in GROUP_M:
                for kind in KINDS:
                    sel = selections(kind, M, ne, k, rng)
                    for R in GROUP_R:
                        got, want = moe_group(cuda_ctx, sel, ne, R), group_ref(sel, ne, R)
                        for name, g, w in zip(("counts", "offsets", "pairs", "tiles"), got, want):
                            assert np.array_equal(g, w), (name, ne, k, M, kind, R)
                        calls += 1
    print("group kernel: %d launches bit for bit" % calls)


@gpu
def test_group_refusals_write_nothing(cuda_ctx):
    lib, h = cuda_ctx.lib, cuda_ctx.h
    sel = np.zeros((4, 8), dtype=np.int32)
    outs = [np.full(4096, -7, dtype=np.int32) for _ in range(5)]
    S = sel.ctypes.data
    O = [o.ctypes.data for o in outs]
    bad = [(0, 8, 2, 16), (-1, 8, 2, 16), (4, 0, 1, 16), (4, 65, 2, 16), (4, 8, 0, 16), (4, 8, 9, 16), (4, 4, 5, 16), (4, 8, 2, 0),
           (4, 8, 2, 65)]
    for n, ne, k, R in bad:
        assert lib.jl_moe_group(h, n, ne, k, R, S, *O) == JL_ERR_INVALID, (n, ne, k, R)
    for v in (-1, 8):
        s2 = np.zeros((4, 2), dtype=np.int32)
        s2[3, 1] = v
        assert lib.jl_moe_group(h, 4, 8, 2, 16, s2.ctypes.data, *O) == JL_ERR_INVALID, v
    for i in range(6):
        args = [S] + O
        args[i] = None
        assert lib.jl_moe_group(h, 4, 8, 2, 16, *args) == JL_ERR_INVALID, i
    assert all((o == -7).all() for o in outs)


# ---- the phases inside models -----------------------------------------------------------------------------------------------
def model_weights(name, wd, zero_router=False):
    """(cfg, synth direct weights); zero_router: every router logit 0, so every row selects experts 0..k-1"""
    from jlama_b200 import synth
    if name == "8x7b":
        return case_weights(dict(cfg="8x7b", wd=wd, router_craft="zero" if zero_router else None))
    cfg = synth.get_config(name)
    w = synth.make_weights(cfg, wdtype=wd, mode="direct")
    if zero_router:
        for L in range(cfg["layers"]):
            dt, data, s = w[rkey(L)]
            w[rkey(L)] = (dt, data, np.zeros_like(s))
    return cfg, w


def check_phases(ref, b, lab):
    """router, selections, gate/up and down + sum of the last layer from the buffers that feed them; every err/bar <= 1"""
    L = ref.cfg["layers"] - 1
    KE = ref.cfg["experts_per_token"]
    lg, e, nat, _ = router_ref(ref, L, b["xb"], True)
    res = {"router": check_probs(b["probs"], lg, e, nat)[0]}
    amb = check_selection(b["probs"], b["sel"], lg, e, KE)
    res["gate/up"] = check_gate_up(ref, L, b["xb"], b["h"], b["sel"], True)[0]
    d, bar, nat_d = down_refs(ref, L, b["h"], b["sel"], True)
    res["down+sum"] = check_sum(b["x"], b["xb"], d, bar, nat_d)[0]
    print("%s: %s, %d ambiguous selection rows" % (lab, ", ".join("%s err/bar %.3f" % kv for kv in res.items()), len(amb)))
    for ph, r in res.items():
        assert r <= 1.0, (lab, ph, r)


STEPS = [2, 8, 9, 16, 63, 64]
PHASE_CASES = [
    dict(id="tiny-Q4", name="tiny-mixtral", wd=Q4, steps=STEPS, prompts=[16, 256]),
    dict(id="tiny-Q8_0", name="tiny-mixtral", wd=I8, steps=STEPS, prompts=[16]),
    dict(id="small-Q4", name="small-mixtral", wd=Q4, steps=STEPS, prompts=[16, 256, 300]),
    dict(id="small-Q8_0", name="small-mixtral", wd=I8, steps=[2, 16, 64], prompts=[300]),
    dict(id="small-Q4-one-expert", name="small-mixtral", wd=Q4, zero=True, steps=[2, 64], prompts=[300]),
    dict(id="tiny-Q8_0-one-expert", name="tiny-mixtral", wd=I8, zero=True, steps=[9, 64], prompts=[256]),
    dict(id="8x7b-Q4", name="8x7b", wd=Q4, steps=[2, 16, 64], prompts=[16]),
    dict(id="8x7b-Q8_0-one-expert", name="8x7b", wd=I8, zero=True, steps=[16], prompts=[]),
]


@gpu
@pytest.mark.parametrize("case", PHASE_CASES, ids=[c["id"] for c in PHASE_CASES])
def test_grouped_phases_against_exact_references(cuda_ctx, case):
    from jlama_b200.model import LlamaModel
    cfg, w = model_weights(case["name"], case["wd"], case.get("zero", False))
    ref = MoeRef(cfg, w)
    KE = cfg["experts_per_token"]
    rng = np.random.default_rng(zlib.crc32(case["id"].encode()))
    gm = LlamaModel(cuda_ctx, cfg, w, working_qtype=I8, max_batch=300, max_sessions=64, max_context=min(cfg["ctx"], 320))
    try:
        for n in case["steps"]:
            decode_step(gm, n, rng, cfg["vocab"])
            b = read_bufs(gm, n)
            check_phases(ref, b, "%s step n=%d" % (case["id"], n))
            if case.get("zero"):
                assert np.array_equal(b["sel"], np.tile(np.arange(KE), (n, 1)))
        for n in case["prompts"]:
            gm.reset_session(0)
            gm.batch_forward(rng.integers(0, cfg["vocab"], n).astype(np.int32), 0, session=0)
            check_phases(ref, read_bufs(gm, n), "%s prompt n=%d" % (case["id"], n))
    finally:
        gm.close()


# ---- companions, graphs, launches -----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n", [16, 64])
def test_row_bits_do_not_depend_on_companions(cuda_ctx, n):
    """a token at position 0 decoded at row 0 of one step and at row n - 5 of another, among other tokens routed to other experts"""
    from jlama_b200.model import LlamaModel
    cfg, w = model_weights("small-mixtral", Q4)
    gm = LlamaModel(cuda_ctx, cfg, w, working_qtype=I8, max_sessions=64, max_context=64)
    try:
        rng = np.random.default_rng(n)
        twin = 17
        a = rng.integers(0, cfg["vocab"], n).astype(np.int32)
        b = rng.integers(0, cfg["vocab"], n).astype(np.int32)
        a[0], b[n - 5] = twin, twin
        sess = np.arange(n, dtype=np.int32)
        _, la = gm.decode(a, np.zeros(n, dtype=np.int32), sessions=sess, want_logits=True)
        sa = read_bufs(gm, n)["sel"]
        _, lb = gm.decode(b, np.zeros(n, dtype=np.int32), sessions=sess[::-1].copy(), want_logits=True)
        sb = read_bufs(gm, n)["sel"]
        ne = cfg["experts"]
        others_a = np.bincount(np.delete(sa, 0, axis=0).reshape(-1), minlength=ne)
        others_b = np.bincount(np.delete(sb, n - 5, axis=0).reshape(-1), minlength=ne)
        assert (others_a != others_b).any(), "the companions should give the experts other row counts"
        assert np.array_equal(la[0].view(np.uint32), lb[n - 5].view(np.uint32)), "the twin's logits depend on its companions"
    finally:
        gm.close()


@gpu
@pytest.mark.parametrize("n", [16, 64])
def test_graph_replay_equals_eager(cuda_ctx, n):
    from jlama_b200.model import LlamaModel
    cfg, w = model_weights("small-mixtral", Q4)
    mk = lambda flags: LlamaModel(cuda_ctx, cfg, w, working_qtype=I8, max_sessions=64, max_context=64, flags=flags)  # noqa: E731
    g, e = mk(0), mk(MODEL_NO_GRAPH)
    try:
        assert g.decode_mode(n) == 1 and e.decode_mode(n) == 0
        rng = np.random.default_rng(100 + n)
        decode_step(g, n, rng, cfg["vocab"])
        a = read_bufs(g, n)
        tb = decode_step(g, n, rng, cfg["vocab"])
        b = read_bufs(g, n)
        assert (a["sel"] != b["sel"]).any(), "the two steps should route some row differently"
        decode_step(e, n, rng, cfg["vocab"], tokens=tb)
        eb = read_bufs(e, n)
        for k in b:
            assert np.array_equal(b[k].view(np.uint32), eb[k].view(np.uint32)), "graph and eager %s differ" % k
    finally:
        g.close()
        e.close()


@gpu
def test_decode_step_launches_do_not_grow_with_rows(cuda_ctx):
    """16 and 64 rows launch the same kernels; 2 rows differ from 16 only where the dense GEMMs change kernel (gemm8 -> gemm64,
    one more prologue launch each), far fewer launches than one more row of the per-row loop would add"""
    from jlama_b200.model import LlamaModel
    cfg, w = model_weights("small-mixtral", Q4)
    gm = LlamaModel(cuda_ctx, cfg, w, working_qtype=I8, max_sessions=64, max_context=64, flags=MODEL_NO_GRAPH)
    try:
        rng = np.random.default_rng(5)
        got = {}
        for n in (2, 16, 64, 16):
            before = cuda_ctx.kernel_launches()
            decode_step(gm, n, rng, cfg["vocab"])
            got[n] = cuda_ctx.kernel_launches() - before
        print("launches per step: %s" % got)
        assert got[16] == got[64]
        per_row = cfg["layers"] * (2 + 2 * cfg["experts_per_token"])
        assert 0 <= got[16] - got[2] < per_row
    finally:
        gm.close()


@gpu
def test_scheduler_sessions_against_the_oracle(cuda_ctx, oracle):
    from jlama_b200 import native, synth
    from jlama_b200.model import LlamaModel
    from jlama_b200.scheduler import SessionScheduler
    cfg = synth.get_config("small-mixtral")
    w = synth.make_weights(cfg)
    gm = LlamaModel(cuda_ctx, cfg, w, working_qtype=I8, max_sessions=16)
    om = oracle.OracleLlama(cfg, w, act_q8=True)
    try:
        work = [(synth.random_prompt(cfg, 3 + (5 * i) % 13, seed=2100 + i), 6 + i % 5) for i in range(16)]
        with SessionScheduler(gm) as sched:
            ids = [sched.submit(p, n) for p, n in work]
            widest = 0
            while True:
                st = sched.step()
                widest = max(widest, st.decode_rows)
                if st.active == 0 and st.queued == 0:
                    break
            results = []
            for rid, (p, n) in zip(ids, work):
                toks, state, _ = sched.result(rid)
                assert state == native.SCHED_FINISHED and len(toks) == n
                results.append((p, n, toks))
        assert widest > 8
        print("16 small-mixtral sessions: %d exact" % _check_against_oracle(om, results))
    finally:
        om.close()
        gm.close()


# ---- the restatement, checked on the CPU ------------------------------------------------------------------------------------
def test_group_restatement():
    """pairs ascend within an expert, tiles cover each expert's list in runs of at most R, and the tile bound holds at its worst"""
    rng = np.random.default_rng(7)
    for ne, k, M, R in ((8, 2, 64, 16), (64, 8, 300, 64), (1, 1, 2, 16), (33, 2, 2048, 48)):
        for kind in KINDS:
            sel = selections(kind, M, ne, k, rng)
            assert all(len(set(r)) == k for r in sel.tolist())
            counts, offsets, pairs, tiles = group_ref(sel, ne, R)
            flat = sel.reshape(-1)
            for e in range(ne):
                p = pairs[offsets[e]:offsets[e] + counts[e]]
                assert (flat[p] == e).all() and (np.diff(p) > 0).all()
            assert len(tiles) <= tile_bound(M * k, ne, R)
            assert (tiles[:, 2] >= 1).all() and (tiles[:, 2] <= R).all() and tiles[:, 2].sum() == M * k
    # the bound is reached: every expert one pair past a multiple of R
    R, ne = 16, 4
    sel = np.repeat(np.arange(ne), R + 1).reshape(-1, 1).astype(np.int32)
    assert len(group_ref(sel, ne, R)[3]) == 2 * ne == tile_bound(len(sel), ne, R)
