"""The numpy statement of the allowed-token mask rule (DESIGN §3.18) in jlama_b200/sampling.py, which the GPU tests compare against:
the packed layout, that a banned token never wins whatever the draw, and that an allow-all mask changes nothing."""
import numpy as np
import pytest

from jlama_b200.sampling import apply_mask, mask_words, pack_mask, sample_topkp, select_constrained, unpack_mask


@pytest.mark.parametrize("V", [1, 31, 32, 33])
def test_pack_mask_round_trips_and_lays_bits_out_little_end_first(V):
    rng = np.random.default_rng(V)
    for _ in range(20):
        a = rng.random(V) < 0.5
        w = pack_mask(a)
        assert w.dtype == np.uint32 and len(w) == mask_words(V) == (V + 31) // 32
        assert np.array_equal(unpack_mask(w, V), a)
        for t in range(V):  # token t is bit t % 32 of word t // 32
            assert bool((int(w[t // 32]) >> (t % 32)) & 1) == a[t]
    # bits at or above the vocabulary are ignored
    w = pack_mask(np.zeros(V, bool))
    if V % 32:
        w[-1] = np.uint32(0xFFFFFFFF ^ ((1 << (V % 32)) - 1))
    assert not unpack_mask(w, V).any()
    assert np.array_equal(apply_mask(np.zeros(V, np.float32), w), np.full(V, -np.inf, np.float32))


def _cases(rng, V):
    row = (rng.standard_normal(V) * 3).astype(np.float32)
    a = rng.random(V) < 0.3
    a[rng.integers(0, V)] = True
    row[~a] += 50.0  # every banned token above every allowed one
    return row, a


@pytest.mark.parametrize("V", [1, 2, 33, 1000])
def test_a_banned_token_never_wins(V):
    rng = np.random.default_rng(V)
    for _ in range(30):
        row, a = _cases(rng, V)
        for T, k, p in ((0.0, 0, 1.0), (0.8, 0, 1.0), (1.5, 3, 1.0), (0.7, 0, 0.5), (1.0, V + 5, 0.9)):
            for u in (0.0, 1.0, float(rng.random())):
                t = select_constrained(row, a, T, k, p, u)
                assert a[t], (V, T, k, p, u, t)
                assert select_constrained(row, pack_mask(a), T, k, p, u) == t
    # the reference's prefix-sum rule would return index 0 at u = 0 and vocab - 1 at the end; the integer rule gives a banned token weight
    # 0 and never draws it
    V = 8
    a = np.zeros(V, bool)
    a[3] = a[5] = True
    row = np.zeros(V, np.float32)
    assert select_constrained(row, a, 1.0, 0, 1.0, 0.0) == 3
    assert select_constrained(row, a, 1.0, 0, 1.0, 1.0) == 5


def test_ties_among_allowed_tokens_take_the_first():
    row = np.array([9, 1, 5, 5, 9, 5], np.float32)
    a = np.array([False, True, False, True, False, True])
    assert select_constrained(row, a, 0.0) == 3
    a[2] = True
    assert select_constrained(row, a, 0.0) == 2


@pytest.mark.parametrize("V", [1, 33, 500])
def test_an_allow_all_mask_changes_nothing(V):
    rng = np.random.default_rng(V)
    for _ in range(20):
        row = (rng.standard_normal(V) * 4).astype(np.float32)
        a = np.ones(V, bool)
        assert np.array_equal(apply_mask(row, a).view(np.int32), row.view(np.int32))
        for T, k, p in ((0.0, 0, 1.0), (0.9, 0, 1.0), (0.8, 7, 0.9), (1.2, 0, 0.4)):
            u = float(rng.random())
            assert select_constrained(row, a, T, k, p, u) == sample_topkp(row, T, k, p, u)
