"""numpy statement of the top-k / top-p sampling rule (DESIGN §3.12) that jl_sample_topkp and the *_topkp model calls implement on the
GPU.  It uses uint64 and float64 exactly as the rule is written, so that it and the kernel agree token for token; the GPU tests compare
against it."""
import numpy as np

TWO40 = np.float64(2.0 ** 40)


def weights(logits, temperature):
    """w_i = (uint64)(e_i * 2^40), e_i = (float) exp(((double) l_i - (double) max) / (double) T); a -inf logit gets 0"""
    l = np.asarray(logits, dtype=np.float32)
    with np.errstate(over="ignore", under="ignore"):
        e = np.exp((l.astype(np.float64) - np.float64(l.max())) / np.float64(np.float32(temperature))).astype(np.float32)
    return (e.astype(np.float64) * TWO40).astype(np.uint64)


def kept_topkp(w, top_k, top_p):
    """boolean mask of the tokens the filter keeps, given the integer weights w"""
    V = len(w)
    keep = np.ones(V, dtype=bool)
    if 1 <= top_k < V:
        t = np.partition(w, V - top_k)[V - top_k]  # the k-th largest weight, counting multiplicity
        keep = w >= t
    p = np.float64(np.float32(top_p))
    if p < 1.0:
        kw = w[keep]
        S = kw.sum(dtype=np.uint64)
        vals, counts = np.unique(kw, return_counts=True)  # ascending distinct weights
        mass = vals * counts.astype(np.uint64)
        G = np.cumsum(mass[::-1], dtype=np.uint64)[::-1] - mass  # mass strictly heavier than each value
        ok = G.astype(np.float64) < p * np.float64(S)
        keep &= w >= vals[ok].min()
    return keep


def sample_topkp(logits, temperature, top_k, top_p, uniform):
    """The token the rule draws from one logits row with uniform u in [0, 1]; temperature 0 is the arg-max (first index on ties)."""
    l = np.asarray(logits, dtype=np.float32)
    if np.float32(temperature) == 0.0:
        return int(np.argmax(l))
    w = weights(l, temperature)
    keep = kept_topkp(w, top_k, top_p)
    kw = np.where(keep, w, np.uint64(0))
    W = kw.sum(dtype=np.uint64)
    r = min(int(W) - 1, int(np.floor(np.float64(np.float32(uniform)) * np.float64(W))))
    return int(np.argmax(np.cumsum(kw, dtype=np.uint64) > np.uint64(r)))


MAX_LOGPROBS = 20  # JL_MAX_LOGPROBS


def logprobs(row, target, top_n):
    """The log-probability rule (DESIGN §3.13) that jl_logprobs and the *_logprobs / score model calls implement on the GPU, for one raw
    logits row (finite, or -inf with at least one finite entry): m = max l, Z = sum exp((double) l_i - (double) m) in double,
    lp_i = (float) (((double) l_i - (double) m) - log Z).  Returns (lp of `target` (NaN for target -1), ids [MAX_LOGPROBS],
    lps [MAX_LOGPROBS]): the top_n tokens of largest logit, ties by lower index, then id -1 and NaN."""
    l = np.asarray(row, dtype=np.float32).astype(np.float64)
    m = l.max()
    with np.errstate(under="ignore"):
        logz = np.log(np.exp(l - m).sum())
    lp = ((l - m) - logz).astype(np.float32)
    ids = np.full(MAX_LOGPROBS, -1, dtype=np.int32)
    lps = np.full(MAX_LOGPROBS, np.nan, dtype=np.float32)
    n = min(int(top_n), len(l))
    if n > 0:
        order = np.lexsort((np.arange(len(l)), -l))[:n]  # l descending, then index ascending
        ids[:n] = order
        lps[:n] = lp[order]
    return (np.float32(np.nan) if target < 0 else lp[target]), ids, lps


def apply_penalties(row, prompt_ids=(), generated_ids=(), presence=0.0, frequency=0.0, repetition=1.0, logit_bias=None):
    """The penalty rule (DESIGN §3.14) that jl_apply_penalties and the *_penalized model calls implement on the GPU, for one raw logits
    row.  logit_bias: {id: value} or (id, value) pairs.  With c = the count of each token among generated_ids and s = whether it occurs
    in prompt_ids or generated_ids, every step one float32 operation:
        b = l + bias;  b = where(s, where(b < 0, b * repetition, b / repetition), b);  b = b - float32(c) * frequency;
        b = where(c > 0, b - presence, b).
    An unpenalised row (presence = frequency = 0, repetition = 1, no bias) is returned as it is."""
    l = np.asarray(row, dtype=np.float32)
    bias = list(logit_bias.items()) if isinstance(logit_bias, dict) else list(logit_bias or ())
    if presence == 0 and frequency == 0 and repetition == 1 and not bias:
        return l.copy()
    V = len(l)
    c = np.bincount(np.asarray(generated_ids, dtype=np.int64), minlength=V)[:V]
    s = c > 0
    s[np.asarray(prompt_ids, dtype=np.int64)] = True
    bias_row = np.zeros(V, dtype=np.float32)
    for t, v in bias:
        bias_row[int(t)] = np.float32(v)
    r, f, p = np.float32(repetition), np.float32(frequency), np.float32(presence)
    with np.errstate(over="ignore", invalid="ignore"):
        b = l + bias_row
        b = np.where(s, np.where(b < 0, b * r, b / r), b).astype(np.float32)
        b = b - c.astype(np.float32) * f
        b = np.where(c > 0, b - p, b).astype(np.float32)
    return b


def mask_words(vocab):
    """the uint32 words of one allowed-token mask row: (vocab + 31) // 32"""
    return (int(vocab) + 31) // 32


def pack_mask(allowed):
    """bool[V] -> uint32[(V + 31) // 32]: token t is allowed when bit t % 32 of word t // 32 is set (DESIGN §3.18)"""
    a = np.asarray(allowed, dtype=bool).reshape(-1)
    bits = np.zeros(mask_words(len(a)) * 32, dtype=np.uint64)
    bits[:len(a)] = a
    return (bits.reshape(-1, 32) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)


def unpack_mask(words, vocab):
    """uint32 words -> bool[vocab]; bits at or above vocab are ignored"""
    w = np.asarray(words, dtype=np.uint32).reshape(-1)
    return ((w[:, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(-1)[:int(vocab)]


def apply_mask(row, allowed):
    """The constrained processed row (DESIGN §3.18): p_t = row_t where t is allowed, else -inf.  `row` is the raw row or the processed row
    of apply_penalties; `allowed` a bool[V] or the packed uint32 words of pack_mask."""
    l = np.asarray(row, dtype=np.float32)
    a = np.asarray(allowed)
    if a.dtype != bool:
        a = unpack_mask(a, len(l))
    return np.where(a, l, np.float32(-np.inf)).astype(np.float32)


def select_constrained(row, allowed, temperature, top_k=0, top_p=1.0, uniform=0.0):
    """The token of one constrained row: temperature 0 takes the arg-max of the masked row (first index on ties); otherwise the top-k /
    top-p rule of sample_topkp draws from it, which gives a banned token weight 0 and never draws one."""
    return sample_topkp(apply_mask(row, allowed), temperature, top_k, top_p, uniform)
