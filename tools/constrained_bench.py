"""Cost of allowed-token masks (DESIGN §3.18) in a greedy decode step on Llama-3-8B.
    greedy decode step at n sessions after 128-token prompts: every row unconstrained (jl_model_decode_penalized, no penalty), every
    row under its own random 50 %-density mask, and every row under a one-token mask (jl_model_decode_constrained)
Run on the GPU box:
    python tools/constrained_bench.py [--n 1,8,64] [--prompt 128] [--rounds 5] [--steps 5] [--out DIR]

Weights are synthetic Q4 ("direct" bytes and scales, the dims of Llama-3-8B), Q8 activations, F32 KV, vocabulary 128,256.  Each
session's prompt is prefilled once; every timed step decodes at the position after the prompt (rewriting that position's K/V), so
every round sees the same context.  The masks (n rows of 4,008 words) are built once and uploaded inside every timed call, as a grammar
engine's masks would be.  The variants call the C ABI directly with their arguments prepared once and alternate round by round in one
process; the minimum over rounds is reported.  Step time: host clock around calls that end with the tokens back on the host.  Card
name, power limit and maximum SM clock are read with nvidia-smi in the same run."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jlama_b200 import native, synth  # noqa: E402
from jlama_b200.model import LlamaModel  # noqa: E402
from jlama_b200.native import ptr  # noqa: E402
from jlama_b200.sampling import pack_mask  # noqa: E402
from logprobs_bench import best  # noqa: E402
from sampling_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", default="1,8,64")
    ap.add_argument("--prompt", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ns = [int(x) for x in a.n.split(",")]
    hw = card()
    print(json.dumps({"card": hw}), flush=True)
    ctx = native.Context(0)
    cfg = synth.get_config("llama-3-8b")
    V = cfg["vocab"]
    w = synth.make_weights(cfg, wdtype=native.Q4, mode="direct")
    m = LlamaModel(ctx, cfg, w, max_context=a.prompt + 16, max_sessions=max(ns), prefill_tensor_core=1, max_batch=2048)
    del w
    rng = np.random.default_rng(0)
    for s in range(max(ns)):
        m.reset_session(s)
        m.batch_forward(synth.random_prompt(cfg, a.prompt, seed=300 + s), 0, session=s)
    records = []
    for n in ns:
        toks = (np.arange(n, dtype=np.int32) * 37 + 11) % V
        pos = np.full(n, a.prompt, dtype=np.int32)
        sess = np.arange(n, dtype=np.int32)
        rows = np.arange(n, dtype=np.int32)
        half = np.ascontiguousarray(np.concatenate([pack_mask(rng.random(V) < 0.5) for _ in range(n)]))
        one = np.ascontiguousarray(np.concatenate([pack_mask(np.arange(V) == int(rng.integers(0, V))) for _ in range(n)]))
        nxt = np.empty(n, np.int32)

        def step(allow):
            if allow is None:
                rc = m.lib.jl_model_decode_penalized(m.h, n, ptr(sess), ptr(toks), ptr(pos), None, None, None, None, None, None, ptr(nxt), None,
                                                     None, None, None)
            else:
                rc = m.lib.jl_model_decode_constrained(m.h, n, ptr(sess), ptr(toks), ptr(pos), None, None, None, None, None, None, n, ptr(allow),
                                                       ptr(rows), ptr(nxt), None, None, None, None)
            ctx.check(rc)

        t = best(ctx, {"free": lambda: step(None), "half": lambda: step(half), "one": lambda: step(one)}, a.rounds, a.steps)
        rec = {"n": n, "prompt": a.prompt, "card": hw, "mode": m.decode_mode(n), "mask_bytes": int(half.nbytes)}
        rec.update({name + "_ms": round(v, 3) for name, v in t.items()})
        rec["half_over_free"] = round(t["half"] / t["free"] - 1.0, 4)
        rec["one_over_free"] = round(t["one"] / t["free"] - 1.0, 4)
        records.append(rec)
        print(json.dumps(rec), flush=True)
    m.close()
    ctx.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "constrained_bench.json"), "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
