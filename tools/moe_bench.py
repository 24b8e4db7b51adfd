"""Mixtral-8x7B decode steps and prompt passes on the grouped mixture-of-experts path (DESIGN §3.8).
    decode: a greedy step of n sessions after 128-token prompts, against the same n sessions as n one-row steps (the M = 1 path,
            which keeps the per-row expert loop), alternated round by round in one process; the expert bytes the step streams
    prompts: time to all first tokens of S sessions x P-token prompts through jl_model_batch_forward_multi + one sampling call
Run on the GPU box:
    python tools/moe_bench.py [--n 1,2,8,16,32,64] [--prompt 128] [--segs 8x512,64x128] [--max-batch 256,2048] [--layers 32]
                              [--rounds 3] [--steps 3] [--out DIR]

Weights are synthetic Q4 ("direct" bytes and scales) with Mixtral-8x7B's dimensions (E 4096, H 14336, 8 experts, top-2, 32
layers: about 26 GB on the card), Q8 activations, F32 KV.  Expert bytes of a step: the distinct experts its rows selected, read
back from the last layer's selections (the one layer the debug read exposes, taken for every layer), times one expert's Q4 bytes
(w1, w2, w3 and their block scales); the bytes/s divide that by the step time.  Step and prompt times: host clock around calls
that end with the tokens back on the host, minimum over rounds.  Card name, power limit and maximum SM clock are read with
nvidia-smi in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jlama_b200 import native, synth  # noqa: E402
from jlama_b200.model import LlamaModel  # noqa: E402
from logprobs_bench import best  # noqa: E402
from sampling_bench import card  # noqa: E402


def expert_bytes(cfg):
    """Q4 bytes of one expert: three E x H tensors, half a byte per weight and one f32 scale per 32"""
    return 3 * (cfg["E"] * cfg["H"] // 2 + cfg["E"] * cfg["H"] // 32 * 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", default="1,2,8,16,32,64")
    ap.add_argument("--prompt", type=int, default=128)
    ap.add_argument("--segs", default="8x512,64x128")
    ap.add_argument("--max-batch", default="256,2048")
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ns = [int(x) for x in a.n.split(",")]
    segs = [tuple(int(v) for v in s.split("x")) for s in a.segs.split(",")]
    hw = card()
    print(json.dumps({"card": hw}), flush=True)
    ctx = native.Context(0)
    cfg = synth.get_config("mixtral-8x7b", layers=a.layers)
    V, L, eb = cfg["vocab"], cfg["layers"], expert_bytes(cfg)
    t0 = time.perf_counter()
    w = synth.make_weights(cfg, wdtype=native.Q4, mode="direct")
    print(json.dumps({"weights_s": round(time.perf_counter() - t0, 1), "layers": L}), flush=True)
    ctx_len = max([a.prompt + 16] + [p + 16 for _, p in segs])
    sessions = max(ns + [s for s, _ in segs])
    records = []
    for mb in [int(x) for x in a.max_batch.split(",")]:
        m = LlamaModel(ctx, cfg, w, max_context=ctx_len, max_sessions=sessions, max_batch=mb)
        for S, P in segs:  # time to all first tokens
            prompts = [synth.random_prompt(cfg, P, seed=700 + s) for s in range(S)]
            sess = np.arange(S, dtype=np.int32)

            def prefill():
                for s in range(S):
                    m.reset_session(s)
                m.batch_forward_multi([(s, prompts[s], 0) for s in range(S)])
                m.sample_multi(sess)

            t = best(ctx, {"prefill": prefill}, a.rounds, 1)["prefill"]
            rec = {"what": "prompts", "sessions": S, "prompt": P, "max_batch": mb, "layers": L, "card": hw, "ms": round(t, 2),
                   "prompt_tokens_per_s": round(S * P / t * 1e3, 1)}
            records.append(rec)
            print(json.dumps(rec), flush=True)
        if mb != int(a.max_batch.split(",")[0]):
            m.close()
            continue
        for s in range(max(ns)):  # decode
            m.reset_session(s)
            m.batch_forward(synth.random_prompt(cfg, a.prompt, seed=300 + s), 0, session=s)
        for n in ns:
            toks = (np.arange(n, dtype=np.int32) * 37 + 11) % V
            pos = np.full(n, a.prompt, dtype=np.int32)
            sess = np.arange(n, dtype=np.int32)

            def grouped():
                m.decode(toks, pos, sessions=sess)

            def rows():
                for i in range(n):
                    m.decode(toks[i:i + 1], pos[i:i + 1], sessions=sess[i:i + 1])

            t = best(ctx, {"step": grouped, "rows": rows}, a.rounds, a.steps)
            grouped()
            sel = m.debug_read(9, n * cfg["experts_per_token"]).view(np.int32)
            distinct = len(np.unique(sel))
            step_bytes = distinct * eb * L
            rec = {"what": "decode", "n": n, "prompt": a.prompt, "layers": L, "card": hw, "mode": m.decode_mode(n),
                   "step_ms": round(t["step"], 3), "rows_ms": round(t["rows"], 3), "rows_over_step": round(t["rows"] / t["step"], 3),
                   "distinct_experts_last_layer": distinct, "expert_gb_per_step": round(step_bytes / 1e9, 2),
                   "expert_gb_per_s": round(step_bytes / t["step"] / 1e6, 1), "tokens_per_s": round(n / t["step"] * 1e3, 1)}
            records.append(rec)
            print(json.dumps(rec), flush=True)
        m.close()
    ctx.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "moe_bench.json"), "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
