"""Decode and prefill of a device-synthesised LLaMA-7B-geometry Q4_0 model with an f16 and an f32 KV cache (B200_SESSION_KV_F32), alternated in one
run on the same card:

  decode@1   ms per token at n_past 512, 1024 and 2048 - 1 (the last past the f32 cluster attention's bound of 1664 positions: the two-kernel
             attention), CUDA-graph replay of one step after a rewind, CUDA events around `steps` tokens
  prefill    ms for 512 tokens from n_past 0 with n_batch 512

For each it reports the launches of one step, the algorithmic bytes of one decode step -- every streamed weight plus K and V of n_kv positions,
2 n_layer n_kv n_embd_gqa x element size -- and that byte count over the time as a share of the data-sheet HBM bandwidth (3.35 TB/s, H100 SXM).
The card's name, power limit and SM clock are read in the same run.  Usage: python tools/kv_f32_bench.py [n_layer]"""
import json
import subprocess
import sys

sys.path.insert(0, ".")
import numpy as np  # noqa: E402

import llm_b200  # noqa: E402
from llm_b200 import ModelKVMemoryType as KV  # noqa: E402
from oracle import synth  # noqa: E402

HBM = 3.35e12


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}


def main():
    n_layer = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    steps, rounds = 32, 3
    hp = dict(synth.CONFIGS["7b"], n_layer=n_layer, wtype=2)                      # Q4_0, n_ctx 2048
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=2048))
    m.synthesize(0x5EED)
    L = m.L
    gqa = hp["n_embd"] // (hp["n_head"] // hp["n_head_kv"])
    toks = synth.make_tokens(hp, 2048)
    top = 2048 - steps - 1

    def fill(s):                                                                     # the cache up to n_past `top`
        s.rewind(0)
        for a in range(0, top, 512):
            s.evaluate(toks[a:min(a + 512, top)])

    sessions = {}
    for name, t in (("f16", KV.Float16), ("f32", KV.Float32)):
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=512, memory_k_type=t, memory_v_type=t))
        fill(s)
        sessions[name] = s
    info = card()
    res = {k: {} for k in sessions}
    for r in range(rounds):                                                          # f16 and f32 alternated
        for name, s in sessions.items():
            elem = 4 if name == "f32" else 2
            for n_past in (top, 1024, 512):                                           # each rewind goes back from where the last left
                s.rewind(n_past)
                s.evaluate(toks[n_past:n_past + 1])                                  # warm the bucket's graph
                s.rewind(n_past)
                L.b200_timing_begin()
                for i in range(steps):
                    s.evaluate(toks[n_past + i:n_past + i + 1])
                ms = L.b200_timing_end_ms() / steps
                n_kv = n_past + steps // 2
                kv_bytes = 2 * n_layer * n_kv * gqa * elem
                byt = m.weight_bytes + kv_bytes
                res[name].setdefault(f"decode@{n_past}", []).append(dict(ms=ms, launches=s.last_launches, bytes=byt, kv_bytes=kv_bytes,
                                                                         hbm_share=byt / (ms * 1e-3) / HBM))
            s.rewind(0)
            L.b200_timing_begin()
            s.evaluate(toks[:512])
            res[name].setdefault("prefill@512", []).append(dict(ms=L.b200_timing_end_ms(), launches=s.last_launches))
            fill(s)
    out = {"card": info, "n_layer": n_layer, "steps": steps, "rounds": rounds, "weight_bytes": m.weight_bytes}
    for name, d in res.items():
        out[name] = {}
        for k, v in d.items():
            ms = float(np.median([x["ms"] for x in v]))                               # the median of the rounds
            out[name][k] = dict(v[-1], ms=ms, ms_all=[round(x["ms"], 4) for x in v])
            if "bytes" in v[-1]:
                out[name][k]["hbm_share"] = v[-1]["bytes"] / (ms * 1e-3) / HBM
    print(json.dumps(out, indent=1))
    for s in sessions.values():
        s.close()
    m.close()


if __name__ == "__main__":
    main()
