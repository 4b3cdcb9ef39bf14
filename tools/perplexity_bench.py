"""Perplexity of a device-synthesised LLaMA-7B-geometry Q4_0 model, per chunk, at context sizes 512 and 2048 with n_batch 512:

  device   InferenceSession.perplexity: the logits stay in HBM and ppl.cu reduces each scored row to one term
  prefill  the same chunk's forward passes alone (every row's logits computed, left in HBM): device - prefill is the cost of the scoring
  host     evaluate(all_logits=True) per batch, every row copied to the host, then the plain-C oracle's softmax loop on the host libm
           (oracle/ppl_oracle.c, the reference's arithmetic) -- what a user had to do before

Each time is CUDA events on the backend's stream around one chunk (the host path's CPU work lies between its two events), after one warm-up chunk,
averaged over 2 chunks.  The card's name and power limit are read in the same run.  The device and host paths' perplexities must be identical.
Usage: python tools/perplexity_bench.py [n_layer]"""
import ctypes as C
import json
import subprocess
import sys

sys.path.insert(0, ".")
import numpy as np  # noqa: E402

import llm_b200  # noqa: E402
from oracle import synth  # noqa: E402
from oracle.ppl import PplOracle  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}


def main():
    n_layer = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    n_batch, reps = 512, 2
    hp = dict(synth.CONFIGS["7b"], n_layer=n_layer, wtype=2)                      # Q4_0
    por = PplOracle()
    info = card()
    results = []
    for C_ in (512, 2048):
        m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=C_))
        m.synthesize(0x5EED)
        L = m.L
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=n_batch))
        toks = synth.make_tokens(hp, C_ * (reps + 1))

        def device(chunk):
            L.b200_timing_begin()
            p = s.perplexity(chunk)
            return L.b200_timing_end_ms(), p[0]

        def prefill(chunk):
            s.rewind(0)
            L.b200_timing_begin()
            for b0 in range(0, C_, n_batch):
                b = np.ascontiguousarray(chunk[b0:b0 + n_batch], np.int32)
                if b0 == 0:
                    b[0] = 1
                # all_logits with no output buffer: every row through the lm_head, nothing copied to the host
                assert L.b200_session_evaluate(s._s, b.ctypes.data_as(C.c_void_p), b.size, None, 1) == 0
            return L.b200_timing_end_ms(), None

        def host(chunk):
            def evaluate(b):
                return s.evaluate(b, all_logits=True)
            L.b200_timing_begin()
            p, _ = por.perplexity(evaluate, lambda: s.rewind(0), chunk, C_, n_batch, 1)
            return L.b200_timing_end_ms(), p[0]

        row = dict(context_size=C_, n_batch=n_batch, scored_rows=C_ - 1 - min(512, C_ // 2))
        for name, fn in (("device", device), ("prefill", prefill), ("host", host)):
            fn(toks[:C_])                                                         # warm-up
            times, ppls = [], []
            for r in range(1, reps + 1):
                ms, p = fn(toks[r * C_:(r + 1) * C_])
                times.append(ms); ppls.append(p)
            row[f"{name}_ms_per_chunk"] = round(float(np.mean(times)), 3)
            if p is not None:
                row[f"{name}_ppl"] = [float(x) for x in ppls]
        assert row["device_ppl"] == row["host_ppl"], (row["device_ppl"], row["host_ppl"])
        row["scoring_ms_per_chunk"] = round(row["device_ms_per_chunk"] - row["prefill_ms_per_chunk"], 3)
        results.append(row)
        s.close(); m.close()
    print(json.dumps(dict(card=info.get("name"), power_limit=info.get("power.limit"), sm_clock_max=info.get("clocks.max.sm"), n_layer=n_layer,
                          model="LLaMA-7B geometry, Q4_0, device-synthesised", results=results)), flush=True)


if __name__ == "__main__":
    main()
