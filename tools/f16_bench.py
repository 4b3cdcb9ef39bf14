"""F16 LLaMA-7B on one GPU: a device-synthesised F16 model (weights N(0, 1/K) rounded to fp16), decode at n_past 512 (CUDA events, 8 warm-up and
64 timed steps), prefill of 512 tokens, and the weight mat-vecs alone (b200_session_probe_matvec).  Bytes and FMAs come from the shapes; the
shares are of the H100 SXM data sheet's 3.35 TB/s HBM3 (decode, mat-vec) and 67 TFLOP/s FP32 (prefill), figures for a 700 W card.  The card's
name, power limit and SM clock are read in the same run.  Usage: python tools/f16_bench.py [n_layer]"""
import ctypes as C
import json
import subprocess
import sys

sys.path.insert(0, ".")
import numpy as np  # noqa: E402

import llm_b200  # noqa: E402
from oracle import synth  # noqa: E402

HBM = 3.35e12
FP32_FMA = 67e12 / 2


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}


def main():
    n_layer = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    hp = dict(synth.CONFIGS["7b"], n_layer=n_layer, wtype=1)
    e, f, v = hp["n_embd"], hp["n_ff"], hp["n_vocab"]
    layer_w = 4 * e * e + 3 * e * f                        # wq wk wv wo, w1 w2 w3
    w_bytes = 2 * (n_layer * layer_w + v * e)              # every streamed weight: the layers and the lm_head
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=2048))
    m.synthesize(0x5EED)
    L = m.L
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=512))
    toks = synth.make_tokens(hp, 1024)
    info = card()

    s.evaluate(toks[:512])                                 # prefill@512, warm-up
    s.rewind(0)
    L.b200_timing_begin()
    s.evaluate(toks[:512])
    prefill_ms = L.b200_timing_end_ms()
    for i in range(8):                                     # decode at n_past 512..
        s.evaluate(toks[512 + i:513 + i])
    launches = s.last_launches
    s.rewind(512)
    L.b200_timing_begin()
    for i in range(64):
        s.evaluate(toks[512 + i:513 + i])
    decode_ms = L.b200_timing_end_ms() / 64

    n = C.c_int64(0); nbytes = C.c_double(0.0)
    reps = 8
    mv_ms = L.b200_session_probe_matvec(s._s, reps, C.byref(n), C.byref(nbytes)) / reps
    prefill_fma_all = 512 * n_layer * layer_w + v * e     # the lm_head runs on the last row only
    out = dict(card=info.get("name"), power_limit=info.get("power.limit"), sm_clock=info.get("clocks.sm"), sm_clock_max=info.get("clocks.max.sm"),
               n_layer=n_layer, weight_bytes_per_token=w_bytes, decode_ms=round(decode_ms, 4), decode_launches_per_token=launches,
               decode_hbm_share=round(w_bytes / (decode_ms * 1e-3) / HBM, 4),
               matvec_ms=round(mv_ms, 4), matvec_bytes=nbytes.value / reps, matvec_hbm_share=round(nbytes.value / reps / (mv_ms * 1e-3) / HBM, 4),
               prefill512_ms=round(prefill_ms, 3), prefill512_weight_fma=prefill_fma_all,
               prefill512_fp32_share=round(prefill_fma_all / (prefill_ms * 1e-3) / FP32_FMA, 4),
               decode_floor_ms=round(w_bytes / HBM * 1e3, 3), prefill_floor_ms=round(prefill_fma_all / FP32_FMA * 1e3, 2))
    print(json.dumps(out), flush=True)
    s.close(); m.close()
    assert np.isfinite(decode_ms)


if __name__ == "__main__":
    main()
