"""BASELINE.json configs[4]: quant-format sweep Q4_0 / Q4_1 / Q5_0 / Q5_1 / Q8_0 on GPT-NeoX-20B geometry (44 layers, n_embd 6144, 64 heads of 96, n_rot 24,
vocab 50432), one H100: decode@1 at n_past = 512 through the native fused schedule (8 kernels per layer from one CUDA graph), device-resident, CUDA events;
tokens/s, ms/token and the fraction of the HBM roofline (every weight byte once + the f16 KV cache read).  Weights are generated on the device.
Usage: python tools/neox_sweep.py [--layers 44] [--steps 32] [--formats q4_0,q8_0] > neox20b_sweep.json"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from llm_b200 import _lib                                    # noqa: E402
from llm_b200.neox import GptNeoX                             # noqa: E402

TYPES = {"q4_0": (2, 18), "q4_1": (3, 20), "q5_0": (6, 22), "q5_1": (7, 24), "q8_0": (8, 34)}
N_PAST = 512


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=44)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--formats", default="q4_0,q4_1,q5_0,q5_1,q8_0")
    args = ap.parse_args()
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {"hbm_gbs": 3350.0}   # H100 SXM data sheet
    L = _lib.lib()
    out = []
    for name in args.formats.split(","):
        t, blk = TYPES[name]
        hp = dict(n_vocab=50432, n_ctx=2048, n_embd=6144, n_head=64, n_layer=args.layers, n_rot=24, use_parallel_residual=1, wtype=t)
        t0 = time.time()
        m = GptNeoX(hp, None, context_size=2048)
        m.synthesize(0x4E580000)
        s = m.start_session(512)
        toks = np.random.default_rng(7).integers(0, hp["n_vocab"], N_PAST + 1, dtype=np.int32)
        L.b200_timing_begin()
        s.evaluate(toks[:N_PAST])                              # prefill@512 (node-by-node exact kernels incl. the wgmma GEMM); fills the KV cache
        pf_ms = L.b200_timing_end_ms()
        logits = s.evaluate(toks[N_PAST:N_PAST + 1])
        assert np.isfinite(logits).all()
        launches = s.last_launches
        for _ in range(4):
            s.rewind(N_PAST); L.b200_neox_evaluate_device(s._s, 1)
        s.sync()
        L.b200_timing_begin()
        for _ in range(args.steps):
            s.rewind(N_PAST); L.b200_neox_evaluate_device(s._s, 1)
        ms = L.b200_timing_end_ms() / args.steps
        e = hp["n_embd"]
        wbytes = m.weight_bytes
        kv = 2 * hp["n_layer"] * (N_PAST + 1) * e * 2
        gbs = (wbytes + kv) / (ms * 1e-3) / 1e9
        rec = {"format": name, "n_layer": hp["n_layer"], "decode_tokens_per_s": 1e3 / ms, "ms_per_token": ms, "launches_per_token": launches, "weight_bytes_per_token": wbytes,
               "kv_bytes_per_token": kv, "achieved_gbs": gbs, "hbm_peak_gbs": peaks["hbm_gbs"], "frac_of_hbm_roofline": gbs / peaks["hbm_gbs"],
               "hbm_floor_tokens_per_s": peaks["hbm_gbs"] * 1e9 / (wbytes + kv), "prefill512_ms_first_call": pf_ms, "setup_s": time.time() - t0}
        print(json.dumps(rec), flush=True)
        out.append(rec)
        s.close(); m.close()
    print(json.dumps({"config": "GPT-NeoX-20B geometry, decode batch=1 n_past=512, 1 x H100, conformant (bit-exact) kernels", "results": out}))


if __name__ == "__main__":
    main()
