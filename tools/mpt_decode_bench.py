"""MPT-7B decode on one H100: 32 layers, n_embd 4096, 32 heads, vocab 50432, Q4_0, weights synthesised on the device.  decode@1 at n_past = 512
through the native fused schedule (8 kernels per layer + 3, ALiBi in the cluster attention, one CUDA graph per context bucket), timed with CUDA events
after a warm-up; the SM clock is read with nvidia-smi right after the timed loop.  Parity is the tests' job (tests/test_gpu_alibi.py), not this script's.
Usage: python tools/mpt_decode_bench.py [--layers 32] [--steps 64] [--warmup 8]   (one JSON line)"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from llm_b200 import _lib                                    # noqa: E402
from llm_b200.neox import Mpt                                 # noqa: E402

N_PAST = 512


def sm_clock():
    """current and maximum SM clock (MHz), GPU name and power limit as nvidia-smi reports them (read only)"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,clocks.sm,clocks.max.sm,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "sm_clock_mhz": float(q[1]), "sm_clock_max_mhz": float(q[2]), "power_limit_w": float(q[3])}
    except Exception as e:                                    # noqa: BLE001 -- the number stands without it, marked as unknown
        return {"sm_clock_mhz": None, "nvidia_smi_error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    L = _lib.lib()
    hp = dict(n_vocab=50432, n_ctx=2048, n_embd=4096, n_head=32, n_layer=args.layers, wtype=2, alibi_bias_max=8.0)
    m = Mpt(hp, None)
    m.synthesize(0x4D500000)
    s = m.start_session(512)
    toks = np.random.default_rng(7).integers(0, hp["n_vocab"], N_PAST + 1, dtype=np.int32)
    s.evaluate(toks[:N_PAST])                                  # prefill@512 fills the KV cache
    assert np.isfinite(s.evaluate(toks[N_PAST:N_PAST + 1])).all()
    launches = s.last_launches
    assert launches == 8 * args.layers + 3, launches
    for _ in range(args.warmup):
        s.rewind(N_PAST); L.b200_neox_evaluate_device(s._s, 1)
    s.sync()
    L.b200_timing_begin()
    for _ in range(args.steps):
        s.rewind(N_PAST); L.b200_neox_evaluate_device(s._s, 1)
    ms = L.b200_timing_end_ms() / args.steps
    clock = sm_clock()
    kv = 2 * args.layers * (N_PAST + 1) * hp["n_embd"] * 2
    print(json.dumps(dict(config="MPT-7B geometry Q4_0, decode batch 1 at n_past 512, 1 GPU, bit-exact kernels", n_layer=args.layers, steps=args.steps,
                          decode_tokens_per_s=1e3 / ms, ms_per_token=ms, launches_per_token=launches, weight_bytes_per_token=m.weight_bytes,
                          kv_bytes_per_token=kv, achieved_gbs=(m.weight_bytes + kv) / (ms * 1e-3) / 1e9, **clock)), flush=True)
    s.close(); m.close()


if __name__ == "__main__":
    main()
