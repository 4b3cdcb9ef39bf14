"""GPT-J 6B on one H100: 28 layers, n_embd 4096, 16 heads of 256, n_rot 64, vocab 50400, Q4_0, weights synthesised on the device.  decode@1 at n_past = 512
through the native fused schedule (6 kernels per layer + 3, the wide cluster attention with 8 CTAs per head, one CUDA graph per context bucket) and
prefill@512, both timed with CUDA events after a warm-up; GPU name, power limit and SM clock are read with nvidia-smi right after the timed loops.
Parity is the tests' job (tests/test_gpu_gptj.py), not this script's.
Usage: python tools/gptj_decode_bench.py [--layers 28] [--steps 64] [--warmup 8] [--prefill-reps 4]   (one JSON line)"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from llm_b200 import _lib                                    # noqa: E402
from llm_b200.neox import GptJ                                # noqa: E402
from mpt_decode_bench import sm_clock                         # noqa: E402

N_PAST = 512


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--prefill-reps", type=int, default=4)
    args = ap.parse_args()
    L = _lib.lib()
    hp = dict(n_vocab=50400, n_ctx=2048, n_embd=4096, n_head=16, n_layer=args.layers, n_rot=64, wtype=2)
    m = GptJ(hp, None)
    m.synthesize(0x47504A00)
    s = m.start_session(512)
    toks = np.random.default_rng(7).integers(0, hp["n_vocab"], N_PAST + 1, dtype=np.int32)
    s.evaluate(toks[:N_PAST])                                  # prefill@512 fills the KV cache (and stages the tokens for the device-side reruns)
    for _ in range(args.warmup // 4 + 1):
        s.rewind(0); L.b200_neox_evaluate_device(s._s, N_PAST)
    s.sync()
    L.b200_timing_begin()
    for _ in range(args.prefill_reps):
        s.rewind(0); L.b200_neox_evaluate_device(s._s, N_PAST)
    prefill_ms = L.b200_timing_end_ms() / args.prefill_reps
    assert np.isfinite(s.evaluate(toks[N_PAST:N_PAST + 1])).all()
    launches = s.last_launches
    assert launches == 6 * args.layers + 3, launches
    for _ in range(args.warmup):
        s.rewind(N_PAST); L.b200_neox_evaluate_device(s._s, 1)
    s.sync()
    L.b200_timing_begin()
    for _ in range(args.steps):
        s.rewind(N_PAST); L.b200_neox_evaluate_device(s._s, 1)
    ms = L.b200_timing_end_ms() / args.steps
    clock = sm_clock()
    kv = 2 * args.layers * (N_PAST + 1) * hp["n_embd"] * 2
    print(json.dumps(dict(config="GPT-J 6B geometry Q4_0, decode batch 1 at n_past 512 and prefill of 512, 1 GPU, bit-exact kernels", n_layer=args.layers,
                          steps=args.steps, decode_tokens_per_s=1e3 / ms, ms_per_token=ms, launches_per_token=launches, weight_bytes_per_token=m.weight_bytes,
                          kv_bytes_per_token=kv, achieved_gbs=(m.weight_bytes + kv) / (ms * 1e-3) / 1e9,
                          prefill_tokens=N_PAST, prefill_ms=prefill_ms, prefill_tokens_per_s=N_PAST * 1e3 / prefill_ms, **clock)), flush=True)
    s.close(); m.close()


if __name__ == "__main__":
    main()
