"""What the norms' in-order fallback costs: the seam's rms_norm / norm kernels (rowops.cu) on rows whose tree sum is settled by row_sum_settled
(random rows) and on rows where it is not, so one thread adds the row again in index order (the adversarial rows of tests/test_gpu_row_sums.py:
every row of the batch takes the fallback).  n = 4096 and 8192; one row (the latency a decode step's norm would pay) and 512 rows (a prefill).
CUDA events around --reps back-to-back launches on the library's stream (b200_op_norm_device), after a warm-up.  The card's name and power limit
are read in the same run.  Usage: python tools/row_sum_bench.py [--reps 200]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}


def time_us(L, op, x, y, n, rows, reps):
    args = (op, x.data_ptr(), y.data_ptr(), n, rows, 5e-6)
    for _ in range(10):
        assert L.b200_op_norm_device(*args) == 0
    L.b200_timing_begin()
    for _ in range(reps):
        L.b200_op_norm_device(*args)
    return L.b200_timing_end_ms() / reps * 1e3


def main():
    import torch

    from llm_b200 import _lib
    from test_gpu_row_sums import f32_row
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    L = _lib.lib()
    assert L.b200_init(0) == 0
    rng = np.random.default_rng(7)
    res = dict(card=card(), reps=a.reps, runs=[])
    for n in (4096, 8192):
        for op, name in ((1, "rms_norm"), (2, "norm")):
            for rows in (1, 512):
                fast = (rng.standard_normal((rows, n)) * 3).astype(np.float32)
                slow = np.stack([f32_row("rms" if op == 1 else "norm", n, n + r) for r in range(min(rows, 8))])
                slow = np.resize(slow, (rows, n)).astype(np.float32)
                t = {}
                for kind, rows_h in (("fast", fast), ("fallback", slow)):
                    x = torch.from_numpy(rows_h).cuda()
                    y = torch.empty_like(x)
                    torch.cuda.synchronize()
                    t[kind] = time_us(L, op, x, y, n, rows, a.reps)
                res["runs"].append(dict(op=name, n=n, rows=rows, fast_us=round(t["fast"], 2), fallback_us=round(t["fallback"], 2),
                                        fallback_extra_us=round(t["fallback"] - t["fast"], 2)))
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
