"""Session snapshots, measured: a LLaMA-7B-geometry Q4_0 model (n_embd 4096, 32 layers, n_vocab 32000) and an MPT-7B-geometry one (V kept by position in
the reference, so memory_v is transposed on the way out and in), synthesized in HBM, context 2048, n_past 2000, f16 and f32 caches.

  get_s      b200_*_get_snapshot into host buffers touched by an untimed call first (the ring's D2H, then a copy out of the pinned slots)
  write_s    write_snapshot to a file in --dir (the page cache: the file is not synced), host clock, ending after the file is closed
  disk_s     writing the same bytes from host memory to a file there with Python (the disk / page-cache leg alone)
  read_s     read_snapshot of that file into a new session (the session's allocation included)
  *_gbs      cache bytes (memory_k + memory_v) / time
  transpose  the transpose kernel alone on one layer of the MPT cache, [4096][2048] -> [2048][4096], CUDA events over --reps2 launches: bytes read +
             written / time, and as a share of the H100 SXM data sheet's 3.35 TB/s
The ring overlaps each chunk's download with the previous chunk's write, so write_s should be close to max(get_s, disk_s), not their sum.  The
card's name and power limit are read in the same run.  Usage: python tools/snapshot_bench.py [--dir DIR] [--reps 3] [--reps2 200]"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35          # H100 SXM5 80 GB data sheet


def card():
    q = "name,power.limit"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), (v.strip() for v in out[0].split(",")))) if out else {}


def session(arch, kv):
    import llm_b200
    from llm_b200.neox import Mpt
    kvt = llm_b200.ModelKVMemoryType.Float32 if kv == "f32" else llm_b200.ModelKVMemoryType.Float16
    if arch == "llama":
        hp = dict(n_vocab=32000, n_embd=4096, n_head=32, n_head_kv=32, n_layer=32, n_rot=128, n_ff=11008, wtype=llm_b200.Q4_0)
        m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=2048))
        m.synthesize()
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=512, memory_k_type=kvt, memory_v_type=kvt))
    else:
        hp = dict(n_vocab=50432, n_ctx=2048, n_embd=4096, n_head=32, n_layer=32, wtype=llm_b200.Q4_0, alibi_bias_max=8.0)
        m = Mpt(hp)
        m.synthesize()
        s = m.start_session(512, memory_k_type=kvt, memory_v_type=kvt)
    toks = (np.arange(2000, dtype=np.int32) * 37) % hp["n_vocab"]
    for a in range(0, 2000, 512):
        s.evaluate(toks[a:a + 512])
    s.sync()
    return m, s


def measure(arch, kv, d, reps):
    from llm_b200 import _lib
    m, s = session(arch, kv)
    get = s.L.b200_session_get_snapshot if arch == "llama" else s.L.b200_neox_get_snapshot
    h = _lib.Snapshot()
    assert get(s._s, C.byref(h)) == 0
    bufs = [np.empty(h.n_tokens, np.uint32), np.empty(h.n_logits, np.float32), np.ones(h.memory_k_bytes, np.uint8), np.ones(h.memory_v_bytes, np.uint8)]
    h.tokens, h.last_logits, h.memory_k, h.memory_v = (b.ctypes.data for b in bufs)
    cache = h.memory_k_bytes + h.memory_v_bytes
    get_s, write_s, disk_s, read_s = [], [], [], []
    path, raw = os.path.join(d, f"{arch}_{kv}.session"), os.path.join(d, "raw.bin")
    for _ in range(reps):
        t = time.perf_counter()
        assert get(s._s, C.byref(h)) == 0
        get_s.append(time.perf_counter() - t)
        t = time.perf_counter()
        s.write_snapshot(path)
        write_s.append(time.perf_counter() - t)
        t = time.perf_counter()
        with open(raw, "wb") as f:
            f.write(bufs[2].data)
            f.write(bufs[3].data)
        disk_s.append(time.perf_counter() - t)
        os.unlink(raw)
        t = time.perf_counter()
        r = type(s).read_snapshot(path, m)
        r.sync()
        read_s.append(time.perf_counter() - t)
        assert r.n_past == 2000
        r.close()
    out = dict(arch=arch, kv=kv, n_past=2000, context=2048, cache_bytes=cache, file_bytes=os.path.getsize(path))
    for k, v in (("get", get_s), ("write", write_s), ("disk", disk_s), ("read", read_s)):
        out[k + "_s"] = round(min(v), 4)
        out[k + "_gbs"] = round(cache / min(v) / 1e9, 2)
    out["write_vs_max_get_disk"] = round(min(write_s) / max(min(get_s), min(disk_s)), 2)
    out["write_vs_sum_get_disk"] = round(min(write_s) / (min(get_s) + min(disk_s)), 2)
    os.unlink(path)
    s.close(); m.close()
    return out


def transpose_kernel(reps):
    import torch
    from llm_b200 import _lib
    L = _lib.lib()
    rows, cols = 4096, 2048                  # one MPT-7B layer of memory_v: [n_embd][n_ctx] -> [n_ctx][n_embd]
    out = {}
    for es, dt in ((2, torch.float16), (4, torch.float32)):
        src = torch.randn(rows * cols, device="cuda").to(dt)
        dst = torch.empty_like(src)
        torch.cuda.synchronize()
        args = (es, src.data_ptr(), cols, dst.data_ptr(), rows, rows, cols)
        assert L.b200_op_transpose_device(*args) == 0
        L.b200_timing_begin()
        for _ in range(reps):
            L.b200_op_transpose_device(*args)
        ms = L.b200_timing_end_ms() / reps
        assert torch.equal(dst.view(cols, rows).cpu(), src.view(rows, cols).t().contiguous().cpu())
        tbs = 2 * rows * cols * es / (ms * 1e-3) / 1e12
        out["f16" if es == 2 else "f32"] = dict(us=round(ms * 1e3, 2), tb_per_s=round(tbs, 3), share_of_hbm=round(tbs / HBM_TBS, 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", default=None, help="where the session files go (default: a temporary directory, removed afterwards)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--reps2", type=int, default=200)
    a = ap.parse_args()
    d = a.dir or tempfile.mkdtemp(prefix="snapshot_bench_")
    os.makedirs(d, exist_ok=True)
    try:
        res = dict(card=card(), runs=[measure(arch, kv, d, a.reps) for arch, kv in (("llama", "f16"), ("llama", "f32"), ("mpt", "f16"), ("mpt", "f32"))],
                   transpose=transpose_kernel(a.reps2))
    finally:
        if not a.dir:
            shutil.rmtree(d, ignore_errors=True)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
