"""Model quantization, measured: a LLaMA-7B-geometry F16 file (n_embd 4096, n_ff 11008, n_vocab 32000, --layers layers; 4 layers is ~2.1 GB)
is synthesized in a temporary directory (deleted afterwards) and quantized to --target.

  end_to_end_s   llm_b200.quantize on the file, host clock, page cache warm (one untimed run first), ending after the output is closed
  kernel         the quantize kernel alone over the same tensors resident in HBM, CUDA events: bytes read + written / kernel time
  reference_s    the reference's ggml_quantize_<target> (oracle/_ref/libggml_ref.so) on one host thread, as its `quantize` runs it: the
                 tensors widened to f32 first (not timed), then one call per tensor (timed)

The card's name and power limit are read in the same run.  Usage: python tools/quantize_bench.py [--layers 4] [--target q4_0] [--reps 3]"""
import argparse
import ctypes as C
import json
import os
import shutil
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), (v.strip() for v in out[0].split(",")))) if out else {}


def shapes(n_layer, e=4096, f=11008, v=32000):
    out = [("tok_embeddings.weight", (v, e)), ("norm.weight", (e,)), ("output.weight", (v, e))]
    for i in range(n_layer):
        p = f"layers.{i}."
        out += [(p + "attention_norm.weight", (e,)), (p + "attention.wq.weight", (e, e)), (p + "attention.wk.weight", (e, e)),
                (p + "attention.wv.weight", (e, e)), (p + "attention.wo.weight", (e, e)), (p + "ffn_norm.weight", (e,)),
                (p + "feed_forward.w1.weight", (f, e)), (p + "feed_forward.w2.weight", (e, f)), (p + "feed_forward.w3.weight", (f, e))]
    return out


def synthesize(path, n_layer):
    """GGJT v3, F16 2-D weights N(0, 1/64) drawn from a 16 Mi-value pool at a different offset per tensor (the timing does not depend on the
    values), f32 norms.  Returns [(name, f16 array view of the weight)] of the 2-D tensors (the pool slices, for the kernel and reference legs)."""
    rng = np.random.default_rng(0)
    pool = (rng.standard_normal(1 << 24, np.float32) / 64).astype(np.float16)
    pool2 = np.concatenate([pool, pool])
    weights = []
    with open(path, "wb") as fp:
        fp.write(struct.pack("<II", 0x67676A74, 3) + struct.pack("<7i", 32000, 4096, 256, 32, n_layer, 128, 1))
        for i in range(32000):
            tok = b"t%d" % i
            fp.write(struct.pack("<I", len(tok)) + tok + struct.pack("<f", 0.0))
        for k, (name, shp) in enumerate(shapes(n_layer)):
            nb = name.encode()
            ne = shp[::-1]
            fp.write(struct.pack("<iiI", len(shp), len(nb), 1 if len(shp) == 2 else 0) + struct.pack(f"<{len(ne)}i", *ne) + nb)
            fp.write(bytes(-fp.tell() % 32))
            if len(shp) == 1:
                fp.write(np.ones(shp, np.float32).tobytes())
                continue
            n = shp[0] * shp[1]
            off = (k * 7919 * 32) % (1 << 24)
            reps = []
            left = n
            while left > 0:                                              # the pool tiled from `off`
                take = min(left, 1 << 24)
                reps.append(pool2[off:off + take])
                left -= take
            w = np.concatenate(reps)
            fp.write(w.tobytes())
            weights.append((name, w))
    return weights


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--target", default="q4_0")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import llm_b200
    from llm_b200 import _lib
    from llm_b200.quantize import TARGETS
    target = TARGETS[a.target]
    L = _lib.lib()
    assert L.b200_init(0) == 0
    tmp = tempfile.mkdtemp(prefix="quantize_bench_")
    try:
        src, dst = os.path.join(tmp, "f16.bin"), os.path.join(tmp, f"{a.target}.bin")
        weights = synthesize(src, a.layers)
        src_bytes = os.path.getsize(src)

        with open(src, "rb") as fp:                                      # page cache warm
            while fp.read(1 << 26):
                pass
        llm_b200.quantize(src, dst, "llama", target)
        e2e = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            llm_b200.quantize(src, dst, "llama", target)
            e2e.append(time.perf_counter() - t0)
        dst_bytes = os.path.getsize(dst)

        import torch
        bb = {2: 18, 3: 20, 6: 22, 7: 24, 8: 34}[target]
        dev = [(torch.from_numpy(w.view(np.int16)).cuda(), torch.empty(w.size // 32 * bb, dtype=torch.uint8, device="cuda")) for _, w in weights]
        hist = torch.zeros(16, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        for s, d in dev:                                                  # warm-up
            L.b200_op_quantize_blocks_device(target, 1, s.data_ptr(), s.numel() // 32, d.data_ptr(), hist.data_ptr())
        kms = []
        for _ in range(a.reps):
            L.b200_timing_begin()
            for s, d in dev:
                L.b200_op_quantize_blocks_device(target, 1, s.data_ptr(), s.numel() // 32, d.data_ptr(), hist.data_ptr())
            kms.append(L.b200_timing_end_ms())
        k_bytes = sum(s.numel() * 2 + d.numel() for s, d in dev)
        del dev
        torch.cuda.empty_cache()

        ref_s = None
        ref_lib = os.path.join(ROOT, "oracle", "_ref", "libggml_ref.so")
        if os.path.exists(ref_lib):
            R = C.CDLL(ref_lib)
            f = getattr(R, f"ggml_quantize_{a.target}")
            f.restype = C.c_size_t
            f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
            h = np.zeros(16, np.int64)
            ref_s = 0.0
            for name, w in weights:
                x = w.astype(np.float32)                                  # the reference's Vec<f32> (not timed)
                out = np.empty(x.size // 32 * bb, np.uint8)
                t0 = time.perf_counter()
                f(x.ctypes.data, out.ctypes.data, x.size, 4096 if "w2" not in name else 11008, h.ctypes.data)
                ref_s += time.perf_counter() - t0
        info = card()
        kbest = min(kms)
        print(json.dumps(dict(card=info.get("name"), power_limit=info.get("power.limit"), layers=a.layers, target=a.target, source_bytes=src_bytes,
                              output_bytes=dst_bytes, end_to_end_s=[round(t, 3) for t in e2e], end_to_end_GBps=round(src_bytes / min(e2e) / 1e9, 2),
                              kernel_ms=[round(t, 3) for t in kms], kernel_bytes=k_bytes, kernel_GBps=round(k_bytes / (kbest * 1e-3) / 1e9, 1),
                              reference_s=None if ref_s is None else round(ref_s, 3),
                              reference_GBps_of_f16=None if ref_s is None else round(sum(w.size * 2 for _, w in weights) / ref_s / 1e9, 3))))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
