"""Per-tensor weight types at LLaMA-7B geometry (32 layers, n_embd 4096, n_ff 11008, 32000 logits), weights synthesised on the device:

  decode@1 at n_past 512 and prefill@512 for   Q4_0 (one type) | Q4_0 + Q6_K output.weight | Q4_K_M (the quantizer's mix)
  the K-quant decode mat-vec alone (every mat-vec of a pure Q4_K / Q6_K model, b200_session_probe_matvec) in GB/s and as a share of 3.35 TB/s

The timed quantities end in a device synchronise (evaluate copies its logits back).  Prints one JSON line per measurement and the GPU's name,
power limit and SM clock.  Usage: python tools/kquant_bench.py [--layers 32] [--steps 32]

--op-sweep [--lib path/to/libllm_b200.so]: instead, the K-quant mat-mul kernels alone through b200_op_mul_mat at K = N = 4096 for B in 1 .. 512,
each kernel's device time from torch.profiler (CUDA activities), of this build or of another build of the library (to compare kernels)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import llm_b200  # noqa: E402
from oracle import kquant as KQ  # noqa: E402
from oracle import synth  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def model(hp, mix):
    base = KQ.MIXES["q4_0" if mix == "q4_0-only" else mix][0]
    types = {} if mix == "q4_0-only" else {k: v for k, v in KQ.mix_types(hp, mix).items() if v != base}
    hp = dict(hp, wtype=base)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), None, tensor_types=types or None)
    m.synthesize(0x5EED)
    return m, types


def time_session(m, hp, steps):
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=512))
    toks = synth.make_tokens(hp, 512 + steps + 8)
    s.evaluate(toks[:512])                                      # warm-up of the prefill shapes
    s.rewind(0)
    t0 = time.perf_counter(); s.evaluate(toks[:512]); t_pre = time.perf_counter() - t0
    for i in range(4):                                          # warm-up: the first step runs eagerly, the next captures the graph
        s.evaluate(toks[512 + i:513 + i])
    s.rewind(512)
    t0 = time.perf_counter()
    for i in range(steps):
        s.evaluate(toks[512 + i:513 + i])
    t_dec = (time.perf_counter() - t0) / steps
    launches = s.last_launches
    s.close()
    return t_pre, t_dec, launches


def op_sweep(lib_path):
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from llm_b200 import _lib
    path = os.path.abspath(lib_path) if lib_path else _lib.LIB_PATH
    L = C.CDLL(path)                                                # only the two entry points every build has
    L.b200_init.argtypes = [C.c_int]
    L.b200_op_mul_mat.argtypes = [C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32]
    assert L.b200_init(0) == 0
    torch.cuda.init()
    K = N = 4096
    rng = np.random.default_rng(1)
    print(json.dumps({"gpu": gpu_info(), "lib": path}), flush=True)
    for t, tname in ((10, "Q2_K"), (12, "Q4_K"), (14, "Q6_K")):
        wq = rng.integers(0, 256, size=(N, K // 256 * KQ.B.SUPER_BLOCK_BYTES[t]), dtype=np.uint8)
        d_off = {10: 80, 12: 0, 14: 208}[t]
        for off in (d_off, d_off + 2) if t != 14 else (d_off,):      # finite fp16 d / dmin
            wq.reshape(N, -1, KQ.B.SUPER_BLOCK_BYTES[t])[:, :, off:off + 2] = np.frombuffer(np.float16(1e-3).tobytes(), np.uint8)
        for Bn in (1, 2, 4, 8, 16, 32, 64, 128, 512):
            x = rng.standard_normal((Bn, K)).astype(np.float32)
            out = np.empty((Bn, N), np.float32)
            for _ in range(3):
                L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, out.ctypes.data, 0)
            reps = 20
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, out.ctypes.data, 0)
            us = {}
            for e in prof.key_averages():
                if "kq" in e.key and "quantize" not in e.key and "get_rows" not in e.key:
                    dt = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    us[e.key.split("(")[0][-60:]] = round(dt / reps, 2)
            print(json.dumps({"type": tname, "K": K, "N": N, "B": Bn, "kernel_us": us}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--op-sweep", action="store_true")
    ap.add_argument("--lib", default=None)
    a = ap.parse_args()
    if a.op_sweep:
        op_sweep(a.lib)
        return
    hp = dict(synth.CONFIGS["7b"], n_layer=a.layers, n_ctx=1024)
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for mix in ("q4_0-only", "q4_0", "q4_K_M"):
        m, types = model(hp, mix)
        t_pre, t_dec, launches = time_session(m, hp, a.steps)
        name = {"q4_0-only": "Q4_0", "q4_0": "Q4_0 + Q6_K output", "q4_K_M": "Q4_K_M"}[mix]
        print(json.dumps({"model": name, "layers": a.layers, "prefill512_ms": round(t_pre * 1e3, 2), "prefill512_tok_s": round(512 / t_pre, 1),
                          "decode_at_512_ms": round(t_dec * 1e3, 3), "decode_launches": launches,
                          "weight_bytes": int(m.L.b200_model_weight_bytes(m._m))}), flush=True)
        m.close()
    for t, tname in ((12, "Q4_K"), (14, "Q6_K")):
        hp1 = dict(hp, wtype=t)
        m = llm_b200.Llama(hp1, llm_b200.ModelParameters(context_size=hp1["n_ctx"]), None)
        m.synthesize(0x5EED)
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=1))
        n, b = C.c_int64(0), C.c_double(0)
        m.L.b200_session_probe_matvec.restype = C.c_float
        m.L.b200_session_probe_matvec.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_double)]
        ms = m.L.b200_session_probe_matvec(s._s, 5, C.byref(n), C.byref(b))
        gbs = b.value / (ms * 1e-3) / 1e9
        print(json.dumps({"matvec": tname, "layers": a.layers, "launches": n.value, "ms": round(ms, 3), "GB_s": round(gbs, 1),
                          "share_of_3.35TB_s": round(gbs / 3350, 3)}), flush=True)
        s.close(); m.close()
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
