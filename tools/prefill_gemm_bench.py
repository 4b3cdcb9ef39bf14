"""Kernel-only timing of the prefill weight mat-muls (7B shapes, 512 tokens) for the exact kernels: mma.sync (exact_mma.cu, impl 6)
vs wgmma (exact_tc5.cu, impl 7) [and the order-free int8 kernel, impl 3].  Prints ms, useful TFLOP/s (2*B*N*K) and the fp32-pipe
fraction (9 fp32 ops per token*row*block on every SM x 128 lanes at the SM clock given, default the H100's 1980 MHz boost).  Usage: python tools/prefill_gemm_bench.py [wtype] [B] [impls] [sm_mhz]"""
import ctypes as C
import sys

sys.path.insert(0, ".")
from llm_b200 import _lib

L = _lib.lib()
L.b200_op_bench_mul_mat.argtypes = [C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.POINTER(C.c_float)]
L.b200_init(0)
n_sm = C.c_int32(0)
assert L.b200_device_info(C.byref(n_sm), None, None) == 0
sm_hz = (float(sys.argv[4]) if len(sys.argv) > 4 else 1980.0) * 1e6
wtype = int(sys.argv[1]) if len(sys.argv) > 1 else 2
B = int(sys.argv[2]) if len(sys.argv) > 2 else 512
impls = [int(a) for a in sys.argv[3].split(",")] if len(sys.argv) > 3 else [6, 7]
shapes = [("qkv", 4096, 12288), ("wo", 4096, 4096), ("w13", 4096, 22016), ("w2", 11008, 4096), ("lm_head", 4096, 32000)]
tot = {i: 0.0 for i in impls}
for name, K, N in shapes:
    for impl in impls:
        ms = C.c_float()
        rc = L.b200_op_bench_mul_mat(wtype, K, N, B, impl, 10, C.byref(ms))
        fl = 2.0 * B * N * K
        fp32 = 9.0 * B * N * (K // 32) / (n_sm.value * 128 * sm_hz)
        print(f"{name:8s} K={K:6d} N={N:6d} B={B} impl={impl} rc={rc} {ms.value:8.3f} ms  {fl / ms.value / 1e9:8.1f} TFLOP/s  fp32-pipe floor {fp32 * 1e3:6.3f} ms ({fp32 * 1e3 / ms.value:5.2f})", flush=True)
        tot[impl] += ms.value * (32 if name != "lm_head" else 1)
for impl in impls:
    print(f"impl {impl}: 32 layers + lm_head = {tot[impl]:.1f} ms")
