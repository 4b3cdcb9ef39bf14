"""Per-op parity of the CUDA kernels against the oracle, called THROUGH the C ABI:
  * the ggml_cuda_* seam with hand-built `struct ggml_tensor`s (llm_b200/ggml.py = the ctypes stub of the plugin API)
  * the b200_op_* host-buffer entry points.
Bars: BIT-EXACT for the default kernels (exact.cu reproduces the AVX2 operation order, rowops.cu the reference's row sums) and for every
integer/byte/LUT result;
the order-free fast kernels (mmvq/mmq/attn.cu) are held to f32 summation noise (<= 2e-6 of the row scale)."""
import ctypes as C

import numpy as np
import pytest

from oracle import bindings as B

pytestmark = pytest.mark.gpu

TYPES = list(B.QUANT_TYPES.items())


def rel(g, c):
    return float(np.abs(g.astype(np.float64) - c).max() / max(np.abs(c).max(), 1e-30))


@pytest.fixture(scope="module")
def ctx():
    from llm_b200 import ggml
    c = ggml.Context()
    yield c
    c.close()


@pytest.fixture(scope="module")
def L():
    from llm_b200 import _lib
    lib = _lib.lib()
    assert lib.b200_init(0) == 0
    return lib


@pytest.mark.parametrize("vdt", [B.Q8_0, B.Q8_1])
def test_quantize_act_bit_exact(L, orc, vdt):
    rng = np.random.default_rng(3)
    K, Bn = 4096, 7
    x = (rng.standard_normal((Bn, K)) * rng.uniform(0.01, 20, (Bn, 1))).astype(np.float32)
    x[2, 64:96] = 0.0
    x[3] = np.round(x[3] * 4) / 4          # many exact .5 products -> exercises round-half-even
    qs = np.empty((Bn, K), np.int8); d = np.empty((Bn, K // 32), np.float32); aux = np.empty_like(d)
    assert L.b200_op_quantize_act(vdt, x.ctypes.data, K, Bn, qs.ctypes.data, d.ctypes.data, aux.ctypes.data) == 0
    for b in range(Bn):
        o = orc.from_float(vdt, x[b])
        if vdt == B.Q8_0:
            blk = o.reshape(-1, 34)
            od = blk[:, :2].copy().view(np.float16).astype(np.float32)[:, 0]
            oq = blk[:, 2:].copy().view(np.int8)
            assert np.array_equal(aux[b], oq.astype(np.int32).sum(1).astype(np.float32))
        else:
            blk = o.reshape(-1, 40)
            od = blk[:, :4].copy().view(np.float32)[:, 0]
            os_ = blk[:, 4:8].copy().view(np.float32)[:, 0]
            oq = blk[:, 8:].copy().view(np.int8)
            assert np.array_equal(aux[b].view(np.uint32), os_.view(np.uint32))
        assert np.array_equal(qs[b].reshape(-1, 32), oq)
        assert np.array_equal(d[b].view(np.uint32), od.view(np.uint32))


@pytest.mark.parametrize("name,t", TYPES)
@pytest.mark.parametrize("K,N,Bn", [(4096, 200, 1), (11008, 96, 1), (256, 33, 5), (4096, 130, 37), (704, 100, 40), (64, 5, 3),
                                     (4096, 257, 9), (5120, 64, 2)])
def test_mul_mat_bit_exact(L, orc, name, t, K, N, Bn):
    """default kernels: same bits as ggml_compute_forward_mul_mat on the reference's x86 build"""
    rng = np.random.default_rng(K * 5 + N + t)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    x = (rng.standard_normal((Bn, K)) * rng.uniform(0.05, 8, (Bn, 1))).astype(np.float32)
    wq = orc.quantize(t, w)
    want = orc.mul_mat(t, wq, x)
    got = np.empty((Bn, N), np.float32)
    assert L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, got.ctypes.data, 4) == 0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, K, N, Bn, rel(got, want))


@pytest.mark.parametrize("name,t", TYPES)
@pytest.mark.parametrize("K,N,Bn", [(4096, 200, 128), (256, 33, 16), (704, 100, 40), (11008, 48, 37), (4096, 17, 300), (64, 16, 129), (2048, 130, 512)])
def test_mul_mat_tensor_core_bit_exact(L, orc, name, t, K, N, Bn):
    """prefill GEMM with the block dots on tensor cores (block-diagonal f16 MMA, exact_mma.cu): same bits as the reference"""
    rng = np.random.default_rng(K * 11 + N + t)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    x = (rng.standard_normal((Bn, K)) * rng.uniform(0.05, 8, (Bn, 1))).astype(np.float32)
    x[Bn // 2, :32] = 0.0
    wq = orc.quantize(t, w)
    want = orc.mul_mat(t, wq, x)
    got = np.empty((Bn, N), np.float32)
    assert L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, got.ctypes.data, 6) == 0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, K, N, Bn, rel(got, want), int((got != want).sum()))


@pytest.mark.parametrize("name,t", TYPES)
@pytest.mark.parametrize("K,N,Bn", [(4096, 200, 128), (256, 33, 16), (704, 100, 40), (11008, 48, 37), (4096, 17, 300), (64, 16, 129), (2048, 130, 512),
                                     (5120, 96, 257), (128, 32, 1)])
def test_mul_mat_tcgen05_bit_exact(L, orc, name, t, K, N, Bn):
    """prefill GEMM on the warpgroup tensor cores (TMA-staged activations, block-diagonal wgmma.mma_async into registers;
    exact_tc5.cu): same bits as ggml_compute_forward_mul_mat, for every format, ragged N / token counts and K tails of the stage ring"""
    rng = np.random.default_rng(K * 13 + N + t)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    x = (rng.standard_normal((Bn, K)) * rng.uniform(0.05, 8, (Bn, 1))).astype(np.float32)
    x[Bn // 2, :32] = 0.0
    wq = orc.quantize(t, w)
    want = orc.mul_mat(t, wq, x)
    got = np.empty((Bn, N), np.float32)
    assert L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, got.ctypes.data, 7) == 0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, K, N, Bn, rel(got, want), int((got != want).sum()))


@pytest.mark.parametrize("name,t", TYPES)
@pytest.mark.parametrize("K,N,Bn", [(4096, 200, 1), (11008, 96, 2), (256, 33, 3), (5120, 1000, 1), (4096, 31, 1), (2048, 32, 1), (13824, 64, 1)])
def test_mul_mat_stream_bit_exact(L, orc, name, t, K, N, Bn):
    """decode mat-vec fed by TMA bulk copies (exact_stream.cu): same bits as the reference, any tile/chunk tail"""
    rng = np.random.default_rng(K * 3 + N + t)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    x = (rng.standard_normal((Bn, K)) * rng.uniform(0.05, 8, (Bn, 1))).astype(np.float32)
    wq = orc.quantize(t, w)
    want = orc.mul_mat(t, wq, x)
    got = np.empty((Bn, N), np.float32)
    assert L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, got.ctypes.data, 5) == 0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, K, N, Bn, rel(got, want))


@pytest.mark.parametrize("name,t", TYPES)
@pytest.mark.parametrize("K,N,Bn,impl", [(4096, 200, 1, 1), (11008, 96, 1, 1), (256, 33, 5, 2), (4096, 130, 37, 3),
                                          (704, 100, 40, 3), (4096, 256, 128, 3), (4096, 64, 3, 1)])
def test_mul_mat_fast_kernels_vs_oracle(L, orc, name, t, K, N, Bn, impl):
    rng = np.random.default_rng(K * 7 + N + t)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    x = (rng.standard_normal((Bn, K)) * 2.5).astype(np.float32)
    wq = orc.quantize(t, w)
    want = orc.mul_mat(t, wq, x)
    got = np.empty((Bn, N), np.float32)
    assert L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, got.ctypes.data, impl) == 0
    assert rel(got, want) <= 2e-6, (name, K, N, Bn, impl, rel(got, want))


@pytest.mark.parametrize("name,t", TYPES)
def test_weight_quantizer_bit_exact(L, orc, name, t):
    """ggml_quantize_q* on the GPU (the call crates/llm-base/src/quantize.rs:365-377 makes per tensor): identical GGML blocks, incl. all-zero blocks,
    blocks whose extreme value is positive / negative / repeated, and large dynamic range"""
    rng = np.random.default_rng(99 + t)
    K, N = 4096, 67
    w = (rng.standard_normal((N, K)) * rng.uniform(1e-3, 30, (N, 1))).astype(np.float32)
    w[3, :64] = 0.0
    w[5, 32:64] = np.abs(w[5, 32:64]); w[5, 40] = w[5, 32:64].max()           # tie for the maximum
    w[6, 0:32] = -np.abs(w[6, 0:32])
    w[7, 96:128] = 1.5
    want = orc.quantize(t, w)
    got = np.empty_like(want)
    assert L.b200_op_quantize_weights(t, w.ctypes.data, K, N, got.ctypes.data) == 0
    assert np.array_equal(got, want), (name, int((got != want).sum()))


@pytest.mark.parametrize("name,t", TYPES)
@pytest.mark.parametrize("K,N,Bn", [(4096, 256, 128), (704, 100, 40), (11008, 300, 200), (2048, 513, 512), (64, 16, 129)])
def test_mul_mat_fast_tcgen05_vs_oracle(L, orc, name, t, K, N, Bn):
    """fused dequant -> wgmma GEMM (mmq_tc5.cu), the order-free fast mode: fp16 operands, f32 accumulation in registers.  Held to 2e-3 of the row scale
    (it is NOT the conformant path: activations are not Q8-quantized and the summation order is the tensor core's)"""
    rng = np.random.default_rng(K * 17 + N + t)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    x = (rng.standard_normal((Bn, K)) * 2.5).astype(np.float32)
    wq = orc.quantize(t, w)
    deq = np.stack([orc.to_float(t, wq[i], K) for i in range(N)])
    want = x.astype(np.float64) @ deq.astype(np.float64).T                    # exact product with the dequantized weights, unquantized activations
    got = np.empty((Bn, N), np.float32)
    assert L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, got.ctypes.data, 8) == 0
    assert rel(got, want) <= 2e-3, (name, K, N, Bn, rel(got, want))


@pytest.mark.parametrize("name,t", TYPES)
def test_mul_mat_three_kernels_agree(L, orc, name, t):
    """decode mat-vec, CUDA-core GEMM and tensor-core GEMM are the same arithmetic up to f32 summation order"""
    rng = np.random.default_rng(11 + t)
    K, N, Bn = 2048, 192, 24
    wq = orc.quantize(t, (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32))
    x = rng.standard_normal((Bn, K)).astype(np.float32)
    outs = []
    for impl in (1, 2, 3):
        o = np.empty((Bn, N), np.float32)
        assert L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, o.ctypes.data, impl) == 0
        outs.append(o)
    assert rel(outs[0], outs[1].astype(np.float64)) <= 2e-6 and rel(outs[2], outs[1].astype(np.float64)) <= 2e-6


@pytest.mark.parametrize("name,t", TYPES)
def test_seam_mul_mat_offloaded_weight(ctx, orc, name, t):
    """The node the reference executor sends for every weight mat-mul: src0 uploaded with transform_tensor (GPU), src1 and
    dst on the host (the lm_head case, llama lib.rs:350-352)."""
    rng = np.random.default_rng(5 + t)
    K, N = 512, 96
    wq = orc.quantize(t, (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32))
    for Bn in (1, 4, 33):
        x = rng.standard_normal((Bn, K)).astype(np.float32)
        w = ctx.transfer_to_gpu(ctx.quantized(t, wq, K))
        xt = ctx.from_numpy(x)
        dst = ctx.op_mul_mat(w, xt)
        assert ctx.compute(dst, nth=4) is True
        got = ctx.host_array(dst).reshape(Bn, N)
        assert np.array_equal(got, orc.mul_mat(t, wq, x))


def _gpu_src(ctx, a):
    t = ctx.from_numpy(a)
    return ctx.transfer_to_gpu(t)


def test_seam_row_ops(ctx, orc, golden_ops):
    g = golden_ops
    x = g["row_x"]
    r = ctx.op_rms_norm(_gpu_src(ctx, x)); assert ctx.compute(r)
    assert np.array_equal(ctx.host_array(r).view(np.uint32), g["rms_norm"].view(np.uint32))
    r = ctx.op_norm(_gpu_src(ctx, x)); assert ctx.compute(r)
    assert np.array_equal(ctx.host_array(r).view(np.uint32), g["norm"].view(np.uint32))
    r = ctx.op_soft_max(_gpu_src(ctx, g["softmax_x"])); assert ctx.compute(r)
    assert np.array_equal(ctx.host_array(r).view(np.uint32), g["softmax"].view(np.uint32))
    r = ctx.op_silu(_gpu_src(ctx, x)); assert ctx.compute(r)
    assert np.array_equal(ctx.host_array(r).view(np.uint32), g["silu"].view(np.uint32))
    r = ctx.op_gelu(_gpu_src(ctx, x)); assert ctx.compute(r)
    assert np.array_equal(ctx.host_array(r).view(np.uint32), g["gelu"].view(np.uint32))


def test_seam_luts_exhaustive(ctx, golden_ops):
    g = golden_ops
    for op, key in ((ctx.op_silu, "lut_silu"), (ctx.op_gelu, "lut_gelu")):
        r = op(_gpu_src(ctx, g["lut_in"])); assert ctx.compute(r)
        assert np.array_equal(ctx.host_array(r).view(np.uint32).ravel(), g[key].view(np.uint32))


def test_seam_attention_chain(ctx, orc, golden_ops):
    g = golden_ops
    a = _gpu_src(ctx, g["chain_x"])
    s = ctx.op_scale(a, 0.125); ctx.offload_no_scratch(s); assert ctx.compute(s)
    m = ctx.op_diag_mask_inf(s, 35); ctx.offload_no_scratch(m); assert ctx.compute(m)
    r = ctx.op_soft_max(m); assert ctx.compute(r)
    assert np.array_equal(ctx.host_array(r).view(np.uint32), g["chain"].view(np.uint32))


@pytest.mark.parametrize("tag", ["llama", "llama511", "neox"])
def test_seam_rope(ctx, golden_ops, tag):
    g = golden_ops
    n_past, nd, mode = (int(v) for v in g[f"rope_{tag}_p"])
    r = ctx.op_rope(_gpu_src(ctx, g[f"rope_{tag}_x"]), n_past, nd, mode); assert ctx.compute(r)
    got = ctx.host_array(r)
    assert np.array_equal(got.view(np.uint32), g[f"rope_{tag}"].view(np.uint32)), np.abs(got - g[f"rope_{tag}"]).max()


def test_seam_mul_mat_f16_bit_exact(ctx, orc):
    """the attention mat-muls: F16 src0 (KV cache views), f32 src1 rounded to fp16, ggml_vec_dot_f16 operation order"""
    from llm_b200 import ggml
    rng = np.random.default_rng(21)
    # n < 8 or unaligned rows: one warp per dot; otherwise the shared-memory tiled kernel (16 x 32 tiles, ragged edges, leftovers k % 32)
    for k, rows, n, heads in ((128, 70, 5, 4), (64, 33, 1, 3), (45, 64, 7, 2), (513, 128, 1, 2), (96, 16, 3, 1),
                              (128, 70, 40, 4), (96, 33, 9, 2), (100, 24, 16, 2), (64, 17, 33, 1), (516, 20, 12, 1)):
        a = rng.standard_normal((heads, rows, k)).astype(np.float16)
        b = (rng.standard_normal((heads, n, k)) * 2).astype(np.float32)
        at = ctx.transfer_to_gpu(ctx.new_tensor(ggml.F16, [k, rows, heads], a))
        bt = ctx.from_numpy(b)
        dst = ctx.op_mul_mat(at, bt)
        assert ctx.compute(dst) is True
        got = ctx.host_array(dst).reshape(heads, n, rows)
        b16 = b.astype(np.float16)
        want = np.empty_like(got)
        for h in range(heads):
            for i in range(n):
                for r in range(rows):
                    want[h, i, r] = orc.vec_dot_f16(a[h, r].view(np.uint16), b16[h, i].view(np.uint16))
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (k, rows, n, heads, rel(got, want))


def test_seam_rows_large(ctx, orc):
    rng = np.random.default_rng(9)
    x = (rng.standard_normal((33, 4096)) * 3).astype(np.float32)
    r = ctx.op_rms_norm(_gpu_src(ctx, x)); assert ctx.compute(r)
    assert np.array_equal(ctx.host_array(r).view(np.uint32), orc.rms_norm(x).view(np.uint32))
    xs = (rng.standard_normal((64, 1537)) * 5).astype(np.float32)
    r = ctx.op_soft_max(_gpu_src(ctx, xs)); assert ctx.compute(r)
    assert np.array_equal(ctx.host_array(r).view(np.uint32), orc.soft_max(xs).view(np.uint32))


def test_seam_add_mul_broadcast_and_cpy(ctx):
    rng = np.random.default_rng(10)
    a = rng.standard_normal((9, 256)).astype(np.float32)
    gsc = rng.standard_normal(256).astype(np.float32)
    r = ctx.op_mul(_gpu_src(ctx, a), _gpu_src(ctx, gsc)); assert ctx.compute(r)
    assert np.array_equal(ctx.host_array(r), a * gsc)
    r = ctx.op_add(_gpu_src(ctx, a), ctx.from_numpy(a[::-1].copy())); assert ctx.compute(r)   # src1 on the host (inpSA at layer 0)
    assert np.array_equal(ctx.host_array(r), a + a[::-1])
    r = ctx.op_cpy_to(_gpu_src(ctx, a), 1); assert ctx.compute(r)                               # f32 -> f16 (KV store)
    assert np.array_equal(ctx.host_array(r, np.float16), a.astype(np.float16))


def test_seam_declines_what_it_does_not_own(ctx):
    """return false == 'CPU, it is yours' is only legal when nothing lives on the device (LC/ggml.c:14589-14590)"""
    a = ctx.from_numpy(np.ones((4, 64), np.float32))
    r = ctx.op_rms_norm(a)
    assert ctx.compute(r) is False
    from llm_b200 import ggml
    w = ctx.new_tensor(ggml.Q4_0, [64, 8])
    assert ctx.L.ggml_cuda_can_mul_mat(C.byref(w), C.byref(a), C.byref(r)) is False
