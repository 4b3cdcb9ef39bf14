"""The arithmetic of an F32 KV cache, pinned on the CPU before any GPU run (no GPU needed):

  * ggml_vec_dot_f32 as the reference's AVX2 build computes it -- 32 FMA chains, the GGML_F32x8_REDUCE tree, the leftovers (n % 32) multiplied in
    vectors of 8 and 4 and added in order, the last n % 4 as scalar FMAs, all into a float -- restated in numpy and checked bit for bit against
    the reference's own vec_dot of GGML_TYPE_F32 for every n in 1..160.  llm_b200/csrc/f32dot.cuh restates the same rule for the kernels.
  * the F32-cache reference (oracle/kv32.mk) really runs on an F32 cache: after one prefill, layer 0 of its cache rounded to fp16 is the F16
    reference's layer 0, and the logits differ."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import bindings as B
from oracle import kv32
from oracle import synth


def fma32(a, b, c):
    """fmaf: a * b + c rounded once to float32 (round to nearest, ties to even)"""
    exact = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    f = np.float32(float(exact))
    cands = [f, np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))]
    return min(cands, key=lambda x: (abs(Fraction(float(x)) - exact), int(np.float32(x).view(np.uint32)) & 1))


def vec_dot_f32(x, y):
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    n = x.size
    np_ = n & ~31
    c = [np.float32(0)] * 32
    for k in range(np_):
        c[k % 32] = fma32(x[k], y[k], c[k % 32])
    for l in range(16):
        c[l] = np.float32(c[l] + c[l + 16])
    for l in range(8):
        c[l] = np.float32(c[l] + c[l + 8])
    for l in range(4):
        c[l] = np.float32(c[l] + c[l + 4])
    s = np.float32(np.float32(c[0] + c[1]) + np.float32(c[2] + c[3]))
    left = n - np_
    nv = left & ~3
    for i in range(np_, np_ + nv):
        s = np.float32(s + np.float32(x[i] * y[i]))
    for i in range(np_ + nv, n):
        s = fma32(x[i], y[i], s)
    return np.float32(s)


def test_vec_dot_f32_restatement_matches_reference(ref):
    rng = np.random.default_rng(0xF32D07)
    for n in range(1, 161):
        for rep in range(2):
            x = (rng.standard_normal(n) * (1 if rep == 0 else 40)).astype(np.float32)
            y = rng.standard_normal(n).astype(np.float32)
            want = ref.vec_dot(B.F32, n, x, y)
            got = vec_dot_f32(x, y)
            assert np.float32(got).view(np.uint32) == np.float32(want).view(np.uint32), (n, rep, got, want)


def test_f32_cache_reaches_the_reference_graph(ref, orc):
    if not kv32.have_ref():
        pytest.skip("oracle/_ref/*_kv32.so not built")
    hp, tens = synth.make_llama(synth.CONFIGS["tiny"], B.Q4_0, ref.quantize)
    toks = synth.make_tokens(hp, 24)
    m16 = ref.llama(hp, tens, n_threads=4, n_batch=32)
    m32 = kv32.ref_lib().llama(hp, tens, n_threads=4, n_batch=32)
    l16, l32 = m16.eval(toks), m32.eval(toks)
    n0 = hp["n_ctx"] * hp["n_embd"]                    # layer 0 of [n_layer][n_ctx][n_embd]
    for which in (0, 1):
        k16 = m16.kv(which)
        k32 = kv32.kv_f32(m32, which)
        assert k16.dtype == np.uint16 and k32.size == k16.size
        assert np.array_equal(k32[:n0].astype(np.float16).view(np.uint16), k16[:n0]), which
        assert np.count_nonzero(k32[:n0]) > 0
    assert not np.array_equal(l16, l32)
    assert np.abs(l16 - l32).max() < 1e-1
    m16.close(); m32.close()
