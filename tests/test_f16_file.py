"""F16 model files without a GPU: an all-F16 LLaMA GGJT file parses as wtype 1 (llama_ftype 1, no quantization-version rule), and the plain-C
ggml_vec_dot_f16 restatement the F16 kernels follow agrees with the reference's own on the edges of fp16."""
import numpy as np
import pytest

from oracle import bindings as B
from oracle import synth


def f16(t, w):
    return np.ascontiguousarray(w, np.float32).astype(np.float16)


def test_f16_llama_file_parses(tmp_path):
    from llm_b200.loader import GgmlFile, write_llama
    hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], B.F16, f16)
    path = str(tmp_path / "f16.bin")
    write_llama(path, hp, tens, synth.tensor_shapes(hp), quantization_version=0)      # no quantized tensor: the version is not checked
    f = GgmlFile(path)
    h = f.llama_hyperparameters()
    f.close()
    assert h["wtype"] == B.F16 and h["llama_ftype"] == 1 and h["n_ff"] == hp["n_ff"]


def edge_rows(rng, K):
    """(weights, activations) as fp16 bits: activations rounded from exact rounding ties, subnormals, and one +-inf per row whose weight is
    nonzero and finite (no inf * 0, no inf - inf in any chain)"""
    w = (rng.standard_normal(K) / np.sqrt(K)).astype(np.float16)
    w[1::5] = (rng.standard_normal(len(range(1, K, 5))) * 2e-5).astype(np.float16)
    x = rng.standard_normal(K).astype(np.float32)
    h = x.astype(np.float16)
    tie = ((h.astype(np.float32) + np.nextafter(h, np.float16(np.inf)).astype(np.float32)) * 0.5).astype(np.float32)
    m = rng.random(K) < 0.3
    x[m] = tie[m]
    s = rng.random(K) < 0.05
    x[s] = (rng.standard_normal(int(s.sum())) * 3e-6).astype(np.float32)
    x[7] = -1e5
    w[7] = np.float16(0.25)
    return w, x


@pytest.mark.parametrize("K", [64, 4096, 11008])
def test_vec_dot_f16_matches_reference(orc, ref, K):
    rng = np.random.default_rng(K)
    for _ in range(4):
        w, x = edge_rows(rng, K)
        xr = ref.from_float(B.F16, x).view(np.uint16)                   # ggml_fp32_to_fp16_row
        assert np.array_equal(xr, x.astype(np.float16).view(np.uint16))
        assert np.array_equal(xr, np.array([orc.fp32_to_fp16(v) for v in x], np.uint16))
        want = np.float32(ref.vec_dot(B.F16, K, w.view(np.uint16), xr))
        got = orc.vec_dot_f16(w.view(np.uint16), xr)
        assert np.isinf(want)
        assert np.array_equal(np.array([got], np.float32).view(np.uint32), np.array([want], np.float32).view(np.uint32))
        x[7] = 0.5                                                        # and a finite row
        xr = ref.from_float(B.F16, x).view(np.uint16)
        want = np.float32(ref.vec_dot(B.F16, K, w.view(np.uint16), xr))
        got = orc.vec_dot_f16(w.view(np.uint16), xr)
        assert np.isfinite(want)
        assert np.array_equal(np.array([got], np.float32).view(np.uint32), np.array([want], np.float32).view(np.uint32))
