"""The sampler chain's plain-C restatement (oracle/sampler_oracle.c), stage by stage on hand-built rows, and the C ABI of the sampler
(b200_sampler, the new entry points) against the ctypes bindings.  CPU only: the GPU kernel is compared with this restatement in
tests/test_gpu_generate.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT

LIB = os.path.join(ROOT, "llm_b200", "libllm_b200.so")


@pytest.fixture(scope="module")
def so():
    from oracle.sampler import SamplerOracle
    return SamplerOracle()


def f32(x):
    return np.float32(x)


# ---- the random stream -------------------------------------------------------------------------------------------------------------------------
def test_splitmix64_known_answers(so):
    assert so.splitmix64(0, 0) == 0xE220A8397B1DCDAF
    assert so.splitmix64(0, 1) == 0x6E789E6AA1B965F4
    assert so.splitmix64(0, 2) == 0x06C45D188009454F
    assert so.splitmix64(1234567, 0) == 0x599ED017FB08FC85       # the published SplitMix64 vector for seed 1234567
    # z of draw d is the (d + 1)-th step of the generator: seed + (d + 1) * golden gamma, then the finalizer
    assert so.splitmix64(0x9E3779B97F4A7C15, 0) == so.splitmix64(0, 1)


def test_uniform_is_the_top_24_bits(so):
    for seed, draw in ((0, 0), (7, 3), (2**64 - 1, 12345)):
        z = so.splitmix64(seed, draw)
        assert so.uniform(seed, draw) == f32((z >> 40) * 2.0**-24)
        assert 0.0 <= so.uniform(seed, draw) < 1.0


# ---- the stages ------------------------------------------------------------------------------------------------------------------------------
def test_repetition_once_per_distinct_id(so):
    row = np.array([2.0, -2.0, 0.0, 4.0, 1.0], np.float32)
    hist = np.array([3, 3, 3, 1, 0, 0], np.int32)              # ids 3 and 0 repeat: each is penalized once
    rc, out = so.repetition(row, hist, hist.size, 64, 2.0)
    assert rc == 0
    assert out.tolist() == [1.0, -4.0, 0.0, 2.0, 1.0]
    assert row.tolist() == [2.0, -2.0, 0.0, 4.0, 1.0], "the row itself is not modified"


def test_repetition_negative_and_zero(so):
    row = np.array([-0.0, 0.0, -3.0, 3.0, -1e-30], np.float32)
    hist = np.arange(5, dtype=np.int32)
    rc, out = so.repetition(row, hist, 5, 64, f32(1.3))
    assert rc == 0
    assert out[0] == 0.0 and not np.signbit(out[0]), "-0 * penalty is -0, then + 0.0f makes it +0"
    assert out[1] == 0.0 and not np.signbit(out[1]), "0 <= 0: multiplied, stays +0"
    assert out[2] == f32(-3.0) * f32(1.3) and out[3] == f32(3.0) / f32(1.3)
    assert out[4] == f32(-1e-30) * f32(1.3)


def test_repetition_window(so):
    row = np.ones(8, np.float32)
    hist = np.array([0, 1, 2, 3, 4, 5], np.int32)
    _, out = so.repetition(row, hist, 6, 2, 2.0)                # only the last two: ids 4 and 5
    assert np.flatnonzero(out != 1.0).tolist() == [4, 5]
    _, out = so.repetition(row, hist, 4, 100, 2.0)              # window past the start: [0, n_past)
    assert np.flatnonzero(out != 1.0).tolist() == [0, 1, 2, 3]
    for pen, last_n in ((1.0, 64), (2.0, 0)):                    # off
        _, out = so.repetition(row, hist, 6, last_n, pen)
        assert (out == 1.0).all()


def test_repetition_nan_fails(so):
    row = np.zeros(4, np.float32)
    row[2] = np.nan
    assert so.repetition(row, None, 0, 64, 1.3)[0] == -1
    assert so.sample(row, None, 0)[0] == -1


def test_top_k_order_and_ties(so):
    row = np.array([1.0, 3.0, 3.0, -np.inf, 2.0, 3.0, 2.0], np.float32)
    ids, vals = so.top_k(row, 5)
    assert ids.tolist() == [1, 2, 5, 4, 6]                       # value descending, ties by ascending id
    assert vals.tolist() == [3.0, 3.0, 3.0, 2.0, 2.0]
    ids, _ = so.top_k(row, 100)                                  # k > n_vocab: every id
    assert ids.tolist() == [1, 2, 5, 4, 6, 0, 3]
    ids, _ = so.top_k(np.zeros(5000, np.float32), 5000)          # capped at 1024
    assert ids.tolist() == list(range(1024))


def test_k1_is_the_argmax_after_the_penalty(so):
    row = np.array([0.5, 5.0, 4.5, -1.0], np.float32)
    hist = np.array([1], np.int32)
    for seed in range(5):
        rc, tok, n_kept, ids, _ = so.sample(row, hist, 1, penalty=1.3, k=1, seed=seed, draw=seed)
        assert rc == 0 and tok == 2 and n_kept == 1 and ids.tolist() == [2]   # 5.0 / 1.3 < 4.5
        rc, tok, *_ = so.sample(row, hist, 1, penalty=1.0, k=1, seed=seed)
        assert tok == 1


def test_top_p_one_keeps_all(so):
    vals = np.linspace(0, -20, 40).astype(np.float32)
    n, probs = so.top_p(vals, 1.0)
    assert n == 40 or np.cumsum(probs, dtype=np.float32)[n - 1] >= 1.0
    n, _ = so.top_p(vals, 2.0)                                   # never reached: all k
    assert n == 40


def test_top_p_cut_on_the_boundary(so):
    vals = np.zeros(4, np.float32)                               # p_i = 1/4 exactly; running sums 0.25, 0.5, 0.75, 1
    assert so.top_p(vals, 0.5)[0] == 2                           # >= p: the prefix that reaches p exactly
    assert so.top_p(vals, np.nextafter(f32(0.5), f32(1)))[0] == 3
    assert so.top_p(vals, 0.0)[0] == 1                           # at least one
    n, probs = so.top_p(vals, 0.95)
    assert n == 4 and probs.tolist() == [0.25] * 4


def test_temperature_divides(so):
    assert so.temperature([1.0, -2.0, 0.3], 0.8).tolist() == [f32(1.0) / f32(0.8), f32(-2.0) / f32(0.8), f32(0.3) / f32(0.8)]


def test_draw_thresholds(so):
    vals = np.zeros(3, np.float32)                               # w = 1, 1, 1; x = 3u
    assert so.draw(vals, 0.0) == 0
    assert so.draw(vals, np.nextafter(f32(1 / 3), f32(0))) == 0
    assert so.draw(vals, f32(1 / 3) + f32(1e-7)) == 1
    assert so.draw(vals, np.nextafter(f32(1), f32(0))) == 2     # u just below 1: the last
    assert so.draw(np.array([5.0], np.float32), np.nextafter(f32(1), f32(0))) == 0
    assert so.draw(np.array([0.0, -np.inf], np.float32), np.nextafter(f32(1), f32(0))) == 0   # a zero weight is never picked


def test_sample_composes_the_stages(so):
    rng = np.random.default_rng(5)
    row = (rng.standard_normal(3000) * 2).astype(np.float32)
    hist = rng.integers(0, 3000, 80).astype(np.int32)
    for k, p, t, seed, draw in ((40, 0.95, 0.8, 1, 0), (1024, 1.0, 1.0, 2, 9), (7, 0.5, 0.1, 3, 4)):
        rc, tok, n_kept, ids, probs = so.sample(row, hist, 80, 1.3, 64, k, p, t, seed, draw)
        _, pen = so.repetition(row, hist, 80, 64, 1.3)
        ids2, vals = so.top_k(pen, k)
        n2, probs2 = so.top_p(vals, p)
        pick = so.draw(so.temperature(vals[:n2], t), so.uniform(seed, draw))
        assert rc == 0 and ids.tolist() == ids2.tolist() and n_kept == n2
        assert np.array_equal(probs.view(np.uint32), probs2.view(np.uint32))
        assert tok == ids2[pick]


# ---- the C ABI ---------------------------------------------------------------------------------------------------------------------------------
SAMPLER_FIELDS = ("repetition_penalty", "repetition_last_n", "top_k", "top_p", "temperature", "seed", "draw")


def test_sampler_struct_layout(tmp_path):
    from llm_b200 import _lib
    prog = ['#include "llm_b200.h"', "#include <stdio.h>", "#include <stddef.h>", "int main(void){",
            'printf("%zu", sizeof(b200_sampler));']
    prog += [f'printf(" %zu", offsetof(b200_sampler, {f}));' for f in SAMPLER_FIELDS]
    prog += ['printf(" %d\\n", B200_ERR_SAMPLER_FAILURE);', "return 0;}"]
    src = tmp_path / "s.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "s"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    S = _lib.SamplerParams
    assert got[0] == C.sizeof(S) == 40
    assert got[1:-1] == [getattr(S, f).offset for f in SAMPLER_FIELDS]
    assert got[-1] == -6
    from llm_b200 import session
    with pytest.raises(session.SamplerFailure):
        session._check(-6, "x")


def test_new_symbols_are_exported_and_bound():
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    from llm_b200 import _lib
    from llm_b200.neox import _bind
    L = _bind(_lib.lib())
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "llm_b200.h")).read(), flags=re.S)
    names = ("b200_session_infer_next_token", "b200_session_read_tokens", "b200_session_last_logits", "b200_neox_infer_next_token",
             "b200_neox_read_tokens", "b200_neox_last_logits", "b200_op_sample")
    for n in names:
        assert re.search(r"\b" + n + r"\s*\(", src), n
        assert getattr(L, n).argtypes is not None, f"{n} has no ctypes signature in llm_b200"
    assert L.b200_session_read_tokens.restype == C.c_int32 and L.b200_neox_read_tokens.restype == C.c_int32


def test_python_defaults_are_the_reference_chain():
    import llm_b200
    s = llm_b200.InferenceParameters().sampler
    assert (s.repetition_penalty, s.repetition_last_n, s.top_k, s.top_p, s.temperature) == (1.30, 64, 40, 0.95, 0.80)
    r = llm_b200.Rng(-1)
    assert (r.seed, r.draw) == (2**64 - 1, 0)
    req = llm_b200.InferenceRequest([1, 2])
    assert req.maximum_token_count is None and req.parameters.sampler == s
