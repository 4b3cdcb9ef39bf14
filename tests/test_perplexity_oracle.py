"""The perplexity checkers on the CPU: the product's restated expf / logf (llm_b200/csrc/libm_f32.h, compiled here by gcc) equals the host libm
on every input the perplexity loop can produce, and the plain-C oracle (oracle/ppl_oracle.c) equals a scalar restatement of the reference's Rust
(util::softmax and InferenceSession::perplexity) in np.float32 arithmetic with libm called through ctypes.

The truth is the host libm: the reference's binary would call the same library.  A host whose glibc takes the non-FMA expf / logf, or predates
the table-driven ones (2.27), fails the exhaustive tests, which name the function."""
import ctypes as C
import ctypes.util

import numpy as np
import pytest

from oracle.ppl import LibmCheck, PplOracle

F = np.float32


def fbits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


@pytest.fixture(scope="module")
def libm():
    L = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
    for f in ("expf", "logf"):
        getattr(L, f).restype = C.c_float
        getattr(L, f).argtypes = [C.c_float]
    return L


@pytest.mark.slow
def test_expf_restatement_equals_libm_on_every_float_in_minus_104_to_minus_0():
    n, first = LibmCheck().mismatches(0, 0x80000000, fbits(-104.0))     # -0 ... -104, every bit pattern in between
    assert n == 0, f"expf: the restatement differs from the host libm on {n} inputs, first {first:#010x}"


@pytest.mark.slow
def test_logf_restatement_equals_libm_on_every_float_in_0_to_1():
    n, first = LibmCheck().mismatches(1, 0x00000001, fbits(1.0))         # the least subnormal ... 1
    assert n == 0, f"logf: the restatement differs from the host libm on {n} inputs, first {first:#010x}"


def test_restatement_special_values(libm):
    chk = LibmCheck().lib
    xs = [0.0, -0.0, 1.0, -1.0, 88.72283935546875, 88.7228394, 89.0, -103.28, -103.9720840454, -104.0, -200.0, np.inf, -np.inf, 1e-45, 1e-40,
          1.1754942e-38, 3.4028235e38, np.nan]
    for x in xs:
        x = float(F(x))
        for mine, ref in ((chk.lm_check_expf, libm.expf), (chk.lm_check_logf, libm.logf)):
            a, b = F(mine(x)), F(ref(x))
            assert (np.isnan(a) and np.isnan(b)) or a.view(np.uint32) == b.view(np.uint32), (mine.__name__, x, a, b)


# ---- the oracle against a scalar restatement of the Rust ----------------------------------------------------------------------------------
def rust_softmax_term(libm, row, target):
    """util::softmax(row)[target] then -p.ln(): max = fold(-inf, f32::max), sum = in-order f32 sum of (v - max).exp(), f32 division"""
    mx = F(-np.inf)
    for v in row:
        mx = v if v > mx else mx
    s = F(0.0)
    for v in row:
        s = F(s + F(libm.expf(float(F(v - mx)))))
    p = F(F(libm.expf(float(F(row[target] - mx)))) / s)
    return F(-F(libm.logf(float(p))))


def rust_perplexity(libm, logits_by_chunk, tokens, C_):
    """the reference's fold: nll (f32) over every chunk, count, expf(nll / count as f32) after each chunk"""
    nll, count, out, terms = F(0.0), 0, [], []
    for i, logits in enumerate(logits_by_chunk):
        for j in range(min(512, C_ // 2), C_ - 1):
            t = rust_softmax_term(libm, logits[j], int(tokens[i * C_ + j + 1]))
            terms.append(t)
            nll = F(nll + t)
            count += 1
        out.append(F(libm.expf(float(F(nll / F(count))))))
    return out, terms


def small_logits(rng, rows, V):
    x = (rng.standard_normal((rows, V)) * 4).astype(np.float32)
    x[0, :3] = x[0].max() + 1                               # ties at the max
    x[1] = rng.uniform(-150, 10, V).astype(np.float32)      # expf underflows to 0 and subnormals
    return x


def test_nll_rows_equals_rust_restatement(libm):
    rng = np.random.default_rng(1)
    x = small_logits(rng, 6, 57)
    t = rng.integers(0, 57, 6).astype(np.int32)
    t[0] = 1
    x[2, t[2]] = x[2].max() - 300                           # p underflows to 0: term +inf
    got = PplOracle().nll_rows(x, t)
    want = np.array([rust_softmax_term(libm, x[r], t[r]) for r in range(6)], np.float32)
    assert np.isposinf(got[2])
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (got, want)


@pytest.mark.parametrize("C_,n_batch", [(8, 3), (9, 9), (16, 1)])
def test_or_perplexity_equals_rust_restatement(libm, C_, n_batch):
    """the loop with a stand-in model: its logits depend on (position in the chunk, token), so the batching, the rewind and the bos replacement
    are all visible in the result"""
    V = 41
    rng = np.random.default_rng(C_ * 100 + n_batch)
    table = small_logits(rng, C_ * V, V).reshape(C_, V, V)
    tokens = rng.integers(0, V, C_ * 5 // 2).astype(np.int32)
    bos = 3
    state = {"n_past": 0, "fed": []}

    def evaluate(batch):
        rows = []
        for tok in batch:
            rows.append(table[state["n_past"], int(tok)])
            state["fed"].append(int(tok))
            state["n_past"] += 1
        return np.stack(rows)

    def reset():
        state["n_past"] = 0

    ppl, terms = PplOracle().perplexity(evaluate, reset, tokens, C_, n_batch, bos)
    n_chunk = tokens.size // C_
    assert len(ppl) == n_chunk and state["fed"][0] == bos and state["fed"][C_] == bos
    assert state["fed"][1:C_] == list(tokens[1:C_]) and state["fed"][C_ + 1:2 * C_] == list(tokens[C_ + 1:2 * C_])
    by_chunk = []
    for i in range(n_chunk):
        chunk = tokens[i * C_:(i + 1) * C_].copy()
        chunk[0] = bos
        by_chunk.append(np.stack([table[j, chunk[j]] for j in range(C_)]))
    want_ppl, want_terms = rust_perplexity(libm, by_chunk, tokens, C_)
    assert np.array_equal(np.asarray(ppl, np.float32).view(np.uint32), np.asarray(want_ppl, np.float32).view(np.uint32)), (ppl, want_ppl)
    assert np.array_equal(terms.ravel().view(np.uint32), np.asarray(want_terms, np.float32).view(np.uint32))
