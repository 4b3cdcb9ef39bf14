"""TEST INFRASTRUCTURE: bindings of the perplexity checkers (oracle/ppl.mk) and the reference's perplexity loop driven over a reference model.

  or_nll_rows / or_perplexity_chunk   ppl_oracle.c: util::softmax and the nll / count fold of InferenceSession::perplexity, libm expf / logf
  lm_check_range                      libm_f32_check.c: the product's restated expf / logf against the host libm, bit for bit
  perplexity(evaluate, reset, ...)    the loop of crates/llm-base/src/inference_session.rs:514-589 with one rewind per chunk, on logits of a model
                                      whose evaluate(tokens) returns all rows (RefLlama / RefGpt2 / RefAlibi / RefGptJ .eval)
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
    path = os.path.join(HERE, name)
    if not os.path.exists(path):
        subprocess.check_call(["make", "-C", HERE, "-f", "ppl.mk", name])
    return C.CDLL(path)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class PplOracle:
    def __init__(self):
        self.lib = L = _load("liboracle_ppl.so")
        L.or_nll_rows.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]
        L.or_perplexity_chunk.restype = C.c_float
        L.or_perplexity_chunk.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int64), C.c_void_p]
        for f in ("or_expf", "or_logf"):
            getattr(L, f).restype = C.c_float
            getattr(L, f).argtypes = [C.c_float]

    def nll_rows(self, logits, targets):
        logits = np.ascontiguousarray(logits, np.float32)
        targets = np.ascontiguousarray(targets, np.int32)
        out = np.empty(logits.shape[0], np.float32)
        self.lib.or_nll_rows(_p(logits), logits.shape[0], logits.shape[1], _p(targets), _p(out))
        return out

    def perplexity(self, evaluate, reset, tokens, context_size, n_batch, bos):
        """(per-chunk perplexities, [n_chunk, scored] terms): each chunk evaluated from n_past 0 (reset()) in batches of n_batch through
        evaluate(tokens) -> [rows, n_vocab] logits, its first token replaced by bos; the softmax and the fold in C on libm."""
        tokens = np.ascontiguousarray(tokens, np.int32)
        Cs = int(context_size)
        n_chunk = tokens.size // Cs
        first = min(512, Cs // 2)
        scored = max(Cs - 1 - first, 0)
        nll, count = C.c_float(0.0), C.c_int64(0)
        ppl, terms = [], np.zeros((n_chunk, scored), np.float32)
        for i in range(n_chunk):
            start = i * Cs
            reset()
            rows = []
            for b0 in range(0, Cs, n_batch):
                batch = tokens[start + b0:start + min(Cs, b0 + n_batch)].copy()
                if b0 == 0:
                    batch[0] = bos
                rows.append(np.asarray(evaluate(batch), np.float32))
            logits = np.ascontiguousarray(np.concatenate(rows, 0))
            chunk = np.ascontiguousarray(tokens[start:start + Cs])
            t = np.empty(max(scored, 1), np.float32)
            ppl.append(self.lib.or_perplexity_chunk(_p(logits), Cs, logits.shape[1], _p(chunk), C.byref(nll), C.byref(count), _p(t)))
            terms[i] = t[:scored]
        return ppl, terms


class LibmCheck:
    """The product header's lm_expf / lm_logf compiled by gcc, compared with the host libm."""

    def __init__(self):
        self.lib = L = _load("liblibm_f32_check.so")
        L.lm_check_range.restype = C.c_int64
        L.lm_check_range.argtypes = [C.c_int, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
        for f in ("lm_check_expf", "lm_check_logf"):
            getattr(L, f).restype = C.c_float
            getattr(L, f).argtypes = [C.c_float]

    def mismatches(self, which, lo_bits, hi_bits):
        """(number of differing inputs, first differing bit pattern or None) over the float bit patterns [lo_bits, hi_bits]; which 0 = expf, 1 = logf"""
        first = C.c_uint32(0)
        n = self.lib.lm_check_range(which, lo_bits, hi_bits, C.byref(first))
        return n, (first.value if n else None)
