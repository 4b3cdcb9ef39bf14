"""TEST INFRASTRUCTURE: bindings of the sampler checker (oracle/sampler.mk): the default sampler chain of b200_sampler in plain C on the host
libm, one function per stage (sampler_oracle.c).

  splitmix64 / uniform            the draw's random stream
  repetition / top_k / top_p      the stages, each on its own
  temperature / draw
  sample                          the whole chain: (status, id, n_kept, candidate ids, candidate top-p probabilities)
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class SamplerOracle:
    def __init__(self):
        path = os.path.join(HERE, "liboracle_sampler.so")
        if not os.path.exists(path):
            subprocess.check_call(["make", "-C", HERE, "-f", "sampler.mk", "liboracle_sampler.so"])
        self.lib = L = C.CDLL(path)
        vp, i32, i64, u64, f = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_float
        L.or_splitmix64.restype = u64
        L.or_splitmix64.argtypes = [u64, u64]
        L.or_uniform.restype = f
        L.or_uniform.argtypes = [u64, u64]
        L.or_repetition.argtypes = [vp, i64, vp, i32, i32, f, vp]
        L.or_top_k.restype = i32
        L.or_top_k.argtypes = [vp, i64, i32, vp, vp]
        L.or_top_p.restype = i32
        L.or_top_p.argtypes = [vp, i32, f, vp]
        L.or_temperature.argtypes = [vp, i32, f]
        L.or_draw.restype = i32
        L.or_draw.argtypes = [vp, i32, f]
        L.or_sample.argtypes = [vp, i64, vp, i32, f, i32, i32, f, f, u64, u64, vp, vp, vp, vp]

    def splitmix64(self, seed, draw):
        return self.lib.or_splitmix64(seed, draw)

    def uniform(self, seed, draw):
        return np.float32(self.lib.or_uniform(seed, draw))

    def repetition(self, row, history, n_past, last_n, penalty):
        row = np.ascontiguousarray(row, np.float32)
        hist = np.ascontiguousarray(history if history is not None and len(history) else [0], np.int32)
        out = np.empty_like(row)
        rc = self.lib.or_repetition(_p(row), row.size, _p(hist), n_past, last_n, penalty, _p(out))
        return rc, out

    def top_k(self, vals, k):
        vals = np.ascontiguousarray(vals, np.float32)
        ids, v = np.empty(1024, np.int32), np.empty(1024, np.float32)
        n = self.lib.or_top_k(_p(vals), vals.size, k, _p(ids), _p(v))
        return ids[:n], v[:n]

    def top_p(self, vals, p):
        vals = np.ascontiguousarray(vals, np.float32)
        probs = np.empty(vals.size, np.float32)
        n = self.lib.or_top_p(_p(vals), vals.size, p, _p(probs))
        return n, probs

    def temperature(self, vals, t):
        vals = np.array(vals, np.float32)
        self.lib.or_temperature(_p(vals), vals.size, t)
        return vals

    def draw(self, vals, u):
        vals = np.ascontiguousarray(vals, np.float32)
        return self.lib.or_draw(_p(vals), vals.size, float(u))

    def sample(self, row, history, n_past, penalty=1.30, last_n=64, k=40, p=0.95, t=0.80, seed=0, draw=0):
        """(status 0 / -1 on a NaN, id, n_kept, candidate ids, their top-p probabilities)"""
        row = np.ascontiguousarray(row, np.float32)
        hist = np.ascontiguousarray(history if history is not None and len(history) else [0], np.int32)
        kk = min(k, row.size, 1024)
        ids, probs = np.empty(kk, np.int32), np.empty(kk, np.float32)
        tok, n_kept = C.c_int32(-1), C.c_int32(0)
        rc = self.lib.or_sample(_p(row), row.size, _p(hist), n_past, penalty, last_n, k, p, t, seed, draw, C.byref(tok), C.byref(n_kept),
                                _p(ids), _p(probs))
        return rc, tok.value, n_kept.value, ids, probs
