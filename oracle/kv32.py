"""The reference graphs on an F32 KV cache (oracle/kv32.mk) -- TEST INFRASTRUCTURE.

  ref_lib()                    RefLib over _ref/libggml_ref_kv32.so: .llama / .gpt2 / .neox as in oracle/bindings.py, memory_k / memory_v F32
  RefAlibiKV32(hp, t, arch)    RefAlibi (oracle/alibi.py) over _ref/libggml_alibi_kv32.so
  RefGptJKV32(hp, t)           RefGptJ (oracle/gptj.py) over _ref/libggml_gptj_kv32.so
  kv_f32(model, which)         the F32 cache of any of them as float32 values (their kv() returns the bytes as uint16 pairs)
"""
import ctypes as C
import os

import numpy as np

from . import alibi, gptj
from .bindings import HERE, RefLib

LIBS = {k: os.path.join(HERE, "_ref", f"libggml_{k}_kv32.so") for k in ("ref", "alibi", "gptj")}


def have_ref():
    return all(os.path.exists(p) for p in LIBS.values())


_ref = None


def ref_lib():
    global _ref
    if _ref is None:
        _ref = RefLib("ref_kv32")
    return _ref


def _bind(key, prefix, params):
    """the F32-cache library of `key`, with the argument types oracle/alibi.py / oracle/gptj.py declare for the f16 one (prefix ra_ / rj_)"""
    if key not in _libs:
        L = C.CDLL(LIBS[key])
        vp = C.c_void_p
        getattr(L, prefix + "new").restype = vp
        getattr(L, prefix + "new").argtypes = [C.POINTER(params)]
        getattr(L, prefix + "tensor").restype = vp
        getattr(L, prefix + "tensor").argtypes = [vp, C.c_char_p, C.POINTER(C.c_size_t)]
        getattr(L, prefix + "finalize").argtypes = [vp]
        getattr(L, prefix + "reset").argtypes = [vp]
        getattr(L, prefix + "eval").argtypes = [vp, vp, C.c_int, vp]
        getattr(L, prefix + "kv").restype = vp
        getattr(L, prefix + "kv").argtypes = [vp, C.c_int, C.POINTER(C.c_size_t)]
        getattr(L, prefix + "free").argtypes = [vp]
        _libs[key] = L
    return _libs[key]


_libs = {}


def _load_tensors(model, new, tensor, finalize, params, tensors):
    """the constructor steps of RefAlibi / RefGptJ: new, copy every named tensor in, finalize"""
    model.m = new(C.byref(params))
    assert model.m, "new failed"
    for name, arr in tensors.items():
        nb = C.c_size_t(0)
        dst = tensor(model.m, name.encode(), C.byref(nb))
        assert dst, name
        arr = np.ascontiguousarray(arr)
        assert arr.nbytes == nb.value, (name, arr.nbytes, nb.value)
        C.memmove(dst, arr.ctypes.data_as(C.c_void_p), arr.nbytes)
    assert finalize(model.m) == 0


class RefAlibiKV32(alibi.RefAlibi):
    """RefAlibi on _ref/libggml_alibi_kv32.so; eval / reset / kv / close are RefAlibi's, on self.L"""

    def __init__(self, hp, tensors, arch, n_threads=8, n_batch=512):
        self.L, self.hp, self.arch = _bind("alibi", "ra_", alibi.RaParams), dict(hp), arch
        bias_max = float(hp.get("alibi_bias_max", 8.0)) if arch == alibi.MPT else 8.0
        p = alibi.RaParams(n_threads=n_threads, n_batch=n_batch, arch=arch, alibi_bias_max=bias_max,
                           **{k: int(hp[k]) for k in ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "wtype")})
        _load_tensors(self, self.L.ra_new, self.L.ra_tensor, self.L.ra_finalize, p, tensors)


class RefGptJKV32(gptj.RefGptJ):
    """RefGptJ on _ref/libggml_gptj_kv32.so; eval / reset / kv / close are RefGptJ's, on self.L"""

    def __init__(self, hp, tensors, n_threads=8, n_batch=512):
        self.L, self.hp = _bind("gptj", "rj_", gptj.RjParams), dict(hp)
        p = gptj.RjParams(n_threads=n_threads, n_batch=n_batch, **{k: int(hp[k]) for k in ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "n_rot", "wtype")})
        _load_tensors(self, self.L.rj_new, self.L.rj_tensor, self.L.rj_finalize, p, tensors)


def kv_f32(model, which):
    """memory_k (0) / memory_v (1) of an F32-cache reference model as float32, in the layout its kv() documents"""
    return np.ascontiguousarray(model.kv(which)).view(np.float32)
