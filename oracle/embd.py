"""The reference graphs with their embeddings exposed (oracle/embd.mk) -- TEST INFRASTRUCTURE.

OutputRequest::embeddings (crates/llm-base/src/model/common.rs:40-59) is the final norm's output.  oracle/embd.mk links copies of the GPT-2 / GPT-NeoX,
MPT / BLOOM and GPT-J harnesses (and of their F32-cache copies) that also hand out every row of that tensor and of the residual stream it reads.
LLaMA needs no copy: ref_harness.c's rh_llama_eval already takes embd_out.

  model(kind, hp, tensors, f32=False, arch=None)   the reference model on these libraries: kind "llama", "gpt2", "neox", "alibi" (arch MPT / BLOOM), "gptj"
  eval_embd(model, tokens)                         (logits [n, n_vocab], embd [n, n_embd], resid [n, n_embd] or None for LLaMA)
"""
import ctypes as C
import os

import numpy as np

from . import alibi, gptj, kv32
from .bindings import HERE, RefLib, RefLlama, _p

KEYS = ("ref", "ref_kv32", "alibi", "alibi_kv32", "gptj", "gptj_kv32")
LIBS = {k: os.path.join(HERE, "_ref", f"libggml_{k}_embd.so") for k in KEYS}


def have_ref():
    return all(os.path.exists(p) for p in LIBS.values())


_libs = {}


def _ref_lib(f32):
    key = "ref_kv32" if f32 else "ref"
    if key not in _libs:
        lib = RefLib(f"{key}_embd")
        lib.lib.rx_set_outputs.argtypes = [C.c_void_p, C.c_void_p]
        _libs[key] = lib
    return _libs[key]


def _bind(key, prefix, params):
    """the MPT / BLOOM or GPT-J library `key`, with the argument types oracle/alibi.py / oracle/gptj.py declare (prefix ra_ / rj_)"""
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
        L.rx_set_outputs.argtypes = [vp, vp]
        _libs[key] = L
    return _libs[key]


class RefAlibiEmbd(alibi.RefAlibi):
    """RefAlibi on _ref/libggml_alibi[_kv32]_embd.so; eval / reset / kv / close are RefAlibi's, on self.L"""

    def __init__(self, hp, tensors, arch, f32=False, n_threads=8, n_batch=512):
        self.L, self.hp, self.arch = _bind("alibi_kv32" if f32 else "alibi", "ra_", alibi.RaParams), dict(hp), arch
        bias_max = float(hp.get("alibi_bias_max", 8.0)) if arch == alibi.MPT else 8.0
        p = alibi.RaParams(n_threads=n_threads, n_batch=n_batch, arch=arch, alibi_bias_max=bias_max,
                           **{k: int(hp[k]) for k in ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "wtype")})
        kv32._load_tensors(self, self.L.ra_new, self.L.ra_tensor, self.L.ra_finalize, p, tensors)


class RefGptJEmbd(gptj.RefGptJ):
    """RefGptJ on _ref/libggml_gptj[_kv32]_embd.so; eval / reset / kv / close are RefGptJ's, on self.L"""

    def __init__(self, hp, tensors, f32=False, n_threads=8, n_batch=512):
        self.L, self.hp = _bind("gptj_kv32" if f32 else "gptj", "rj_", gptj.RjParams), dict(hp)
        p = gptj.RjParams(n_threads=n_threads, n_batch=n_batch, **{k: int(hp[k]) for k in ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "n_rot", "wtype")})
        kv32._load_tensors(self, self.L.rj_new, self.L.rj_tensor, self.L.rj_finalize, p, tensors)


def model(kind, hp, tensors, f32=False, arch=None, n_threads=8, n_batch=128):
    if kind in ("llama", "gpt2", "neox"):
        return getattr(_ref_lib(f32), kind)(hp, tensors, n_threads=n_threads, n_batch=n_batch)
    if kind == "alibi":
        return RefAlibiEmbd(hp, tensors, arch, f32, n_threads=n_threads, n_batch=n_batch)
    assert kind == "gptj", kind
    return RefGptJEmbd(hp, tensors, f32, n_threads=n_threads, n_batch=n_batch)


def eval_embd(m, tokens):
    """one eval of `tokens` on a model of model(): its logits, and every row of the final norm's output (OutputRequest::embeddings keeps the
    last) and of the residual stream that norm reads (None for LLaMA)"""
    tokens = np.ascontiguousarray(tokens, np.int32)
    n = tokens.size
    embd = np.empty((n, m.hp["n_embd"]), np.float32)
    if isinstance(m, RefLlama):                                 # rh_llama_eval's embd_out
        logits = np.empty((n, m.hp["n_vocab"]), np.float32)
        assert m.ref.lib.rh_llama_eval(m.m, _p(tokens), n, _p(logits), _p(embd)) == 0
        return logits, embd, None
    L = m.ref.lib if hasattr(m, "ref") else m.L
    resid = np.empty_like(embd)
    L.rx_set_outputs(_p(embd), _p(resid))
    try:
        logits = m.eval(tokens)
    finally:
        L.rx_set_outputs(None, None)
    return logits, embd, resid
