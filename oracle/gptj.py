"""GPT-J on the reference's own ggml (oracle/ref_gptj.c, built by oracle/gptj.mk), and seeded synthetic models for it -- TEST INFRASTRUCTURE.

  RefGptJ(hp, tensors)   _ref/libggml_gptj.so: the reference graph of crates/models/gptj on the CPU
  make_gptj              tensors named as the loader names them (gptj/src/lib.rs:59-103)
"""
import ctypes as C
import os

import numpy as np

from .alibi import _make
from .bindings import HERE, _p

LIB = os.path.join(HERE, "_ref", "libggml_gptj.so")


def have_ref():
    return os.path.exists(LIB)


class RjParams(C.Structure):
    """rj_params (oracle/ref_gptj.c)"""
    _fields_ = [(n, C.c_int32) for n in ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "n_rot", "wtype", "n_threads", "n_batch")]


_lib = None


def _load():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        vp = C.c_void_p
        L.rj_new.restype = vp
        L.rj_new.argtypes = [C.POINTER(RjParams)]
        L.rj_tensor.restype = vp
        L.rj_tensor.argtypes = [vp, C.c_char_p, C.POINTER(C.c_size_t)]
        L.rj_finalize.argtypes = [vp]
        L.rj_reset.argtypes = [vp]
        L.rj_eval.argtypes = [vp, vp, C.c_int, vp]
        L.rj_kv.restype = vp
        L.rj_kv.argtypes = [vp, C.c_int, C.POINTER(C.c_size_t)]
        L.rj_free.argtypes = [vp]
        _lib = L
    return _lib


class RefGptJ:
    """The reference's GPT-J graph on the reference ggml (CPU).  hp: n_vocab, n_ctx, n_embd, n_head, n_layer, n_rot, wtype."""

    def __init__(self, hp, tensors, n_threads=8, n_batch=512):
        self.L, self.hp = _load(), dict(hp)
        p = RjParams(n_threads=n_threads, n_batch=n_batch, **{k: int(hp[k]) for k in ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "n_rot", "wtype")})
        self.m = self.L.rj_new(C.byref(p))
        assert self.m, "rj_new failed"
        for name, arr in tensors.items():
            nb = C.c_size_t(0)
            dst = self.L.rj_tensor(self.m, name.encode(), C.byref(nb))
            assert dst, name
            arr = np.ascontiguousarray(arr)
            assert arr.nbytes == nb.value, (name, arr.nbytes, nb.value)
            C.memmove(dst, _p(arr), arr.nbytes)
        assert self.L.rj_finalize(self.m) == 0

    def eval(self, tokens):
        tokens = np.ascontiguousarray(tokens, np.int32)
        logits = np.empty((tokens.size, self.hp["n_vocab"]), np.float32)
        assert self.L.rj_eval(self.m, _p(tokens), tokens.size, _p(logits)) == 0
        return logits

    def reset(self):
        self.L.rj_reset(self.m)

    def kv(self, which):
        """f16 bits of memory_k (0) [n_layer][n_ctx][n_embd] / memory_v (1) [n_layer][n_embd][n_ctx] -- the native layout, no transpose"""
        nb = C.c_size_t(0)
        ptr = self.L.rj_kv(self.m, which, C.byref(nb))
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint16)), (nb.value // 2,)).copy()

    def close(self):
        if self.m:
            self.L.rj_free(self.m)
            self.m = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- synthetic models ---------------------------------------------------------------------------------------------------------------------
GPTJ_CONFIGS = {
    "gptj-tiny": dict(n_vocab=320, n_ctx=128, n_embd=512, n_head=2, n_layer=2, n_rot=64),       # hd 256: clusters of 8 CTAs (the wide attention)
    "gptj-hd192": dict(n_vocab=320, n_ctx=128, n_embd=768, n_head=4, n_layer=2, n_rot=32),      # hd 192: clusters of 6 (not a power of two)
    "gptj-hd64": dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2, n_rot=16),       # hd 64: the attention kernel of hd <= 128
    "gptj-6b": dict(n_vocab=50400, n_ctx=2048, n_embd=4096, n_head=16, n_layer=28, n_rot=64),   # GPT-J 6B
}


def gptj_tensor_shapes(hp):
    e, v = hp["n_embd"], hp["n_vocab"]
    shapes = {"transformer.wte.weight": (v, e), "transformer.ln_f.weight": (e,), "transformer.ln_f.bias": (e,), "lm_head.weight": (v, e), "lm_head.bias": (v,)}
    for i in range(hp["n_layer"]):
        p = f"transformer.h.{i}."
        shapes.update({p + "ln_1.weight": (e,), p + "ln_1.bias": (e,),
                       p + "attn.q_proj.weight": (e, e), p + "attn.k_proj.weight": (e, e), p + "attn.v_proj.weight": (e, e), p + "attn.out_proj.weight": (e, e),
                       p + "mlp.fc_in.weight": (4 * e, e), p + "mlp.fc_in.bias": (4 * e,), p + "mlp.fc_out.weight": (e, 4 * e), p + "mlp.fc_out.bias": (e,)})
    return shapes


def make_gptj(hp, wtype, quantize, seed=0x47504A00):
    """2-D weights N(0, 1/K) quantized with the given quantizer, LayerNorm gains 1 + 0.1 N(0,1), biases (LayerNorm, MLP, lm_head) 0.01 N(0,1)"""
    return _make(gptj_tensor_shapes, hp, wtype, quantize, seed, lambda name: name.endswith(("ln_1.weight", "ln_f.weight")))
