"""MPT and BLOOM on the reference's own ggml (oracle/ref_alibi.c, built by oracle/alibi.mk), and seeded synthetic models for them -- TEST INFRASTRUCTURE.

  RefAlibi(hp, tensors, arch)   _ref/libggml_alibi.so: the reference graph of crates/models/mpt (arch 2) or crates/models/bloom (arch 3) on the CPU
  make_mpt / make_bloom         tensors named as the loaders name them (mpt/src/lib.rs:50-65, bloom/src/lib.rs:56-83)
"""
import ctypes as C
import os

import numpy as np

from .bindings import HERE, _p

MPT, BLOOM = 2, 3
LIB = os.path.join(HERE, "_ref", "libggml_alibi.so")


def have_ref():
    return os.path.exists(LIB)


class RaParams(C.Structure):
    """ra_params (oracle/ref_alibi.c)"""
    _fields_ = [(n, C.c_int32) for n in ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "wtype", "n_threads", "n_batch", "arch")] + [("alibi_bias_max", C.c_float)]


_lib = None


def _load():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        vp = C.c_void_p
        L.ra_new.restype = vp
        L.ra_new.argtypes = [C.POINTER(RaParams)]
        L.ra_tensor.restype = vp
        L.ra_tensor.argtypes = [vp, C.c_char_p, C.POINTER(C.c_size_t)]
        L.ra_finalize.argtypes = [vp]
        L.ra_reset.argtypes = [vp]
        L.ra_eval.argtypes = [vp, vp, C.c_int, vp]
        L.ra_kv.restype = vp
        L.ra_kv.argtypes = [vp, C.c_int, C.POINTER(C.c_size_t)]
        L.ra_free.argtypes = [vp]
        _lib = L
    return _lib


class RefAlibi:
    """The reference's MPT / BLOOM graph on the reference ggml (CPU).  hp: n_vocab, n_ctx, n_embd, n_head, n_layer, wtype (+ alibi_bias_max for MPT)."""

    def __init__(self, hp, tensors, arch, n_threads=8, n_batch=512):
        self.L, self.hp, self.arch = _load(), dict(hp), arch
        bias_max = float(hp.get("alibi_bias_max", 8.0)) if arch == MPT else 8.0
        p = RaParams(n_threads=n_threads, n_batch=n_batch, arch=arch, alibi_bias_max=bias_max,
                     **{k: int(hp[k]) for k in ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "wtype")})
        self.m = self.L.ra_new(C.byref(p))
        assert self.m, "ra_new failed"
        for name, arr in tensors.items():
            nb = C.c_size_t(0)
            dst = self.L.ra_tensor(self.m, name.encode(), C.byref(nb))
            assert dst, name
            arr = np.ascontiguousarray(arr)
            assert arr.nbytes == nb.value, (name, arr.nbytes, nb.value)
            C.memmove(dst, _p(arr), arr.nbytes)
        assert self.L.ra_finalize(self.m) == 0

    def eval(self, tokens):
        tokens = np.ascontiguousarray(tokens, np.int32)
        logits = np.empty((tokens.size, self.hp["n_vocab"]), np.float32)
        assert self.L.ra_eval(self.m, _p(tokens), tokens.size, _p(logits)) == 0
        return logits

    def reset(self):
        self.L.ra_reset(self.m)

    def kv(self, which):
        """f16 bits of memory_k (0) / memory_v (1), both [n_layer][n_ctx][n_embd] (the reference keeps V by position)"""
        nb = C.c_size_t(0)
        ptr = self.L.ra_kv(self.m, which, C.byref(nb))
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint16)), (nb.value // 2,)).copy()

    def close(self):
        if self.m:
            self.L.ra_free(self.m)
            self.m = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- synthetic models ---------------------------------------------------------------------------------------------------------------------
MPT_CONFIGS = {
    "mpt-tiny": dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2, alibi_bias_max=8.0),        # hd 64, 4 heads (a power of two)
    "mpt-24h": dict(n_vocab=320, n_ctx=128, n_embd=768, n_head=24, n_layer=2, alibi_bias_max=8.0),        # hd 32, 24 heads: 8 on the m1 branch
    "mpt-7b": dict(n_vocab=50432, n_ctx=2048, n_embd=4096, n_head=32, n_layer=32, alibi_bias_max=8.0),
}
BLOOM_CONFIGS = {
    "bloom-tiny": dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2),
    "bloom-12h": dict(n_vocab=320, n_ctx=128, n_embd=768, n_head=12, n_layer=2),                          # 12 heads: 4 on the m1 branch
    "bloom-560m": dict(n_vocab=250880, n_ctx=2048, n_embd=1024, n_head=16, n_layer=24),
}


def mpt_tensor_shapes(hp):
    e, v = hp["n_embd"], hp["n_vocab"]
    shapes = {"transformer.wte.weight": (v, e), "transformer.norm_f.weight": (e,)}
    for i in range(hp["n_layer"]):
        p = f"transformer.blocks.{i}."
        shapes.update({p + "norm_1.weight": (e,), p + "attn.Wqkv.weight": (3 * e, e), p + "attn.out_proj.weight": (e, e),
                       p + "norm_2.weight": (e,), p + "ffn.up_proj.weight": (4 * e, e), p + "ffn.down_proj.weight": (e, 4 * e)})
    return shapes


def bloom_tensor_shapes(hp):
    e, v = hp["n_embd"], hp["n_vocab"]
    shapes = {"tok_embeddings.weight": (v, e), "norm.weight": (e,), "norm.bias": (e,), "output_norm.weight": (e,), "output_norm.bias": (e,), "output.weight": (v, e)}
    for i in range(hp["n_layer"]):
        p = f"layers.{i}."
        shapes.update({p + "attention_norm.weight": (e,), p + "attention_norm.bias": (e,),
                       p + "attention.query_key_value.weight": (3 * e, e), p + "attention.query_key_value.bias": (3 * e,),
                       p + "attention.wo.weight": (e, e), p + "attention.wo.bias": (e,),
                       p + "ffn_norm.weight": (e,), p + "ffn_norm.bias": (e,),
                       p + "feed_forward.w1.weight": (4 * e, e), p + "feed_forward.w1.bias": (4 * e,),
                       p + "feed_forward.w2.weight": (e, 4 * e), p + "feed_forward.w2.bias": (e,)})
    return shapes


def _make(shapes, hp, wtype, quantize, seed, gain_of):
    hp = dict(hp, wtype=wtype)
    out = {}
    for idx, (name, shp) in enumerate(shapes(hp).items()):
        rng = np.random.default_rng(seed + idx)
        if len(shp) == 1:
            g = gain_of(name)
            out[name] = ((1.0 if g else 0.0) + (0.1 if g else 0.01) * rng.standard_normal(shp)).astype(np.float32)
        else:
            n, k = shp
            out[name] = quantize(wtype, (rng.standard_normal((n, k)) / np.sqrt(k)).astype(np.float32))
    return hp, out


def make_mpt(hp, wtype, quantize, seed=0x4D500000):
    """2-D weights N(0, 1/K) quantized with the given quantizer, norm gains 1 + 0.1 N(0,1) (MPT has no biases)"""
    return _make(mpt_tensor_shapes, hp, wtype, quantize, seed, lambda name: True)


def make_bloom(hp, wtype, quantize, seed=0x424C0000):
    """as make_mpt; biases 0.01 N(0,1)"""
    return _make(bloom_tensor_shapes, hp, wtype, quantize, seed, lambda name: name.endswith("norm.weight"))
