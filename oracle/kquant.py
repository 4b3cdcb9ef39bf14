"""Mixed-type LLaMA models: the reference quantizer's per-tensor type rules and the reference graph on such a model -- TEST INFRASTRUCTURE.

mix_types(hp, mix) restates the type choice of the reference's vendored quantizer (LC/llama.cpp:2938-2965, GGML_USE_K_QUANTS, QK_K = 256) tensor
by tensor: output.weight becomes Q6_K when both its dimensions are multiples of 256 (every file type); attention.wv / feed_forward.w2 take Q6_K in
the layers use_more_bits picks (Q4_K_M, Q5_K_M) or Q4_K (Q3_K_M, Q2_K); attention.wo takes Q4_K (Q3_K_M, Q2_K); a K-quant choice on a tensor with a
dimension that is not a multiple of 256 falls back to F16 (output), Q4_0 (tok_embeddings) or is refused (any other tensor).
make_llama_mixed quantizes a synthetic model (oracle.synth's draws) with each tensor's type through the reference's own from_float
(quantize_row_q*_K for the K-quants).  ref_llama runs the reference's LLaMA graph on it: oracle/kquant.mk's _ref/libggml_ref_kq.so.
"""
import ctypes as C
import os

import numpy as np

from . import bindings as B
from . import synth

HERE = os.path.dirname(os.path.abspath(__file__))
F16 = B.F16
# mix name -> (base type of the 2-D weights, llama_ftype of the file header, LC/llama.h)
MIXES = {"q4_0": (B.Q4_0, 2), "q4_1": (B.Q4_1, 3), "q5_0": (B.Q5_0, 8), "q5_1": (B.Q5_1, 9), "q8_0": (B.Q8_0, 7),
         "q2_K": (B.Q2_K, 10), "q3_K_M": (B.Q3_K, 12), "q4_K_M": (B.Q4_K, 15), "q5_K_M": (B.Q5_K, 17), "q6_K": (B.Q6_K, 18)}
KQUANTS = (B.Q2_K, B.Q3_K, B.Q4_K, B.Q5_K, B.Q6_K)


def use_more_bits(i_layer, num_layers):
    return i_layer < num_layers // 8 or i_layer >= 7 * num_layers // 8 or (i_layer - num_layers // 8) % 3 == 2


def mix_types(hp, mix):
    """{name: enum ggml_type} of every 2-D weight of a LLaMA model of `hp` quantized as `mix` (the quantizer's file order: wv / w2 counted in
    layer order).  Raises ValueError where the quantizer throws (a K-quant choice on a tensor it cannot split into super-blocks)."""
    base, _ = MIXES[mix]
    n = hp["n_layer"]
    out = {}
    for name, shp in synth.tensor_shapes(hp).items():
        if len(shp) != 2:
            continue
        t = base
        il = int(name.split(".")[1]) if name.startswith("layers.") else -1
        if name == "output.weight":
            if shp[0] % 256 == 0 and shp[1] % 256 == 0:
                t = B.Q6_K
        elif name.endswith("attention.wv.weight") or name.endswith("feed_forward.w2.weight"):
            if mix in ("q3_K_M", "q2_K"):
                t = B.Q4_K
            elif mix in ("q4_K_M", "q5_K_M") and use_more_bits(il, n):
                t = B.Q6_K
        elif name.endswith("attention.wo.weight"):
            if mix in ("q3_K_M", "q2_K"):
                t = B.Q4_K
        if t in KQUANTS and (shp[0] % 256 or shp[1] % 256):
            if name == "output.weight":
                t = F16
            elif name == "tok_embeddings.weight":
                t = B.Q4_0
            else:
                raise ValueError(f"{name} {shp}: not divisible by 256, required for k-quants")
        out[name] = t
    return out


def quantize_as(ref, t, w):
    """[N, K] f32 -> the type's GGML rows: quantize_row_q*_K (from_float) for K-quants, ggml_quantize_* for the classic formats, fp16 for F16"""
    w = np.ascontiguousarray(w, np.float32)
    if t == F16:
        return w.astype(np.float16)
    if t in KQUANTS:
        return np.stack([ref.from_float(t, row) for row in w])
    return ref.quantize(t, w)


def make_llama_mixed(hp, mix, ref, seed=0x5EED0000, overrides=None):
    """(hp with wtype = the mix's base type, tensors, types): oracle.synth.make_llama's draws, each 2-D weight quantized with its own type.
    overrides: {name: type} applied on top of the mix (e.g. to make one tensor refusable)."""
    types = mix_types(hp, mix)
    types.update(overrides or {})
    base = MIXES[mix][0]
    hp2, f32 = synth.make_llama(hp, base, lambda t, w: w, seed=seed)
    tensors = {name: (quantize_as(ref, types[name], a) if name in types else a) for name, a in f32.items()}
    return hp2, tensors, types


class RefKq(B.RefLib):
    """the reference ggml + a copy of ref_harness.c whose LLaMA model takes a type per 2-D weight"""

    def __init__(self):
        super().__init__("ref_kq")
        self.lib.rk_set_types.argtypes = [C.c_void_p, C.c_int]

    def llama_typed(self, hp, tensors, types, n_threads=8, n_batch=512):
        # allocation order of rh_llama_new: tok_embeddings, output, then per layer wq wk wv wo w1 w2 w3
        order = ["tok_embeddings.weight", "output.weight"] + [n for i in range(hp["n_layer"]) for n in
                             (f"layers.{i}.attention.wq.weight", f"layers.{i}.attention.wk.weight", f"layers.{i}.attention.wv.weight",
                              f"layers.{i}.attention.wo.weight", f"layers.{i}.feed_forward.w1.weight", f"layers.{i}.feed_forward.w2.weight",
                              f"layers.{i}.feed_forward.w3.weight")]
        tab = np.array([types.get(n, hp["wtype"]) for n in order], np.int32)
        self.lib.rk_set_types(tab.ctypes.data, tab.size)
        try:
            return B.RefLlama(self, hp, tensors, 0, n_threads, n_batch)
        finally:
            self.lib.rk_set_types(None, 0)


def have_ref_kq():
    return os.path.exists(os.path.join(HERE, "_ref", "libggml_ref_kq.so"))
