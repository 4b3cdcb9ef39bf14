"""GPT-NeoX, GPT-2, MPT, BLOOM and GPT-J models whose 2-D weights each have their own element type, and the reference graphs on them with and
without ModelParameters::rope_overrides -- TEST INFRASTRUCTURE.

make_typed(arch, hp, types, ref) draws the architecture's synthetic model (oracle.synth / alibi / gptj, the same draws as their one-type makers) and
quantizes each 2-D weight with its own type through the reference's own quantizers (kquant.quantize_as).  ref_typed(arch, hp, tensors, types, rope)
runs the reference graph of the architecture on it: oracle/neox_kquant.mk's libraries, copies of ref_gpt2.c / ref_alibi.c / ref_gptj.c whose 2-D
weights take their types from kquant_types.inc and whose RoPE nodes take the overrides of rope_custom.inc.  kv32=True: the same graphs on an F32
KV cache (oracle/kquant_kv32.mk's _ref/*_kq_kv32.so; read their caches with oracle.kv32.kv_f32).
"""
import ctypes as C
import os

import numpy as np

from . import alibi, gptj, kquant, kv32, synth
from .bindings import HERE, RefGpt2, RefLib

LIBS = {k + s: os.path.join(HERE, "_ref", f"libggml_{k}{s}.so") for k in ("ref_nxkq", "alibi_kq", "gptj_kq") for s in ("", "_kv32")}
ARCHS = ("gptneox", "gpt2", "mpt", "bloom", "gptj")


def _kv(kv32):
    return "_kv32" if kv32 else ""


def have_ref(kv32=False):
    return all(os.path.exists(p) for k, p in LIBS.items() if k.endswith("_kv32") == kv32)


def tensor_shapes(arch, hp, lm_head=False):
    return {"gptneox": synth.neox_tensor_shapes, "gpt2": lambda h: synth.gpt2_tensor_shapes(h, lm_head), "mpt": alibi.mpt_tensor_shapes,
            "bloom": alibi.bloom_tensor_shapes, "gptj": gptj.gptj_tensor_shapes}[arch](hp)


def matrices(arch, hp, lm_head=False):
    """the 2-D weights in the order the harness allocates them (the order kquant_types.inc's table is read in)"""
    L = range(hp["n_layer"])
    if arch == "gpt2":
        return ["model/wte"] + (["model/lm_head"] if lm_head else []) + [f"model/h{i}/{s}" for i in L for s in ("attn/c_attn/w", "attn/c_proj/w", "mlp/c_fc/w", "mlp/c_proj/w")]
    if arch == "gptneox":
        return ["gpt_neox.embed_in.weight", "embed_out.weight"] + [f"gpt_neox.layers.{i}.{s}" for i in L for s in (
            "attention.query_key_value.weight", "attention.dense.weight", "mlp.dense_h_to_4h.weight", "mlp.dense_4h_to_h.weight")]
    if arch == "mpt":
        return ["transformer.wte.weight"] + [f"transformer.blocks.{i}.{s}" for i in L for s in ("attn.Wqkv.weight", "attn.out_proj.weight", "ffn.up_proj.weight",
                                                                                                  "ffn.down_proj.weight")]
    if arch == "bloom":
        return ["tok_embeddings.weight", "output.weight"] + [f"layers.{i}.{s}" for i in L for s in ("attention.query_key_value.weight", "attention.wo.weight",
                                                                                                     "feed_forward.w1.weight", "feed_forward.w2.weight")]
    return ["transformer.wte.weight", "lm_head.weight"] + [f"transformer.h.{i}.{s}" for i in L for s in (
        "attn.q_proj.weight", "attn.k_proj.weight", "attn.v_proj.weight", "attn.out_proj.weight", "mlp.fc_in.weight", "mlp.fc_out.weight")]


def make_typed(arch, hp, base, ref, types=None, lm_head=False, seed=None):
    """(hp with wtype = base, tensors, types): the architecture's synthetic draws, every 2-D weight quantized with types.get(name, base) (F16: fp16
    rows).  `types` is completed to every matrix of the model."""
    ident = lambda t, w: w
    kw = {} if seed is None else {"seed": seed}
    hp2, f32 = {"gptneox": lambda: synth.make_neox(hp, base, ident, **kw), "gpt2": lambda: synth.make_gpt2(hp, base, ident, lm_head=lm_head, **kw),
                "mpt": lambda: alibi.make_mpt(hp, base, ident, **kw), "bloom": lambda: alibi.make_bloom(hp, base, ident, **kw),
                "gptj": lambda: gptj.make_gptj(hp, base, ident, **kw)}[arch]()
    types = {n: int((types or {}).get(n, base)) for n in matrices(arch, hp2, lm_head)}
    tensors = {name: (kquant.quantize_as(ref, types[name], a) if name in types else a) for name, a in f32.items()}
    return hp2, tensors, types


_libs = {}


def ref_lib(kv32=False):
    """RefLib over _ref/libggml_ref_nxkq.so (kv32: _ref/libggml_ref_nxkq_kv32.so): the reference's quantizers and the GPT-2 / GPT-NeoX graphs of
    the typed copy"""
    key = "ref_nxkq" + _kv(kv32)
    if key not in _libs:
        r = RefLib(key)
        r.lib.rk_set_types.argtypes = [C.c_void_p, C.c_int]
        r.lib.rk_set_rope.argtypes = [C.c_float, C.c_float]
        _libs[key] = r
    return _libs[key]


def _lib(key, prefix, params):
    """the typed copy of ref_alibi.c (ra_) or ref_gptj.c (rj_), with the argument types oracle/alibi.py / oracle/gptj.py declare"""
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
        L.rk_set_types.argtypes = [C.c_void_p, C.c_int]
        if prefix == "rj_":
            L.rk_set_rope.argtypes = [C.c_float, C.c_float]
        _libs[key] = L
    return _libs[key]


class _Alibi(alibi.RefAlibi):
    def __init__(self, hp, tensors, arch, n_threads=8, n_batch=512, f32_cache=False):
        self.L, self.hp, self.arch = _lib("alibi_kq" + _kv(f32_cache), "ra_", alibi.RaParams), dict(hp), arch
        bias_max = float(hp.get("alibi_bias_max", 8.0)) if arch == alibi.MPT else 8.0
        p = alibi.RaParams(n_threads=n_threads, n_batch=n_batch, arch=arch, alibi_bias_max=bias_max,
                           **{k: int(hp[k]) for k in ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "wtype")})
        kv32._load_tensors(self, self.L.ra_new, self.L.ra_tensor, self.L.ra_finalize, p, tensors)


class _GptJ(gptj.RefGptJ):
    def __init__(self, hp, tensors, n_threads=8, n_batch=512, f32_cache=False):
        self.L, self.hp = _lib("gptj_kq" + _kv(f32_cache), "rj_", gptj.RjParams), dict(hp)
        p = gptj.RjParams(n_threads=n_threads, n_batch=n_batch, **{k: int(hp[k]) for k in ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "n_rot", "wtype")})
        kv32._load_tensors(self, self.L.rj_new, self.L.rj_tensor, self.L.rj_finalize, p, tensors)


class RefTyped:
    """the reference graph of `arch` on a typed model; rope = (base, scale): the RoPE nodes are ggml_rope_custom_inplace with them (GPT-NeoX, GPT-J).
    kv32: the graph on an F32 KV cache.  eval / reset / kv / close as the one-type reference models."""

    def __init__(self, arch, hp, tensors, types, rope=None, n_threads=8, n_batch=512, kv32=False):
        self.arch, self.rope = arch, rope if arch in ("gptneox", "gptj") else None      # the others have no RoPE
        lm_head = "model/lm_head" in tensors
        tab = np.array([types.get(n, hp["wtype"]) for n in matrices(arch, hp, lm_head)], np.int32)
        if arch in ("gpt2", "gptneox"):
            self.L = ref_lib(kv32).lib
        else:
            self.L = _lib("gptj_kq" + _kv(kv32), "rj_", gptj.RjParams) if arch == "gptj" else _lib("alibi_kq" + _kv(kv32), "ra_", alibi.RaParams)
        self.L.rk_set_types(tab.ctypes.data, tab.size)
        try:
            if arch in ("gpt2", "gptneox"):
                self.m = RefGpt2(ref_lib(kv32), hp, tensors, 0, n_threads, n_batch, arch=1 if arch == "gptneox" else 0)
            elif arch == "gptj":
                self.m = _GptJ(hp, tensors, n_threads, n_batch, kv32)
            else:
                self.m = _Alibi(hp, tensors, alibi.MPT if arch == "mpt" else alibi.BLOOM, n_threads, n_batch, kv32)
        finally:
            self.L.rk_set_types(None, 0)

    def eval(self, tokens):
        if self.rope is None:
            return self.m.eval(tokens)
        self.L.rk_set_rope(*self.rope)
        try:
            return self.m.eval(tokens)
        finally:
            self.L.rk_set_rope(0.0, 1.0)

    def reset(self):
        self.m.reset()

    def kv(self, which):
        return self.m.kv(which)

    def close(self):
        self.m.close()
