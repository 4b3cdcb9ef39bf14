"""Host-side mirror of the reference's GPT-NeoX model / session over the native C ABI (include/llm_b200.h: b200_neox_*).

  GptNeoX(KnownModel)     crates/models/gptneox/src/lib.rs:36-140     new / start_session / evaluate
  Hyperparameters         crates/models/gptneox/src/lib.rs (n_vocab, n_ctx, n_embd, n_head, n_layer, n_rot, use_parallel_residual, file_type)
  Gpt2 / Mpt / Bloom      crates/models/{gpt2,mpt,bloom} on the same runtime (Mpt, Bloom: ALiBi attention, b200_neox_new_alibi)
  InferenceSession        crates/llm-base/src/inference_session.rs     evaluate / n_past / rewind
No arithmetic happens in Python."""
import ctypes as C
from typing import Dict

import numpy as np

from . import _lib
from .session import _check, _Native


class NeoxHparams(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_vocab", "n_embd", "n_head", "n_layer", "n_rot", "use_parallel_residual", "wtype", "context_size", "arch", "has_lm_head")]


def _bind(L):
    if getattr(L, "_neox_ready", False):
        return L
    vp, i32 = C.c_void_p, C.c_int32
    L.b200_neox_new.restype = vp
    L.b200_neox_new.argtypes = [C.POINTER(NeoxHparams)]
    L.b200_neox_new_alibi.restype = vp
    L.b200_neox_new_alibi.argtypes = [C.POINTER(NeoxHparams), C.c_float]
    L.b200_neox_load_tensor.argtypes = [vp, C.c_char_p, i32, vp, C.c_size_t]
    L.b200_neox_synthesize.argtypes = [vp, C.c_uint64]
    L.b200_neox_weight_bytes.restype = C.c_size_t
    L.b200_neox_weight_bytes.argtypes = [vp]
    L.b200_neox_free.argtypes = [vp]
    L.b200_neox_start_session.restype = vp
    L.b200_neox_start_session.argtypes = [vp, i32]
    L.b200_neox_evaluate.argtypes = [vp, vp, i32, vp, i32]
    L.b200_neox_evaluate_device.argtypes = [vp, i32]
    L.b200_neox_n_past.argtypes = [vp]
    L.b200_neox_set_n_past.argtypes = [vp, i32]
    L.b200_neox_read_kv.argtypes = [vp, i32, vp, C.c_size_t]
    L.b200_neox_last_launches.argtypes = [vp]
    L.b200_neox_sync.argtypes = [vp]
    L.b200_neox_session_free.argtypes = [vp]
    L._neox_ready = True
    return L


class GptNeoX(_Native):
    """hyperparameters: n_vocab, n_ctx, n_embd, n_head, n_layer, n_rot, use_parallel_residual, wtype"""

    ARCH = 0
    _HANDLE, _FREE = "_m", "b200_neox_free"

    def __init__(self, hyperparameters: Dict[str, int], tensors: Dict[str, np.ndarray] = None, context_size: int = None, device: int = 0):
        self.L = _bind(_lib.lib())
        _check(self.L.b200_init(device), "b200_init")
        self.hyperparameters = dict(hyperparameters)
        self.context_size = context_size or hyperparameters["n_ctx"]
        hp = NeoxHparams(n_vocab=hyperparameters["n_vocab"], n_embd=hyperparameters["n_embd"], n_head=hyperparameters["n_head"], n_layer=hyperparameters["n_layer"],
                         n_rot=int(hyperparameters.get("n_rot", 0)), use_parallel_residual=int(hyperparameters.get("use_parallel_residual", 1)), wtype=hyperparameters["wtype"],
                         context_size=self.context_size, arch=self.ARCH, has_lm_head=int(bool(tensors) and "model/lm_head" in tensors))
        self._m = self._new(hp)
        if not self._m:
            raise ValueError(f"b200_neox_new rejected {hyperparameters}")
        for name, arr in (tensors or {}).items():
            arr = np.ascontiguousarray(arr)
            typ = 0 if arr.dtype == np.float32 else int(hyperparameters["wtype"])
            _check(self.L.b200_neox_load_tensor(self._m, name.encode(), typ, arr.ctypes.data_as(C.c_void_p), arr.nbytes), f"load_tensor({name})")

    def _new(self, hp):
        return self.L.b200_neox_new(C.byref(hp))

    def synthesize(self, seed: int = 0x4E580000):
        _check(self.L.b200_neox_synthesize(self._m, seed), "synthesize")

    @property
    def weight_bytes(self) -> int:
        return self.L.b200_neox_weight_bytes(self._m)

    def start_session(self, n_batch: int = 8) -> "NeoxSession":
        return NeoxSession(self, n_batch)


class Gpt2(GptNeoX):
    """KnownModel for GPT-2 (crates/models/gpt2/src/lib.rs): hyperparameters n_vocab, n_ctx, n_embd, n_head, n_layer, wtype; tensors "model/wte",
    "model/wpe" (f32), "model/ln_f/g|b", optional "model/lm_head", "model/hN/{ln_1,ln_2}/{g,b}", "model/hN/attn/{c_attn,c_proj}/{w,b}",
    "model/hN/mlp/{c_fc,c_proj}/{w,b}".  context_size is the model's n_ctx (the rows of wpe)."""
    ARCH = 1


class Mpt(GptNeoX):
    """KnownModel for MPT (crates/models/mpt): hyperparameters n_vocab, n_ctx, n_embd, n_head, n_layer, wtype, alibi_bias_max (the header's float;
    clip_kqv is read by the reference but never applied); tensors "transformer.wte.weight" (also the output projection), "transformer.norm_f.weight",
    "transformer.blocks.N.{norm_1,norm_2}.weight", "transformer.blocks.N.attn.{Wqkv,out_proj}.weight", "transformer.blocks.N.ffn.{up_proj,down_proj}.weight"."""
    ARCH = 2

    def _alibi_bias_max(self):
        return float(self.hyperparameters["alibi_bias_max"])

    def _new(self, hp):
        return self.L.b200_neox_new_alibi(C.byref(hp), self._alibi_bias_max())


class Bloom(Mpt):
    """KnownModel for BLOOM (crates/models/bloom): hyperparameters n_vocab, n_ctx, n_embd, n_head, n_layer, wtype; ALiBi bias 8 (bloom lib.rs:240);
    tensors "tok_embeddings.weight", "norm.{weight,bias}", "output_norm.{weight,bias}", "output.weight", "layers.N.{attention_norm,ffn_norm}.{weight,bias}",
    "layers.N.attention.{query_key_value,wo}.{weight,bias}", "layers.N.feed_forward.{w1,w2}.{weight,bias}"."""
    ARCH = 3

    def _alibi_bias_max(self):
        return 8.0


class NeoxSession(_Native):
    _HANDLE, _FREE = "_s", "b200_neox_session_free"

    def __init__(self, model: GptNeoX, n_batch: int):
        self.model, self.L = model, model.L
        self._s = self.L.b200_neox_start_session(model._m, n_batch)
        if not self._s:
            raise RuntimeError("b200_neox_start_session failed (all tensors loaded?)")
        self.n_vocab = int(model.hyperparameters["n_vocab"])

    @property
    def n_past(self) -> int:
        return self.L.b200_neox_n_past(self._s)

    @property
    def last_launches(self) -> int:
        return self.L.b200_neox_last_launches(self._s)

    def evaluate(self, tokens, all_logits: bool = False) -> np.ndarray:
        tokens = np.ascontiguousarray(tokens, np.int32)
        out = np.empty((tokens.size if all_logits else 1, self.n_vocab), np.float32)
        _check(self.L.b200_neox_evaluate(self._s, tokens.ctypes.data_as(C.c_void_p), tokens.size, out.ctypes.data_as(C.c_void_p), 1 if all_logits else 0), "evaluate")
        return out if all_logits else out[0]

    def rewind(self, n_past: int):
        _check(self.L.b200_neox_set_n_past(self._s, n_past), "rewind")

    def kv(self, which: int) -> np.ndarray:
        """the f16 cache as raw bits: K [n_layer][n_ctx][n_embd] (which = 0), V [n_layer][n_embd][n_ctx] (which = 1)"""
        hp = self.model.hyperparameters
        out = np.empty(hp["n_layer"] * self.model.context_size * hp["n_embd"], np.uint16)
        _check(self.L.b200_neox_read_kv(self._s, which, out.ctypes.data_as(C.c_void_p), out.nbytes), "read_kv")
        return out

    def sync(self):
        self.L.b200_neox_sync(self._s)
