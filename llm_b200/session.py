"""Host-side mirror of the reference's model/session interface for LLaMA over the native C ABI (include/llm_b200.h).

Names follow the reference so that the parity tests read like its own integration tests (binaries/llm-test):
  Llama(KnownModel)                crates/models/llama/src/lib.rs:17-140   new / start_session / evaluate
  ModelParameters                  crates/llm-base/src/model/mod.rs:197-229
  InferenceSessionConfig           crates/llm-base/src/inference_session.rs:799-841
  InferenceSession                 crates/llm-base/src/inference_session.rs:43-512  feed_prompt / n_past / last_logits
  OutputRequest                    crates/llm-base/src/lib.rs (all_logits), model/common.rs:22-39
  InferenceError::ContextFull      crates/llm-base/src/inference_session.rs:311-313
"""
import ctypes as C
import enum
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from . import _lib


class ContextFull(Exception):
    """InferenceError::ContextFull."""


@dataclass
class ModelParameters:
    context_size: int = 2048          # model/mod.rs:214
    use_gpu: bool = True              # this backend IS the GPU path; False is rejected (no CPU fallback)
    rope_freq_base: float = 10000.0   # RoPEOverrides
    rope_freq_scale: float = 1.0
    lora_adapters: Optional[List[str]] = None   # model/mod.rs:205-206: LoRA adapter files, applied in this order to every tensor they name


class ModelKVMemoryType(enum.Enum):
    """ModelKVMemoryType (inference_session.rs:907-922): the element type of memory_k / memory_v"""
    Float16 = 1                       # GGML_TYPE_F16, the default
    Float32 = 0                       # GGML_TYPE_F32 (the CLI's --no-float16): twice the bytes, no fp16 rounding in the attention


SESSION_KV_F32 = 8                    # B200_SESSION_KV_F32 (include/llm_b200.h)


def kv_flags(memory_k_type: ModelKVMemoryType, memory_v_type: ModelKVMemoryType) -> int:
    """The B200_SESSION_* bits of a (memory_k_type, memory_v_type) pair: one type for both caches, as the reference CLI always sets them"""
    if memory_k_type != memory_v_type:
        raise ValueError(f"memory_k_type {memory_k_type} and memory_v_type {memory_v_type} differ: only equal KV types are supported")
    return SESSION_KV_F32 if memory_k_type == ModelKVMemoryType.Float32 else 0


def kv_array(raw: np.ndarray, kv_f32: bool) -> np.ndarray:
    """a cache read back as raw bytes: float32 values of an f32 cache, the f16 bits (uint16) otherwise"""
    return raw.view(np.float32) if kv_f32 else raw.view(np.uint16)


@dataclass
class InferenceSessionConfig:
    n_batch: int = 8                  # inference_session.rs:837
    flags: int = 0
    memory_k_type: ModelKVMemoryType = ModelKVMemoryType.Float16      # inference_session.rs:838-839
    memory_v_type: ModelKVMemoryType = ModelKVMemoryType.Float16

    def __post_init__(self):
        kv_flags(self.memory_k_type, self.memory_v_type)


@dataclass
class OutputRequest:
    all_logits: Optional[np.ndarray] = None     # set to an empty array to request all rows (OutputRequest::all_logits)
    want_all_logits: bool = False


_HP_KEYS = ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_rot", "n_ff")


def llama_tensor_shapes(hp: Dict[str, int]) -> Dict[str, tuple]:
    """tensor name -> (rows N, cols K) for 2-D weights, (n,) for norm gains: the names the reference's loader asks for
    (crates/models/llama/src/lib.rs:52-91)"""
    e, f, v = hp["n_embd"], hp["n_ff"], hp["n_vocab"]
    gqa = e // (hp["n_head"] // hp["n_head_kv"])
    shapes = {"tok_embeddings.weight": (v, e), "norm.weight": (e,), "output.weight": (v, e)}
    for i in range(hp["n_layer"]):
        p = f"layers.{i}."
        shapes.update({p + "attention_norm.weight": (e,), p + "attention.wq.weight": (e, e), p + "attention.wk.weight": (gqa, e),
                       p + "attention.wv.weight": (gqa, e), p + "attention.wo.weight": (e, e), p + "ffn_norm.weight": (e,),
                       p + "feed_forward.w1.weight": (f, e), p + "feed_forward.w2.weight": (e, f), p + "feed_forward.w3.weight": (f, e)})
    return shapes


def _check(rc, what):
    if rc == -1:
        raise ContextFull(what)
    if rc != 0:
        raise RuntimeError(f"{what} failed with code {rc}")


def _perplexity(entry, handle, tokens, bos: int, context_size: int, callback, return_terms: bool):
    """InferenceSession::perplexity through b200_session_perplexity / b200_neox_perplexity: the per-chunk perplexities (and, with return_terms,
    the [n_chunk, scored rows] -ln p terms); callback(chunk, ppl) is called for each chunk in order, as the reference's perplexity_callback"""
    tokens = np.ascontiguousarray(tokens, np.int32).ravel()
    n_chunk_max = tokens.size // context_size
    first = min(512, context_size // 2)
    scored = max(context_size - 1 - first, 0)
    ppl = np.empty(max(n_chunk_max, 1), np.float32)
    terms = np.empty((max(n_chunk_max, 1), max(scored, 1)), np.float32)
    n_chunk = C.c_int32(0)
    _check(entry(handle, tokens.ctypes.data_as(C.c_void_p), tokens.size, int(bos), ppl.ctypes.data_as(C.c_void_p),
                 terms.ctypes.data_as(C.c_void_p) if return_terms else None, C.byref(n_chunk)), "perplexity")
    out = [float(p) for p in ppl[:n_chunk.value]]
    if callback is not None:
        for i, p in enumerate(out):
            callback(i, p)
    return (out, terms[:n_chunk.value, :scored]) if return_terms else out


class _Native:
    """Owner of one native handle (attribute `_HANDLE`, released by the library function `_FREE`): close() frees it once, and so does
    garbage collection."""
    _HANDLE, _FREE = "", ""

    def close(self):
        h = getattr(self, self._HANDLE, None)
        if h:
            getattr(self.L, self._FREE)(h)
            setattr(self, self._HANDLE, None)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class LoraAdapters:
    """The adapter files of ModelParameters::lora_adapters, opened as LoRA containers (r, alpha, no vocabulary) for the span of a load:
    `handles` is the array the b200_*_load_tensor_lora entry points take."""
    LORA_ARCH = 6                                 # B200_ARCH_LORA

    def __init__(self, L, paths: Optional[List[str]]):
        self.L, self._open = L, []
        for p in paths or []:
            err = C.c_int(0)
            f = L.b200_ggml_open_arch(p.encode(), self.LORA_ARCH, C.byref(err))
            if not f:
                self.close()
                from .loader import LoadError
                raise LoadError(err.value, f"open LoRA adapter {p}")
            self._open.append(f)
        self.handles = (C.c_void_p * max(1, len(self._open)))(*self._open)
        self.n = len(self._open)

    def close(self):
        for f in self._open:
            self.L.b200_ggml_close(f)
        self._open = []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def ggml_dims(arr: np.ndarray, wtype: int):
    """(n_dims, ne0, ne1) of a tensor given as GGML-layout block rows (uint8 [rows][row bytes]) or f32 ([n] or [rows][cols])"""
    if arr.dtype == np.float32:
        return (1, arr.shape[0], 1) if arr.ndim == 1 else (2, arr.shape[-1], arr.size // arr.shape[-1])
    if arr.dtype == np.float16:                  # F16 weights: [rows][cols] halves
        return 2, arr.shape[-1], arr.size // arr.shape[-1]
    block = {2: 18, 3: 20, 6: 22, 7: 24, 8: 34}[wtype]
    return 2, arr.shape[-1] // block * 32, arr.size // arr.shape[-1]


class Llama(_Native):
    """KnownModel for LLaMA.  `hyperparameters` is a dict with n_vocab, n_embd, n_head, n_head_kv, n_layer, n_rot, n_ff, wtype."""
    _HANDLE, _FREE = "_m", "b200_model_free"

    def __init__(self, hyperparameters: Dict[str, int], params: ModelParameters = None, tensors: Dict[str, np.ndarray] = None,
                 device: int = 0):
        params = params or ModelParameters()
        if not params.use_gpu:
            raise ValueError("llm_b200 has no CPU path: ModelParameters.use_gpu must be True")
        self.L = _lib.lib()
        _check(self.L.b200_init(device), "b200_init")
        self.hyperparameters = dict(hyperparameters)
        self.params = params
        hp = _lib.LlamaHparams(**{k: int(hyperparameters[k]) for k in _HP_KEYS}, wtype=int(hyperparameters["wtype"]),
                               context_size=params.context_size, rope_freq_base=params.rope_freq_base,
                               rope_freq_scale=params.rope_freq_scale)
        self._m = self.L.b200_llama_new(C.byref(hp))
        if not self._m:
            raise ValueError(f"b200_llama_new rejected hyperparameters {hyperparameters}")
        if tensors is not None and params.lora_adapters:
            shapes = llama_tensor_shapes(self.hyperparameters)
            with LoraAdapters(self.L, params.lora_adapters) as ad:
                for name, arr in tensors.items():
                    self.load_tensor(name, arr, ad, shapes.get(name))
        elif tensors is not None:
            for name, arr in tensors.items():
                self.load_tensor(name, arr)

    # TensorLoader::load + transfer_to(Backend::Gpu)
    def load_tensor(self, name: str, arr: np.ndarray, adapters: "LoraAdapters" = None, shape: tuple = None):
        """`adapters`: patch the tensor with them (LoraAdapter::patch); `shape` is then its (rows, cols) / (n,) as in llama_tensor_shapes"""
        arr = np.ascontiguousarray(arr)
        typ = 0 if arr.dtype == np.float32 else 1 if arr.dtype == np.float16 else int(self.hyperparameters["wtype"])
        if adapters is None:
            _check(self.L.b200_model_load_tensor(self._m, name.encode(), typ, arr.ctypes.data_as(C.c_void_p), arr.nbytes),
                   f"load_tensor({name})")
            return
        nd, ne0, ne1 = (len(shape), shape[-1], shape[0] if len(shape) == 2 else 1) if shape else ggml_dims(arr, typ)
        rc = self.L.b200_model_load_tensor_lora(self._m, name.encode(), typ, nd, ne0, ne1, arr.ctypes.data_as(C.c_void_p), arr.nbytes,
                                                adapters.handles, adapters.n)
        if rc != 0:
            from .loader import LoadError
            raise LoadError(rc, f"load_tensor({name})")

    def synthesize(self, seed: int = 0x5EED0000):
        _check(self.L.b200_model_synthesize(self._m, seed), "synthesize")

    def read_tensor(self, name: str) -> np.ndarray:
        nb = self.L.b200_model_tensor_nbytes(self._m, name.encode())
        if nb == 0:
            raise KeyError(name)
        is_f32 = name.endswith("norm.weight")
        out = np.empty(nb // 4, np.float32) if is_f32 else np.empty(nb, np.uint8)
        _check(self.L.b200_model_read_tensor(self._m, name.encode(), out.ctypes.data_as(C.c_void_p), nb), f"read_tensor({name})")
        return out

    @property
    def weight_bytes(self) -> int:
        return self.L.b200_model_weight_bytes(self._m)

    def start_session(self, config: InferenceSessionConfig = None) -> "InferenceSession":
        return InferenceSession(self, config or InferenceSessionConfig())

    def context_size(self) -> int:
        return self.params.context_size

    def bot_token_id(self) -> Optional[int]:
        """KnownModel::bot_token_id: LLaMA has none (llama lib.rs:382-384)"""
        return None


class InferenceSession(_Native):
    _HANDLE, _FREE = "_s", "b200_session_free"

    def __init__(self, model: Llama, config: InferenceSessionConfig):
        self.model, self.config, self.L = model, config, model.L
        self.kv_f32 = kv_flags(config.memory_k_type, config.memory_v_type) != 0
        cfg = _lib.SessionConfig(n_batch=config.n_batch, flags=config.flags | (SESSION_KV_F32 if self.kv_f32 else 0))
        self._s = self.L.b200_model_start_session(model._m, C.byref(cfg))
        if not self._s:
            raise RuntimeError("b200_model_start_session failed (all tensors loaded?)")
        self.n_vocab = int(model.hyperparameters["n_vocab"])
        self.last_logits = np.zeros(self.n_vocab, np.float32)

    @property
    def n_past(self) -> int:
        return self.L.b200_session_n_past(self._s)

    def top_k(self, k: int):
        """Sampler hand-off: (token ids, logits) of the k largest logits of the last evaluated row, selected on the device."""
        ids, vals = np.empty(k, np.int32), np.empty(k, np.float32)
        _check(self.L.b200_session_top_k(self._s, k, ids.ctypes.data_as(C.c_void_p), vals.ctypes.data_as(C.c_void_p)), "top_k")
        return ids, vals

    def evaluate(self, tokens, all_logits: bool = False) -> np.ndarray:
        """Model::evaluate: one forward pass over `tokens` (<= n_batch) appended at n_past; returns logits
        ([n, n_vocab] when all_logits else the last row, which is also kept in self.last_logits)."""
        tokens = np.ascontiguousarray(tokens, np.int32)
        n = tokens.size
        out = np.empty((n if all_logits else 1, self.n_vocab), np.float32)
        _check(self.L.b200_session_evaluate(self._s, tokens.ctypes.data_as(C.c_void_p), n, out.ctypes.data_as(C.c_void_p),
                                            1 if all_logits else 0), "evaluate")
        self.last_logits = out[-1].copy()
        return out if all_logits else out[0]

    def feed_prompt(self, tokens) -> np.ndarray:
        tokens = np.ascontiguousarray(tokens, np.int32)
        if tokens.size == 0:                      # the reference leaves last_logits untouched for an empty prompt (inference_session.rs:299-350)
            return self.last_logits
        out = np.empty(self.n_vocab, np.float32)
        _check(self.L.b200_session_feed_prompt(self._s, tokens.ctypes.data_as(C.c_void_p), tokens.size,
                                               out.ctypes.data_as(C.c_void_p)), "feed_prompt")
        self.last_logits = out
        return out

    def perplexity(self, tokens, callback=None, bos: Optional[int] = None, return_terms: bool = False):
        """InferenceSession::perplexity on token ids (tokenization is the caller's), computed on the device: one perplexity per chunk of
        context_size tokens, callback(chunk, ppl) after each.  bos replaces each chunk's first token (default: bot_token_id() or 1).  Every chunk
        starts at n_past 0; afterwards n_past is context_size (unchanged when there are fewer tokens than that).  See include/llm_b200.h."""
        bot = self.model.bot_token_id()
        bos = (1 if bot is None else bot) if bos is None else bos
        return _perplexity(self.L.b200_session_perplexity, self._s, tokens, bos, self.model.params.context_size, callback, return_terms)

    def rewind(self, n_past: int):
        _check(self.L.b200_session_set_n_past(self._s, n_past), "rewind")

    def kv(self, which: int) -> np.ndarray:
        """memory_k (0) / memory_v (1): float32 values of an f32 cache (or a session started with the B200_SESSION_KV_F32 flag), else the f16 bits"""
        hp = self.model.hyperparameters
        gqa = hp["n_embd"] // (hp["n_head"] // hp["n_head_kv"])
        n = hp["n_layer"] * self.model.params.context_size * gqa
        f32 = self.kv_f32 or bool(self.config.flags & SESSION_KV_F32)
        out = np.empty(n * (4 if f32 else 2), np.uint8)
        _check(self.L.b200_session_read_kv(self._s, which, out.ctypes.data_as(C.c_void_p), out.nbytes), "read_kv")
        return kv_array(out, f32)

    def sync(self):
        self.L.b200_session_sync(self._s)

    @property
    def last_launches(self) -> int:
        return self.L.b200_session_last_launches(self._s)
