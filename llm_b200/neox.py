"""Host-side mirror of the reference's GPT-NeoX model / session over the native C ABI (include/llm_b200.h: b200_neox_*).

  GptNeoX(KnownModel)     crates/models/gptneox/src/lib.rs:36-140     new / start_session / evaluate
  Hyperparameters         crates/models/gptneox/src/lib.rs (n_vocab, n_ctx, n_embd, n_head, n_layer, n_rot, use_parallel_residual, file_type)
  Gpt2 / Mpt / Bloom      crates/models/{gpt2,mpt,bloom} on the same runtime (Mpt, Bloom: ALiBi attention, b200_neox_new_alibi)
  GptJ                    crates/models/gptj on the same runtime (RoPE mode 0 over the whole head, heads up to 256 wide)
  InferenceSession        crates/llm-base/src/inference_session.rs     evaluate / n_past / rewind
No arithmetic happens in Python."""
import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _lib
from .session import (ContextFull, InferenceSnapshot, LoraAdapters, ModelKVMemoryType, OutputRequest, _BatchedSessions, _check, _embeddings_buffer,
                      _Generation, _Native, _perplexity, _ref_cache_bytes, _Snapshots, _vocab_id, ggml_dims, kv_array, kv_flags)


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
    L.b200_neox_new_typed.restype = vp
    L.b200_neox_new_typed.argtypes = [C.POINTER(NeoxHparams), C.c_float, C.c_float, C.c_float, C.POINTER(_lib.TensorType), i32, C.POINTER(C.c_int)]
    L.b200_neox_is_loaded.argtypes = [vp]
    L.b200_neox_load_file.restype = vp
    L.b200_neox_load_file.argtypes = [C.c_char_p, i32, i32, C.c_float, C.c_float, C.POINTER(C.c_char_p), i32, C.POINTER(C.c_int)]
    L.b200_ggml_neox_hparams.argtypes = [vp, C.POINTER(NeoxHparams), C.POINTER(C.c_float), C.POINTER(i32)]
    L.b200_ggml_weight_types.restype = C.c_int64
    L.b200_ggml_weight_types.argtypes = [vp, C.POINTER(_lib.TensorType), C.c_int64]
    L.b200_neox_load_tensor.argtypes = [vp, C.c_char_p, i32, vp, C.c_size_t]
    L.b200_neox_load_tensor_lora.argtypes = [vp, C.c_char_p, i32, i32, C.c_int64, C.c_int64, vp, C.c_size_t, C.POINTER(vp), i32]
    L.b200_neox_synthesize.argtypes = [vp, C.c_uint64]
    L.b200_neox_weight_bytes.restype = C.c_size_t
    L.b200_neox_weight_bytes.argtypes = [vp]
    L.b200_neox_free.argtypes = [vp]
    L.b200_neox_start_session.restype = vp
    L.b200_neox_start_session.argtypes = [vp, i32]
    L.b200_neox_start_session_flags.restype = vp
    L.b200_neox_start_session_flags.argtypes = [vp, i32, i32]
    L.b200_neox_evaluate.argtypes = [vp, vp, i32, vp, i32]
    L.b200_neox_evaluate_output.argtypes = [vp, vp, i32, vp, i32, vp]
    L.b200_neox_evaluate_device.argtypes = [vp, i32]
    L.b200_neox_n_past.argtypes = [vp]
    L.b200_neox_set_n_past.argtypes = [vp, i32]
    L.b200_neox_read_kv.argtypes = [vp, i32, vp, C.c_size_t]
    L.b200_neox_last_launches.argtypes = [vp]
    L.b200_neox_sync.argtypes = [vp]
    L.b200_neox_perplexity.argtypes = [vp, vp, C.c_int64, i32, vp, vp, C.POINTER(i32)]
    L.b200_neox_infer_next_token.argtypes = [vp, C.POINTER(_lib.SamplerParams), C.POINTER(i32)]
    L.b200_neox_evaluate_sessions.argtypes = [vp, C.POINTER(vp), i32, vp, vp]
    L.b200_neox_infer_next_tokens.argtypes = [vp, C.POINTER(vp), i32, C.POINTER(_lib.SamplerParams), vp, vp]
    L.b200_neox_evaluate_ragged.argtypes = [vp, C.POINTER(vp), i32, vp, vp, vp, i32]
    L.b200_neox_read_tokens.restype = i32
    L.b200_neox_read_tokens.argtypes = [vp, vp, i32]
    L.b200_neox_last_logits.argtypes = [vp, vp]
    L.b200_neox_session_free.argtypes = [vp]
    L.b200_neox_get_snapshot.argtypes = [vp, C.POINTER(_lib.Snapshot)]
    L.b200_neox_write_snapshot.argtypes = [vp, C.c_char_p]
    L.b200_neox_session_from_snapshot.restype = vp
    L.b200_neox_session_from_snapshot.argtypes = [vp, C.POINTER(_lib.Snapshot), C.POINTER(C.c_int)]
    L.b200_neox_session_read_snapshot.restype = vp
    L.b200_neox_session_read_snapshot.argtypes = [vp, C.c_char_p, C.POINTER(C.c_int)]
    L._neox_ready = True
    return L


class GptNeoX(_BatchedSessions, _Native):
    """hyperparameters: n_vocab, n_ctx, n_embd, n_head, n_layer, n_rot, use_parallel_residual, wtype.  lora_adapters: LoRA adapter files applied in
    order to every tensor they name (ModelParameters::lora_adapters).  tensor_types: {name: enum ggml_type} of 2-D weights whose type is not wtype
    (mixed-type and K-quant files, b200_neox_new_typed).  rope_freq_base / rope_freq_scale: ModelParameters::rope_overrides (GPT-NeoX and GPT-J)."""

    ARCH = 0
    _HANDLE, _FREE = "_m", "b200_neox_free"
    _EVAL_SESSIONS, _INFER_SESSIONS = "b200_neox_evaluate_sessions", "b200_neox_infer_next_tokens"
    _EVAL_RAGGED = "b200_neox_evaluate_ragged"

    BOT_TOKEN: Optional[bytes] = None       # the vocabulary entry bot_token_id() names (MPT, BLOOM); None: the model has no BOS token
    EOT_TOKEN: bytes = b"<|endoftext|>"     # the entry eot_token_id() names (gptneox lib.rs:376-378, gpt2 :353-355, gptj :329-331, mpt :277-279)

    tensor_types: Dict[str, int] = {}           # models loaded from a file: their types are in the C model

    def __init__(self, hyperparameters: Dict[str, int], tensors: Dict[str, np.ndarray] = None, context_size: int = None, device: int = 0,
                 lora_adapters: Optional[List[str]] = None, vocabulary: Optional[Sequence] = None, tensor_types: Optional[Dict[str, int]] = None,
                 rope_freq_base: float = 10000.0, rope_freq_scale: float = 1.0):
        """vocabulary: the model file's tokens (GgmlFile.vocabulary(): (bytes, score) pairs, or bytes), consulted by bot_token_id()"""
        self.L = _bind(_lib.lib())
        _check(self.L.b200_init(device), "b200_init")
        self.hyperparameters = dict(hyperparameters)
        self.tensor_types = dict(tensor_types or {})
        self.rope = (float(rope_freq_base), float(rope_freq_scale))
        self.vocabulary = [t[0] if isinstance(t, tuple) else bytes(t) for t in vocabulary] if vocabulary is not None else None
        self.context_size = context_size or hyperparameters["n_ctx"]
        hp = NeoxHparams(n_vocab=hyperparameters["n_vocab"], n_embd=hyperparameters["n_embd"], n_head=hyperparameters["n_head"], n_layer=hyperparameters["n_layer"],
                         n_rot=int(hyperparameters.get("n_rot", 0)), use_parallel_residual=int(hyperparameters.get("use_parallel_residual", 1)), wtype=hyperparameters["wtype"],
                         context_size=self.context_size, arch=self.ARCH, has_lm_head=int(bool(tensors) and "model/lm_head" in tensors))
        self._m = self._new(hp)
        if not self._m:
            raise ValueError(f"b200_neox_new rejected {hyperparameters}")
        if lora_adapters:
            with LoraAdapters(self.L, lora_adapters) as ad:
                for name, arr in (tensors or {}).items():
                    self._load_lora(name, np.ascontiguousarray(arr), ad)
            return
        for name, arr in (tensors or {}).items():
            arr = np.ascontiguousarray(arr)
            typ = 0 if arr.dtype == np.float32 else 1 if arr.dtype == np.float16 else int(self.tensor_types.get(name, hyperparameters["wtype"]))
            _check(self.L.b200_neox_load_tensor(self._m, name.encode(), typ, arr.ctypes.data_as(C.c_void_p), arr.nbytes), f"load_tensor({name})")

    def _load_lora(self, name, arr, ad):
        typ = 0 if arr.dtype == np.float32 else 1 if arr.dtype == np.float16 else int(self.tensor_types.get(name, self.hyperparameters["wtype"]))
        nd, ne0, ne1 = ggml_dims(arr, typ)
        rc = self.L.b200_neox_load_tensor_lora(self._m, name.encode(), typ, nd, ne0, ne1, arr.ctypes.data_as(C.c_void_p), arr.nbytes, ad.handles, ad.n)
        if rc != 0:
            from .loader import LoadError
            raise LoadError(rc, f"load_tensor({name})")

    def _new(self, hp):
        names = [n.encode() for n in self.tensor_types]
        table = (_lib.TensorType * max(1, len(names)))(*[_lib.TensorType(n, int(t)) for n, t in zip(names, self.tensor_types.values())])
        err = C.c_int(0)
        m = self.L.b200_neox_new_typed(C.byref(hp), self._alibi_bias_max(), self.rope[0], self.rope[1], table, len(names), C.byref(err))
        if not m and err.value != -2:               # B200_ERR_BAD_ARG: hyperparameters the untyped forms refuse too (ValueError below)
            from .loader import LoadError
            raise LoadError(err.value, "b200_neox_new_typed")
        return m

    def _alibi_bias_max(self):
        return 0.0

    def synthesize(self, seed: int = 0x4E580000):
        _check(self.L.b200_neox_synthesize(self._m, seed), "synthesize")

    @property
    def weight_bytes(self) -> int:
        return self.L.b200_neox_weight_bytes(self._m)

    def start_session(self, n_batch: int = 8, memory_k_type: ModelKVMemoryType = ModelKVMemoryType.Float16,
                      memory_v_type: ModelKVMemoryType = ModelKVMemoryType.Float16) -> "NeoxSession":
        """InferenceSessionConfig's n_batch and KV types (equal types only: ValueError otherwise)"""
        return NeoxSession(self, n_batch, kv_flags(memory_k_type, memory_v_type))

    def bot_token_id(self) -> Optional[int]:
        """KnownModel::bot_token_id: GPT-NeoX, GPT-2 and GPT-J have none; MPT's is "<|padding|>" and BLOOM's "<s>" when the vocabulary has it
        (mpt lib.rs:273-275, bloom lib.rs:356-358).  Without a vocabulary there is nothing to look up: None."""
        if self.BOT_TOKEN is None or self.vocabulary is None:
            return None
        return _vocab_id(self.vocabulary, self.BOT_TOKEN)

    def eot_token_id(self) -> Optional[int]:
        """KnownModel::eot_token_id: "<|endoftext|>" (BLOOM: "</s>") in the vocabulary.  The reference panics when it is missing; here that, and
        a model without a vocabulary, give None (no end of text)."""
        return None if self.vocabulary is None else _vocab_id(self.vocabulary, self.EOT_TOKEN)


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
    BOT_TOKEN = b"<|padding|>"

    def _alibi_bias_max(self):
        return float(self.hyperparameters["alibi_bias_max"])


class Bloom(Mpt):
    """KnownModel for BLOOM (crates/models/bloom): hyperparameters n_vocab, n_ctx, n_embd, n_head, n_layer, wtype; ALiBi bias 8 (bloom lib.rs:240);
    tensors "tok_embeddings.weight", "norm.{weight,bias}", "output_norm.{weight,bias}", "output.weight", "layers.N.{attention_norm,ffn_norm}.{weight,bias}",
    "layers.N.attention.{query_key_value,wo}.{weight,bias}", "layers.N.feed_forward.{w1,w2}.{weight,bias}"."""
    ARCH = 3
    BOT_TOKEN = b"<s>"
    EOT_TOKEN = b"</s>"                     # bloom lib.rs:360-362

    def _alibi_bias_max(self):
        return 8.0


class GptJ(GptNeoX):
    """KnownModel for GPT-J (crates/models/gptj): hyperparameters n_vocab, n_ctx, n_embd, n_head, n_layer, n_rot, wtype; tensors "transformer.wte.weight",
    "transformer.ln_f.{weight,bias}", "lm_head.{weight,bias}", "transformer.h.N.ln_1.{weight,bias}", "transformer.h.N.attn.{q_proj,k_proj,v_proj,out_proj}.weight",
    "transformer.h.N.mlp.{fc_in,fc_out}.{weight,bias}".  n_rot is the angle step of RoPE mode 0, which rotates every pair of the head."""
    ARCH = 4


class NeoxSession(_Generation, _Snapshots, _Native):
    _HANDLE, _FREE = "_s", "b200_neox_session_free"
    _INFER, _TOKENS, _LAST = "b200_neox_infer_next_token", "b200_neox_read_tokens", "b200_neox_last_logits"
    _GET_SNAP, _WRITE_SNAP = "b200_neox_get_snapshot", "b200_neox_write_snapshot"
    _FROM_SNAP, _READ_SNAP = "b200_neox_session_from_snapshot", "b200_neox_session_read_snapshot"

    def __init__(self, model: GptNeoX, n_batch: int, flags: int = 0, _handle=None):
        self.model, self.L = model, model.L
        self.kv_f32 = flags != 0
        self.n_batch = n_batch
        self._s = _handle or self.L.b200_neox_start_session_flags(model._m, n_batch, flags)
        if not self._s:
            raise RuntimeError("b200_neox_start_session failed (all tensors loaded?)")
        self.n_vocab = int(model.hyperparameters["n_vocab"])
        self._last_logits = None if _handle else np.zeros(self.n_vocab, np.float32)

    @classmethod
    def from_snapshot(cls, snapshot: InferenceSnapshot, model: GptNeoX) -> "NeoxSession":
        """InferenceSession::from_snapshot for every architecture of this runtime (see InferenceSession.from_snapshot)"""
        return cls._from(snapshot, model, 0)

    @classmethod
    def read_snapshot(cls, path: str, model: GptNeoX) -> "NeoxSession":
        """from_snapshot of a session file, streamed into HBM"""
        return cls._read(path, model, 0)

    @staticmethod
    def _start_args(flags):
        return ()

    @staticmethod
    def _cache_bytes(model, variant):
        hp = model.hyperparameters
        return _ref_cache_bytes(hp["n_layer"], model.context_size, hp["n_embd"], variant)

    @classmethod
    def _adopt(cls, model, handle, config):
        return cls(model, config.n_batch, 8 if config.memory_k_type == ModelKVMemoryType.Float32 else 0, _handle=handle)

    @property
    def n_past(self) -> int:
        return self.L.b200_neox_n_past(self._s)

    @property
    def last_launches(self) -> int:
        return self.L.b200_neox_last_launches(self._s)

    def evaluate(self, tokens, all_logits: bool = False, output_request: Optional[OutputRequest] = None) -> np.ndarray:
        """Model::evaluate; output_request.embeddings, when not None, is replaced with the n_embd f32 of the last row of the final LayerNorm's output"""
        tokens = np.ascontiguousarray(tokens, np.int32)
        out = np.empty((tokens.size if all_logits else 1, self.n_vocab), np.float32)
        embd = _embeddings_buffer(output_request, self.model.hyperparameters["n_embd"])
        _check(self.L.b200_neox_evaluate_output(self._s, tokens.ctypes.data_as(C.c_void_p), tokens.size, out.ctypes.data_as(C.c_void_p), 1 if all_logits else 0,
                                                None if embd is None else embd.ctypes.data_as(C.c_void_p)), "evaluate")
        if embd is not None:
            output_request.embeddings = embd
        self._last_logits = out[-1].copy()
        return out if all_logits else out[0]

    def feed_prompt(self, tokens, output_request: Optional[OutputRequest] = None) -> np.ndarray:
        """InferenceSession::feed_prompt (inference_session.rs:299-350): the prompt in chunks of n_batch, each evaluated with output_request (so its
        embeddings are the last chunk's last row); returns last_logits.  ContextFull if it does not fit (nothing is evaluated then); an empty prompt
        leaves last_logits and output_request untouched."""
        tokens = np.ascontiguousarray(tokens, np.int32).ravel()
        if tokens.size == 0:
            return self.last_logits
        if self.n_past + tokens.size > self.model.context_size:
            raise ContextFull("feed_prompt")
        for i in range(0, tokens.size, self.n_batch):
            last = i + self.n_batch >= tokens.size
            self.evaluate(tokens[i:i + self.n_batch], output_request=output_request if last else None)
        return self.last_logits

    def perplexity(self, tokens, callback=None, bos: Optional[int] = None, return_terms: bool = False):
        """InferenceSession::perplexity on the device (see InferenceSession.perplexity); bos defaults to bot_token_id() or 1"""
        bot = self.model.bot_token_id()
        bos = (1 if bot is None else bot) if bos is None else bos
        self._last_logits = None
        return _perplexity(self.L.b200_neox_perplexity, self._s, tokens, bos, self.model.context_size, callback, return_terms)

    def rewind(self, n_past: int):
        _check(self.L.b200_neox_set_n_past(self._s, n_past), "rewind")

    def kv(self, which: int) -> np.ndarray:
        """the cache: K [n_layer][n_ctx][n_embd] (which = 0), V [n_layer][n_embd][n_ctx] (which = 1); float32 values of an f32 cache, else the f16 bits"""
        hp = self.model.hyperparameters
        out = np.empty(hp["n_layer"] * self.model.context_size * hp["n_embd"] * (4 if self.kv_f32 else 2), np.uint8)
        _check(self.L.b200_neox_read_kv(self._s, which, out.ctypes.data_as(C.c_void_p), out.nbytes), "read_kv")
        return kv_array(out, self.kv_f32)

    def sync(self):
        self.L.b200_neox_sync(self._s)


GptNeoX._SESSION = NeoxSession
