"""Host-side mirror of the reference's model/session interface for LLaMA over the native C ABI (include/llm_b200.h).

Names follow the reference so that the parity tests read like its own integration tests (binaries/llm-test):
  Llama(KnownModel)                crates/models/llama/src/lib.rs:17-140   new / start_session / evaluate
  ModelParameters                  crates/llm-base/src/model/mod.rs:197-229
  InferenceSessionConfig           crates/llm-base/src/inference_session.rs:799-841
  InferenceSession                 crates/llm-base/src/inference_session.rs:43-512  feed_prompt / n_past / last_logits
  OutputRequest                    crates/llm-base/src/lib.rs (all_logits), model/common.rs:22-39
  InferenceError::ContextFull      crates/llm-base/src/inference_session.rs:311-313
  infer_next_token / infer         crates/llm-base/src/inference_session.rs:381-512, InferenceRequest / InferenceStats / InferenceFeedback
  InferenceParameters / Sampler    crates/llm-base/src/inference_session.rs, samplers.rs:97-211 (the default chain, run on the device)
  get_snapshot / from_snapshot     crates/llm-base/src/inference_session.rs:591-646, InferenceSnapshot / SnapshotError :733-792; session files as
                                   the CLI's --save-session / --load-session (binaries/llm-cli/src/snapshot.rs)
"""
import ctypes as C
import enum
import time
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

from . import _lib


class ContextFull(Exception):
    """InferenceError::ContextFull."""


class EndOfText(Exception):
    """InferenceError::EndOfText: the sampled token is the model's end-of-text token.  It has been evaluated (n_past counts it), as in the
    reference; `token` is its id."""

    def __init__(self, token: int):
        super().__init__(f"end of text (token {token})")
        self.token = token


class SamplerFailure(Exception):
    """InferenceError::SamplerFailure: the last logits row holds a NaN.  n_past, tokens() and last_logits are as they were before the call."""


class SnapshotError(Exception):
    """SnapshotError, and a session file this library cannot read (B200_ERR_SNAPSHOT_FORMAT: see b200_snapshot in include/llm_b200.h)"""


class MemorySizeMismatch(SnapshotError):
    """SnapshotError::MemorySizeMismatch: the snapshot's memory_k (or, when that fits, memory_v) is not the size of this model's cache"""

    def __init__(self, self_size: int, input_size: int):
        super().__init__(f"memory size mismatch: session {self_size} bytes, snapshot {input_size} bytes")
        self.self_size, self.input_size = self_size, input_size


@dataclass
class Sampler:
    """The reference's default sampler chain (samplers.rs:97-211, ensure_default_slots), in this order: repetition penalty over the last
    `repetition_last_n` tokens, top-k, top-p, temperature, one random draw.  Its arithmetic is fixed in include/llm_b200.h (b200_sampler);
    top_k = 1 is greedy decoding."""
    repetition_penalty: float = 1.30
    repetition_last_n: int = 64
    top_k: int = 40
    top_p: float = 0.95
    temperature: float = 0.80


@dataclass
class InferenceParameters:
    sampler: Sampler = field(default_factory=Sampler)


class Rng:
    """The random stream of the draw: SplitMix64 seeded with `seed`; `draw` is the index of the next uniform.  The caller owns the counter:
    after a rewind by r tokens, `draw -= r` replays the same draws."""

    def __init__(self, seed: int = 0):
        self.seed, self.draw = int(seed) & 0xFFFFFFFFFFFFFFFF, 0


@dataclass
class InferenceRequest:
    prompt: Sequence[int] = ()                      # token ids (tokenization is the caller's)
    parameters: InferenceParameters = field(default_factory=InferenceParameters)
    maximum_token_count: Optional[int] = None       # None: until end of text (or ContextFull)
    play_back_previous_tokens: bool = False         # infer first calls callback(id) for every id of tokens() (a restored session's history)


@dataclass
class InferenceStats:
    feed_prompt_duration: float = 0.0               # seconds
    prompt_tokens: int = 0                          # n_past after the prompt
    predict_duration: float = 0.0                   # seconds, from the start of infer
    predict_tokens: int = 0                         # n_past at the end


class InferenceFeedback(enum.Enum):
    Continue = 0
    Halt = 1


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


# ModelKVMemoryType as the snapshot encodes it: bincode's enum variant index (Float16 = 0, Float32 = 1), neither enum ggml_type nor .value above
KV_VARIANT = {ModelKVMemoryType.Float16: 0, ModelKVMemoryType.Float32: 1}
KV_FROM_VARIANT = {v: k for k, v in KV_VARIANT.items()}
SNAPSHOT_SIZE_MISMATCH, SNAPSHOT_FORMAT = -18, -19


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
    # OutputRequest::embeddings (model/common.rs:40-59): set to any array (an empty one will do) to request them; evaluate / feed_prompt replace it
    # with the n_embd f32 of the last row of the final norm's output
    embeddings: Optional[np.ndarray] = None


def _embeddings_buffer(request: Optional[OutputRequest], n_embd: int) -> Optional[np.ndarray]:
    """the host row an evaluate fills when `request` asks for embeddings, else None"""
    return None if request is None or request.embeddings is None else np.empty(n_embd, np.float32)


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
    if rc == -6:
        raise SamplerFailure(what)
    if rc != 0:
        raise RuntimeError(f"{what} failed with code {rc}")


@dataclass
class InferenceSnapshot:
    """InferenceSnapshot: the session at npast, with memory_k / memory_v as the reference's bytes (include/llm_b200.h: b200_snapshot)"""
    npast: int
    config: InferenceSessionConfig                  # n_batch and the KV types
    n_threads: int
    tokens: np.ndarray                              # np.uint32, the ids at positions [0, npast)
    last_logits: np.ndarray                         # np.float32, n_vocab
    memory_k: np.ndarray                            # np.uint8
    memory_v: np.ndarray


def _snapshot_struct(snap: InferenceSnapshot):
    """the b200_snapshot of `snap`, and the arrays it points into (to be kept alive for the call)"""
    kt, vt = KV_VARIANT[snap.config.memory_k_type], KV_VARIANT[snap.config.memory_v_type]
    arrs = [np.ascontiguousarray(snap.tokens, np.uint32), np.ascontiguousarray(snap.last_logits, np.float32),
            np.ascontiguousarray(snap.memory_k, np.uint8).ravel(), np.ascontiguousarray(snap.memory_v, np.uint8).ravel()]
    c = _lib.Snapshot(npast=snap.npast, memory_k_type=kt, memory_v_type=vt, n_batch=snap.config.n_batch, n_threads=snap.n_threads,
                      n_tokens=arrs[0].size, tokens=arrs[0].ctypes.data, n_logits=arrs[1].size, last_logits=arrs[1].ctypes.data,
                      memory_k_bytes=arrs[2].nbytes, memory_v_bytes=arrs[3].nbytes, memory_k=arrs[2].ctypes.data, memory_v=arrs[3].ctypes.data)
    return c, arrs


def _snapshot_refused(rc: int, what: str, self_bytes, k_bytes: int, v_bytes: int):
    """the exception of a from_snapshot refusal: self_bytes(variant) is the model's cache size for a KV type"""
    if rc == SNAPSHOT_SIZE_MISMATCH:
        raise MemorySizeMismatch(self_bytes, k_bytes if k_bytes != self_bytes else v_bytes)
    if rc == SNAPSHOT_FORMAT:
        raise SnapshotError(f"{what}: not a session file this library reads (code {rc})")
    _check(rc, what)
    raise RuntimeError(f"{what} failed")


def _snapshot_file_header(L, path: str) -> "_lib.Snapshot":
    h = _lib.Snapshot()
    rc = L.b200_snapshot_read_header(str(path).encode(), C.byref(h))
    if rc != 0:
        _snapshot_refused(rc, f"read_snapshot({path})", 0, 0, 0)
    return h


def _ref_cache_bytes(n_layer: int, context_size: int, n_embd: int, variant: int) -> int:
    """the reference's memory_k / memory_v size: n_layer x context_size x n_embd values (also with grouped-query attention)"""
    return n_layer * context_size * n_embd * (4 if variant == 1 else 2)


class _Snapshots:
    """get_snapshot / write_snapshot and the from_snapshot / read_snapshot constructors of a native session: `_GET_SNAP`, `_WRITE_SNAP`,
    `_FROM_SNAP`, `_READ_SNAP` name the library's entry points; `_adopt(model, handle, config)` wraps a session handle, `_start_args(flags)` are
    the extra arguments of the constructors, `_cache_bytes(model, variant)` the size a snapshot's memory must have."""
    _GET_SNAP = _WRITE_SNAP = _FROM_SNAP = _READ_SNAP = ""

    def get_snapshot(self) -> InferenceSnapshot:
        """InferenceSession::get_snapshot: a copy of the session, the cache in the reference's layout (after the work queued so far)"""
        get = getattr(self.L, self._GET_SNAP)
        h = _lib.Snapshot()
        _check(get(self._s, C.byref(h)), "get_snapshot")
        tok, lg = np.empty(h.n_tokens, np.uint32), np.empty(h.n_logits, np.float32)
        mk, mv = np.empty(h.memory_k_bytes, np.uint8), np.empty(h.memory_v_bytes, np.uint8)
        h.tokens, h.last_logits, h.memory_k, h.memory_v = tok.ctypes.data, lg.ctypes.data, mk.ctypes.data, mv.ctypes.data
        _check(get(self._s, C.byref(h)), "get_snapshot")
        cfg = InferenceSessionConfig(n_batch=h.n_batch, memory_k_type=KV_FROM_VARIANT[h.memory_k_type], memory_v_type=KV_FROM_VARIANT[h.memory_v_type])
        return InferenceSnapshot(npast=h.npast, config=cfg, n_threads=h.n_threads, tokens=tok, last_logits=lg, memory_k=mk, memory_v=mv)

    def write_snapshot(self, path: str):
        """the snapshot as the CLI's session file (bincode in a zstd frame of raw blocks), streamed from HBM"""
        _check(getattr(self.L, self._WRITE_SNAP)(self._s, str(path).encode()), f"write_snapshot({path})")

    @classmethod
    def _restore(cls, model, entry, source, flags, sizes, config):
        err = C.c_int(0)
        h = entry(model._m, source, *cls._start_args(flags), C.byref(err))
        if not h:
            kt, kb, vb = sizes()
            _snapshot_refused(err.value, "from_snapshot", cls._cache_bytes(model, kt), kb, vb)
        return cls._adopt(model, h, config())

    @classmethod
    def _from(cls, snapshot: InferenceSnapshot, model, flags: int):
        c, keep = _snapshot_struct(snapshot)
        return cls._restore(model, getattr(model.L, cls._FROM_SNAP), C.byref(c), flags,
                            lambda: (KV_VARIANT[snapshot.config.memory_k_type], keep[2].nbytes, keep[3].nbytes),
                            lambda: InferenceSessionConfig(n_batch=snapshot.config.n_batch, flags=flags, memory_k_type=snapshot.config.memory_k_type,
                                                           memory_v_type=snapshot.config.memory_v_type))

    @classmethod
    def _read(cls, path: str, model, flags: int):
        hdr = {}

        def header():
            if not hdr:
                hdr["h"] = _snapshot_file_header(model.L, path)
            return hdr["h"]

        def sizes():
            h = header()
            return h.memory_k_type, h.memory_k_bytes, h.memory_v_bytes

        def config():
            h = header()
            kv = KV_FROM_VARIANT[h.memory_k_type]
            return InferenceSessionConfig(n_batch=h.n_batch, flags=flags, memory_k_type=kv, memory_v_type=kv)

        return cls._restore(model, getattr(model.L, cls._READ_SNAP), str(path).encode(), flags, sizes, config)


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


class _Generation:
    """Text generation on a native session (InferenceSession::infer_next_token / infer): `_INFER`, `_TOKENS` and `_LAST` name the library's
    entry points; the session keeps `model`, `n_vocab`, `L`, `_s`, `_last_logits` (host copy of the last row, None: read it from the device)."""
    _INFER, _TOKENS, _LAST = "", "", ""

    @property
    def last_logits(self) -> np.ndarray:
        """the last evaluated row (zeros before the first evaluate); read from the device on access after generation"""
        if self._last_logits is None:
            out = np.zeros(self.n_vocab, np.float32)
            if getattr(self.L, self._LAST)(self._s, out.ctypes.data_as(C.c_void_p)) != 0:
                out[:] = 0.0                        # nothing evaluated yet
            self._last_logits = out
        return self._last_logits

    def tokens(self) -> np.ndarray:
        """InferenceSession::tokens: the ids at positions [0, n_past)"""
        n = self.n_past
        out = np.empty(max(n, 1), np.int32)
        got = getattr(self.L, self._TOKENS)(self._s, out.ctypes.data_as(C.c_void_p), n)
        if got < 0:
            _check(got, "read_tokens")
        return out[:min(got, n)].copy()

    def infer_next_token(self, params: Optional[InferenceParameters], rng: Rng) -> int:
        """Sample the next token from last_logits on the device, append it and evaluate it; returns its id and advances rng.draw.
        Raises ContextFull (n_past + 1 >= context size; nothing changes), SamplerFailure (nothing changes), or EndOfText (the token is the
        model's eot_token_id(); it has been evaluated and rng.draw advanced)."""
        sp = (params or InferenceParameters()).sampler
        c = _lib.SamplerParams(repetition_penalty=sp.repetition_penalty, repetition_last_n=sp.repetition_last_n, top_k=sp.top_k, top_p=sp.top_p,
                               temperature=sp.temperature, seed=rng.seed, draw=rng.draw)
        tok = C.c_int32(-1)
        _check(getattr(self.L, self._INFER)(self._s, C.byref(c), C.byref(tok)), "infer_next_token")
        rng.draw += 1
        self._last_logits = None
        eot = self.model.eot_token_id()
        if eot is not None and tok.value == eot:
            raise EndOfText(tok.value)
        return tok.value

    def infer(self, request: InferenceRequest, rng: Rng, callback: Optional[Callable[[int], Optional[InferenceFeedback]]] = None) -> InferenceStats:
        """InferenceSession::infer: feed the prompt, then generate until end of text, maximum_token_count tokens or a callback that returns
        InferenceFeedback.Halt.  callback(token_id) is called for each generated token but the end-of-text one.  ContextFull is raised, as the
        reference returns it."""
        stats = InferenceStats()
        t0 = time.perf_counter()
        if request.play_back_previous_tokens and callback is not None:
            for tok in self.tokens():               # inference_session.rs:443-457: the feedback is ignored, as for SnapshotToken
                callback(int(tok))
        if len(request.prompt):
            self.feed_prompt(request.prompt)
        stats.feed_prompt_duration = time.perf_counter() - t0
        stats.prompt_tokens = self.n_past
        limit = request.maximum_token_count
        done = 0
        while limit is None or done < limit:
            try:
                tok = self.infer_next_token(request.parameters, rng)
            except EndOfText:
                break
            if callback is not None and callback(tok) == InferenceFeedback.Halt:
                break
            done += 1
        stats.predict_duration = time.perf_counter() - t0
        stats.predict_tokens = self.n_past
        return stats


class _BatchedSessions:
    """Batched steps over the sessions of one model (include/llm_b200.h: b200_model_evaluate_ragged / b200_neox_evaluate_ragged and the decode
    steps b200_*_evaluate_sessions, b200_*_infer_next_tokens): `_EVAL_SESSIONS`, `_INFER_SESSIONS` and `_EVAL_RAGGED` name the library's entry
    points, `_SESSION` the model's session class; the model keeps `L`, `_m`, `hyperparameters` and its context size."""
    _EVAL_SESSIONS, _INFER_SESSIONS, _EVAL_RAGGED = "", "", ""
    _SESSION: type = type(None)
    MAX_SESSIONS = 64                           # B200_MAX_SESSIONS
    MAX_BATCH_ROWS = 4096                       # B200_MAX_BATCH_ROWS: the tokens of one ragged step

    def _session_handles(self, sessions):
        return (C.c_void_p * max(1, len(sessions)))(*[s._s for s in sessions])

    def _own(self, sessions, what):
        """the library cannot tell one runtime's session handle from another's, nor check a handle it was not given by this model's runtime"""
        for s in sessions:
            if not isinstance(s, self._SESSION):
                raise TypeError(f"{what}: {type(s).__name__} is not a {self._SESSION.__name__}")
            if s.model is not self:
                raise RuntimeError(f"{what}: a session of another model")

    def evaluate_sessions(self, sessions: Sequence["InferenceSession"], tokens) -> np.ndarray:
        """One decode step for several sessions of this model: session i evaluates tokens[i] at its own n_past, reading the weights once for
        all of them.  Each session ends exactly as after session.evaluate([tokens[i]]) alone, bit for bit.  Returns the [n, n_vocab] logits.
        Refused as a whole, nothing changed (RuntimeError, or ContextFull when a session has no room): 0 or more than 64 sessions, a session of
        another model, the same session twice, FAST sessions (LLaMA), mixed KV cache types, an id outside the vocabulary; TypeError for a session that
        is not of this model's runtime.  See include/llm_b200.h."""
        tokens = np.ascontiguousarray(tokens, np.int32).ravel()
        n = len(sessions)
        if tokens.size != n:
            raise ValueError(f"{n} sessions, {tokens.size} tokens")
        self._own(sessions, "evaluate_sessions")
        out = np.empty((max(n, 1), int(self.hyperparameters["n_vocab"])), np.float32)
        _check(getattr(self.L, self._EVAL_SESSIONS)(self._m, self._session_handles(sessions), n, tokens.ctypes.data_as(C.c_void_p),
                                                   out.ctypes.data_as(C.c_void_p)), "evaluate_sessions")
        for i, s in enumerate(sessions):
            s._last_logits = None
        return out[:n]

    def evaluate_ragged(self, sessions: Sequence["InferenceSession"], chunks, all_logits: bool = False) -> List[np.ndarray]:
        """One step for several sessions of this model, each evaluating a chunk of its own: session i evaluates chunks[i] (1 to its n_batch ids)
        at its own n_past, reading the weights once for all of them -- new sessions prefill while others decode.  Each session ends exactly as
        after session.evaluate(chunks[i], all_logits) alone, bit for bit.  Returns one array per session: its last row [n_vocab], or with
        all_logits every row [len(chunks[i]), n_vocab].  Refused as a whole, nothing changed (RuntimeError, or ContextFull when a chunk does not
        fit): evaluate_sessions' refusals, an empty chunk or one longer than its session's n_batch, more than 4096 ids in all; TypeError for a
        session that is not of this model's runtime.  See include/llm_b200.h."""
        n = len(sessions)
        if len(chunks) != n:
            raise ValueError(f"{n} sessions, {len(chunks)} chunks")
        arrs = [np.ascontiguousarray(c, np.int32).ravel() for c in chunks]
        counts = np.array([a.size for a in arrs] or [0], np.int32)
        toks = np.ascontiguousarray(np.concatenate(arrs) if arrs else np.zeros(1, np.int32), np.int32)
        self._own(sessions, "evaluate_ragged")
        rows = int(counts[:n].sum()) if all_logits else n
        out = np.empty((max(rows, 1), int(self.hyperparameters["n_vocab"])), np.float32)
        _check(getattr(self.L, self._EVAL_RAGGED)(self._m, self._session_handles(sessions), n, counts.ctypes.data_as(C.c_void_p),
                                                 toks.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), 1 if all_logits else 0),
               "evaluate_ragged")
        for s in sessions:
            s._last_logits = None
        if not all_logits:
            return [out[i] for i in range(n)]
        ends = np.cumsum(counts[:n])
        return [out[e - c:e] for e, c in zip(ends, counts[:n])]

    def feed_prompts(self, sessions: Sequence["InferenceSession"], prompts) -> List[np.ndarray]:
        """InferenceSession::feed_prompt for several sessions of this model: each prompt is cut into chunks of its own session's n_batch, and step
        k evaluates chunk k of every session that still has one (evaluate_ragged), so each session ends bit-identical to feed_prompt alone.  A
        step of more than 4096 ids is split across sessions; each session's chunks stay the same.  Returns each session's last_logits (an empty
        prompt leaves its session untouched).  ContextFull, before anything is evaluated, when a prompt does not fit its session."""
        n = len(sessions)
        if len(prompts) != n:
            raise ValueError(f"{n} sessions, {len(prompts)} prompts")
        self._own(sessions, "feed_prompts")
        ps = [np.ascontiguousarray(p, np.int32).ravel() for p in prompts]
        cs = self.context_size
        n_ctx = cs() if callable(cs) else cs
        for s, p in zip(sessions, ps):
            if s.n_past + p.size > n_ctx:              # feed_prompt's check (inference_session.rs:311-313), for every session first
                raise ContextFull("feed_prompts")
            if min(p.size, s.n_batch) > self.MAX_BATCH_ROWS:
                raise ValueError(f"feed_prompts: a chunk of {s.n_batch} ids is more than one step takes ({self.MAX_BATCH_ROWS})")
        done = [0] * n
        while True:
            step = [(i, ps[i][done[i]:done[i] + sessions[i].n_batch]) for i in range(n) if done[i] < ps[i].size]
            if not step:
                break
            while step:
                rows, k = 0, 0
                while k < len(step) and rows + step[k][1].size <= self.MAX_BATCH_ROWS:
                    rows += step[k][1].size
                    k += 1
                part, step = step[:k], step[k:]
                got = self.evaluate_ragged([sessions[i] for i, _ in part], [c for _, c in part])
                for (i, c), row in zip(part, got):
                    done[i] += c.size
                    sessions[i]._last_logits = row.copy()
        return [s.last_logits for s in sessions]

    def infer_next_tokens(self, sessions: Sequence["InferenceSession"], params, rngs: Sequence[Rng]) -> List[int]:
        """infer_next_token for several sessions at once: session i samples from its last row with its own parameters and rngs[i], then one
        batched step evaluates every sampled id.  `params`: one InferenceParameters (or None) for all, or one per session.  Returns the ids; each
        rngs[i].draw advances by one for every session that sampled.  End of text is NOT raised: the id is returned (and has been evaluated), and
        the caller compares it with eot_token_id().  A session whose row holds a NaN is left as it was; once the others have advanced,
        SamplerFailure is raised with `.sessions`, the failed indices, and `.tokens`, the ids (-1 at the failed ones)."""
        n = len(sessions)
        plist = list(params) if isinstance(params, (list, tuple)) else [params] * n
        if len(plist) != n or len(rngs) != n:
            raise ValueError(f"{n} sessions, {len(plist)} parameters, {len(rngs)} rngs")
        table = (_lib.SamplerParams * max(n, 1))()
        for i, (p, rng) in enumerate(zip(plist, rngs)):
            sp = (p or InferenceParameters()).sampler
            table[i] = _lib.SamplerParams(repetition_penalty=sp.repetition_penalty, repetition_last_n=sp.repetition_last_n, top_k=sp.top_k,
                                          top_p=sp.top_p, temperature=sp.temperature, seed=rng.seed, draw=rng.draw)
        self._own(sessions, "infer_next_tokens")
        toks, status = np.full(max(n, 1), -1, np.int32), np.zeros(max(n, 1), np.int32)
        _check(getattr(self.L, self._INFER_SESSIONS)(self._m, self._session_handles(sessions), n, table, toks.ctypes.data_as(C.c_void_p),
                                                   status.ctypes.data_as(C.c_void_p)), "infer_next_tokens")
        failed = []
        for i, (s, rng) in enumerate(zip(sessions, rngs)):
            if status[i] == 0:
                rng.draw += 1
                s._last_logits = None
            else:
                failed.append(i)
        ids = [int(t) for t in toks[:n]]
        if failed:
            err = SamplerFailure(f"infer_next_tokens: sampler failure in sessions {failed}")
            err.sessions, err.tokens = failed, ids
            raise err
        return ids


def _vocab_id(vocabulary, token: bytes) -> Optional[int]:
    try:
        return vocabulary.index(token)
    except ValueError:
        return None


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


KQUANT_BLOCK_BYTES = {10: 84, 11: 110, 12: 144, 13: 176, 14: 210}      # Q2_K .. Q6_K super-block bytes (LC/k_quants.h)


def ggml_dims(arr: np.ndarray, wtype: int):
    """(n_dims, ne0, ne1) of a tensor given as GGML-layout block rows (uint8 [rows][row bytes]) or f32 ([n] or [rows][cols])"""
    if arr.dtype == np.float32:
        return (1, arr.shape[0], 1) if arr.ndim == 1 else (2, arr.shape[-1], arr.size // arr.shape[-1])
    if arr.dtype == np.float16:                  # F16 weights: [rows][cols] halves
        return 2, arr.shape[-1], arr.size // arr.shape[-1]
    if wtype in KQUANT_BLOCK_BYTES:              # K-quants: 256-element super-blocks
        return 2, arr.shape[-1] // KQUANT_BLOCK_BYTES[wtype] * 256, arr.size // arr.shape[-1]
    block = {2: 18, 3: 20, 6: 22, 7: 24, 8: 34}[wtype]
    return 2, arr.shape[-1] // block * 32, arr.size // arr.shape[-1]


class Llama(_BatchedSessions, _Native):
    """KnownModel for LLaMA.  `hyperparameters` is a dict with n_vocab, n_embd, n_head, n_head_kv, n_layer, n_rot, n_ff, wtype.
    `tensor_types`: {name: enum ggml_type} of 2-D weights whose type is not `wtype` (mixed-type files, b200_llama_new_typed)."""
    _HANDLE, _FREE = "_m", "b200_model_free"
    _EVAL_SESSIONS, _INFER_SESSIONS = "b200_model_evaluate_sessions", "b200_model_infer_next_tokens"
    _EVAL_RAGGED = "b200_model_evaluate_ragged"
    tensor_types: Dict[str, int] = {}           # models loaded from a file or cut into shards: their types are in the C model

    def __init__(self, hyperparameters: Dict[str, int], params: ModelParameters = None, tensors: Dict[str, np.ndarray] = None,
                 device: int = 0, vocabulary: Optional[Sequence] = None, tensor_types: Optional[Dict[str, int]] = None):
        """vocabulary: the model file's tokens ((bytes, score) pairs, or bytes), consulted by eot_token_id()"""
        params = params or ModelParameters()
        self.vocabulary = [t[0] if isinstance(t, tuple) else bytes(t) for t in vocabulary] if vocabulary is not None else None
        if not params.use_gpu:
            raise ValueError("llm_b200 has no CPU path: ModelParameters.use_gpu must be True")
        self.L = _lib.lib()
        _check(self.L.b200_init(device), "b200_init")
        self.hyperparameters = dict(hyperparameters)
        self.params = params
        hp = _lib.LlamaHparams(**{k: int(hyperparameters[k]) for k in _HP_KEYS}, wtype=int(hyperparameters["wtype"]),
                               context_size=params.context_size, rope_freq_base=params.rope_freq_base,
                               rope_freq_scale=params.rope_freq_scale)
        self.tensor_types = dict(tensor_types or {})
        if self.tensor_types:
            names = [n.encode() for n in self.tensor_types]
            table = (_lib.TensorType * len(names))(*[_lib.TensorType(n, int(t)) for n, t in zip(names, self.tensor_types.values())])
            err = C.c_int(0)
            self._m = self.L.b200_llama_new_typed(C.byref(hp), table, len(names), C.byref(err))
            if not self._m:
                from .loader import LoadError
                raise LoadError(err.value, "b200_llama_new_typed")
        else:
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
        typ = 0 if arr.dtype == np.float32 else 1 if arr.dtype == np.float16 else int(self.tensor_types.get(name, self.hyperparameters["wtype"]))
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

    def eot_token_id(self) -> Optional[int]:
        """KnownModel::eot_token_id: "</s>" in the vocabulary, else 2 (llama lib.rs:386-388).  Without a vocabulary: None (no end of text)."""
        vocab = getattr(self, "vocabulary", None)
        if vocab is None:
            return None
        eot = _vocab_id(vocab, b"</s>")
        return 2 if eot is None else eot


class InferenceSession(_Generation, _Snapshots, _Native):
    _HANDLE, _FREE = "_s", "b200_session_free"
    _INFER, _TOKENS, _LAST = "b200_session_infer_next_token", "b200_session_read_tokens", "b200_session_last_logits"
    _GET_SNAP, _WRITE_SNAP = "b200_session_get_snapshot", "b200_session_write_snapshot"
    _FROM_SNAP, _READ_SNAP = "b200_model_session_from_snapshot", "b200_model_session_read_snapshot"

    def __init__(self, model: Llama, config: InferenceSessionConfig, _handle=None):
        self.model, self.config, self.L = model, config, model.L
        self.kv_f32 = kv_flags(config.memory_k_type, config.memory_v_type) != 0
        cfg = _lib.SessionConfig(n_batch=config.n_batch, flags=config.flags | (SESSION_KV_F32 if self.kv_f32 else 0))
        self._s = _handle or self.L.b200_model_start_session(model._m, C.byref(cfg))
        if not self._s:
            raise RuntimeError("b200_model_start_session failed (all tensors loaded?)")
        self.n_vocab = int(model.hyperparameters["n_vocab"])
        self._last_logits = None if _handle else np.zeros(self.n_vocab, np.float32)

    @classmethod
    def from_snapshot(cls, snapshot: InferenceSnapshot, model: Llama, flags: int = 0) -> "InferenceSession":
        """InferenceSession::from_snapshot: a session of `model` with the snapshot's n_batch and KV types, cache, history and last row.  flags may
        add B200_SESSION_NO_GRAPH / UNFUSED / FAST.  Raises MemorySizeMismatch for another geometry, context size or KV type."""
        return cls._from(snapshot, model, flags)

    @classmethod
    def read_snapshot(cls, path: str, model: Llama, flags: int = 0) -> "InferenceSession":
        """from_snapshot of a session file (the CLI's --load-session), streamed into HBM; SnapshotError if the file cannot be read"""
        return cls._read(path, model, flags)

    @staticmethod
    def _start_args(flags):
        return (flags,)

    @staticmethod
    def _cache_bytes(model, variant):
        hp = model.hyperparameters
        return _ref_cache_bytes(hp["n_layer"], model.params.context_size, hp["n_embd"], variant)

    @classmethod
    def _adopt(cls, model, handle, config):
        return cls(model, config, _handle=handle)

    @property
    def n_past(self) -> int:
        return self.L.b200_session_n_past(self._s)

    @property
    def n_batch(self) -> int:
        return self.config.n_batch

    def top_k(self, k: int):
        """Sampler hand-off: (token ids, logits) of the k largest logits of the last evaluated row, selected on the device."""
        ids, vals = np.empty(k, np.int32), np.empty(k, np.float32)
        _check(self.L.b200_session_top_k(self._s, k, ids.ctypes.data_as(C.c_void_p), vals.ctypes.data_as(C.c_void_p)), "top_k")
        return ids, vals

    def evaluate(self, tokens, all_logits: bool = False, output_request: Optional[OutputRequest] = None) -> np.ndarray:
        """Model::evaluate: one forward pass over `tokens` (<= n_batch) appended at n_past; returns logits
        ([n, n_vocab] when all_logits else the last row, which is also kept in self.last_logits).  output_request.embeddings, when not None,
        is replaced with the n_embd f32 of the last row of the final norm's output (a tensor-parallel session refuses that request: RuntimeError)."""
        tokens = np.ascontiguousarray(tokens, np.int32)
        n = tokens.size
        out = np.empty((n if all_logits else 1, self.n_vocab), np.float32)
        embd = _embeddings_buffer(output_request, self.model.hyperparameters["n_embd"])
        _check(self.L.b200_session_evaluate_output(self._s, tokens.ctypes.data_as(C.c_void_p), n, out.ctypes.data_as(C.c_void_p),
                                                   1 if all_logits else 0, None if embd is None else embd.ctypes.data_as(C.c_void_p)), "evaluate")
        if embd is not None:
            output_request.embeddings = embd
        self._last_logits = out[-1].copy()
        return out if all_logits else out[0]

    def feed_prompt(self, tokens, output_request: Optional[OutputRequest] = None) -> np.ndarray:
        """InferenceSession::feed_prompt: the prompt in chunks of n_batch, each evaluated with output_request (so its embeddings are the last
        chunk's last row); returns last_logits."""
        tokens = np.ascontiguousarray(tokens, np.int32)
        if tokens.size == 0:                      # the reference leaves last_logits untouched for an empty prompt (inference_session.rs:299-350)
            return self.last_logits
        out = np.empty(self.n_vocab, np.float32)
        embd = _embeddings_buffer(output_request, self.model.hyperparameters["n_embd"])
        _check(self.L.b200_session_feed_prompt_output(self._s, tokens.ctypes.data_as(C.c_void_p), tokens.size, out.ctypes.data_as(C.c_void_p),
                                                      None if embd is None else embd.ctypes.data_as(C.c_void_p)), "feed_prompt")
        if embd is not None:
            output_request.embeddings = embd
        self._last_logits = out
        return out

    def perplexity(self, tokens, callback=None, bos: Optional[int] = None, return_terms: bool = False):
        """InferenceSession::perplexity on token ids (tokenization is the caller's), computed on the device: one perplexity per chunk of
        context_size tokens, callback(chunk, ppl) after each.  bos replaces each chunk's first token (default: bot_token_id() or 1).  Every chunk
        starts at n_past 0; afterwards n_past is context_size (unchanged when there are fewer tokens than that).  See include/llm_b200.h."""
        bot = self.model.bot_token_id()
        bos = (1 if bot is None else bot) if bos is None else bos
        self._last_logits = None
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


Llama._SESSION = InferenceSession
