"""GGML / GGMF / GGJT model files over the C ABI (include/llm_b200.h, csrc/ggml_file.cu) -- SURVEY.md §8f-2.

Mirrors the reference's loading surface:
  ggml::format::load / TensorLoadInfo     crates/ggml/src/format/loader.rs:160-281          -> GgmlFile
  ggml::format::save                       crates/ggml/src/format/saver.rs:86-160            -> write_llama
  llm::load::<Llama>(path, params)         crates/llm-base/src/loader.rs:419-567             -> load
  LoadError variants                       crates/ggml/src/format/loader.rs:38-70            -> LoadError.kind
The parser runs without a GPU; `load` needs one (the tensors go straight from the file mapping to HBM).
"""
import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .session import Llama, ModelParameters

MAGIC = {0x67676d6c: "ggml", 0x67676d66: "ggmf", 0x67676a74: "ggjt", 0x67676c61: "ggla"}
ERRORS = {-10: "Io", -11: "InvalidMagic", -12: "InvalidFormatVersion", -13: "InvariantBroken", -14: "UnsupportedElementType",
          -15: "QuantizationVersion", -3: "UnknownTensor", -4: "TensorWrongSize", -5: "NotLoaded", -2: "BadArgument"}


class LoadError(Exception):
    def __init__(self, code: int, what: str):
        self.code, self.kind = code, ERRORS.get(code, str(code))
        super().__init__(f"{what}: {self.kind}")


ARCH = {"llama": 0, "gpt2": 1, "gptneox": 2, "mpt": 3, "bloom": 4, "gptj": 5, "lora": 6}
HPARAM_NAMES = {
    "llama": ("n_vocab", "n_embd", "n_mult", "n_head", "n_layer", "n_rot", "file_type"),                                   # llama lib.rs:425-447
    "gpt2": ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "file_type", "n_vocab_again"),                              # gpt2 lib.rs:394-416
    "gptneox": ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "n_rot", "use_parallel_residual", "file_type"),          # gptneox lib.rs:431-442
    "mpt": ("n_embd", "max_seq_len", "n_head", "n_layer", "n_vocab", "alibi_bias_max", "clip_kqv", "file_type"),          # mpt lib.rs:317-330
    "bloom": ("n_vocab", "n_embd", "n_mult", "n_head", "n_layer", "file_type"),                                           # bloom lib.rs
    "gptj": ("n_vocab", "n_ctx", "n_embd", "n_head", "n_layer", "n_rot", "file_type", "n_vocab_again"),                    # gptj lib.rs:366-401
    "lora": ("r", "alpha"),                                                                                                 # LoraParameters, lora.rs:27-35
}
FLOAT_WORDS = {"alibi_bias_max", "clip_kqv"}                                                                             # f32 in the header (read_f32)


def _f32_bits(x) -> int:
    return int(np.array([x], np.float32).view(np.int32)[0])


class GgmlFile:
    """A parsed container: ContainerType, the architecture's hyperparameters, vocabulary, tensor table (name, dims, type, file offset)."""

    def __init__(self, path: str, arch: str = "llama"):
        self.L = _lib.lib()
        err = C.c_int(0)
        self.arch = arch
        self._f = self.L.b200_ggml_open_arch(path.encode(), ARCH[arch], C.byref(err))
        if not self._f:
            raise LoadError(err.value, f"open {path}")
        self.path = path

    def hyperparameters(self) -> Dict[str, int]:
        """The header words of the file, named after the architecture's Hyperparameters struct."""
        arch, words, n = C.c_int32(), (C.c_int32 * 8)(), C.c_int32()
        self.L.b200_ggml_hparams(self._f, C.byref(arch), C.byref(words), C.byref(n))
        out = dict(zip(HPARAM_NAMES[self.arch], list(words)[:n.value]))
        for k in FLOAT_WORDS & out.keys():
            out[k] = float(np.array([out[k]], np.int32).view(np.float32)[0])
        return out

    @property
    def container(self) -> Tuple[str, int]:
        m, v = C.c_uint32(), C.c_uint32()
        self.L.b200_ggml_container(self._f, C.byref(m), C.byref(v))
        return MAGIC[m.value], v.value

    def llama_hyperparameters(self) -> Dict[str, int]:
        hp, n_mult, ftype, qv = _lib.LlamaHparams(), C.c_int32(), C.c_int32(), C.c_int32()
        rc = self.L.b200_ggml_llama_hparams(self._f, C.byref(hp), C.byref(n_mult), C.byref(ftype), C.byref(qv))
        if rc != 0:
            raise LoadError(rc, f"hyperparameters of {self.path}")
        out = {k: getattr(hp, k) for k in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_rot", "n_ff", "wtype")}
        out.update(n_mult=n_mult.value, llama_ftype=ftype.value, quantization_version=qv.value)
        return out

    def tensors(self) -> List[dict]:
        out = []
        for i in range(self.L.b200_ggml_n_tensors(self._f)):
            ti = _lib.GgmlTensorInfo()
            self.L.b200_ggml_tensor(self._f, i, C.byref(ti))
            out.append(dict(name=ti.name.decode(), type=ti.type, n_dims=ti.n_dims, ne=(ti.ne[0], ti.ne[1]), offset=ti.offset, nbytes=ti.nbytes))
        return out

    def tensor_bytes(self, i: int) -> np.ndarray:
        ti = _lib.GgmlTensorInfo()
        self.L.b200_ggml_tensor(self._f, i, C.byref(ti))
        p = self.L.b200_ggml_tensor_data(self._f, i)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(ti.nbytes,)).copy()

    def vocabulary(self) -> List[Tuple[bytes, float]]:
        out = []
        for i in range(self.L.b200_ggml_n_vocab(self._f)):
            b, n, s = C.POINTER(C.c_uint8)(), C.c_uint32(), C.c_float()
            self.L.b200_ggml_token(self._f, i, C.byref(b), C.byref(n), C.byref(s))
            out.append((bytes(b[:n.value]), s.value))
        return out

    def close(self):
        if getattr(self, "_f", None):
            self.L.b200_ggml_close(self._f)
            self._f = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def write_llama(path: str, hyperparameters: Dict[str, int], tensors: Dict[str, np.ndarray], shapes: Dict[str, Tuple[int, ...]],
                vocabulary: Optional[Sequence[Tuple[bytes, float]]] = None, n_mult: int = 256, quantization_version: int = 2):
    """ggml::format::save for LLaMA (GGJT v3).  `tensors`: name -> GGML-layout bytes (uint8 block rows) or f32 arrays; `shapes`: name ->
    (rows, cols) / (n,) as in oracle.synth.tensor_shapes (ggml order is reversed: ne0 = cols)."""
    L = _lib.lib()
    wtype = int(hyperparameters["wtype"])
    llama_ftype = {0: 0, 1: 1, 2: 2, 3: 3, 8: 7, 6: 8, 7: 9}[wtype]               # llama_ftype of an all-<wtype> file (LC/llama.h)
    hp = _lib.LlamaHparams(**{k: int(hyperparameters[k]) for k in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_rot", "n_ff")}, wtype=wtype)
    infos = (_lib.GgmlTensorInfo * len(tensors))()
    datas = (C.c_void_p * len(tensors))()
    keep = []
    for i, (name, arr) in enumerate(tensors.items()):
        a = np.ascontiguousarray(arr)
        keep.append(a)
        shp = shapes[name]
        infos[i].name = name.encode()
        infos[i].type = 0 if a.dtype == np.float32 else wtype
        infos[i].n_dims = len(shp)
        infos[i].ne[0] = shp[-1]
        infos[i].ne[1] = shp[0] if len(shp) == 2 else 1
        infos[i].nbytes = a.nbytes
        datas[i] = a.ctypes.data
    nv = int(hyperparameters["n_vocab"])
    tb = tl = ts = None
    if vocabulary is not None:
        assert len(vocabulary) == nv
        bufs = [C.create_string_buffer(t, len(t)) for t, _ in vocabulary]
        keep.append(bufs)
        tb = (C.c_void_p * nv)(*[C.cast(b, C.c_void_p) for b in bufs])
        tl = (C.c_uint32 * nv)(*[len(t) for t, _ in vocabulary])
        ts = (C.c_float * nv)(*[s for _, s in vocabulary])
    rc = L.b200_ggml_write_llama(path.encode(), C.byref(hp), n_mult, quantization_version * 1000 + llama_ftype, tb, tl, ts, infos, datas, len(tensors))
    if rc != 0:
        raise LoadError(rc, f"write {path}")


def write_model(path: str, arch: str, header: Dict[str, int], tensors: Dict[str, np.ndarray], shapes: Dict[str, Tuple[int, ...]], wtype: int,
                vocabulary: Optional[Sequence[Tuple[bytes, float]]] = None):
    """ggml::format::save for any of the architectures: `header` holds the words of HPARAM_NAMES[arch] (FLOAT_WORDS as floats)."""
    L = _lib.lib()
    words = [_f32_bits(header[k]) if k in FLOAT_WORDS else int(header["n_vocab"]) if k == "n_vocab_again" else int(header[k]) for k in HPARAM_NAMES[arch]]
    infos = (_lib.GgmlTensorInfo * len(tensors))()
    datas = (C.c_void_p * len(tensors))()
    keep = []
    for i, (name, arr) in enumerate(tensors.items()):
        a = np.ascontiguousarray(arr)
        keep.append(a)
        shp = shapes[name]
        infos[i].name = name.encode()
        infos[i].type = 0 if a.dtype == np.float32 else wtype
        infos[i].n_dims = len(shp)
        infos[i].ne[0] = shp[-1]
        infos[i].ne[1] = shp[0] if len(shp) == 2 else 1
        infos[i].nbytes = a.nbytes
        datas[i] = a.ctypes.data
    nv = int(header["n_vocab"])
    tb = tl = ts = None
    if vocabulary is not None:
        assert len(vocabulary) == nv
        bufs = [C.create_string_buffer(t, len(t)) for t, _ in vocabulary]
        keep.append(bufs)
        tb = (C.c_void_p * nv)(*[C.cast(b, C.c_void_p) for b in bufs])
        tl = (C.c_uint32 * nv)(*[len(t) for t, _ in vocabulary])
        ts = (C.c_float * nv)(*[s for _, s in vocabulary])
    rc = L.b200_ggml_write(path.encode(), (C.c_int32 * len(words))(*words), len(words), nv, tb, tl, ts, infos, datas, len(tensors))
    if rc != 0:
        raise LoadError(rc, f"write {path}")


def load(path: str, params: ModelParameters = None, device: int = 0) -> Llama:
    """llm::load::<Llama>: parse the file, create the model for its geometry, upload every tensor from the mapping to HBM, patched by
    params.lora_adapters (in order) where they name it."""
    params = params or ModelParameters()
    if not params.use_gpu:
        raise ValueError("llm_b200 has no CPU path: ModelParameters.use_gpu must be True")
    L = _lib.lib()
    rc = L.b200_init(device)
    if rc != 0:
        raise RuntimeError(f"b200_init failed with code {rc}")
    with_hp = GgmlFile(path)
    hp = with_hp.llama_hyperparameters()
    vocabulary = [t for t, _ in with_hp.vocabulary()]
    with_hp.close()
    err = C.c_int(0)
    if params.lora_adapters:
        paths = (C.c_char_p * len(params.lora_adapters))(*[p.encode() for p in params.lora_adapters])
        m = L.b200_llama_load_file_lora(path.encode(), params.context_size, params.rope_freq_base, params.rope_freq_scale, 1, paths,
                                        len(params.lora_adapters), C.byref(err))
    else:
        m = L.b200_llama_load_file(path.encode(), params.context_size, params.rope_freq_base, params.rope_freq_scale, C.byref(err))
    if not m:
        raise LoadError(err.value, f"load {path}")
    model = Llama.__new__(Llama)
    model.L, model.hyperparameters, model.params, model._m = L, hp, params, m
    model.vocabulary = vocabulary                                  # eot_token_id()
    return model
