"""The reference's model quantization restated in Python over the reference's own quantizers -- TEST INFRASTRUCTURE.

  quantize()        llm_base::quantize + QuantizeSaver::tensor_data   crates/llm-base/src/quantize.rs:139-414
                    ggml::format::save                                crates/ggml/src/format/saver.rs:86-160 (its own writer, both containers)
  ggml_quantize()   ggml_quantize_q{4_0,4_1,5_0,5_1,8_0}, called unmodified from oracle/_ref/libggml_ref.so (LC/ggml.c:18083-18208), with its
                    16-bin histogram
  write_file()      a GGJT v3 / GGML writer for source files: header words, vocabulary, tensor records
  model()           small F16 / F32 model files of each architecture (the loaders' tensor names)
Tensors are taken in the order given (the reference's HashMap order is not deterministic; the native quantizer keeps the source file's order).
"""
import ctypes as C
import os
import re
import struct

import numpy as np

from . import alibi, gptj, synth

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libggml_ref.so")

F32, F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0 = 0, 1, 2, 3, 6, 7, 8
TARGETS = (Q4_0, Q4_1, Q5_0, Q5_1, Q8_0)
BLOCK_BYTES = {Q4_0: 18, Q4_1: 20, Q5_0: 22, Q5_1: 24, Q8_0: 34}
LLAMA_FTYPE = {Q4_0: 2, Q4_1: 3, Q5_0: 8, Q5_1: 9, Q8_0: 7}                # FileTypeFormat::MostlyQ* (crates/llm-base/src/loader.rs:32-50)
ARCHS = ("llama", "gpt2", "gptneox", "mpt", "bloom", "gptj")
FILE_TYPE_WORD = {"llama": 6, "gpt2": 5, "gptneox": 7, "mpt": 7, "bloom": 5, "gptj": 6}      # the file_type word of each write_ggml
QUANTIZE_TENSORS = {a: [".*weight"] for a in ARCHS}                                        # KnownModel::quantize_tensors()
QUANTIZE_TENSORS["gpt2"] = ["model/wte", "model/lm_head", "model/h.*/attn/c_attn/w", "model/h.*/attn/c_proj/w", "model/h.*/mlp/c_fc/w",
                            "model/h.*/mlp/c_proj/w"]                                      # gpt2 lib.rs:357-369
MAGIC_GGJT, MAGIC_GGML = 0x67676A74, 0x67676D6C

_lib = None


def have_ref():
    return os.path.exists(LIB)


def _load():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        for t in ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0"):
            f = getattr(L, f"ggml_quantize_{t}")
            f.restype = C.c_size_t
            f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        _lib = L
    return _lib


class OracleQuantizeError(Exception):
    def __init__(self, kind):
        self.kind = kind
        super().__init__(kind)


def ggml_quantize(target, x, ne0):
    """ggml_quantize_<target>(src, dst, n_elements, ne0, hist) -> (bytes, hist int64[16]) -- what ggml::quantize_q* calls (crates/ggml/src/lib.rs:423-483)."""
    x = np.ascontiguousarray(x, np.float32).ravel()
    name = {Q4_0: "q4_0", Q4_1: "q4_1", Q5_0: "q5_0", Q5_1: "q5_1", Q8_0: "q8_0"}[target]
    out = np.zeros(x.size // 32 * BLOCK_BYTES[target], np.uint8)
    hist = np.zeros(16, np.int64)
    n = getattr(_load(), f"ggml_quantize_{name}")(x.ctypes.data, out.ctypes.data, x.size, ne0, hist.ctypes.data)
    assert n == out.size, (n, out.size)
    return out.tobytes(), hist


def selected(arch, name, n_dims):
    """QuantizeSaver::tensor_data's rule: 2-D, and some quantize_tensors() pattern matches anywhere in the name (Regex::is_match)"""
    return n_dims == 2 and any(re.search(p, name) for p in QUANTIZE_TENSORS[arch])


def _f32_history(hist, total):
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.asarray(hist, np.int64).astype(np.float32) / np.float32(total)


def write_file(words, vocabulary, tensors, container="ggjt-v3"):
    """ggml::format::save: the container's magic (+ version 3), the header words, the vocabulary (scores only in GGJT), then per tensor n_dims,
    name length, element type, dims, name, [GGJT: zeros to the next multiple of 32], data.  tensors: dicts name / n_dims / ne / type / data."""
    ggjt = container == "ggjt-v3"
    out = bytearray(struct.pack("<II", MAGIC_GGJT, 3) if ggjt else struct.pack("<I", MAGIC_GGML))
    out += struct.pack(f"<{len(words)}i", *words)
    for tok, score in vocabulary:
        out += struct.pack("<I", len(tok)) + tok
        if ggjt:
            out += struct.pack("<f", score)
    for t in tensors:
        name = t["name"].encode()
        out += struct.pack("<iiI", t["n_dims"], len(name), t["type"]) + struct.pack(f"<{t['n_dims']}i", *t["ne"][:t["n_dims"]]) + name
        if ggjt:
            out += bytes(-len(out) % 32)
        out += t["data"]
    return bytes(out)


def quantize(arch, words, vocabulary, tensors, target, container="ggjt-v3"):
    """llm_base::quantize::<arch> of a source with these header words, vocabulary and tensors (in this order).  Returns dict(file, events,
    reports, original_size, reduced_size, hist): events are tuples named after QuantizeProgress; reports the per-tensor fields of
    b200_quantize_report.  Raises OracleQuantizeError(kind) where the reference returns an error."""
    if target not in TARGETS:
        raise OracleQuantizeError("InvalidQuantizationTarget")
    if container == "ggml" and any(s != 0.0 for _, s in vocabulary):
        raise OracleQuantizeError("VocabularyScoringNotSupported")
    words = list(words)
    words[FILE_TYPE_WORD[arch]] = 2 * 1000 + LLAMA_FTYPE[target]              # quantization_version = QNT_VERSION, format = MostlyQ*
    events, reports, written = [("HyperparametersLoaded",)], [], []
    total_in = total_out = 0
    hist_all = np.zeros(16, np.int64)
    for t in tensors:
        ne0, ne1 = t["ne"]
        n_el = ne0 * ne1
        events.append(("TensorLoading", t["name"], (ne0, ne1), t["type"], n_el))
        q = selected(arch, t["name"], t["n_dims"])
        if q and t["type"] not in (F32, F16):
            raise OracleQuantizeError("UnsupportedElementType")
        total_in += len(t["data"])
        if q:
            events.append(("TensorQuantizing", t["name"]))
            x = np.frombuffer(t["data"], np.float16 if t["type"] == F16 else np.float32).astype(np.float32)     # half::f16::to_f32 is exact
            if ne0 % 32:
                raise OracleQuantizeError("InvariantBroken")                  # the reference's C assert
            data, hist = ggml_quantize(target, x, ne0)
            hist_all += hist
            events.append(("TensorQuantized", t["name"], len(t["data"]), len(data), _f32_history(hist, n_el)))
            out_type = target
            if target in (Q4_0, Q4_1) and ne0 % 64:
                raise OracleQuantizeError("InvariantBroken")                  # saver.rs:124-131
        else:
            events.append(("TensorSkipped", t["name"], len(t["data"])))
            data, hist, out_type = t["data"], np.zeros(16, np.int64), t["type"]
        total_out += len(data)
        reports.append(dict(name=t["name"], n_dims=t["n_dims"], src_type=t["type"], dst_type=out_type, ne=(ne0, ne1), n_elements=n_el,
                            original_size=len(t["data"]), reduced_size=len(data), hist=hist))
        written.append(dict(t, type=out_type, data=data))
    events.append(("Finished", total_in, total_out, _f32_history(hist_all, hist_all.sum())))
    return dict(file=write_file(words, vocabulary, written, container), events=events, reports=reports, original_size=total_in,
                reduced_size=total_out, hist=hist_all)


# ---- small source models --------------------------------------------------------------------------------------------------------------------
CONFIGS = {
    "llama": dict(n_vocab=320, n_embd=256, n_head=4, n_head_kv=4, n_layer=2, n_ff=768, n_rot=64, n_ctx=128),
    "llama-gqa": dict(n_vocab=352, n_embd=512, n_head=8, n_head_kv=2, n_layer=2, n_ff=1024, n_rot=64, n_ctx=128),
    "gpt2": dict(n_vocab=320, n_ctx=64, n_embd=128, n_head=4, n_layer=2),
    "gptneox": dict(n_vocab=384, n_ctx=64, n_embd=128, n_head=4, n_layer=2, n_rot=8, use_parallel_residual=1),
    "mpt": dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2, alibi_bias_max=8.0),
    "bloom": dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2),
    "gptj": dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2, n_rot=16),
}


def header_words(arch, hp, file_type):
    """the words of each architecture's write_ggml, in file order (MPT's alibi_bias_max and clip_kqv as f32 bits)"""
    f32 = lambda x: int(np.array([x], np.float32).view(np.int32)[0])
    v = hp["n_vocab"]
    return {"llama": lambda: [v, hp["n_embd"], 256, hp["n_head"], hp["n_layer"], hp["n_rot"], file_type],
            "gpt2": lambda: [v, hp["n_ctx"], hp["n_embd"], hp["n_head"], hp["n_layer"], file_type, v],
            "gptneox": lambda: [v, hp["n_ctx"], hp["n_embd"], hp["n_head"], hp["n_layer"], hp["n_rot"], hp["use_parallel_residual"], file_type],
            "mpt": lambda: [hp["n_embd"], hp["n_ctx"], hp["n_head"], hp["n_layer"], v, f32(hp["alibi_bias_max"]), f32(0.0), file_type],
            "bloom": lambda: [v, hp["n_embd"], 256, hp["n_head"], hp["n_layer"], file_type],
            "gptj": lambda: [v, hp["n_ctx"], hp["n_embd"], hp["n_head"], hp["n_layer"], hp["n_rot"], file_type, v]}[arch]()


def shapes(arch, hp, lm_head=False):
    return {"llama": synth.tensor_shapes, "gptneox": synth.neox_tensor_shapes, "mpt": alibi.mpt_tensor_shapes, "bloom": alibi.bloom_tensor_shapes,
            "gptj": gptj.gptj_tensor_shapes, "gpt2": lambda h: synth.gpt2_tensor_shapes(h, lm_head)}[arch](hp)


def vocabulary(n, scored=True):
    return [(b"t%d" % i if i % 7 else bytes([i % 256]) * (i % 5), (-0.25 * i) if scored else 0.0) for i in range(n)]


def tensor(name, x, src_type):
    """a tensor dict of the values x ([ne1, ne0] or [ne0]): 2-D tensors stored as src_type, 1-D as F32"""
    x = np.asarray(x, np.float32)
    t = src_type if x.ndim == 2 else F32
    data = (x.astype(np.float16) if t == F16 else x).tobytes()
    return dict(name=name, n_dims=x.ndim, ne=(x.shape[-1], x.shape[0] if x.ndim == 2 else 1), type=t, data=data)


def model(arch, cfg, src_type, seed=0x51A0, lm_head=False, scored=True):
    """(hp, header words, vocabulary, tensors) of a small model file: 2-D weights N(0, 1/K) stored as src_type, 1-D tensors 1 + 0.1 N(0, 1) in F32"""
    hp = CONFIGS[cfg]
    words = header_words(arch, hp, src_type)                      # file type: MostlyF32 (0) / MostlyF16 (1), quantization version 0
    out = []
    for idx, (name, shp) in enumerate(shapes(arch, hp, lm_head).items()):
        rng = np.random.default_rng(seed + idx)
        x = rng.standard_normal(shp) / np.sqrt(shp[-1]) if len(shp) == 2 else 1.0 + 0.1 * rng.standard_normal(shp)
        out.append(tensor(name, x, src_type))
    return hp, words, vocabulary(hp["n_vocab"], scored), out
