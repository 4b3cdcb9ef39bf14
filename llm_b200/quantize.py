"""Model quantization over the C ABI (b200_quantize_file, include/llm_b200.h; csrc/quantize_file.cu): llm_base::quantize
(crates/llm-base/src/quantize.rs:139-414) for every native architecture -- an F16 / F32 model file to Q4_0 / Q4_1 / Q5_0 / Q5_1 / Q8_0, with the
quantization on the GPU and the output byte-identical with the reference's given the same tensor order (this one writes the source file's order).

  QuantizeProgress  crates/llm-base/src/quantize.rs:18-67    -> HyperparametersLoaded, TensorLoading, TensorQuantizing, TensorQuantized,
                                                                TensorSkipped, Finished
  QuantizeError     crates/llm-base/src/quantize.rs:69-121   -> QuantizeError.kind
  SaveContainerType crates/ggml/src/format/saver.rs:62-80    -> container "ggjt-v3" | "ggml"
Everything is checked before the destination is created, so a refused call leaves no file and reports no tensor events.
"""
import ctypes as C
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Tuple, Union

import numpy as np

from . import _lib
from .loader import ARCH, GgmlFile, LoadError

TARGETS = {"q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8}          # QuantizationTarget -> enum ggml_type
CONTAINERS = {"ggjt-v3": 0, "ggml": 1}
ERRORS = {-10: "Io", -13: "InvariantBroken", -14: "UnsupportedElementType", -16: "InvalidQuantizationTarget", -17: "VocabularyScoringNotSupported"}


class QuantizeError(Exception):
    """llm_base::QuantizeError: `kind` is the variant name ("Load" carries the LoadError in `load_error`)."""

    def __init__(self, kind: str, what: str, load_error: Optional[LoadError] = None, element_type: Optional[int] = None):
        self.kind, self.load_error, self.element_type = kind, load_error, element_type
        super().__init__(f"{what}: {kind}")


# ---- QuantizeProgress ----------------------------------------------------------------------------------------------------------------------
@dataclass
class HyperparametersLoaded:
    pass


@dataclass
class TensorLoading:
    name: str
    dims: Tuple[int, int]
    element_type: int
    n_elements: int


@dataclass
class TensorQuantizing:
    name: str


@dataclass
class TensorQuantized:
    name: str
    original_size: int
    reduced_size: int
    history: List[float] = field(default_factory=list)


@dataclass
class TensorSkipped:
    name: str
    size: int


@dataclass
class Finished:
    original_size: int
    reduced_size: int
    history: List[float] = field(default_factory=list)


def _history(hist, total) -> List[float]:
    """`hist as f32 / total as f32` for each bin, in f32 (0 / 0 is NaN, as in the reference)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return [float(v) for v in np.asarray(hist, np.int64).astype(np.float32) / np.float32(total)]


def _ggml_type(target: Union[int, str]) -> int:
    if isinstance(target, str):
        if target.lower() not in TARGETS:
            raise QuantizeError("InvalidQuantizationTarget", f"target {target!r}")
        return TARGETS[target.lower()]
    if int(target) not in TARGETS.values():
        raise QuantizeError("InvalidQuantizationTarget", f"target {target}", element_type=int(target))
    return int(target)


def quantize(source: str, destination: str, architecture: str, target: Union[int, str], container: str = "ggjt-v3",
             progress: Optional[Callable[[object], None]] = None) -> None:
    """llm_base::quantize::<M>(source -> destination): `architecture` one of "llama", "gpt2", "gptneox", "mpt", "bloom", "gptj"; `target` an
    enum ggml_type (2, 3, 6, 7, 8) or its name ("q4_0" ...); `progress` receives the QuantizeProgress events in the reference's order:
    HyperparametersLoaded, per tensor TensorLoading then TensorQuantizing + TensorQuantized or TensorSkipped, and Finished."""
    if architecture not in ARCH or architecture == "lora":
        raise ValueError(f"unknown architecture {architecture!r}: one of {', '.join(a for a in ARCH if a != 'lora')}")
    if container not in CONTAINERS:
        raise ValueError(f"unknown container {container!r}: one of {', '.join(CONTAINERS)}")
    ttype = _ggml_type(target)
    emit = progress or (lambda event: None)
    try:                                                             # ggml::format::load of the source: its errors are QuantizeError::Load
        GgmlFile(source, architecture).close()
    except LoadError as e:
        raise QuantizeError("Load", f"load {source}", load_error=e) from e
    emit(HyperparametersLoaded())

    failure = []

    def on_tensor(_user, rp):
        r = rp.contents
        if failure:
            return
        try:
            name = r.name.decode()
            emit(TensorLoading(name, (int(r.ne[0]), int(r.ne[1])), int(r.src_type), int(r.n_elements)))
            if r.dst_type != r.src_type:
                emit(TensorQuantizing(name))
                emit(TensorQuantized(name, int(r.original_size), int(r.reduced_size), _history(list(r.hist), r.n_elements)))
            else:
                emit(TensorSkipped(name, int(r.original_size)))
        except BaseException as e:                                   # re-raised once the C call returns
            failure.append(e)

    cb = _lib.QUANTIZE_CALLBACK(on_tensor)
    original, reduced, hist = C.c_int64(), C.c_int64(), (C.c_int64 * 16)()
    rc = _lib.lib().b200_quantize_file(source.encode(), destination.encode(), ARCH[architecture], ttype, CONTAINERS[container], cb, None,
                                       C.byref(original), C.byref(reduced), C.byref(hist))
    if rc == -2:
        raise ValueError(f"quantize {source} -> {destination}: the destination is the source file, or an argument is out of range")
    if rc != 0:
        raise QuantizeError(ERRORS.get(rc, str(rc)), f"quantize {source} -> {destination}")
    if failure:
        raise failure[0]
    emit(Finished(original.value, reduced.value, _history(list(hist), sum(hist))))
