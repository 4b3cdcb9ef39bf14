"""llm_b200 -- H100-native quantized-inference backend behind the rustformers/llm accelerator seam.

The product is the C-ABI shared library llm_b200/libllm_b200.so (sources in llm_b200/csrc, headers in include/):
  * include/ggml_b200.h : the ggml_cuda_* seam the reference's ggml.c and crates/ggml call (drop-in boundary)
  * include/llm_b200.h  : native model/session runtime mirroring llm-base's InferenceSession / KnownModel for LLaMA
This Python package is only the host-side mirror of that interface over ctypes (tests, bench.py); it contains no
arithmetic and no fallback path.
"""
from .session import ContextFull, InferenceSession, InferenceSessionConfig, Llama, ModelKVMemoryType, ModelParameters, OutputRequest  # noqa: F401
from .session import (EndOfText, InferenceFeedback, InferenceParameters, InferenceRequest, InferenceStats, Rng, Sampler,  # noqa: F401
                      SamplerFailure)
from .session import InferenceSnapshot, MemorySizeMismatch, SnapshotError  # noqa: F401
from . import ggml  # noqa: F401

# enum ggml_type values of the five block formats on the hot path (LC/ggml.h:262-285)
Q4_0, Q4_1, Q5_0, Q5_1, Q8_0 = 2, 3, 6, 7, 8
F32, F16 = 0, 1
from . import loader  # noqa: F401
from .quantize import QuantizeError, quantize  # noqa: F401
from . import tp  # noqa: F401
from .neox import GptJ, NeoxSession  # noqa: F401
