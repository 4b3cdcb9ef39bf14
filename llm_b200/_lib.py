"""Loader of the C-ABI product library (llm_b200/libllm_b200.so).

There is no Python/NumPy/CPU implementation of anything in this package: if the CUDA library is missing or no CUDA device
is present, calls fail loudly (ImportError here, exit(1) inside the library -- the reference backend's error behaviour,
LC/ggml-cuda.cu:24-53)."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libllm_b200.so")

_lib = None


class LlamaHparams(C.Structure):
    """b200_llama_hparams (include/llm_b200.h) <- Hyperparameters, crates/models/llama/src/lib.rs:403-447."""
    _fields_ = [("n_vocab", C.c_int32), ("n_embd", C.c_int32), ("n_head", C.c_int32), ("n_head_kv", C.c_int32),
                ("n_layer", C.c_int32), ("n_rot", C.c_int32), ("n_ff", C.c_int32), ("wtype", C.c_int32),
                ("context_size", C.c_int32), ("rope_freq_base", C.c_float), ("rope_freq_scale", C.c_float)]


class TensorType(C.Structure):
    """b200_tensor_type: one 2-D weight's enum ggml_type (b200_llama_new_typed)"""
    _fields_ = [("name", C.c_char_p), ("type", C.c_int32)]


class GgmlTensorInfo(C.Structure):
    """b200_ggml_tensor_info <- TensorLoadInfo, crates/ggml/src/format/loader.rs:72-86."""
    _fields_ = [("name", C.c_char * 96), ("type", C.c_int32), ("n_dims", C.c_int32), ("ne", C.c_int64 * 2), ("offset", C.c_uint64), ("nbytes", C.c_uint64)]


class SessionConfig(C.Structure):
    """b200_session_config <- InferenceSessionConfig, crates/llm-base/src/inference_session.rs:799-841."""
    _fields_ = [("n_batch", C.c_int32), ("flags", C.c_int32)]


class SamplerParams(C.Structure):
    """b200_sampler (include/llm_b200.h) <- the default chain of crates/llm-base/src/samplers.rs:97-211, with the caller's seed and draw index."""
    _fields_ = [("repetition_penalty", C.c_float), ("repetition_last_n", C.c_int32), ("top_k", C.c_int32), ("top_p", C.c_float),
                ("temperature", C.c_float), ("seed", C.c_uint64), ("draw", C.c_uint64)]


class QuantizeReport(C.Structure):
    """b200_quantize_report (include/llm_b200.h): one tensor of b200_quantize_file, as written."""
    _fields_ = [("name", C.c_char * 96), ("n_dims", C.c_int32), ("src_type", C.c_int32), ("dst_type", C.c_int32), ("ne", C.c_int64 * 2),
                ("n_elements", C.c_int64), ("original_size", C.c_int64), ("reduced_size", C.c_int64), ("hist", C.c_int64 * 16)]


class Snapshot(C.Structure):
    """b200_snapshot (include/llm_b200.h) <- InferenceSnapshot, crates/llm-base/src/inference_session.rs:733-792."""
    _fields_ = [("npast", C.c_int64), ("memory_k_type", C.c_int32), ("memory_v_type", C.c_int32), ("n_batch", C.c_int64), ("n_threads", C.c_int64),
                ("n_tokens", C.c_int64), ("tokens", C.c_void_p), ("n_logits", C.c_int64), ("last_logits", C.c_void_p),
                ("memory_k_bytes", C.c_uint64), ("memory_v_bytes", C.c_uint64), ("memory_k", C.c_void_p), ("memory_v", C.c_void_p)]


QUANTIZE_CALLBACK = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(QuantizeReport))


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(nvcc, sm_90a). llm_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t
    L.b200_init.argtypes = [C.c_int]
    L.b200_device_info.argtypes = [C.POINTER(i32), C.POINTER(sz), C.POINTER(sz)]
    L.b200_stream.restype = vp
    L.b200_llama_new.restype = vp
    L.b200_llama_new.argtypes = [C.POINTER(LlamaHparams)]
    L.b200_llama_new_typed.restype = vp
    L.b200_llama_new_typed.argtypes = [C.POINTER(LlamaHparams), C.POINTER(TensorType), i32, C.POINTER(C.c_int)]
    L.b200_llama_new_tp.restype = vp
    L.b200_llama_new_tp.argtypes = [C.POINTER(LlamaHparams), i32, i32]
    L.b200_session_tp_handle.argtypes = [vp, vp]
    L.b200_session_tp_connect.argtypes = [vp, C.c_char_p]
    L.b200_session_tp_set_nowait.argtypes = [vp, i32]
    L.b200_session_tp_timeouts.restype = i32
    L.b200_session_tp_timeouts.argtypes = [vp]
    L.b200_model_load_tensor.argtypes = [vp, C.c_char_p, i32, vp, sz]
    L.b200_model_synthesize.argtypes = [vp, C.c_uint64]
    L.b200_model_read_tensor.argtypes = [vp, C.c_char_p, vp, sz]
    L.b200_model_tensor_nbytes.restype = sz
    L.b200_model_tensor_nbytes.argtypes = [vp, C.c_char_p]
    L.b200_model_weight_bytes.restype = sz
    L.b200_model_weight_bytes.argtypes = [vp]
    L.b200_model_free.argtypes = [vp]
    L.b200_model_start_session.restype = vp
    L.b200_model_start_session.argtypes = [vp, C.POINTER(SessionConfig)]
    L.b200_session_evaluate.argtypes = [vp, vp, i32, vp, i32]
    L.b200_session_feed_prompt.argtypes = [vp, vp, i32, vp]
    L.b200_session_evaluate_output.argtypes = [vp, vp, i32, vp, i32, vp]
    L.b200_session_feed_prompt_output.argtypes = [vp, vp, i32, vp, vp]
    L.b200_session_perplexity.argtypes = [vp, vp, i64, i32, vp, vp, C.POINTER(i32)]
    L.b200_op_nll_rows.argtypes = [vp, i64, i64, vp, vp]
    L.b200_session_top_k.argtypes = [vp, i32, vp, vp]
    L.b200_session_infer_next_token.argtypes = [vp, C.POINTER(SamplerParams), C.POINTER(i32)]
    L.b200_session_read_tokens.restype = i32
    L.b200_session_read_tokens.argtypes = [vp, vp, i32]
    L.b200_session_last_logits.argtypes = [vp, vp]
    L.b200_op_sample.argtypes = [vp, i64, vp, i32, C.POINTER(SamplerParams), C.POINTER(i32), C.POINTER(i32), vp, vp]
    L.b200_session_evaluate_device.argtypes = [vp, vp, i32]
    L.b200_session_device_logits.restype = vp
    L.b200_session_device_logits.argtypes = [vp]
    L.b200_session_n_past.argtypes = [vp]
    L.b200_session_set_n_past.argtypes = [vp, i32]
    L.b200_session_read_kv.argtypes = [vp, i32, vp, sz]
    L.b200_session_sync.argtypes = [vp]
    L.b200_session_decode_timeline.argtypes = [vp, vp, C.c_int, C.c_int]
    L.b200_session_set_tap.argtypes = [vp, i32, i32]
    L.b200_session_read_tap.restype = i64
    L.b200_session_read_tap.argtypes = [vp, vp, i64]
    L.b200_session_last_launches.argtypes = [vp]
    L.b200_session_free.argtypes = [vp]
    L.b200_timing_begin.argtypes = []
    L.b200_timing_end_ms.restype = C.c_float
    L.b200_session_probe_matvec.restype = C.c_float
    L.b200_session_probe_matvec.argtypes = [vp, i32, C.POINTER(i64), C.POINTER(C.c_double)]
    L.b200_model_is_loaded.argtypes = [vp]
    L.b200_ggml_open.restype = vp
    L.b200_ggml_open.argtypes = [C.c_char_p, C.POINTER(C.c_int)]
    L.b200_ggml_open_arch.restype = vp
    L.b200_ggml_open_arch.argtypes = [C.c_char_p, i32, C.POINTER(C.c_int)]
    L.b200_ggml_hparams.argtypes = [vp, C.POINTER(i32), C.POINTER(i32 * 8), C.POINTER(i32)]
    L.b200_ggml_write.argtypes = [C.c_char_p, C.POINTER(i32), i32, i32, vp, vp, vp, C.POINTER(GgmlTensorInfo), vp, i64]
    L.b200_ggml_close.argtypes = [vp]
    L.b200_ggml_container.argtypes = [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.b200_ggml_n_tensors.restype = i64
    L.b200_ggml_n_tensors.argtypes = [vp]
    L.b200_ggml_tensor.argtypes = [vp, i64, C.POINTER(GgmlTensorInfo)]
    L.b200_ggml_tensor_data.restype = vp
    L.b200_ggml_tensor_data.argtypes = [vp, i64]
    L.b200_ggml_n_vocab.restype = i64
    L.b200_ggml_n_vocab.argtypes = [vp]
    L.b200_ggml_token.argtypes = [vp, i64, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_uint32), C.POINTER(C.c_float)]
    L.b200_ggml_llama_hparams.argtypes = [vp, C.POINTER(LlamaHparams), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.b200_ggml_write_llama.argtypes = [C.c_char_p, C.POINTER(LlamaHparams), i32, i32, vp, vp, vp, C.POINTER(GgmlTensorInfo), vp, i64]
    L.b200_llama_load_file.restype = vp
    L.b200_llama_load_file.argtypes = [C.c_char_p, i32, C.c_float, C.c_float, C.POINTER(C.c_int)]
    L.b200_op_quantize_act.argtypes = [i32, vp, i64, i64, vp, vp, vp]
    L.b200_op_quantize_weights.argtypes = [i32, vp, i64, i64, vp]
    L.b200_op_quantize_blocks_device.argtypes = [i32, i32, vp, i64, vp, vp]
    L.b200_op_mul_mat.argtypes = [i32, vp, i64, i64, vp, i64, vp, i32]
    L.b200_op_mul_mat_kv.argtypes = [i32, vp, i64, i64, i64, i64, i64, vp, i64, i64, i64, i64, vp, i64, i64, i32]
    L.b200_op_quantize_q8_K.argtypes = [vp, i64, i64, vp]
    L.b200_op_lora_patch.argtypes = [i32, vp, i64, i64, i32, vp, vp, i64, C.c_float]
    L.b200_model_load_tensor_lora.argtypes = [vp, C.c_char_p, i32, i32, i64, i64, vp, sz, C.POINTER(vp), i32]
    L.b200_llama_load_file_lora.restype = vp
    L.b200_llama_load_file_lora.argtypes = [C.c_char_p, i32, C.c_float, C.c_float, i32, C.POINTER(C.c_char_p), i32, C.POINTER(C.c_int)]
    L.b200_quantize_file.argtypes = [C.c_char_p, C.c_char_p, i32, i32, i32, QUANTIZE_CALLBACK, vp, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64 * 16)]
    L.b200_session_get_snapshot.argtypes = [vp, C.POINTER(Snapshot)]
    L.b200_session_write_snapshot.argtypes = [vp, C.c_char_p]
    L.b200_model_session_from_snapshot.restype = vp
    L.b200_model_session_from_snapshot.argtypes = [vp, C.POINTER(Snapshot), i32, C.POINTER(C.c_int)]
    L.b200_model_session_read_snapshot.restype = vp
    L.b200_model_session_read_snapshot.argtypes = [vp, C.c_char_p, i32, C.POINTER(C.c_int)]
    L.b200_snapshot_read_header.argtypes = [C.c_char_p, C.POINTER(Snapshot)]
    L.b200_op_transpose_device.argtypes = [i32, vp, i64, vp, i64, i64, i64]
    L.b200_op_norm_device.argtypes = [i32, vp, vp, i64, i64, C.c_float]
    _lib = L
    return L
