"""LoRA adapters for tests -- TEST INFRASTRUCTURE.

  RefLora()            _ref/libggml_lora.so: LoraAdapter::patch (crates/llm-base/src/lora.rs:71-140) on the reference's own ggml (oracle/ref_lora.c)
  OracleLora()         liboracle_lora.so: the same patch restated in plain C (oracle/lora_oracle.c)
  write_ggla           a GGLA v1 adapter file (the container ggml::format::load reads with LoraParameters: r, alpha, no vocabulary)
  make_adapter         seeded A / B factors for a set of target tensors
"""
import ctypes as C
import os
import struct
import subprocess

import numpy as np

from .bindings import HERE, _p, row_bytes

MAGIC_GGLA = 0x67676C61
REF_LIB = os.path.join(HERE, "_ref", "libggml_lora.so")
ORACLE_LIB = os.path.join(HERE, "liboracle_lora.so")


def have_ref():
    return os.path.exists(REF_LIB)


def _patch_args(w, K, N, a, b):
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b, np.float32)
    out = np.array(w, copy=True)
    assert a.shape[0] == K and a.shape[1] == b.shape[1], (a.shape, b.shape, K)
    return out, a, b


class RefLora:
    """The reference's patch graph: W = W + scaling * (A x B) with ggml_mul_mat / ggml_scale / ggml_add, 8 threads."""

    def __init__(self):
        self.L = L = C.CDLL(REF_LIB)
        L.rl_patch.argtypes = [C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_float, C.c_int32]

    def patch(self, wtype, w, K, N, a, b, scaling):
        """w: N rows of the target in GGML layout (uint8 block rows, or f32 [N][K]); a: [K][r] f32 or uint16 (f16 bits); b: [NB][r] f32."""
        out, a, b = _patch_args(w, K, N, a, b)
        assert self.L.rl_patch(wtype, _p(out), K, N, 1 if a.dtype == np.uint16 else 0, _p(a), _p(b), a.shape[1], b.shape[0], scaling, 8) == 0
        return out


class OracleLora:
    """The plain-C restatement (builds without the reference sources)."""

    def __init__(self):
        if not os.path.exists(ORACLE_LIB):
            subprocess.check_call(["make", "-C", HERE, "-f", "lora.mk", "liboracle_lora.so"])
        self.L = L = C.CDLL(ORACLE_LIB)
        L.or_lora_patch.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_float]
        L.or_vec_dot_f32.restype = C.c_float
        L.or_vec_dot_f32.argtypes = [C.c_int64, C.c_void_p, C.c_void_p]

    def vec_dot_f32(self, x, y):
        x, y = np.ascontiguousarray(x, np.float32), np.ascontiguousarray(y, np.float32)
        return np.float32(self.L.or_vec_dot_f32(x.size, _p(x), _p(y)))

    def patch(self, wtype, w, K, N, a, b, scaling):
        out, a, b = _patch_args(w, K, N, a, b)
        self.L.or_lora_patch(wtype, _p(out), K, N, 1 if a.dtype == np.uint16 else 0, _p(a), _p(b), a.shape[1], b.shape[0], scaling)
        return out


def scaling(r, alpha):
    """LoraParameters::calculate_scaling: (f32)alpha / (f32)r"""
    return float(np.float32(alpha) / np.float32(r))


def factors(rng, K, N, r, a_f16=False, sigma=0.05):
    """A [K][r] (f32, or f16 bits) and B [N][r] f32 -- ggml shapes A [ne0 = r, ne1 = K], B [ne0 = r, ne1 = N]"""
    a = (rng.standard_normal((K, r)) * sigma).astype(np.float32)
    b = (rng.standard_normal((N, r)) * sigma).astype(np.float32)
    return (a.astype(np.float16).view(np.uint16) if a_f16 else a), b


def write_ggla(path, r, alpha, tensors):
    """GGLA v1: magic, version, r, alpha, then per tensor n_dims, name_len, type, dims (ne0 first), name, padding to 32 bytes, data.
    tensors: name -> (type, (ne0[, ne1]), bytes-like)"""
    with open(path, "wb") as f:
        f.write(struct.pack("<IIii", MAGIC_GGLA, 1, r, alpha))
        for name, (typ, ne, data) in tensors.items():
            nm = name.encode()
            data = np.ascontiguousarray(data).tobytes()
            f.write(struct.pack("<iiI", len(ne), len(nm), typ) + struct.pack(f"<{len(ne)}i", *ne) + nm)
            f.write(b"\0" * (-f.tell() % 32))
            f.write(data)


def adapter_tensors(targets, r, rng, a_f16=False, b_type=0):
    """targets: name -> (K, N).  Returns (GGLA tensor table, {name: (a, b)})"""
    table, fac = {}, {}
    for name, (K, N) in targets.items():
        a, b = factors(rng, K, N, r, a_f16)
        fac[name] = (a, b)
        table[name + ".loraA"] = (1 if a_f16 else 0, (r, K), a)
        bb = b.astype(np.float16).view(np.uint16) if b_type == 1 else b
        table[name + ".loraB"] = (b_type, (r, N), bb)
    return table, fac


def target_bytes(wtype, K, N):
    return N * row_bytes(wtype, K)
