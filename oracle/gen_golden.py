"""Generate tests/golden/*.npz from the reference's OWN compiled ggml.c (oracle/_ref/libggml_ref.so).

TEST INFRASTRUCTURE. Run here (where /root/reference exists):  python -m oracle.gen_golden
The fixtures travel with the repo; nothing at test time reads /root/reference.

The reference holds no static golden tensors for this path (SURVEY.md §8c): its only KAT input is the
generator of LC/tests/test-quantize-fns.cpp:26-30 (x_i = 0.1 + 2 cos(i + offset), n = 4096), reused below;
everything else is produced by executing the reference on seeded inputs.

tests/golden/reference_pin.json holds one SHA-256 digest of the reference's outputs per larger pinning case of
tests/test_oracle_pin.py (the pin_* functions below, run on the reference here and on the plain-C oracle by the tests).
"""
import hashlib
import json
import os

import numpy as np

from . import bindings as B
from . import synth

OUT = os.path.join(os.path.dirname(B.HERE), "tests", "golden")

MICRO = dict(n_vocab=96, n_embd=128, n_head=4, n_head_kv=4, n_layer=2, n_ff=384, n_rot=32, n_ctx=64)


def synthetic_cos(n, offset):  # LC/tests/test-quantize-fns.cpp:26-30
    return (0.1 + 2.0 * np.cos(np.arange(n, dtype=np.float32) + np.float32(offset))).astype(np.float32)


def digest(outs):
    """bit patterns of one case's outputs (name -> array) in name order: floats as f32 bits, integers widened, names and shapes included"""
    h = hashlib.sha256()
    for k in sorted(outs):
        a = np.asarray(outs[k])
        a = a.astype(np.float32).view(np.uint32) if a.dtype.kind == "f" else a.astype(np.int64)
        h.update(k.encode() + repr(a.shape).encode() + np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:32]


def pin_fp16(to_half, to_float):
    """fp32 -> fp16 over a spread of magnitudes and the specials, fp16 -> fp32 over every finite half"""
    rng = np.random.default_rng(7)
    xs = np.concatenate([rng.standard_normal(4000).astype(np.float32) * s for s in (1e-8, 1e-6, 1e-4, 1, 300, 7e4)] +
                        [np.array([0, -0.0, 65504, 65519.9, 65520, 1e-7, 5.96e-8, 2.98e-8, 3e-8, np.inf, -np.inf], np.float32)])
    hs = [h for h in range(65536) if (h & 0x7c00) != 0x7c00]
    return {"fp16_from_f32": np.array([to_half(float(x)) for x in xs], np.int64),
            "fp16_to_f32": np.array([to_float(h) for h in hs], np.float32)}


def pin_rows(lib, name, t, K, **kw):
    rng = np.random.default_rng(K + t)
    w = (rng.standard_normal((16, K)) / np.sqrt(K)).astype(np.float32)
    x = (rng.standard_normal((3, K)) * rng.uniform(0.01, 30)).astype(np.float32)
    wq = lib.quantize(t, w)
    return {f"rows_{name}_{K}_wq": wq, f"rows_{name}_{K}_xq": lib.from_float(B.VEC_DOT_TYPE[t], x[0]), f"rows_{name}_{K}_mm": lib.mul_mat(t, wq, x, **kw)}


def pin_llama(lib, cfg, name, single_rows, **kw):
    """prefill 33 + decode 1 + batch 3 and both KV caches; then the first 8 tokens again from an empty cache (`single_rows(hp, tens, toks)`:
    the reference evaluates them one token at a time on one thread, the oracle as one batch -- the result must not depend on either)"""
    hp, tens = synth.make_llama(synth.CONFIGS[cfg], B.QUANT_TYPES[name], lib.quantize)
    toks = synth.make_tokens(hp, 37)
    m = lib.llama(hp, tens, **kw)
    p = f"llama_{cfg}_{name}_"
    out = {p + "prefill": m.eval(toks[:33]), p + "decode": m.eval(toks[33:34]), p + "batch": m.eval(toks[34:37]), p + "k": m.kv(0), p + "v": m.kv(1)}
    m.close()
    out[p + "rows8"] = single_rows(hp, tens, toks)
    return out


def pin_rope(lib, **kw):
    """RoPEOverrides then a rewind to position 12"""
    hp, tens = synth.make_llama(synth.CONFIGS["tiny"], B.Q4_0, lib.quantize)
    toks = synth.make_tokens(hp, 30)
    m = lib.llama(hp, tens, **kw)
    m.set_rope(26000.0, 0.5)
    out = {"rope_prefill": m.eval(toks[:20]), "rope_decode": m.eval(toks[20:21])}
    m.set_n_past(12)
    out["rope_rewound"] = m.eval(toks[12:15])
    m.close()
    return out


PIN_LLAMA = [("tiny", "q4_0"), ("tiny", "q4_1"), ("tiny", "q5_0"), ("small", "q5_1"), ("small", "q8_0")]


def reference_pin(ref):
    out = {"fp16": digest(pin_fp16(ref.lib.rh_fp32_to_fp16, ref.lib.rh_fp16_to_fp32))}
    for name, t in B.QUANT_TYPES.items():
        for K in (64, 4096, 11008):
            out[f"rows_{name}_{K}"] = digest(pin_rows(ref, name, t, K, n_threads=3))

    def single_rows(hp, tens, toks):
        m1 = ref.llama(hp, tens, n_threads=1, n_batch=64)
        rows = np.concatenate([m1.eval(toks[i:i + 1]) for i in range(8)])
        m1.close()
        return rows
    for cfg, name in PIN_LLAMA:
        out[f"llama_{cfg}_{name}"] = digest(pin_llama(ref, cfg, name, single_rows, n_threads=4, n_batch=64))
    out["rope"] = digest(pin_rope(ref, n_threads=3, n_batch=64))
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    ref = B.RefLib("ref")
    with open(os.path.join(OUT, "reference_pin.json"), "w") as f:
        json.dump(reference_pin(ref), f, indent=0, sort_keys=True)
    rng = np.random.default_rng(0xC0FFEE)
    g = {}
    # --- test-quantize-fns KAT: quantize both vectors, vec_dot (LC/tests/test-quantize-fns.cpp:95-113)
    n = 4096
    a, b = synthetic_cos(n, 0.0), synthetic_cos(n, 1.0)
    g["kat_a"], g["kat_b"] = a, b
    for name, t in B.QUANT_TYPES.items():
        vt = B.VEC_DOT_TYPE[t]
        wq = ref.quantize(t, a[None, :])
        xq = ref.from_float(vt, b)
        g[f"kat_{name}_wq"] = wq
        g[f"kat_{name}_xq"] = xq
        g[f"kat_{name}_dot"] = np.float32(ref.vec_dot(t, n, wq[0], xq))
        g[f"kat_{name}_deq"] = ref.to_float(t, wq[0], n)
    # --- seeded small matmuls, every format, ragged B
    K, N = 256, 24
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    x = (rng.standard_normal((5, K)) * 2.0).astype(np.float32)
    x[3, 32:64] = 0.0        # an all-zero activation block (id = 0 branch, LC/ggml.c:1242)
    x[4, :] *= 1e-3
    g["mm_w"], g["mm_x"] = w, x
    for name, t in B.QUANT_TYPES.items():
        wq = ref.quantize(t, w)
        g[f"mm_{name}_wq"] = wq
        g[f"mm_{name}_out"] = ref.mul_mat(t, wq, x)
    # --- row ops
    xr = (rng.standard_normal((6, 320)) * 3.0).astype(np.float32)
    g["row_x"] = xr
    g["rms_norm"] = ref.op(1, 0, None, xr, (320, 6, 1), fparams=(5e-6, 0), out_shape=(6, 320))
    g["norm"] = ref.op(2, 0, None, xr, (320, 6, 1), out_shape=(6, 320))
    xs = xr.copy()
    xs[1, 200:] = -np.inf
    g["softmax_x"] = xs
    g["softmax"] = ref.op(3, 0, None, xs, (320, 6, 1), out_shape=(6, 320))
    g["silu"] = ref.op(4, 0, None, xr, (320, 6, 1), out_shape=(6, 320))
    g["gelu"] = ref.op(5, 0, None, xr, (320, 6, 1), out_shape=(6, 320))
    allh = np.arange(65536, dtype=np.uint16).view(np.float16).astype(np.float32)
    allh = allh[np.isfinite(allh)]
    g["lut_in"] = allh
    g["lut_silu"] = ref.op(4, 0, None, allh, (allh.size, 1, 1), out_shape=(allh.size,))
    g["lut_gelu"] = ref.op(5, 0, None, allh, (allh.size, 1, 1), out_shape=(allh.size,))
    xk = rng.standard_normal((3, 5, 40)).astype(np.float32)
    g["chain_x"] = xk
    g["chain"] = ref.op(7, 0, None, xk, (40, 5, 3), iparams=(35, 0, 0, 0), fparams=(0.125, 0), out_shape=(3, 5, 40))
    for tag, (mode, nd, ne0, n_past) in {"llama": (0, 32, 32, 13), "llama511": (0, 128, 128, 511),
                                         "neox": (2, 24, 96, 7)}.items():
        xp = rng.standard_normal((4, 3, ne0)).astype(np.float32)
        g[f"rope_{tag}_x"] = xp
        g[f"rope_{tag}_p"] = np.array([n_past, nd, mode], np.int32)
        g[f"rope_{tag}"] = ref.op(6, 0, None, xp, (ne0, 3, 4), iparams=(n_past, nd, mode, 0), out_shape=(4, 3, ne0))
    np.savez_compressed(os.path.join(OUT, "ops.npz"), **g)

    # --- whole-model goldens: micro LLaMA, prefill 12 + decode 1 + decode-batch 2
    for name in ("q4_0", "q5_1"):
        t = B.QUANT_TYPES[name]
        hp, tens = synth.make_llama(MICRO, t, ref.quantize, seed=0x5EED0000)
        toks = synth.make_tokens(hp, 15)
        m = ref.llama(hp, tens, n_threads=2, n_batch=16)
        out = {"tokens": toks, "hp": np.array([hp[k] for k in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer",
                                                               "n_ff", "n_rot", "n_ctx", "wtype")], np.int32)}
        out["logits_prefill"] = m.eval(toks[:12])
        out["logits_decode"] = m.eval(toks[12:13])
        out["logits_tail"] = m.eval(toks[13:15])
        for k, v in tens.items():
            out["w:" + k] = v
        np.savez_compressed(os.path.join(OUT, f"llama_micro_{name}.npz"), **out)
        m.close()
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
