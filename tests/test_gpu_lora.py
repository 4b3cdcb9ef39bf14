"""LoRA adapters on the GPU: the fused patch kernel (lora.cu) and the load hook, bit-identical to the reference's own ggml.c running
LoraAdapter::patch (oracle/ref_lora.c), and whole models loaded with adapters bit-identical to the reference graphs fed the reference-patched tensors."""
import ctypes as C

import numpy as np
import pytest

from oracle import bindings as B
from oracle import lora as Lo
from oracle import synth

pytestmark = pytest.mark.gpu

TARGETS = {"f32": B.F32, **B.QUANT_TYPES}


@pytest.fixture(scope="module")
def rl():
    if not Lo.have_ref():
        pytest.skip("oracle/_ref/libggml_lora.so not built (the reference's ggml running the LoRA patch graph)")
    return Lo.RefLora()


def bits(x):
    return np.ascontiguousarray(x).view(np.uint8).ravel()


def op_patch(wtype, w, K, N, a, b, scaling):
    from llm_b200 import _lib
    L = _lib.lib()
    assert L.b200_init(0) == 0
    out = np.array(w, copy=True)
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b, np.float32)
    rc = L.b200_op_lora_patch(wtype, out.ctypes.data_as(C.c_void_p), K, N, 1 if a.dtype == np.uint16 else 0, a.ctypes.data_as(C.c_void_p),
                              b.ctypes.data_as(C.c_void_p), a.shape[1], scaling)
    assert rc == 0, rc
    return out


def target(orc, wtype, K, N, rng):
    w = (rng.standard_normal((N, K)) * 0.1).astype(np.float32)
    return w if wtype == B.F32 else orc.quantize(wtype, w)


# ---- op level -----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", ["r", 3])
@pytest.mark.parametrize("r", [7, 8, 31, 32, 40, 64])
@pytest.mark.parametrize("a_f16", [False, True], ids=["A_f32", "A_f16"])
@pytest.mark.parametrize("tname", list(TARGETS))
def test_op_patch_matches_reference(orc, rl, tname, a_f16, r, alpha):
    wtype = TARGETS[tname]
    alpha = r if alpha == "r" else alpha
    rng = np.random.default_rng(1000 * r + wtype + 7 * a_f16)
    K, N = (96, 1) if wtype == B.F32 else (128, 37)      # 37 rows: three CTA tiles of 16, the last one partial
    w = target(orc, wtype, K, N, rng)
    a, b = Lo.factors(rng, K, N, r, a_f16)
    s = Lo.scaling(r, alpha)
    want = rl.patch(wtype, w, K, N, a, b, s)
    assert np.array_equal(bits(op_patch(wtype, w, K, N, a, b, s)), bits(want))


@pytest.mark.parametrize("tname", ["q4_0", "q8_0"])
def test_op_patch_4096_square(orc, rl, tname):
    wtype = TARGETS[tname]
    rng = np.random.default_rng(4096)
    K = N = 4096
    w = target(orc, wtype, K, N, rng)
    a, b = Lo.factors(rng, K, N, 16)
    s = Lo.scaling(16, 32)
    assert np.array_equal(bits(op_patch(wtype, w, K, N, a, b, s)), bits(rl.patch(wtype, w, K, N, a, b, s)))


def test_op_patch_f32_matrix_rows_not_a_tile_multiple(orc, rl):
    rng = np.random.default_rng(21)
    K, N, r = 200, 21, 35                                  # K not a multiple of 32 either (f32 targets have no blocks)
    w = target(orc, B.F32, K, N, rng)
    a, b = Lo.factors(rng, K, N, r, True)
    s = Lo.scaling(r, 5)
    assert np.array_equal(bits(op_patch(B.F32, w, K, N, a, b, s)), bits(rl.patch(B.F32, w, K, N, a, b, s)))


# ---- LLaMA from a file ------------------------------------------------------------------------------------------------------------------
LLAMA_TARGETS = ["layers.0.attention.wq.weight", "layers.1.attention.wv.weight", "layers.0.feed_forward.w1.weight", "output.weight",
                 "layers.1.attention_norm.weight"]


def kn(shape):
    return (shape[-1], shape[0] if len(shape) == 2 else 1)


def make_adapters(tmp_path, shapes, names, specs):
    """specs: [(file name, r, alpha, A as f16, extra GGLA tensors)] -> [(path, scaling, {target: (a, b)})]"""
    out = []
    for i, (fname, r, alpha, a_f16, extra) in enumerate(specs):
        rng = np.random.default_rng(0xA0 + i)
        table, fac = Lo.adapter_tensors({n: kn(shapes[n]) for n in names}, r, rng, a_f16)
        table.update(extra)
        path = str(tmp_path / fname)
        Lo.write_ggla(path, r, alpha, table)
        out.append((path, Lo.scaling(r, alpha), fac))
    return out


def ref_patched(rl, tens, shapes, wtype, adapters):
    out = dict(tens)
    for _, s, fac in adapters:
        for name, (a, b) in fac.items():
            K, N = kn(shapes[name])
            t = wtype if out[name].dtype == np.uint8 else B.F32
            out[name] = rl.patch(t, np.asarray(out[name]).reshape(N, -1), K, N, a, b, s).reshape(np.shape(tens[name]))
    return out


def llama_case(orc, tmp_path, wtype=B.Q4_1):
    from llm_b200 import loader
    hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], wtype, orc.quantize)
    shapes = synth.tensor_shapes(hp)
    path = str(tmp_path / "model.ggjt")
    loader.write_llama(path, hp, tens, shapes)
    unrelated = {"layers.7.attention.wq.weight.loraA": (0, (4, 256), np.zeros((256, 4), np.float32)),
                 "layers.7.attention.wq.weight.loraB": (0, (4, 256), np.zeros((256, 4), np.float32))}
    adapters = make_adapters(tmp_path, shapes, LLAMA_TARGETS, [("a1.ggla", 8, 16, False, unrelated), ("a2.ggla", 40, 3, True, {})])
    return hp, tens, shapes, path, adapters


def check_logits(g, c, what):
    assert np.array_equal(np.asarray(g, np.float32).view(np.uint32).ravel(), np.asarray(c, np.float32).view(np.uint32).ravel()), what


def test_llama_file_with_two_adapters(orc, ref, rl, tmp_path):
    import llm_b200
    from llm_b200 import loader
    hp, tens, shapes, path, adapters = llama_case(orc, tmp_path)
    params = lambda ad: llm_b200.ModelParameters(context_size=hp["n_ctx"], lora_adapters=[p for p, _, _ in ad])
    want = ref_patched(rl, tens, shapes, hp["wtype"], adapters)
    want_swapped = ref_patched(rl, tens, shapes, hp["wtype"], adapters[::-1])
    m = loader.load(path, params(adapters))
    for name in tens:
        assert np.array_equal(bits(m.read_tensor(name)), bits(want[name])), name
        if name not in LLAMA_TARGETS:
            assert np.array_equal(bits(want[name]), bits(tens[name])), name
    ms = loader.load(path, params(adapters[::-1]))
    assert all(np.array_equal(bits(ms.read_tensor(n)), bits(want_swapped[n])) for n in tens)
    assert any(not np.array_equal(bits(want[n]), bits(want_swapped[n])) for n in LLAMA_TARGETS)
    ms.close()

    # the per-tensor entry point gives the same weights
    mt = llm_b200.Llama(hp, params(adapters), tens)
    assert all(np.array_equal(bits(mt.read_tensor(n)), bits(want[n])) for n in tens)
    mt.close()

    cpu = ref.llama(hp, want, n_threads=8)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64))
    toks = synth.make_tokens(hp, 60)
    check_logits(s.evaluate(toks[:20], all_logits=True), cpu.eval(toks[:20]), "prefill 20")
    for i in range(20, 28):
        check_logits(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at {i}")
    check_logits(s.evaluate(toks[28:45], all_logits=True), cpu.eval(toks[28:45]), "batch of 17")
    check_logits(s.evaluate(toks[45:46], all_logits=True), cpu.eval(toks[45:46]), "decode after the batch")
    assert np.array_equal(s.kv(0), cpu.kv(0)) and np.array_equal(s.kv(1), cpu.kv(1))
    s.close(); m.close(); cpu.close()


def test_llama_loads_without_adapters_are_unchanged(orc, tmp_path):
    import llm_b200
    from llm_b200 import loader
    hp, tens, shapes, path, adapters = llama_case(orc, tmp_path, B.Q8_0)
    for lora in (None, []):
        m = loader.load(path, llm_b200.ModelParameters(context_size=hp["n_ctx"], lora_adapters=lora))
        assert all(np.array_equal(bits(m.read_tensor(n)), bits(tens[n])) for n in tens)
        m.close()
    # an adapter whose patch set names no tensor of the model changes nothing
    other = str(tmp_path / "other.ggla")
    Lo.write_ggla(other, 4, 4, {"layers.9.attention.wq.weight.loraA": (0, (4, 256), np.ones((256, 4), np.float32)),
                                "layers.9.attention.wq.weight.loraB": (0, (4, 256), np.ones((256, 4), np.float32))})
    m = loader.load(path, llm_b200.ModelParameters(context_size=hp["n_ctx"], lora_adapters=[other]))
    assert all(np.array_equal(bits(m.read_tensor(n)), bits(tens[n])) for n in tens)
    m.close()


# ---- errors ---------------------------------------------------------------------------------------------------------------------------------
def _load_err(path, hp, adapter):
    import llm_b200
    from llm_b200 import loader
    with pytest.raises(loader.LoadError) as e:
        loader.load(path, llm_b200.ModelParameters(context_size=hp["n_ctx"], lora_adapters=[adapter]))
    return e.value.kind


def test_adapter_errors(orc, tmp_path):
    hp, tens, shapes, path, _ = llama_case(orc, tmp_path, B.Q4_0)
    name = "layers.0.attention.wq.weight"
    rng = np.random.default_rng(3)
    a, b = Lo.factors(rng, 256, 256, 8)
    cases = {
        "UnknownTensor": {name + ".loraA": (0, (8, 256), a)},                                                        # no .loraB
        "TensorWrongSize": {name + ".loraA": (0, (8, 256), a), name + ".loraB": (0, (4, 256), b[:, :4].copy())},      # r of A != r of B
        "UnsupportedElementType": {name + ".loraA": (0, (8, 256), a), name + ".loraB": (1, (8, 256), b.astype(np.float16).view(np.uint16))},
    }
    for kind, table in cases.items():
        p = str(tmp_path / f"{kind}.ggla")
        Lo.write_ggla(p, 8, 8, table)
        assert _load_err(path, hp, p) == kind
    p = str(tmp_path / "rows.ggla")                                                                                   # B has the wrong number of rows
    Lo.write_ggla(p, 8, 8, {name + ".loraA": (0, (8, 256), a), name + ".loraB": (0, (8, 128), b[:128].copy())})
    assert _load_err(path, hp, p) == "TensorWrongSize"


def test_tensor_parallel_models_take_no_adapters(orc, tmp_path):
    from llm_b200 import _lib
    from llm_b200.session import LoraAdapters
    hp, tens, shapes, path, adapters = llama_case(orc, tmp_path, B.Q4_0)
    L = _lib.lib()
    assert L.b200_init(0) == 0
    h = _lib.LlamaHparams(**{k: hp[k] for k in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_rot", "n_ff")}, wtype=hp["wtype"],
                          context_size=hp["n_ctx"], rope_freq_base=10000.0, rope_freq_scale=1.0)
    m = L.b200_llama_new_tp(C.byref(h), 0, 2)
    assert m
    w = np.ascontiguousarray(tens["norm.weight"])
    with LoraAdapters(L, [adapters[0][0]]) as ad:
        assert L.b200_model_load_tensor_lora(m, b"norm.weight", 0, 1, w.size, 1, w.ctypes.data_as(C.c_void_p), w.nbytes, ad.handles, ad.n) == -2
    L.b200_model_free(m)


# ---- GPT-J (separate q_proj / k_proj / v_proj targets, rows of one fused matrix) --------------------------------------------------------------
def test_gptj_with_two_adapters(orc, rl, tmp_path):
    from oracle import gptj as J
    from llm_b200 import GptJ
    if not J.have_ref():
        pytest.skip("oracle/_ref/libggml_gptj.so not built")
    hp, tens = J.make_gptj(J.GPTJ_CONFIGS["gptj-hd64"], B.Q5_0, orc.quantize)
    shapes = J.gptj_tensor_shapes(hp)
    names = ["transformer.h.0.attn.q_proj.weight", "transformer.h.0.attn.k_proj.weight", "transformer.h.1.attn.v_proj.weight",
             "transformer.h.1.mlp.fc_in.weight", "transformer.h.0.ln_1.bias", "lm_head.bias"]
    adapters = make_adapters(tmp_path, shapes, names, [("j1.ggla", 16, 32, False, {}), ("j2.ggla", 33, 5, True, {})])
    want = ref_patched(rl, tens, shapes, hp["wtype"], adapters)
    cpu = J.RefGptJ(hp, want, n_threads=8, n_batch=64)
    m = GptJ(hp, tens, lora_adapters=[p for p, _, _ in adapters])
    s = m.start_session(64)
    toks = np.random.default_rng(0x10A).integers(0, hp["n_vocab"], size=48, dtype=np.int32)
    check_logits(s.evaluate(toks[:20], all_logits=True), cpu.eval(toks[:20]), "prefill 20")
    for i in range(20, 26):
        check_logits(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at {i}")
    check_logits(s.evaluate(toks[26:43], all_logits=True), cpu.eval(toks[26:43]), "batch of 17")
    assert np.array_equal(s.kv(0), cpu.kv(0)) and np.array_equal(s.kv(1), cpu.kv(1))
    s.close(); m.close(); cpu.close()
