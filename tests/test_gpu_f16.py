"""F16 model files on the GPU (exact_f16.cu: the streaming F16 mat-vec and the ordered-FMA GEMM), bit-identical to the reference's own ggml.c
on the CPU: the op against ggml_mul_mat with an F16 weight, LLaMA files loaded through the loader, the GPT-NeoX family, LoRA on F16 targets,
and the refusals (tensor parallelism, B200_SESSION_FAST)."""
import ctypes as C

import numpy as np
import pytest

from oracle import bindings as B
from oracle import synth

pytestmark = pytest.mark.gpu

F16 = B.F16


def f16(t, w):
    """the `quantize` of the synth helpers for F16 weights: the file's halves (numpy rounds to nearest even, as ggml_fp32_to_fp16)"""
    return np.ascontiguousarray(w, np.float32).astype(np.float16)


def check(g, c, what):
    c = np.asarray(c, np.float32).reshape(np.shape(g))
    g = np.asarray(g, np.float32)
    assert np.array_equal(g.view(np.uint32), c.view(np.uint32)), (what, float(np.abs(g - c).max() / max(np.abs(c).max(), 1e-30)), int((g != c).sum()), g.size)


def lib():
    from llm_b200 import _lib
    L = _lib.lib()
    assert L.b200_init(0) == 0
    return L


def op_mul_mat(w16, x, impl):
    L = lib()
    N, K = w16.shape
    Bn = x.shape[0]
    out = np.empty((Bn, N), np.float32)
    w16, x = np.ascontiguousarray(w16), np.ascontiguousarray(x, np.float32)
    rc = L.b200_op_mul_mat(F16, w16.ctypes.data_as(C.c_void_p), K, N, x.ctypes.data_as(C.c_void_p), Bn, out.ctypes.data_as(C.c_void_p), impl)
    assert rc == 0, rc
    return out


def edge_operands(rng, K, N, Bn):
    """weights and activations on the edges of fp16: activations exactly halfway between two halves (the rounding ties), values that become
    fp16 subnormals, and values that round to +-inf, paired with weights that keep every chain free of inf * 0 and inf - inf."""
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    x = rng.standard_normal((Bn, K)).astype(np.float32)
    h = x.astype(np.float16)
    up = np.nextafter(h, np.float16(np.inf))
    tie = ((h.astype(np.float32) + up.astype(np.float32)) * 0.5).astype(np.float32)         # exact in f32
    m = rng.random((Bn, K)) < 0.25
    x[m] = tie[m]
    sub = rng.random((Bn, K)) < 0.05
    x[sub] = (rng.standard_normal(int(sub.sum())) * 3e-6).astype(np.float32)               # fp16 subnormals (< 6.1e-5)
    w16 = w.astype(np.float16)
    w16[:, 1::7] = (rng.standard_normal((N, len(range(1, K, 7)))) * 2e-5).astype(np.float16)  # subnormal weights too
    if Bn > 1:                                          # row 1: one overflowing activation in chain 3 and none elsewhere; its weights nonzero
        x[1, 3] = 70000.0
        w16[:, 3] = np.where(w16[:, 3] == 0, np.float16(0.5), w16[:, 3])
    return w16, x


SHAPES = [(64, 33), (4096, 4096), (11008, 4096), (4096, 11008), (5120, 13824)]
BATCHES = [1, 2, 7, 15, 16, 95, 96, 97, 512]


@pytest.mark.parametrize("K,N", SHAPES)
def test_op_mul_mat_matches_reference(ref, K, N):
    rng = np.random.default_rng(K * 7 + N)
    bmax = max(BATCHES) if K * N <= 4096 * 4096 else 97
    w16, x = edge_operands(rng, K, N, bmax)
    for Bn in BATCHES:
        if Bn > bmax:
            continue
        want = ref.mul_mat(F16, w16.view(np.uint16), x[:Bn], n_threads=16)
        for impl in (0, 4):                              # B200_MM_AUTO (exact_f16.cu), B200_MM_EXACT (mul_mat_f16_exact)
            got = op_mul_mat(w16, x[:Bn], impl)
            fin = np.isfinite(want)
            assert np.array_equal(np.isfinite(got), fin), (K, N, Bn, impl)
            check(got[fin], want[fin], f"K={K} N={N} B={Bn} impl={impl}")


@pytest.mark.slow
@pytest.mark.parametrize("K,N", [(4096, 4096), (11008, 4096)])
def test_op_mul_mat_512_tokens_7b_shapes(ref, K, N):
    rng = np.random.default_rng(K + N)
    w16, x = edge_operands(rng, K, N, 512)
    want = ref.mul_mat(F16, w16.view(np.uint16), x, n_threads=32)
    got = op_mul_mat(w16, x, 0)
    fin = np.isfinite(want)
    check(got[fin], want[fin], "512 tokens")


def test_op_rejects_other_impls():
    L = lib()
    w = np.zeros((8, 64), np.float16)
    x = np.zeros((1, 64), np.float32)
    out = np.empty((1, 8), np.float32)
    for impl in (1, 2, 3, 5, 6, 7, 8):
        assert L.b200_op_mul_mat(F16, w.ctypes.data_as(C.c_void_p), 64, 8, x.ctypes.data_as(C.c_void_p), 1, out.ctypes.data_as(C.c_void_p), impl) == -2
    assert L.b200_op_mul_mat(F16, w.ctypes.data_as(C.c_void_p), 32, 16, x.ctypes.data_as(C.c_void_p), 1, out.ctypes.data_as(C.c_void_p), 0) == -2   # K % 64


# ---- LLaMA --------------------------------------------------------------------------------------------------------------------------------
def llama_launches(hp):
    """the per-op schedule of one token: get_rows, 17 launches per layer, the final norm and the lm_head (2)"""
    return 17 * hp["n_layer"] + 4


def write_f16_llama(tmp_path, cfg, name):
    from llm_b200.loader import write_llama
    hp, tens = synth.make_llama(synth.CONFIGS[cfg], F16, f16)
    path = str(tmp_path / f"{name}.bin")
    write_llama(path, hp, tens, synth.tensor_shapes(hp))
    return hp, tens, path


@pytest.mark.parametrize("cfg", ["tiny8", "gqa8"])
def test_llama_file_matches_reference(ref, tmp_path, cfg):
    import llm_b200
    from llm_b200.loader import load
    hp, tens, path = write_f16_llama(tmp_path, cfg, cfg)
    mr = ref.llama(hp, tens, n_threads=8)
    params = llm_b200.ModelParameters(context_size=hp["n_ctx"])
    # a GGJT header has no n_head_kv (LLaMA-2 70B's n_gqa is a load parameter): the grouped-query model takes its tensors directly
    m = load(path, params) if hp["n_head_kv"] == hp["n_head"] else llm_b200.Llama(hp, params, tens)
    assert m.hyperparameters["wtype"] == F16
    for name in ("layers.0.attention.wk.weight", "layers.1.feed_forward.w3.weight", "output.weight"):
        assert np.array_equal(m.read_tensor(name), tens[name].view(np.uint8).ravel()), name
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64))
    toks = synth.make_tokens(hp, 80)
    check(s.evaluate(toks[:21], all_logits=True), mr.eval(toks[:21]), "prefill 21")
    for i in range(21, 29):
        check(s.evaluate(toks[i:i + 1], all_logits=True), mr.eval(toks[i:i + 1]), f"decode {i}")
        assert s.last_launches == llama_launches(hp), s.last_launches
    check(s.evaluate(toks[29:34], all_logits=True), mr.eval(toks[29:34]), "batch of 5")
    check(s.evaluate(toks[34:50]), mr.eval(toks[34:50])[-1], "last row only")
    s.rewind(40); mr.set_n_past(40)
    check(s.evaluate(toks[50:53], all_logits=True), mr.eval(toks[50:53]), "re-feed after rewind")
    check(s.evaluate(toks[53:54], all_logits=True), mr.eval(toks[53:54]), "decode after rewind")
    for which in (0, 1):        # the CPU model sizes its cache by n_embd; with GQA only the first n_layer * n_ctx * n_embd_gqa values are used
        a = s.kv(which)
        assert np.array_equal(a, mr.kv(which)[:a.size]), which
    s.close(); m.close(); mr.close()


def test_llama_long_context(ref, tmp_path):
    """decode across positions 3072 / 3264 (the fused attention's limits) up to the last slot of a 4096 context, per op"""
    import llm_b200
    from llm_b200.loader import load, write_llama
    hp, tens = synth.make_llama(dict(synth.CONFIGS["tiny8"], n_layer=1, n_ctx=4096), F16, f16)
    path = str(tmp_path / "long.bin")
    write_llama(path, hp, tens, synth.tensor_shapes(hp))
    mr = ref.llama(hp, tens, n_threads=16, n_batch=512)
    m = load(path, llm_b200.ModelParameters(context_size=4096))
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=512))
    toks = synth.make_tokens(hp, 4096)

    def feed(to):                                       # both sides to n_past `to`, in chunks of 512
        while s.n_past < to:
            p = s.n_past
            c = min(512, to - p)
            s.evaluate(toks[p:p + c]); mr.eval(toks[p:p + c])

    for i in list(range(3068, 3076)) + list(range(3260, 3268)) + [4095]:
        feed(i)
        check(s.evaluate(toks[i:i + 1], all_logits=True), mr.eval(toks[i:i + 1]), f"decode at n_past {i}")
    assert s.n_past == 4096
    assert np.array_equal(s.kv(0), mr.kv(0)) and np.array_equal(s.kv(1), mr.kv(1))
    s.close(); m.close(); mr.close()


@pytest.mark.slow
def test_llama_7b_layers(ref):
    """LLaMA-7B layer geometry, two layers: prefill of 512 tokens (the GEMM on 4096 x 12288 / 4096 / 22016 and 11008 x 4096) and decode at n_past 512"""
    import llm_b200
    hp, tens = synth.make_llama(dict(synth.CONFIGS["7b-2l"], n_ctx=1024), F16, f16)
    mr = ref.llama(hp, tens, n_threads=32, n_batch=512)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=1024), tens)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=512))
    toks = synth.make_tokens(hp, 520)
    check(s.evaluate(toks[:512]), mr.eval(toks[:512])[-1], "prefill 512")
    for i in range(512, 514):
        check(s.evaluate(toks[i:i + 1]), mr.eval(toks[i:i + 1])[-1], f"decode {i}")
    s.close(); m.close(); mr.close()


def test_llama_synthesized_reads_back_as_fp16(ref):
    """a device-synthesised F16 model holds fp16 values; read back and given to the reference, both compute the same logits"""
    import llm_b200
    hp = dict(synth.CONFIGS["tiny8"], wtype=F16)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]))
    m.synthesize(0x5EED)
    tens = {}
    for name, shp in synth.tensor_shapes(hp).items():
        a = m.read_tensor(name)
        tens[name] = a if len(shp) == 1 else a.view(np.float16).reshape(shp)
    w = tens["layers.0.attention.wq.weight"].astype(np.float32)
    assert np.isfinite(w).all() and 0.5 < float(w.std() * np.sqrt(hp["n_embd"])) < 2.0
    mr = ref.llama(hp, tens, n_threads=8)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=32))
    toks = synth.make_tokens(hp, 24)
    check(s.evaluate(toks[:20], all_logits=True), mr.eval(toks[:20]), "prefill")
    check(s.evaluate(toks[20:21], all_logits=True), mr.eval(toks[20:21]), "decode")
    s.close(); m.close(); mr.close()


def test_llama_refusals(tmp_path):
    import llm_b200
    from llm_b200 import _lib
    L = lib()
    hp = dict(synth.CONFIGS["tiny8"], wtype=F16)
    h = _lib.LlamaHparams(**{k: int(hp[k]) for k in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_rot", "n_ff")}, wtype=F16, context_size=128)
    assert not L.b200_llama_new_tp(C.byref(h), 0, 2), "tensor-parallel shards need the fused schedule"
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=128))
    m.synthesize()
    cfg = _lib.SessionConfig(n_batch=8, flags=4)                     # B200_SESSION_FAST
    assert not L.b200_model_start_session(m._m, C.byref(cfg))
    m.close()


def test_llama_mixed_and_f32_files_refused(orc, tmp_path):
    from llm_b200.loader import LoadError, load, write_llama
    hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], F16, f16)
    shapes = synth.tensor_shapes(hp)
    path = str(tmp_path / "f16.bin")
    write_llama(path, hp, tens, shapes)
    load(path).close()
    t32 = {k: v.astype(np.float32) for k, v in tens.items()}
    write_llama(str(tmp_path / "f32.bin"), dict(hp, wtype=B.F32), t32, shapes)
    with pytest.raises(LoadError) as e:
        load(str(tmp_path / "f32.bin"))
    assert e.value.code == -14                           # UnsupportedElementType
    # one quantized matrix in an F16 file: the writer types every non-f32 array as the model's type, so the Q8_0 tensor goes in as a second file
    # written with wtype Q8_0 whose wq is F16 is not expressible here; instead a Q8_0 model with one F16 matrix
    q8 = {k: (v if v.dtype == np.float32 else orc.quantize(B.Q8_0, v.astype(np.float32))) for k, v in tens.items()}
    mixed = dict(q8, **{"layers.1.attention.wo.weight": tens["layers.1.attention.wo.weight"]})
    from llm_b200 import _lib
    L = _lib.lib()
    infos = (_lib.GgmlTensorInfo * len(mixed))()
    datas = (C.c_void_p * len(mixed))()
    keep = []
    for i, (name, a) in enumerate(mixed.items()):
        a = np.ascontiguousarray(a); keep.append(a)
        shp = shapes[name]
        infos[i].name = name.encode()
        infos[i].type = 0 if a.dtype == np.float32 else F16 if a.dtype == np.float16 else B.Q8_0
        infos[i].n_dims = len(shp)
        infos[i].ne[0] = shp[-1]
        infos[i].ne[1] = shp[0] if len(shp) == 2 else 1
        infos[i].nbytes = a.nbytes
        datas[i] = a.ctypes.data
    h = _lib.LlamaHparams(**{k: int(hp[k]) for k in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_rot", "n_ff")}, wtype=B.Q8_0)
    mpath = str(tmp_path / "mixed.bin")
    assert L.b200_ggml_write_llama(mpath.encode(), C.byref(h), 256, 2007, None, None, None, infos, datas, len(mixed)) == 0
    with pytest.raises(LoadError) as e:
        load(mpath)
    assert e.value.code == -14


def test_lora_wrong_loraB_rows_on_f16_target(tmp_path):
    """a loraB whose row count is not the F16 target's: TensorWrongSize (the reference asserts in ggml_add)"""
    import llm_b200
    from oracle import lora as Lo
    hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], F16, f16)
    rng = np.random.default_rng(5)
    e = hp["n_embd"]
    a, b = Lo.factors(rng, e, e + 32, 8)
    path = str(tmp_path / "bad.ggla")
    Lo.write_ggla(path, 8, 8, {"layers.0.attention.wo.weight.loraA": (0, (8, e), a), "layers.0.attention.wo.weight.loraB": (0, (8, e + 32), b)})
    from llm_b200.loader import LoadError
    with pytest.raises(LoadError) as err:
        llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"], lora_adapters=[path]), tens)
    assert err.value.code == -4


# ---- the GPT-NeoX family ------------------------------------------------------------------------------------------------------------------
def run_neox_like(s, mr, toks):
    check(s.evaluate(toks[:20], all_logits=True), mr.eval(toks[:20]), "prefill 20")
    for i in range(20, 26):
        check(s.evaluate(toks[i:i + 1], all_logits=True), mr.eval(toks[i:i + 1]), f"decode {i}")
    check(s.evaluate(toks[26:43], all_logits=True), mr.eval(toks[26:43]), "batch 17 after decode")
    check(s.evaluate(toks[43:44], all_logits=True), mr.eval(toks[43:44]), "decode after batch")


def ref_or_skip():
    if not B.have_ref("ref"):
        pytest.skip("oracle/_ref/libggml_ref.so not built")


@pytest.mark.parametrize("cfg", ["par", "seq"])
def test_neox_f16(cfg):
    from llm_b200.neox import GptNeoX
    ref_or_skip()
    c = {"par": dict(n_vocab=384, n_ctx=128, n_embd=256, n_head=4, n_layer=2, n_rot=16, use_parallel_residual=1),
         "seq": dict(n_vocab=384, n_ctx=128, n_embd=256, n_head=8, n_layer=2, n_rot=32, use_parallel_residual=0)}[cfg]
    hp, tens = synth.make_neox(c, F16, f16)
    mr = B.RefLib("ref").neox(hp, tens, n_threads=8, n_batch=64)
    m = GptNeoX(hp, tens)
    s = m.start_session(64)
    run_neox_like(s, mr, synth.make_tokens(hp, 60))
    assert np.array_equal(s.kv(0), mr.kv(0)), "K"
    s.close(); m.close(); mr.close()


@pytest.mark.parametrize("lm_head", [False, True])
def test_gpt2_f16_with_f16_wpe(lm_head):
    from llm_b200.neox import Gpt2
    ref_or_skip()
    hp, tens = synth.make_gpt2(dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2), F16, f16, lm_head=lm_head)
    wpe16 = tens["model/wpe"].astype(np.float16)
    ref_tens = dict(tens, **{"model/wpe": wpe16.astype(np.float32)})   # the reference's F16 get_rows widens exactly
    mr = B.RefLib("ref").gpt2(hp, ref_tens, n_threads=8, n_batch=64)
    m = Gpt2(hp, dict(tens, **{"model/wpe": wpe16}))
    s = m.start_session(64)
    run_neox_like(s, mr, synth.make_tokens(hp, 60))
    s.close(); m.close(); mr.close()


def test_mpt_bloom_f16():
    from oracle import alibi as A
    from llm_b200.neox import Bloom, Mpt
    if not A.have_ref():
        pytest.skip("oracle/_ref/libggml_alibi.so not built")
    for arch, cls, make, cfg in ((A.MPT, Mpt, A.make_mpt, "mpt-tiny"), (A.BLOOM, Bloom, A.make_bloom, "bloom-tiny")):
        hp, tens = make(A.MPT_CONFIGS[cfg] if arch == A.MPT else A.BLOOM_CONFIGS[cfg], F16, f16)
        cpu = A.RefAlibi(hp, tens, arch, n_threads=8, n_batch=512)
        m = cls(hp, tens)
        s = m.start_session(512)
        run_neox_like(s, cpu, np.random.default_rng(0xA11B1).integers(0, hp["n_vocab"], size=64, dtype=np.int32))
        assert np.array_equal(s.kv(0), cpu.kv(0)), "K"
        s.close(); m.close(); cpu.close()


def test_gptj_f16():
    from oracle import gptj as J
    from llm_b200 import GptJ
    if not J.have_ref():
        pytest.skip("oracle/_ref/libggml_gptj.so not built")
    hp, tens = J.make_gptj(J.GPTJ_CONFIGS["gptj-tiny"], F16, f16)
    cpu = J.RefGptJ(hp, tens, n_threads=8, n_batch=512)
    m = GptJ(hp, tens)
    s = m.start_session(512)
    run_neox_like(s, cpu, np.random.default_rng(0x6D71).integers(0, hp["n_vocab"], size=64, dtype=np.int32))
    assert np.array_equal(s.kv(0), cpu.kv(0)) and np.array_equal(s.kv(1), cpu.kv(1))
    s.close(); m.close(); cpu.close()


# ---- LoRA on F16 targets ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [8, 31])
@pytest.mark.parametrize("a_f16", [False, True])
def test_lora_patch_f16_target(r, a_f16):
    from oracle import lora as Lo
    if not Lo.have_ref():
        pytest.skip("oracle/_ref/libggml_lora.so not built")
    rl = Lo.RefLora()
    rng = np.random.default_rng(77 + r + a_f16)
    K, N = 128, 37
    w = (rng.standard_normal((N, K)) * 0.1).astype(np.float16)
    a, b = Lo.factors(rng, K, N, r, a_f16)
    sc = Lo.scaling(r, 3)
    want = rl.patch(F16, w, K, N, a, b, sc)
    L = lib()
    out = np.array(w, copy=True)
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b, np.float32)
    rc = L.b200_op_lora_patch(F16, out.ctypes.data_as(C.c_void_p), K, N, 1 if a.dtype == np.uint16 else 0, a.ctypes.data_as(C.c_void_p),
                              b.ctypes.data_as(C.c_void_p), a.shape[1], sc)
    assert rc == 0, rc
    assert np.array_equal(out.view(np.uint8).ravel(), np.ascontiguousarray(want).view(np.uint8).ravel())
