"""GPT-NeoX, GPT-2, MPT, BLOOM and GPT-J model files loaded with llm_b200.load_dynamic, bit for bit against the reference graphs on the same
per-tensor types (oracle/neox_kquant.mk: the reference's ggml.c + k_quants.c, a type per 2-D weight, RoPE overrides through ggml_rope_custom_inplace).

Each model is synthetic (oracle/neox_kquant.py: make_typed), written as a GGJT v3 file with loader.write_model and loaded through b200_neox_load_file.
Each case prefills in batches of 7 (K-quants: the warp kernel), 40 and 100 tokens (the tiled GEMM; the classic formats' exact GEMMs), decodes five
single tokens comparing every logit and the launch count of each step with the same model built from the tensor dict, and compares both KV caches
with the reference at the end.  Then: files of llm_b200.quantize, RoPE overrides, session features on a loaded mixed model, and the refusals."""
import ctypes as C
import re

import numpy as np
import pytest

import llm_b200
from llm_b200 import _lib, loader, neox
from oracle import bindings as B
from oracle import neox_kquant as NK

pytestmark = pytest.mark.gpu

PREFILL = (7, 40, 100)
DECODE = 5
GEOM = dict(n_vocab=320, n_ctx=256, n_embd=256, n_head=4, n_layer=2)
HP = {"gptneox": dict(GEOM, n_rot=16, use_parallel_residual=1), "gpt2": GEOM, "mpt": dict(GEOM, alibi_bias_max=8.0), "bloom": GEOM,
      "gptj": dict(GEOM, n_rot=16)}
CLASS = {"gptneox": neox.GptNeoX, "gpt2": neox.Gpt2, "mpt": neox.Mpt, "bloom": neox.Bloom, "gptj": neox.GptJ}
KQ = (B.Q2_K, B.Q3_K, B.Q4_K, B.Q5_K, B.Q6_K)
VOCAB = [(b"<|endoftext|>", 0.0), (b"<s>", 0.0), (b"</s>", 0.0), (b"<|padding|>", 0.0)] + [(f"t{i}".encode(), 0.0) for i in range(GEOM["n_vocab"] - 4)]

# (arch, hp overrides, base type, lm_head (GPT-2)): every architecture, each of Q4_0 .. Q8_0 at least once, F16 for each
CLASSIC = {"gptneox-parallel-q4_0": ("gptneox", {}, B.Q4_0, False), "gptneox-sequential-q5_1": ("gptneox", {"use_parallel_residual": 0}, B.Q5_1, False),
           "gpt2-tied-q4_1": ("gpt2", {}, B.Q4_1, False), "gpt2-lm_head-q8_0": ("gpt2", {}, B.Q8_0, True), "mpt-q5_0": ("mpt", {}, B.Q5_0, False),
           "bloom-q8_0": ("bloom", {}, B.Q8_0, False), "gptj-q4_0": ("gptj", {}, B.Q4_0, False),
           **{f"{a}-f16": (a, {}, B.F16, a == "gpt2") for a in NK.ARCHS}}


def check(g, c, what):
    g = np.asarray(g, np.float32)
    c = np.asarray(c, np.float32).reshape(g.shape)
    bad = g.view(np.uint32) != c.view(np.uint32)
    assert not bad.any(), (what, int(bad.sum()), g.size, int(np.argmax(bad.ravel())), float(np.abs(g - c).max()))


@pytest.fixture(scope="module")
def ref():
    if not NK.have_ref():
        pytest.skip("oracle/_ref/*_kq.so not built")
    return NK.ref_lib()


def header(arch, hp, file_type):
    h = dict(hp, file_type=file_type)
    if arch == "mpt":
        h.update(max_seq_len=hp["n_ctx"], clip_kqv=0.0)
    if arch == "bloom":
        h.update(n_mult=1)
    return h


def write(tmp_path, name, arch, hp, tensors, types, file_type=2002):
    path = str(tmp_path / f"{name}.ggjt")
    shapes = NK.tensor_shapes(arch, hp, "model/lm_head" in tensors)
    shapes.update({k: a.shape for k, a in tensors.items() if k not in shapes})          # a tensor the model does not hold (a refusal)
    loader.write_model(path, arch, header(arch, hp, file_type), tensors, shapes, hp["wtype"], vocabulary=VOCAB, tensor_types=types)
    return path


def dict_model(arch, hp, tensors, types, **kw):
    return CLASS[arch](hp, tensors, context_size=hp["n_ctx"], tensor_types=types, **kw)


def kv_equal(s, cpu):
    """both caches whole; GPT-2, MPT and BLOOM keep V by position in the reference, the native cache by channel"""
    hp = s.model.hyperparameters
    for which in (0, 1):
        got = s.kv(which)
        want = np.ascontiguousarray(cpu.kv(which)[:got.size])
        if which and cpu.arch in ("gpt2", "mpt", "bloom"):
            want = want.reshape(hp["n_layer"], s.model.context_size, hp["n_embd"]).transpose(0, 2, 1).ravel()
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), ("cache", which)


def run_and_compare(m, cpu, twin=None, seed=0):
    """prefill batches and decode steps of the loaded model against the reference (and, with twin, against the tensor-dict model: logits and launches)"""
    s = m.start_session(n_batch=128)
    t = twin.start_session(n_batch=128) if twin else None
    toks = np.random.default_rng(seed).integers(4, GEOM["n_vocab"], sum(PREFILL) + DECODE).astype(np.int32)
    at = 0
    for i, n in enumerate(PREFILL + (1,) * DECODE):
        g = s.evaluate(toks[at:at + n], all_logits=True)
        check(g, cpu.eval(toks[at:at + n]), f"{n} tokens at n_past {at}")
        if t:
            check(t.evaluate(toks[at:at + n], all_logits=True), g, f"tensor-dict model, {n} tokens at {at}")
            assert s.last_launches == t.last_launches, (at, s.last_launches, t.last_launches)
        at += n
    kv_equal(s, cpu)
    launches = s.last_launches
    s.close()
    if t:
        t.close()
    return launches


@pytest.mark.parametrize("name", list(CLASSIC))
def test_classic_and_f16_files(ref, tmp_path, name):
    arch, over, base, lm_head = CLASSIC[name]
    hp, tens, types = NK.make_typed(arch, dict(HP[arch], **over), base, ref, lm_head=lm_head)
    path = write(tmp_path, name, arch, hp, tens, None, 1 if base == B.F16 else 2002)
    m = llm_b200.load_dynamic(arch, path, llm_b200.ModelParameters(context_size=hp["n_ctx"]))
    assert type(m) is CLASS[arch] and m.eot_token_id() == (2 if arch == "bloom" else 0)
    cpu = NK.RefTyped(arch, hp, tens, types)
    twin = dict_model(arch, hp, tens, None)
    launches = run_and_compare(m, cpu, twin)
    if base != B.F16:                                        # one classic type: the decode graph
        assert launches < 12 * hp["n_layer"], launches
    m.close(); twin.close(); cpu.close()


def file_tensors(path, arch):
    """every tensor of a file as the reference harness takes it (f32 values, or the GGML bytes) and the file's type table"""
    f = loader.GgmlFile(path, arch)
    out = {}
    for i, t in enumerate(f.tensors()):
        b = f.tensor_bytes(i)
        out[t["name"]] = b.view(np.float32) if t["type"] == B.F32 else b.view(np.float16) if t["type"] == B.F16 else b
    types = loader.weight_types(f)
    f.close()
    return out, types


@pytest.mark.parametrize("arch,target", [("gptneox", B.Q4_0), ("gpt2", B.Q4_1), ("mpt", B.Q5_0), ("bloom", B.Q5_1), ("gptj", B.Q8_0)])
def test_quantizer_round_trip(ref, tmp_path, arch, target):
    """an F16 file quantized by llm_b200.quantize loads back and matches the reference on the quantized file's tensors"""
    hp, tens, _ = NK.make_typed(arch, HP[arch], B.F16, ref)
    src = write(tmp_path, "f16", arch, hp, tens, None, 1)
    dst = str(tmp_path / "q.ggjt")
    llm_b200.quantize(src, dst, arch, target)
    m = llm_b200.load_dynamic(arch, dst, llm_b200.ModelParameters(context_size=hp["n_ctx"]))
    qt, types = file_tensors(dst, arch)
    cpu = NK.RefTyped(arch, dict(hp, wtype=target), qt, types)
    run_and_compare(m, cpu, seed=1)
    m.close(); cpu.close()


def mixed_types(arch, hp, kind):
    """a pure K-quant type throughout; "mixed": Q4_K layer 0, Q5_0 layer 1, a Q6_K output matrix (or tied wte) beside a Q8_0 wte; "vproj": Q4_K
    with GPT-J layer 0's v_proj Q8_0 (its own matrix)"""
    names = NK.matrices(arch, hp, False)
    if kind in KQ:
        return {n: kind for n in names}
    if kind == "vproj":
        return dict({n: B.Q4_K for n in names}, **{"transformer.h.0.attn.v_proj.weight": B.Q8_0})
    t = {}
    for n in names:
        layer = re.search(r"(?:layers\.|blocks\.|/h|\.h\.)(\d+)", n)
        t[n] = B.Q6_K if layer is None else B.Q4_K if layer.group(1) == "0" else B.Q5_0
    if arch in ("gptneox", "bloom", "gptj"):                 # an output matrix of its own: the gathered-only embedding table is classic
        t[names[0]] = B.Q8_0
    return t


KCASES = {"gptneox-q2_K": ("gptneox", B.Q2_K), "gpt2-q3_K": ("gpt2", B.Q3_K), "mpt-q4_K": ("mpt", B.Q4_K), "bloom-q5_K": ("bloom", B.Q5_K),
          "gptj-q6_K": ("gptj", B.Q6_K), **{f"{a}-mixed": (a, "mixed") for a in NK.ARCHS}, "gptj-v_proj-q8_0": ("gptj", "vproj")}


@pytest.mark.parametrize("name", list(KCASES))
def test_kquant_and_mixed_files(ref, tmp_path, name):
    arch, kind = KCASES[name]
    hp0 = HP[arch]
    types = mixed_types(arch, dict(hp0, wtype=0), kind)
    base = types[NK.matrices(arch, dict(hp0, wtype=0))[-1]]
    hp, tens, types = NK.make_typed(arch, hp0, base, ref, types=types)
    path = write(tmp_path, name, arch, hp, tens, types)
    m = llm_b200.load_dynamic(arch, path, llm_b200.ModelParameters(context_size=hp["n_ctx"]))
    cpu = NK.RefTyped(arch, hp, tens, types)
    twin = dict_model(arch, hp, tens, types)
    run_and_compare(m, cpu, twin, seed=2)
    m.close(); twin.close(); cpu.close()


@pytest.mark.parametrize("arch,base", [("gptneox", B.Q4_0), ("gptj", B.Q8_0)])
def test_rope_overrides(ref, tmp_path, arch, base):
    """base 20000, scale 0.5: the graph decode and the per-op prefill match ggml_rope_custom_inplace; the explicit defaults are bit-identical to none"""
    hp, tens, types = NK.make_typed(arch, HP[arch], base, ref)
    path = write(tmp_path, arch, arch, hp, tens, None)
    m = llm_b200.load_dynamic(arch, path, llm_b200.ModelParameters(context_size=hp["n_ctx"], rope_freq_base=20000.0, rope_freq_scale=0.5))
    cpu = NK.RefTyped(arch, hp, tens, types, rope=(20000.0, 0.5))
    twin = dict_model(arch, hp, tens, None, rope_freq_base=20000.0, rope_freq_scale=0.5)
    launches = run_and_compare(m, cpu, twin, seed=3)
    assert launches < 12 * hp["n_layer"], launches             # the decode graph ran
    m.close(); twin.close(); cpu.close()
    plain = NK.RefTyped(arch, hp, tens, types)
    d = llm_b200.load_dynamic(arch, path, llm_b200.ModelParameters(context_size=hp["n_ctx"], rope_freq_base=10000.0, rope_freq_scale=1.0))
    run_and_compare(d, plain, dict_model(arch, hp, tens, None), seed=3)
    d.close(); plain.close()


def test_session_features_on_a_loaded_mixed_model(ref, tmp_path):
    """GPT-NeoX with a Q4_K layer, a Q5_0 layer and a Q6_K embed_out: embeddings, greedy infer_next_token, one perplexity chunk, a snapshot round
    trip and a LoRA adapter on the classic layer's dense weight, each equal to the tensor-dict model's"""
    from oracle import lora
    arch = "gptneox"
    types = mixed_types(arch, dict(HP[arch], wtype=0), "mixed")
    hp, tens, types = NK.make_typed(arch, HP[arch], B.Q5_0, ref, types=types)
    path = write(tmp_path, "mixed", arch, hp, tens, types)
    m = llm_b200.load_dynamic(arch, path, llm_b200.ModelParameters(context_size=hp["n_ctx"]))
    twin = dict_model(arch, hp, tens, types)
    toks = np.random.default_rng(4).integers(4, GEOM["n_vocab"], 40).astype(np.int32)
    out = []
    for model in (m, twin):
        s = model.start_session(n_batch=64)
        req = llm_b200.OutputRequest(embeddings=np.empty(0, np.float32))
        lg = s.evaluate(toks[:33], all_logits=True, output_request=req)
        greedy = llm_b200.InferenceParameters(llm_b200.Sampler(repetition_penalty=1.0, top_k=1))
        rng = llm_b200.Rng(1)
        ids = [s.infer_next_token(greedy, rng) for _ in range(3)]
        snap = s.get_snapshot()
        r = neox.NeoxSession.from_snapshot(snap, model)
        after = r.evaluate(toks[33:34], all_logits=True)
        r.close(); s.close()
        sp = model.start_session(n_batch=64)
        ppl, terms = sp.perplexity(np.random.default_rng(9).integers(4, GEOM["n_vocab"], hp["n_ctx"] + 8).astype(np.int32), return_terms=True, bos=1)
        sp.close()
        out.append((lg, req.embeddings, ids, after, terms, ppl))
    for a, b, what in zip(out[0], out[1], ("logits", "embeddings", "ids", "after snapshot", "perplexity terms", "perplexity")):
        check(np.asarray(a, np.float32), np.asarray(b, np.float32), what)
    m.close(); twin.close()
    ad = str(tmp_path / "lora.ggla")
    table, _ = lora.adapter_tensors({"gpt_neox.layers.1.attention.dense.weight": (256, 256)}, 4, np.random.default_rng(1))
    lora.write_ggla(ad, 4, 8, table)
    m = llm_b200.load_dynamic(arch, path, llm_b200.ModelParameters(context_size=hp["n_ctx"], lora_adapters=[ad]))
    twin = dict_model(arch, hp, tens, types, lora_adapters=[ad])
    plain = dict_model(arch, hp, tens, types)
    got = [x.start_session(n_batch=64).evaluate(toks, all_logits=True) for x in (m, twin, plain)]
    check(got[0], got[1], "LoRA through load_dynamic")
    assert not np.array_equal(got[0], got[2])               # the adapter changed the model
    m.close(); twin.close(); plain.close()


def free_bytes():
    f = C.c_size_t(0)
    _lib.lib().b200_device_info(None, C.byref(f), None)
    return int(f.value)


def test_refusals(ref, tmp_path):
    """each refusal with its LoadError.kind; afterwards the device's free memory is where it was"""
    from oracle import lora

    def refused(path, arch, kind, **kw):
        with pytest.raises(loader.LoadError) as e:
            llm_b200.load_dynamic(arch, path, llm_b200.ModelParameters(context_size=GEOM["n_ctx"], **kw))
        assert e.value.kind == kind, (path, e.value.kind, kind)

    hp, tens, types = NK.make_typed("gptj", HP["gptj"], B.Q4_K, ref)
    ok = write(tmp_path, "ok", "gptj", hp, tens, types)
    llm_b200.load_dynamic("gptj", ok, llm_b200.ModelParameters(context_size=GEOM["n_ctx"])).close()      # warm: the runtime's own buffers exist
    free0 = free_bytes()
    # GPT-J q_proj and k_proj of different types, refused four times
    t = dict(types, **{"transformer.h.1.attn.k_proj.weight": B.Q5_K})
    hp2, tn, t = NK.make_typed("gptj", HP["gptj"], B.Q4_K, ref, types=t)
    qk = write(tmp_path, "qk", "gptj", hp2, tn, t)
    for _ in range(4):
        refused(qk, "gptj", "UnsupportedElementType")
    # an F32 2-D weight
    tn = dict(tens, **{"transformer.h.0.mlp.fc_in.weight": np.zeros((4 * 256, 256), np.float32)})
    refused(write(tmp_path, "f32", "gptj", hp, tn, types), "gptj", "UnsupportedElementType")
    # an F16 weight beside K-quant ones
    tn = dict(tens, **{"transformer.h.0.attn.out_proj.weight": np.zeros((256, 256), np.float16)})
    refused(write(tmp_path, "f16", "gptj", hp, tn, dict(types, **{"transformer.h.0.attn.out_proj.weight": B.F16})), "gptj", "UnsupportedElementType")
    # a LoRA adapter onto a K-quant tensor
    ad = str(tmp_path / "lora.ggla")
    table, _ = lora.adapter_tensors({"transformer.h.0.attn.q_proj.weight": (256, 256)}, 4, np.random.default_rng(1))
    lora.write_ggla(ad, 4, 8, table)
    refused(ok, "gptj", "UnsupportedElementType", lora_adapters=[ad])
    # a K-quant row that is not whole super-blocks: GPT-2 with n_embd 320, attn/c_proj/w Q4_K (a 320-element row: 1.25 super-blocks)
    hp3 = dict(GEOM, n_embd=320, n_head=5)
    hp3, tn, t = NK.make_typed("gpt2", hp3, B.Q8_0, ref)
    tn["model/h0/attn/c_proj/w"] = np.zeros(320 * 320 // 256 * 144, np.uint8)
    t["model/h0/attn/c_proj/w"] = B.Q4_K
    refused(write(tmp_path, "ragged", "gpt2", hp3, tn, t), "gpt2", "InvariantBroken")
    # quantization version 1 with quantized tensors
    hp4, tn, t = NK.make_typed("mpt", HP["mpt"], B.Q4_0, ref)
    refused(write(tmp_path, "qv1", "mpt", hp4, tn, t, file_type=1002), "mpt", "QuantizationVersion")
    # an unknown tensor, a missing tensor
    refused(write(tmp_path, "unknown", "mpt", hp4, dict(tn, **{"transformer.blocks.0.extra.weight": np.zeros(256, np.float32)}), t), "mpt", "UnknownTensor")
    tn2 = dict(tn)
    del tn2["transformer.blocks.1.norm_2.weight"]
    refused(write(tmp_path, "missing", "mpt", hp4, tn2, t), "mpt", "NotLoaded")
    assert abs(free0 - free_bytes()) < (64 << 20), (free0, free_bytes())
