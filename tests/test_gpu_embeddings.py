"""OutputRequest::embeddings on every native session (crates/llm-base/src/model/common.rs:40-59): the last row of the final norm's output, against the
reference's own ggml.c running the same graphs (oracle/embd.py: the harnesses of oracle/ with the final norm's rows handed out), bit for bit on uint32
views.

  LLaMA        MHA and GQA with head sizes 64 and 128; Q4_0, Q5_1, Q8_0 and F16 weights; both KV caches: batches of 1, 5, 20 and 100 tokens, 40 graph
               decode steps (and the same steps on NO_GRAPH and UNFUSED sessions), a rewind and a re-evaluate; feed_prompt across n_batch chunks;
               a LoRA-patched model; a 4096-token context decoded across position 3072 to its last slot
  GPT-NeoX     GPT-NeoX (both residual forms), GPT-2 (tied and untied lm_head), MPT (no bias: signed zeros), BLOOM, GPT-J, both KV caches:
  family       a prefill and graph decode steps
Every step also runs on a second session of the same model without the request: logits, both caches, n_past, last_logits and last_launches are
the same bits.
  edges        NULL pointers, an empty feed_prompt (the buffer is untouched), a tensor-parallel session (B200_ERR_BAD_ARG; needs 2 GPUs), FAST"""
import ctypes as C

import numpy as np
import pytest

import llm_b200
from llm_b200 import ModelKVMemoryType as KV
from llm_b200 import OutputRequest
from llm_b200.neox import Bloom, Gpt2, GptJ, GptNeoX, Mpt
from oracle import alibi as A
from oracle import bindings as B
from oracle import gptj as J
from oracle import embd as E
from oracle import synth
from oracle import lora as Lo

pytestmark = pytest.mark.gpu

BAD_ARG = -2
NO_GRAPH, UNFUSED, FAST = 1, 2, 4
KVS = {"kv16": KV.Float16, "kv32": KV.Float32}


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def check(g, c, what):
    g, c = bits(g).ravel(), bits(c).ravel()
    assert g.size == c.size, (what, g.size, c.size)
    bad = g != c
    assert not bad.any(), (what, int(bad.sum()), g.size)


def ref_or_skip():
    if not E.have_ref():
        pytest.skip("oracle/_ref/*_embd.so not built (the reference graphs on the reference's ggml, oracle/embd.mk)")


def step(req, plain, cpu, toks, what, others=()):
    """one evaluate of `toks` on `req` (and on `others`) with embeddings requested and on `plain` without; all against the oracle"""
    want_logits, want_embd = E.eval_embd(cpu, toks)[:2]
    r = OutputRequest(embeddings=np.empty(0, np.float32))
    got = req.evaluate(toks, all_logits=True, output_request=r)
    check(got, want_logits, f"{what}: logits")
    check(r.embeddings, want_embd[-1], f"{what}: embeddings")
    assert r.embeddings.shape == (want_embd.shape[1],) and r.embeddings.dtype == np.float32
    check(plain.evaluate(toks, all_logits=True), got, f"{what}: logits without the request")
    assert req.last_launches == plain.last_launches, (what, req.last_launches, plain.last_launches)
    assert req.n_past == plain.n_past
    check(req.last_logits, plain.last_logits, f"{what}: last_logits")
    for which in (0, 1):
        assert np.array_equal(req.kv(which), plain.kv(which)), (what, "cache", which)
    for s in others:
        o = OutputRequest(embeddings=np.empty(0, np.float32))
        check(s.evaluate(toks, all_logits=True, output_request=o), want_logits, f"{what}: logits, flags {s.config.flags}")
        check(o.embeddings, want_embd[-1], f"{what}: embeddings, flags {s.config.flags}")


# ---- LLaMA ----------------------------------------------------------------------------------------------------------------------------------------
LLAMA = {"mha": dict(synth.CONFIGS["tiny8"], n_ctx=256),
         "gqa-hd64": synth.CONFIGS["gqa8"],
         "gqa-hd128": dict(n_vocab=352, n_embd=512, n_head=4, n_head_kv=2, n_layer=2, n_ff=1024, n_rot=128, n_ctx=256)}
WTYPES = {"q4_0": B.Q4_0, "q5_1": B.Q5_1, "q8_0": B.Q8_0, "f16": B.F16}


def llama_model(orc, base, wtype):
    quant = (lambda t, w: np.ascontiguousarray(w, np.float32).astype(np.float16)) if wtype == B.F16 else orc.quantize
    return synth.make_llama(base, wtype, quant)


def llama_sessions(m, kv, n_batch=128, flags=(0, 0, NO_GRAPH, UNFUSED)):
    return [m.start_session(llm_b200.InferenceSessionConfig(n_batch=n_batch, flags=f, memory_k_type=kv, memory_v_type=kv)) for f in flags]


def llama_oracle(hp, tens, kv, n_batch=128):
    return E.model("llama", hp, tens, kv == KV.Float32, n_batch=n_batch)


@pytest.mark.parametrize("kv", list(KVS))
@pytest.mark.parametrize("wname", list(WTYPES))
@pytest.mark.parametrize("cfg", list(LLAMA))
def test_llama(orc, cfg, wname, kv):
    ref_or_skip()
    hp, tens = llama_model(orc, LLAMA[cfg], WTYPES[wname])
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens)
    req, plain, nog, unf = sessions = llama_sessions(m, KVS[kv])
    cpu = llama_oracle(hp, tens, KVS[kv])
    toks = synth.make_tokens(hp, 170)
    i = 0
    for n in (1, 5, 20, 100):
        step(req, plain, cpu, toks[i:i + n], f"batch of {n} at {i}", (nog, unf))
        i += n
    for i in range(126, 166):
        step(req, plain, cpu, toks[i:i + 1], f"decode at {i}", (nog, unf))
    if WTYPES[wname] != B.F16:                                   # the step ran the graph schedule: fewer launches than the per-op one
        assert req.last_launches < unf.last_launches
    for s in sessions:
        s.rewind(150)
    cpu.set_n_past(150)
    other = synth.make_tokens(hp, 160, seed=11)
    step(req, plain, cpu, other[150:157], "re-evaluate 7 after a rewind to 150", (nog, unf))
    for i in range(157, 160):
        step(req, plain, cpu, other[i:i + 1], f"decode at {i} after the rewind", (nog, unf))
    for s in sessions:
        s.close()
    m.close(); cpu.close()


@pytest.mark.parametrize("kv", list(KVS))
def test_llama_feed_prompt(orc, kv):
    """feed_prompt passes the request to every chunk of n_batch (inference_session.rs:315-317): the last chunk's last row; an empty prompt leaves
    the request as it was"""
    ref_or_skip()
    hp, tens = llama_model(orc, synth.CONFIGS["gqa8"], B.Q4_0)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens)
    req, plain = llama_sessions(m, KVS[kv], n_batch=16, flags=(0, 0))
    cpu = llama_oracle(hp, tens, KVS[kv], n_batch=16)
    toks = synth.make_tokens(hp, 140)
    for a, b in ((0, 70), (70, 71), (71, 119)):                 # 5 chunks (the last one of 6), a one-token prompt (the graph step), 3 chunks
        r = OutputRequest(embeddings=np.empty(0, np.float32))
        got = req.feed_prompt(toks[a:b], output_request=r)
        for c in range(a, b, 16):
            want_logits, want_embd, _ = E.eval_embd(cpu, toks[c:min(c + 16, b)])
        check(got, want_logits[-1], f"feed_prompt {a}..{b}: last logits")
        check(r.embeddings, want_embd[-1], f"feed_prompt {a}..{b}: embeddings")
        check(plain.feed_prompt(toks[a:b]), got, f"feed_prompt {a}..{b}: without the request")
        assert req.n_past == plain.n_past == b
        for which in (0, 1):
            assert np.array_equal(req.kv(which), plain.kv(which)), (a, which)
    sentinel = np.full(hp["n_embd"], 7.0, np.float32)
    r = OutputRequest(embeddings=sentinel)
    req.feed_prompt(np.zeros(0, np.int32), output_request=r)
    assert r.embeddings is sentinel and np.all(sentinel == 7.0)
    buf = np.full(hp["n_embd"], 7.0, np.float32)
    L = req.L
    assert L.b200_session_feed_prompt_output(req._s, toks.ctypes.data_as(C.c_void_p), 0, None, buf.ctypes.data_as(C.c_void_p)) == 0
    assert np.all(buf == 7.0) and req.n_past == 119
    req.close(); plain.close(); m.close(); cpu.close()


def test_llama_lora(orc, tmp_path):
    """a model patched by two adapters at load time; the oracle runs the patched weights the model holds (tests/test_gpu_lora.py pins those to the
    reference's own LoRA graph)"""
    ref_or_skip()
    from llm_b200 import loader
    hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], B.Q4_1, orc.quantize)
    shapes = synth.tensor_shapes(hp)
    path = str(tmp_path / "model.ggjt")
    loader.write_llama(path, hp, tens, shapes)
    targets = ["layers.0.attention.wq.weight", "layers.1.feed_forward.w2.weight", "norm.weight"]
    adapters = []
    for i, (r, alpha) in enumerate(((8, 16), (4, 3))):
        kn = {n: (shapes[n][-1], shapes[n][0] if len(shapes[n]) == 2 else 1) for n in targets}
        table, _ = Lo.adapter_tensors(kn, r, np.random.default_rng(0xE0 + i))
        adapters.append(str(tmp_path / f"a{i}.ggla"))
        Lo.write_ggla(adapters[-1], r, alpha, table)
    m = loader.load(path, llm_b200.ModelParameters(context_size=hp["n_ctx"], lora_adapters=adapters))
    patched = {n: m.read_tensor(n).reshape(np.shape(tens[n])) for n in tens}
    assert not np.array_equal(patched["norm.weight"], tens["norm.weight"])
    req, plain = llama_sessions(m, KV.Float16, flags=(0, 0))
    cpu = llama_oracle(hp, patched, KV.Float16)
    toks = synth.make_tokens(hp, 40)
    step(req, plain, cpu, toks[:20], "prefill 20")
    for i in range(20, 30):
        step(req, plain, cpu, toks[i:i + 1], f"decode at {i}")
    req.close(); plain.close(); m.close(); cpu.close()


@pytest.mark.slow
def test_llama_long_context(orc):
    """n_ctx 4096: graph steps below 3072 (fused attention), across 3072 (the two-kernel attention) to the last slot"""
    ref_or_skip()
    hp, tens = synth.make_llama(dict(n_vocab=1024, n_embd=512, n_head=4, n_head_kv=4, n_layer=2, n_ff=1536, n_rot=128, n_ctx=4096), B.Q4_0, orc.quantize)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=4096), tens)
    req, plain = llama_sessions(m, KV.Float16, n_batch=512, flags=(0, 0))
    cpu = llama_oracle(hp, tens, KV.Float16, n_batch=512)
    toks = synth.make_tokens(hp, 4096)
    for a in range(0, 3068, 512):
        b = min(a + 512, 3068)
        step(req, plain, cpu, toks[a:b], f"prefill {a}..{b}")
    for i in range(3068, 3076):
        step(req, plain, cpu, toks[i:i + 1], f"decode at {i}")
    for a in range(3076, 4090, 512):
        b = min(a + 512, 4090)
        step(req, plain, cpu, toks[a:b], f"prefill {a}..{b}")
    for i in range(4090, 4096):
        step(req, plain, cpu, toks[i:i + 1], f"decode at {i}")
    req.close(); plain.close(); m.close(); cpu.close()


# ---- GPT-NeoX family ------------------------------------------------------------------------------------------------------------------------------
NEOX = {"neox-par": dict(n_vocab=384, n_ctx=200, n_embd=256, n_head=4, n_layer=2, n_rot=16, use_parallel_residual=1),
        "neox-seq": dict(n_vocab=384, n_ctx=200, n_embd=256, n_head=8, n_layer=2, n_rot=32, use_parallel_residual=0)}
ARCHS = ["neox-par", "neox-seq", "gpt2-tied", "gpt2-untied", "mpt", "bloom", "gptj"]


def neox_case(orc, name, kv):
    """(native model, oracle)"""
    f32 = kv == KV.Float32
    if name in NEOX:
        hp, t = synth.make_neox(NEOX[name], B.Q4_0, orc.quantize)
        return GptNeoX(hp, t), E.model("neox", hp, t, f32)
    if name.startswith("gpt2"):
        hp, t = synth.make_gpt2(dict(n_vocab=320, n_ctx=200, n_embd=256, n_head=4, n_layer=2), B.Q4_0, orc.quantize, lm_head=name == "gpt2-untied")
        return Gpt2(hp, t), E.model("gpt2", hp, t, f32)
    if name in ("mpt", "bloom"):
        make, base, arch, cls = (A.make_mpt, A.MPT_CONFIGS["mpt-tiny"], A.MPT, Mpt) if name == "mpt" else \
                                (A.make_bloom, A.BLOOM_CONFIGS["bloom-tiny"], A.BLOOM, Bloom)
        hp, t = make(dict(base, n_ctx=200), B.Q4_0, orc.quantize)
        return cls(hp, t), E.model("alibi", hp, t, f32, arch)
    hp, t = J.make_gptj(dict(J.GPTJ_CONFIGS["gptj-tiny"], n_ctx=200), B.Q4_0, orc.quantize)
    return GptJ(hp, t), E.model("gptj", hp, t, f32)


@pytest.mark.parametrize("kv", list(KVS))
@pytest.mark.parametrize("name", ARCHS)
def test_neox_family(orc, name, kv):
    ref_or_skip()
    m, cpu = neox_case(orc, name, KVS[kv])
    req, plain = (m.start_session(128, memory_k_type=KVS[kv], memory_v_type=KVS[kv]) for _ in range(2))
    toks = synth.make_tokens(m.hyperparameters, 200)
    step(req, plain, cpu, toks[:37], "prefill 37")
    step(req, plain, cpu, toks[37:100], "prefill 63")
    launches = []
    for i in range(100, 140):
        step(req, plain, cpu, toks[i:i + 1], f"decode at {i}")
        launches.append(req.last_launches)
    assert len(set(launches)) == 1 and launches[0] < 20 * m.hyperparameters["n_layer"], launches    # the graph schedule
    r = OutputRequest(embeddings=np.empty(0, np.float32))
    req.feed_prompt(toks[140:150], output_request=r)
    check(r.embeddings, E.eval_embd(cpu, toks[140:150])[1][-1], "feed_prompt")
    plain.feed_prompt(toks[140:150])
    sentinel = np.full(m.hyperparameters["n_embd"], 7.0, np.float32)
    r = OutputRequest(embeddings=sentinel)
    req.feed_prompt(np.zeros(0, np.int32), output_request=r)
    assert r.embeddings is sentinel and np.all(sentinel == 7.0)
    step(req, plain, cpu, toks[150:151], "decode after feed_prompt")
    req.close(); plain.close(); m.close(); cpu.close()


def test_mpt_keeps_signed_zeros(orc):
    """MPT's final norm has no add node: where the gain is -0 the embedding is a zero whose sign is the product's (a bias add would make it +0)"""
    ref_or_skip()
    hp, t = A.make_mpt(dict(A.MPT_CONFIGS["mpt-tiny"], n_ctx=200), B.Q4_0, orc.quantize)
    g = np.array(t["transformer.norm_f.weight"], np.float32)
    g[::3] = -0.0
    g[1::3] = 0.0
    t = dict(t, **{"transformer.norm_f.weight": g})
    m, cpu = Mpt(hp, t), E.model("alibi", hp, t, arch=A.MPT)
    req, plain = m.start_session(128), m.start_session(128)
    toks = synth.make_tokens(hp, 60)
    step(req, plain, cpu, toks[:30], "prefill 30")
    for i in range(30, 40):
        step(req, plain, cpu, toks[i:i + 1], f"decode at {i}")
    r = OutputRequest(embeddings=np.empty(0, np.float32))
    req.evaluate(toks[40:41], output_request=r)
    z = bits(r.embeddings)[::3]
    assert (z == 0x80000000).any() and (z == 0).any()               # both zeros occur
    req.close(); plain.close(); m.close(); cpu.close()


# ---- edges ----------------------------------------------------------------------------------------------------------------------------------------
def test_null_pointers(orc):
    ref_or_skip()
    hp, tens = llama_model(orc, synth.CONFIGS["tiny8"], B.Q4_0)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens)
    (s,) = llama_sessions(m, KV.Float16, flags=(0,))
    cpu = llama_oracle(hp, tens, KV.Float16)
    L = s.L
    toks = synth.make_tokens(hp, 10)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    buf = np.full(hp["n_embd"], 7.0, np.float32)
    logits = np.empty(hp["n_vocab"], np.float32)
    assert L.b200_session_evaluate_output(None, p(toks), 1, None, 0, p(buf)) == BAD_ARG
    assert L.b200_session_evaluate_output(s._s, None, 1, None, 0, p(buf)) == BAD_ARG
    assert L.b200_session_feed_prompt_output(None, p(toks), 1, None, p(buf)) == BAD_ARG
    assert L.b200_session_feed_prompt_output(s._s, None, 1, None, p(buf)) == BAD_ARG
    assert L.b200_neox_evaluate_output(None, p(toks), 1, None, 0, p(buf)) == BAD_ARG
    assert np.all(buf == 7.0) and s.n_past == 0
    # logits_out NULL: the embeddings alone; embeddings_out NULL: b200_session_evaluate
    assert L.b200_session_evaluate_output(s._s, p(toks), 4, None, 0, p(buf)) == 0
    want_logits, want_embd, _ = E.eval_embd(cpu, toks[:4])
    check(buf, want_embd[-1], "logits_out NULL")
    assert L.b200_session_evaluate_output(s._s, p(toks[4:]), 1, p(logits), 0, None) == 0
    check(logits, cpu.eval(toks[4:5])[-1], "embeddings_out NULL")
    assert L.b200_session_feed_prompt_output(s._s, p(toks[5:]), 3, None, p(buf)) == 0
    check(buf, E.eval_embd(cpu, toks[5:8])[1][-1], "feed_prompt, last_logits_out NULL")
    s.close(); m.close(); cpu.close()


def test_fast_session(orc):
    """a FAST session returns its own order-free numbers (activations quantized for its kernels, other summation orders): n_embd finite values
    pointing the way the conformant row points"""
    ref_or_skip()
    hp, tens = llama_model(orc, synth.CONFIGS["gqa8"], B.Q4_0)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens)
    (s,) = llama_sessions(m, KV.Float16, flags=(FAST,))
    cpu = llama_oracle(hp, tens, KV.Float16)
    toks = synth.make_tokens(hp, 30)
    for a, b in ((0, 20), (20, 21), (21, 22)):
        r = OutputRequest(embeddings=np.empty(0, np.float32))
        s.evaluate(toks[a:b], output_request=r)
        want = E.eval_embd(cpu, toks[a:b])[1][-1]
        assert r.embeddings.shape == want.shape and np.isfinite(r.embeddings).all()
        cos = float(np.dot(r.embeddings, want) / (np.linalg.norm(r.embeddings) * np.linalg.norm(want)))
        assert cos > 0.999, (a, b, cos)
    s.close(); m.close(); cpu.close()


def _gpu_count():
    n = C.c_int(0)
    return n.value if C.CDLL("libcudart.so").cudaGetDeviceCount(C.byref(n)) == 0 else 0


def test_tensor_parallel_refused(orc):
    if _gpu_count() < 2:
        pytest.skip("a tensor-parallel model needs 2 GPUs")
    from llm_b200 import _lib
    from llm_b200.tp import TpLlama
    hp, tens = llama_model(orc, synth.CONFIGS["tiny8"], B.Q4_0)
    m = TpLlama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens, rank=0, world=2, device=0)
    L = m.L
    cfg = _lib.SessionConfig(n_batch=8, flags=0)
    s = L.b200_model_start_session(m._m, C.byref(cfg))
    assert s
    toks = synth.make_tokens(hp, 4)
    buf = np.full(hp["n_embd"], 7.0, np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert L.b200_session_evaluate_output(s, p(toks), 1, None, 0, p(buf)) == BAD_ARG
    assert L.b200_session_feed_prompt_output(s, p(toks), 4, None, p(buf)) == BAD_ARG
    assert np.all(buf == 7.0) and L.b200_session_n_past(s) == 0
    L.b200_session_free(s)
    m.close()
