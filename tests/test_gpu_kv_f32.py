"""F32 KV caches (B200_SESSION_KV_F32; InferenceSessionConfig::memory_k_type = memory_v_type = Float32, the reference CLI's --no-float16) on every
native session, bit for bit against the reference's own ggml.c running the same graphs with an F32 cache (oracle/kv32.mk).

Every case checks the logits of every step and both caches, whole:
  LLaMA            MHA and GQA, Q4_0, Q5_1 and an F16 model; prompt batches of 5, 20 and 100 tokens (the weight GEMM regimes < 16, 16-95, >= 96
                   and both attention mat-mul kernels), then 40 graph decode steps (n_kv covers every residue mod 32 of the KQV dot); a rewind;
                   one case each with B200_SESSION_NO_GRAPH and B200_SESSION_UNFUSED
  GPT-NeoX family  GPT-NeoX (partial rotary; parallel and sequential residual), GPT-2, MPT, BLOOM, GPT-J (256-wide heads)
  head sizes       64 and 128 (the LLaMA-7B head: 4-CTA clusters) for LLaMA, 32 and 64 for GPT-NeoX, 64 for MPT / BLOOM, 256 for GPT-J
  fused bound      a 2048-position LLaMA (hd 64 and 128) and MPT: prefill to just below the f32 cluster attention's bound, then decode across it;
                   a 27648-position LLaMA, past what the two-kernel f32 attention holds, decodes per op
  perplexity       one F32 session against the reference's loop on the reference's logits
  refusals         unequal K / V types, an f32 cache on a tensor-parallel model, an unknown flag"""
import ctypes as C

import numpy as np
import pytest

import llm_b200
from llm_b200 import ModelKVMemoryType as KV
from oracle import alibi as A
from oracle import bindings as B
from oracle import gptj as J
from oracle import kv32
from oracle import synth

pytestmark = pytest.mark.gpu

F32CFG = dict(memory_k_type=KV.Float32, memory_v_type=KV.Float32)


def check(g, c, what):
    g = np.asarray(g, np.float32)
    c = np.asarray(c, np.float32).reshape(g.shape)
    bad = g.view(np.uint32) != c.view(np.uint32)
    assert not bad.any(), (what, int(bad.sum()), g.size, float(np.abs(g - c).max()))


def ref_or_skip():
    if not kv32.have_ref():
        pytest.skip("oracle/_ref/*_kv32.so not built (the F32-cache oracle is the reference graph on the reference's ggml)")


def f16(t, w):
    return np.ascontiguousarray(w, np.float32).astype(np.float16)


def llama_kv_equal(s, cpu):
    for which in (0, 1):            # the reference sizes the cache by n_embd; with GQA only the first n_layer*n_ctx*n_embd_gqa values are used
        a = s.kv(which)
        assert a.dtype == np.float32
        assert np.array_equal(a.view(np.uint32), kv32.kv_f32(cpu, which)[:a.size].view(np.uint32)), which


# hd128: the LLaMA-7B head size (4-CTA clusters, attn_kq_kernel<128, float>); the others have 64-wide heads
LLAMA_CFGS = dict(synth.CONFIGS, hd128=dict(synth.CONFIGS["tiny8"], n_head=2, n_head_kv=2, n_rot=128))


def llama_case(orc, cfg, wtype, flags=0, n_ctx=256, n_batch=128):
    ref_or_skip()
    quant = f16 if wtype == B.F16 else orc.quantize
    hp, tens = synth.make_llama(dict(LLAMA_CFGS[cfg], n_ctx=n_ctx), wtype, quant)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=n_ctx), tens)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=n_batch, flags=flags, **F32CFG))
    cpu = kv32.ref_lib().llama(hp, tens, n_threads=16, n_batch=n_batch)
    return hp, m, s, cpu


@pytest.mark.parametrize("cfg,wtype", [("tiny8", B.Q4_0), ("tiny8", B.Q5_1), ("tiny8", B.F16), ("gqa8", B.Q4_0), ("gqa8", B.Q5_1), ("gqa8", B.F16),
                                       ("hd128", B.Q4_0), ("hd128", B.Q8_0)])
def test_llama_matches_reference(orc, cfg, wtype):
    hp, m, s, cpu = llama_case(orc, cfg, wtype)
    toks = synth.make_tokens(hp, 180)
    at = 0
    for n in (5, 20, 100):
        check(s.evaluate(toks[at:at + n], all_logits=True), cpu.eval(toks[at:at + n]), f"prompt batch of {n}")
        at += n
    graph = 7 * hp["n_layer"] + 3
    for i in range(at, at + 40):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        if wtype != B.F16:          # F16 weights decode per op
            assert s.last_launches == graph, ("graph schedule", i, s.last_launches)
    llama_kv_equal(s, cpu)
    # rewind, then re-evaluate: the same logits as the first time
    s.rewind(130)
    cpu.set_n_past(130)
    first = cpu.eval(toks[130:131])
    check(s.evaluate(toks[130:131], all_logits=True), first, "decode after a rewind")
    s.rewind(130)
    check(s.evaluate(toks[130:131], all_logits=True), first, "the same step again")
    check(s.evaluate(toks[131:140], all_logits=True), cpu.eval(toks[131:140]), "batch after the rewind")
    s.close(); m.close(); cpu.close()


@pytest.mark.parametrize("flag", [1, 2])                 # B200_SESSION_NO_GRAPH, B200_SESSION_UNFUSED
def test_llama_decode_switches(orc, flag):
    hp, m, s, cpu = llama_case(orc, "gqa8", B.Q4_0, flags=flag)
    toks = synth.make_tokens(hp, 80, seed=flag)
    check(s.evaluate(toks[:30], all_logits=True), cpu.eval(toks[:30]), "prompt")
    for i in range(30, 70):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
    llama_kv_equal(s, cpu)
    s.close(); m.close(); cpu.close()


def test_llama_fast_session_runs(orc):
    """B200_SESSION_FAST with an f32 cache: the weight mat-muls go order-free (so the logits are not the reference's and are not compared), the
    attention runs the exact f32 kernels; checked to run and to keep f32 values in the cache"""
    ref_or_skip()
    hp, tens = synth.make_llama(dict(synth.CONFIGS["tiny8"], n_ctx=128), B.Q4_0, orc.quantize)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=128), tens)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64, flags=4, **F32CFG))
    toks = synth.make_tokens(hp, 40)
    assert np.isfinite(s.evaluate(toks[:30], all_logits=True)).all()
    for i in range(30, 40):
        assert np.isfinite(s.evaluate(toks[i:i + 1])).all()
    k = s.kv(0)
    assert k.dtype == np.float32 and np.isfinite(k).all() and np.count_nonzero(k) > 0
    s.close(); m.close()


# ---- the GPT-NeoX family -----------------------------------------------------------------------------------------------------------------------
NEOX_CFGS = {
    "neox-par": dict(n_vocab=384, n_ctx=128, n_embd=256, n_head=4, n_layer=2, n_rot=16, use_parallel_residual=1),
    "neox-seq": dict(n_vocab=384, n_ctx=128, n_embd=256, n_head=8, n_layer=2, n_rot=32, use_parallel_residual=0),
}


def neox_model(orc, arch, wtype=B.Q4_0, n_ctx=None):
    """(native model, reference on an F32 cache, V transposed in the reference: True for GPT-2 / MPT / BLOOM)"""
    from llm_b200.neox import Bloom, Gpt2, GptJ, GptNeoX, Mpt
    ref_or_skip()
    if arch in NEOX_CFGS:
        hp, tens = synth.make_neox(dict(NEOX_CFGS[arch], **({"n_ctx": n_ctx} if n_ctx else {})), wtype, orc.quantize)
        return GptNeoX(hp, tens), kv32.ref_lib().neox(hp, tens, n_threads=8, n_batch=64), hp, False
    if arch == "gpt2":
        hp, tens = synth.make_gpt2(dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2), wtype, orc.quantize)
        return Gpt2(hp, tens), kv32.ref_lib().gpt2(hp, tens, n_threads=8, n_batch=64), hp, True
    if arch in ("mpt", "bloom"):
        a = A.MPT if arch == "mpt" else A.BLOOM
        base = A.MPT_CONFIGS["mpt-tiny"] if arch == "mpt" else A.BLOOM_CONFIGS["bloom-tiny"]
        hp, tens = (A.make_mpt if arch == "mpt" else A.make_bloom)(dict(base, **({"n_ctx": n_ctx} if n_ctx else {})), wtype, orc.quantize)
        return (Mpt if arch == "mpt" else Bloom)(hp, tens), kv32.RefAlibiKV32(hp, tens, a, n_threads=8, n_batch=512), hp, True
    hp, tens = J.make_gptj(J.GPTJ_CONFIGS["gptj-tiny"], wtype, orc.quantize)
    return GptJ(hp, tens), kv32.RefGptJKV32(hp, tens, n_threads=8, n_batch=512), hp, False


def neox_kv_equal(s, cpu, hp, v_by_position):
    nl, n_ctx, e = hp["n_layer"], s.model.context_size, hp["n_embd"]
    k, v = kv32.kv_f32(cpu, 0), kv32.kv_f32(cpu, 1)
    if v_by_position:               # the native cache keeps V by channel
        v = v.reshape(nl, n_ctx, e).transpose(0, 2, 1).ravel()
    assert s.kv(0).dtype == np.float32
    assert np.array_equal(s.kv(0).view(np.uint32), k.view(np.uint32)), "K"
    assert np.array_equal(s.kv(1).view(np.uint32), v.view(np.uint32)), "V"


@pytest.mark.parametrize("arch", ["neox-par", "neox-seq", "gpt2", "mpt", "bloom", "gptj"])
def test_neox_family_matches_reference(orc, arch):
    m, cpu, hp, vpos = neox_model(orc, arch)
    s = m.start_session(64, **F32CFG)
    toks = np.random.default_rng(0xF32).integers(0, hp["n_vocab"], size=80, dtype=np.int32)
    check(s.evaluate(toks[:20], all_logits=True), cpu.eval(toks[:20]), "prefill 20")
    for i in range(20, 60):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
    check(s.evaluate(toks[60:77], all_logits=True), cpu.eval(toks[60:77]), "batch of 17")
    check(s.evaluate(toks[77:78], all_logits=True), cpu.eval(toks[77:78]), "decode after the batch")
    neox_kv_equal(s, cpu, hp, vpos)
    s.close(); m.close(); cpu.close()


# ---- across the f32 cluster attention's bound (1664 positions: buckets up to 1536 fuse, 1792 runs the fallback) -------------------------------------
@pytest.mark.parametrize("cfg", ["tiny8", "hd128"])
def test_llama_decodes_across_the_fused_bound(orc, cfg):
    hp, m, s, cpu = llama_case(orc, cfg, B.Q4_0, n_ctx=2048, n_batch=512)
    toks = synth.make_tokens(hp, 1560)
    for a in range(0, 1530, 512):
        b = min(a + 512, 1530)
        check(s.evaluate(toks[a:b]), cpu.eval(toks[a:b])[-1], f"prefill to {b}")
    for i in range(1530, 1545):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        fused = i + 1 <= 1536
        assert s.last_launches == (7 if fused else 8) * hp["n_layer"] + 3, (i, s.last_launches)
    llama_kv_equal(s, cpu)
    s.close(); m.close(); cpu.close()


def test_llama_context_past_the_f32_fallback_decodes_per_op(orc):
    """past 27520 positions the two-kernel f32 attention's shared memory no longer holds the context: such a session decodes per op from the
    first step (the f16 cache keeps the graph schedule)"""
    n_ctx = 27648
    hp, m, s, cpu = llama_case(orc, "tiny8", B.Q4_0, n_ctx=n_ctx, n_batch=32)
    toks = synth.make_tokens(hp, 40)
    check(s.evaluate(toks[:20], all_logits=True), cpu.eval(toks[:20]), "prompt")
    for i in range(20, 24):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        assert s.last_launches != 7 * hp["n_layer"] + 3, ("per-op decode", s.last_launches)
    llama_kv_equal(s, cpu)
    s.close(); cpu.close()
    s16 = m.start_session(llm_b200.InferenceSessionConfig(n_batch=32))
    s16.evaluate(toks[:20])
    s16.evaluate(toks[20:21])
    assert s16.last_launches == 7 * hp["n_layer"] + 3, s16.last_launches
    s16.close(); m.close()


def test_mpt_decodes_across_the_fused_bound(orc):
    m, cpu, hp, vpos = neox_model(orc, "mpt", n_ctx=2048)
    s = m.start_session(512, **F32CFG)
    toks = np.random.default_rng(0xB0).integers(0, hp["n_vocab"], size=1560, dtype=np.int32)
    for a in range(0, 1530, 512):
        b = min(a + 512, 1530)
        check(s.evaluate(toks[a:b]), cpu.eval(toks[a:b])[-1], f"prefill to {b}")
    graph = 8 * hp["n_layer"] + 3
    for i in range(1530, 1545):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        assert (s.last_launches == graph) == (i + 1 <= 1536), (i, s.last_launches)
    neox_kv_equal(s, cpu, hp, vpos)
    s.close(); m.close(); cpu.close()


# ---- perplexity ---------------------------------------------------------------------------------------------------------------------------------
def test_llama_perplexity(orc):
    from oracle.ppl import PplOracle
    hp, m, s, cpu = llama_case(orc, "gqa8", B.Q5_1, n_ctx=64, n_batch=16)
    toks = synth.make_tokens(hp, 160, seed=0x99)
    got_ppl, got_terms = s.perplexity(toks, return_terms=True, bos=1)
    want_ppl, want_terms = PplOracle().perplexity(cpu.eval, cpu.reset, toks, 64, 16, 1)
    assert len(got_ppl) == len(want_ppl) == 2
    check(got_terms, want_terms, "terms")
    check(got_ppl, want_ppl, "perplexities")
    s.close(); m.close(); cpu.close()


# ---- refusals -------------------------------------------------------------------------------------------------------------------------------------
def test_refusals(orc):
    from llm_b200 import _lib
    from llm_b200.neox import GptNeoX
    from llm_b200.tp import TpLlama
    with pytest.raises(ValueError):
        llm_b200.InferenceSessionConfig(memory_k_type=KV.Float32, memory_v_type=KV.Float16)
    hp, tens = synth.make_neox(NEOX_CFGS["neox-par"], B.Q4_0, orc.quantize)
    mn = GptNeoX(hp, tens)
    with pytest.raises(ValueError):
        mn.start_session(8, memory_k_type=KV.Float16, memory_v_type=KV.Float32)
    L = mn.L
    for flags in (1, 2, 4, 16, 8 | 4):
        assert not L.b200_neox_start_session_flags(mn._m, 8, flags), flags
    ok = L.b200_neox_start_session_flags(mn._m, 8, 8)
    assert ok
    L.b200_neox_session_free(ok)
    mn.close()
    # an f32 cache on a tensor-parallel shard: NULL; the same shard starts an f16 session
    hp2, tens2 = synth.make_llama(synth.CONFIGS["tiny8"], B.Q4_0, orc.quantize)
    mt = TpLlama(hp2, llm_b200.ModelParameters(context_size=hp2["n_ctx"]), tens2, rank=0, world=2, device=0)
    assert not L.b200_model_start_session(mt._m, C.byref(_lib.SessionConfig(n_batch=1, flags=8)))
    s = L.b200_model_start_session(mt._m, C.byref(_lib.SessionConfig(n_batch=1, flags=0)))
    assert s
    L.b200_session_free(s)
    mt.close()
