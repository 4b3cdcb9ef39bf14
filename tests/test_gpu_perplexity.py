"""Perplexity on the GPU (ppl.cu, SessionCore::perplexity), bit for bit against the reference's loop: the plain-C softmax / log-likelihood of
oracle/ppl_oracle.c on the host libm, over logits the reference's own ggml.c computes (oracle/_ref), one rewind per chunk.

  b200_op_nll_rows    vocabularies of 32000 / 32001 / 50257 / 65024 entries, 1-2048 rows, targets at the max and on ties, rows spread wider than
                      104 (expf values of 0 and subnormals), a target whose probability underflows (term +inf), and 2^24 random expf arguments
  whole sessions      LLaMA (MHA Q4_0, GQA Q5_1, an F16 file), GPT-NeoX, GPT-2, MPT, BLOOM, GPT-J; 2.5 chunks; n_batch 1 / 8 / 32 / C; C = 64 and
                      C = 1280 (scoring from row 512): per-position terms, per-chunk perplexities, n_past, and an evaluate afterwards
  FAST sessions       run and give finite values (not the reference's logits, so not compared)
  refusals            tensor parallelism, bos or token ids out of range, null pointers"""
import ctypes as C

import numpy as np
import pytest

import llm_b200
from oracle import bindings as B
from oracle import synth
from oracle.ppl import PplOracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def por():
    return PplOracle()


def lib():
    from llm_b200 import _lib
    L = _lib.lib()
    assert L.b200_init(0) == 0
    return L


def same_bits(got, want, what):
    g, w = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = g.view(np.uint32) != w.view(np.uint32)
    assert not bad.any(), (what, int(bad.sum()), g.size, g[bad][:4], w[bad][:4])


def op_nll(logits, targets):
    L = lib()
    logits = np.ascontiguousarray(logits, np.float32)
    targets = np.ascontiguousarray(targets, np.int32)
    out = np.empty(logits.shape[0], np.float32)
    rc = L.b200_op_nll_rows(logits.ctypes.data_as(C.c_void_p), logits.shape[0], logits.shape[1], targets.ctypes.data_as(C.c_void_p),
                            out.ctypes.data_as(C.c_void_p))
    assert rc == 0, rc
    return out


# ---- the row reduction -------------------------------------------------------------------------------------------------------------------
def edge_rows(rng, rows, V):
    """random logits, with (when there are enough rows) the target at the row's max, the target among five ties at the max, a row spread over
    [-150, 10] (expf(v - max) underflows to 0 or a subnormal for most entries), and a target 200 below the max (p = 0, term = +inf)"""
    x = (rng.standard_normal((rows, V)) * 3).astype(np.float32)
    t = rng.integers(0, V, rows).astype(np.int32)
    t[0] = int(np.argmax(x[0]))
    if rows > 1:
        idx = rng.choice(V, 5, replace=False)
        x[1, idx] = np.float32(x[1].max() + 1)
        t[1] = idx[2]
    if rows > 2:
        x[2] = rng.uniform(-150, 10, V).astype(np.float32)
    if rows > 3:
        x[3, t[3]] = np.float32(x[3].max() - 200)
    return x, t


@pytest.mark.parametrize("V", [32000, 32001, 50257, 65024])
@pytest.mark.parametrize("rows", [1, 5, 37, 512])
def test_op_nll_rows_matches_oracle(por, V, rows):
    rng = np.random.default_rng(V * 31 + rows)
    x, t = edge_rows(rng, rows, V)
    got, want = op_nll(x, t), por.nll_rows(x, t)
    same_bits(got, want, f"V={V} rows={rows}")
    if rows > 3:
        assert np.isposinf(got[3]), got[3]
    assert got[0] >= 0 and np.isfinite(got[:2]).all()


def test_op_nll_rows_2048_rows(por):
    rng = np.random.default_rng(2048)
    x, t = edge_rows(rng, 2048, 32000)
    same_bits(op_nll(x, t), por.nll_rows(x, t), "2048 rows")


def test_op_nll_rows_2_24_expf_arguments(por):
    """2^24 uniform arguments in [-104, 0]: 512 rows of 32768 values whose max is 0 (one entry per row), so every value is an expf argument of
    the row's in-order sum -- the sum and the terms equal the oracle's, which calls the host libm"""
    rng = np.random.default_rng(0xE4F)
    x = rng.uniform(-104, 0, (512, 32768)).astype(np.float32)
    x[np.arange(512), rng.integers(0, 32768, 512)] = 0.0
    t = rng.integers(0, 32768, 512).astype(np.int32)
    same_bits(op_nll(x, t), por.nll_rows(x, t), "2^24 arguments")


def test_op_nll_rows_refusals():
    L = lib()
    x = np.zeros((2, 8), np.float32)
    t = np.array([0, 8], np.int32)
    out = np.empty(2, np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert L.b200_op_nll_rows(p(x), 2, 8, p(t), p(out)) == -2                           # target 8 of 8
    assert L.b200_op_nll_rows(None, 2, 8, p(t), p(out)) == -2
    assert L.b200_op_nll_rows(p(x), 0, 8, p(t), p(out)) == -2


# ---- whole sessions ------------------------------------------------------------------------------------------------------------------------
def check_session(por, s, ref_eval, ref_reset, toks, C_, n_batch, bos, what, ppl_kwargs=None):
    got_ppl, got_terms = s.perplexity(toks, return_terms=True, **(ppl_kwargs if ppl_kwargs is not None else {"bos": bos}))
    want_ppl, want_terms = por.perplexity(ref_eval, ref_reset, toks, C_, n_batch, bos)
    assert len(got_ppl) == len(want_ppl) == toks.size // C_, (what, len(got_ppl))
    same_bits(got_terms, want_terms, what + " terms")
    same_bits(got_ppl, want_ppl, what + " perplexities")
    assert s.n_past == C_, (what, s.n_past)
    assert np.isfinite(got_ppl).all() and min(got_ppl) > 1.0, got_ppl
    return got_ppl


def tokens_for(hp, C_, seed=0x99):
    return synth.make_tokens(hp, C_ * 5 // 2, seed=seed)       # 2.5 chunks: the half chunk is not scored


LLAMA_CASES = [("tiny8", B.Q4_0, 128, 1), ("tiny8", B.Q4_0, 64, 1), ("tiny8", B.Q4_0, 64, 8),
               ("tiny8", B.Q4_0, 64, 32), ("tiny8", B.Q4_0, 64, 64),
               ("gqa8", B.Q5_1, 64, 8), ("gqa8", B.Q5_1, 64, 64), ("tiny8", B.Q4_0, 1280, 32), ("tiny8", B.Q4_0, 1280, 1280)]


@pytest.mark.parametrize("cfg,wtype,C_,n_batch", LLAMA_CASES)
def test_llama_perplexity(ref, orc, por, cfg, wtype, C_, n_batch):
    hp, tens = synth.make_llama(dict(synth.CONFIGS[cfg], n_ctx=C_), wtype, orc.quantize)
    mr = ref.llama(hp, tens, n_threads=8, n_batch=max(n_batch, 8))
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=C_), tens)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=n_batch))
    toks = tokens_for(hp, C_)
    seen = []
    got = check_session(por, s, mr.eval, mr.reset, toks, C_, n_batch, 1, f"{cfg} C={C_} n_batch={n_batch}",
                        ppl_kwargs=dict(callback=lambda i, p: seen.append((i, p))))                # the default bos: LLaMA has none -> 1
    assert seen == list(enumerate(got))
    # the session goes on: rewind into the last chunk and evaluate, as the reference does after its loop
    half = C_ // 2
    s.rewind(half); mr.set_n_past(half)
    nxt = synth.make_tokens(hp, min(3, n_batch), seed=5)
    same_bits(s.evaluate(nxt, all_logits=True), mr.eval(nxt), "evaluate after perplexity")
    s.close(); m.close(); mr.close()


def test_llama_f16_file_perplexity(ref, por, tmp_path):
    from llm_b200.loader import load, write_llama
    f16 = lambda t, w: np.ascontiguousarray(w, np.float32).astype(np.float16)
    hp, tens = synth.make_llama(dict(synth.CONFIGS["tiny8"], n_ctx=64), B.F16, f16)
    path = str(tmp_path / "f16.bin")
    write_llama(path, hp, tens, synth.tensor_shapes(hp))
    mr = ref.llama(hp, tens, n_threads=8, n_batch=32)
    m = load(path, llm_b200.ModelParameters(context_size=64))
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=32))
    check_session(por, s, mr.eval, mr.reset, tokens_for(hp, 64), 64, 32, 1, "F16 file")
    s.close(); m.close(); mr.close()


def test_zero_chunks_leave_the_session_alone(orc):
    hp, tens = synth.make_llama(dict(synth.CONFIGS["tiny8"], n_ctx=64), B.Q4_0, orc.quantize)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=64), tens)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=16))
    s.evaluate(synth.make_tokens(hp, 5))
    assert s.perplexity(synth.make_tokens(hp, 63)) == [] and s.n_past == 5
    s.close(); m.close()


# the GPT-NeoX family at C = 64: (name, model class, make(hp) -> (hp, tensors), reference constructor)
def _neox_family(orc, name, n_ctx):
    from llm_b200.neox import Bloom, GptJ, GptNeoX, Gpt2, Mpt
    q = orc.quantize
    if name in ("neox", "neox-seq"):
        hp, tens = synth.make_neox(dict(synth.NEOX_CONFIGS["neox-tiny" if name == "neox" else "neox-tiny-seq"], n_ctx=n_ctx), B.Q4_0, q)
        return GptNeoX, hp, tens, lambda nb: B.RefLib("ref").neox(hp, tens, n_threads=8, n_batch=nb)
    if name == "gpt2":
        hp, tens = synth.make_gpt2(dict(synth.GPT2_CONFIGS["gpt2-tiny"], n_ctx=n_ctx), B.Q8_0, q)
        return Gpt2, hp, tens, lambda nb: B.RefLib("ref").gpt2(hp, tens, n_threads=8, n_batch=nb)
    if name in ("mpt", "bloom"):
        from oracle import alibi as A
        if not A.have_ref():
            pytest.skip("oracle/_ref/libggml_alibi.so not built")
        arch, cls, make, cfg = (A.MPT, Mpt, A.make_mpt, A.MPT_CONFIGS["mpt-tiny"]) if name == "mpt" else (A.BLOOM, Bloom, A.make_bloom, A.BLOOM_CONFIGS["bloom-tiny"])
        hp, tens = make(dict(cfg, n_ctx=n_ctx), B.Q5_0, q)
        return cls, hp, tens, lambda nb: A.RefAlibi(hp, tens, arch, n_threads=8, n_batch=nb)
    from oracle import gptj as J
    if not J.have_ref():
        pytest.skip("oracle/_ref/libggml_gptj.so not built")
    hp, tens = J.make_gptj(dict(J.GPTJ_CONFIGS["gptj-hd64"], n_ctx=n_ctx), B.Q4_1, q)
    return GptJ, hp, tens, lambda nb: J.RefGptJ(hp, tens, n_threads=8, n_batch=nb)


@pytest.mark.parametrize("n_batch", [1, 8, 32, 64])
@pytest.mark.parametrize("name", ["neox", "neox-seq", "gpt2", "mpt", "bloom", "gptj"])
def test_neox_family_perplexity(ref, orc, por, name, n_batch):
    cls, hp, tens, make_ref = _neox_family(orc, name, 64)
    cpu = make_ref(max(n_batch, 8))
    m = cls(hp, tens)
    s = m.start_session(n_batch)
    check_session(por, s, cpu.eval, cpu.reset, tokens_for(hp, 64, seed=0x4E + n_batch), 64, n_batch, 1, f"{name} n_batch={n_batch}")
    s.rewind(0); cpu.reset()
    nxt = synth.make_tokens(hp, min(5, n_batch), seed=6)
    same_bits(s.evaluate(nxt, all_logits=True), cpu.eval(nxt), "evaluate after perplexity")
    s.close(); m.close(); cpu.close()


@pytest.mark.parametrize("n_batch", [32, 1280])
def test_neox_perplexity_1280(ref, orc, por, n_batch):
    cls, hp, tens, make_ref = _neox_family(orc, "neox", 1280)
    cpu = make_ref(n_batch)
    m = cls(hp, tens)
    s = m.start_session(n_batch)
    check_session(por, s, cpu.eval, cpu.reset, tokens_for(hp, 1280), 1280, n_batch, 1, f"neox C=1280 n_batch={n_batch}")
    s.close(); m.close(); cpu.close()


@pytest.mark.parametrize("name,token", [("mpt", b"<|padding|>"), ("bloom", b"<s>")])
def test_default_bos_from_the_vocabulary(ref, orc, por, name, token):
    """MPT and BLOOM replace each chunk's first token by their vocabulary's <|padding|> / <s> (bot_token_id); without a vocabulary, by 1"""
    cls, hp, tens, make_ref = _neox_family(orc, name, 64)
    vocab = [b"tok%d" % i for i in range(hp["n_vocab"])]
    vocab[7] = token
    cpu = make_ref(32)
    m = cls(hp, tens, vocabulary=[(t, 0.0) for t in vocab])
    assert m.bot_token_id() == 7
    s = m.start_session(32)
    check_session(por, s, cpu.eval, cpu.reset, tokens_for(hp, 64), 64, 32, 7, f"{name} default bos", ppl_kwargs={})
    s.close(); m.close(); cpu.close()
    m = cls(hp, tens)
    assert m.bot_token_id() is None
    m.close()


def test_fast_session_runs(orc, capsys):
    """B200_SESSION_FAST: not the reference's logits, so its perplexity is reported, not compared"""
    hp, tens = synth.make_llama(dict(synth.CONFIGS["tiny8"], n_ctx=64), B.Q4_0, orc.quantize)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=64), tens)
    toks = tokens_for(hp, 64)
    out = {}
    for flags in (0, 4):
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=32, flags=flags))
        out[flags] = s.perplexity(toks)
        assert np.isfinite(out[flags]).all() and s.n_past == 64
        s.close()
    with capsys.disabled():
        print(f"\nperplexity per chunk, tiny8 Q4_0 C=64: exact {out[0]}  FAST {out[4]}")
    m.close()


def test_refusals(orc):
    L = lib()
    hp, tens = synth.make_llama(dict(synth.CONFIGS["tiny8"], n_ctx=64), B.Q4_0, orc.quantize)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=64), tens)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=16))
    s.evaluate(synth.make_tokens(hp, 3))
    toks = tokens_for(hp, 64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    ppl, n_chunk = np.empty(4, np.float32), C.c_int32(-1)
    V = hp["n_vocab"]
    for bos in (-1, V):
        assert L.b200_session_perplexity(s._s, p(toks), toks.size, bos, p(ppl), None, C.byref(n_chunk)) == -2
    for bad in (-1, V):
        t = toks.copy(); t[100] = bad
        assert L.b200_session_perplexity(s._s, p(t), t.size, 1, p(ppl), None, C.byref(n_chunk)) == -2
    assert L.b200_session_perplexity(s._s, None, toks.size, 1, p(ppl), None, C.byref(n_chunk)) == -2
    assert L.b200_session_perplexity(s._s, p(toks), toks.size, 1, None, None, C.byref(n_chunk)) == -2
    assert L.b200_session_perplexity(s._s, p(toks), toks.size, 1, p(ppl), None, None) == -2
    assert L.b200_session_perplexity(s._s, p(toks), -1, 1, p(ppl), None, C.byref(n_chunk)) == -2
    assert L.b200_session_perplexity(None, p(toks), toks.size, 1, p(ppl), None, C.byref(n_chunk)) == -2
    assert s.n_past == 3, "a refused call changes nothing"
    with pytest.raises(RuntimeError):
        s.perplexity(toks, bos=V)
    s.close(); m.close()
    from llm_b200.neox import GptNeoX
    hp2, tens2 = synth.make_neox(synth.NEOX_CONFIGS["neox-tiny"], B.Q4_0, orc.quantize)
    mn = GptNeoX(hp2, tens2)
    sn = mn.start_session(8)
    assert L.b200_neox_perplexity(sn._s, p(toks), toks.size, hp2["n_vocab"], p(ppl), None, C.byref(n_chunk)) == -2
    assert L.b200_neox_perplexity(None, p(toks), toks.size, 1, p(ppl), None, C.byref(n_chunk)) == -2
    sn.close(); mn.close()


def test_tensor_parallel_refused(orc):
    from llm_b200 import _lib
    from llm_b200.tp import TpLlama
    L = lib()
    hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], B.Q4_0, orc.quantize)
    m = TpLlama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens, rank=0, world=2, device=0)
    cfg = _lib.SessionConfig(n_batch=8, flags=0)
    sp = L.b200_model_start_session(m._m, C.byref(cfg))
    assert sp
    toks = synth.make_tokens(hp, 2 * hp["n_ctx"])
    ppl, n_chunk = np.empty(2, np.float32), C.c_int32(-1)
    assert L.b200_session_perplexity(sp, toks.ctypes.data_as(C.c_void_p), toks.size, 1, ppl.ctypes.data_as(C.c_void_p), None, C.byref(n_chunk)) == -2
    L.b200_session_free(sp)
    m.close()
