"""Text generation on the device (sample.cu, SessionCore::infer_next_token): the sampler against its plain-C restatement
(oracle/sampler_oracle.c) bit for bit, and generation against the reference's own graphs (oracle/_ref).

  b200_op_sample      vocabularies of 32000 / 32001 / 50257 / 65024 / 250880 entries; k 1 / 40 / 1024, p 0.95 / 1.0, T 0.1 / 0.8 / 1.0,
                      last_n 0 / 64 / > n_past; ties at the max and across the k-th place; -inf entries; a NaN row (SamplerFailure)
  greedy parity       LLaMA (MHA Q4_0, GQA Q5_1, an F16 file, an F32 cache), GPT-NeoX, GPT-2, MPT, BLOOM, GPT-J: a prompt, then k = 1 steps across a
                      256-position decode-graph bucket; every id is the argmax of the reference's row, the last row and both caches are the
                      reference's, tokens() is prompt + ids
  default chain       three seeds, 64 steps: every id is the C restatement on the reference's row with the same history and draw index
  stopping            end of text, maximum_token_count, a callback Halt, ContextFull at n_past = n_ctx - 1
  rewind              replaying the draws after a rewind gives the same ids, and a fresh session fed the same prefix agrees
  other sessions      FAST sessions generate; tensor-parallel sessions are refused"""
import ctypes as C

import numpy as np
import pytest

import llm_b200
from llm_b200 import ModelKVMemoryType as KV
from llm_b200 import _lib
from oracle import bindings as B
from oracle import synth

pytestmark = pytest.mark.gpu

GREEDY = llm_b200.InferenceParameters(llm_b200.Sampler(repetition_penalty=1.0, top_k=1))


@pytest.fixture(scope="module")
def so():
    from oracle.sampler import SamplerOracle
    return SamplerOracle()


def lib():
    L = _lib.lib()
    assert L.b200_init(0) == 0
    return L


def op_sample(row, hist, n_past, penalty=1.30, last_n=64, k=40, p=0.95, t=0.80, seed=0, draw=0):
    L = lib()
    row = np.ascontiguousarray(row, np.float32)
    hist = np.ascontiguousarray(hist if hist is not None and len(hist) else [0], np.int32)
    sp = _lib.SamplerParams(penalty, last_n, k, p, t, seed, draw)
    kk = min(k, row.size, 1024)
    ids, probs = np.empty(kk, np.int32), np.empty(kk, np.float32)
    tok, n_kept = C.c_int32(-1), C.c_int32(0)
    rc = L.b200_op_sample(row.ctypes.data_as(C.c_void_p), row.size, hist.ctypes.data_as(C.c_void_p), n_past, C.byref(sp), C.byref(tok),
                          C.byref(n_kept), ids.ctypes.data_as(C.c_void_p), probs.ctypes.data_as(C.c_void_p))
    return rc, tok.value, n_kept.value, ids, probs


def same_bits(got, want, what):
    g, w = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = g.view(np.uint32) != w.view(np.uint32)
    assert not bad.any(), (what, int(bad.sum()), g[bad][:4], w[bad][:4])


# ---- the sampler on host rows ------------------------------------------------------------------------------------------------------------------
def edge_row(rng, V, k):
    """normal logits with three ties at the max, a run of ties across the k-th place, and some -inf entries"""
    x = (rng.standard_normal(V) * 3).astype(np.float32)
    order = np.argsort(-x, kind="stable")
    x[order[:3]] = x[order[0]]
    kk = min(k, V, 1024)
    lo, hi = max(kk - 3, 3), min(kk + 3, V)
    if hi > lo:
        x[order[lo:hi]] = x[order[lo]]
    x[rng.choice(V, 17, replace=False)] = -np.inf
    return x


PARAMS = [dict(k=1, p=0.95, t=0.8, last_n=64), dict(k=40, p=0.95, t=0.8, last_n=64), dict(k=40, p=1.0, t=0.1, last_n=0),
          dict(k=1024, p=0.95, t=1.0, last_n=64), dict(k=1024, p=1.0, t=0.8, last_n=500), dict(k=40, p=0.95, t=1.0, last_n=500)]


@pytest.mark.parametrize("V", [32000, 32001, 50257, 65024, 250880])
@pytest.mark.parametrize("pi", range(len(PARAMS)))
def test_op_sample_matches_oracle(so, V, pi):
    prm = PARAMS[pi]
    rng = np.random.default_rng(V + 97 * pi)
    x = edge_row(rng, V, prm["k"])
    top = np.argsort(-x, kind="stable")[:50]
    hist = np.concatenate([rng.choice(top, 60), rng.integers(0, V, 60)]).astype(np.int32)      # repeated ids, many of them near the top
    n_past = hist.size
    for seed, draw in ((0, 0), (11, 5), (2**63 + 3, 1000)):
        kw = dict(penalty=1.30, last_n=prm["last_n"], k=prm["k"], p=prm["p"], t=prm["t"], seed=seed, draw=draw)
        rc, tok, n_kept, ids, probs = op_sample(x, hist, n_past, **kw)
        orc, otok, on_kept, oids, oprobs = so.sample(x, hist, n_past, **kw)
        assert rc == 0 and orc == 0
        assert ids.tolist() == oids.tolist(), (V, prm)
        same_bits(probs, oprobs, f"V={V} {prm} probabilities")
        assert (tok, n_kept) == (otok, on_kept), (V, prm, seed, draw)


def test_op_sample_small_vocabulary_and_no_history(so):
    rng = np.random.default_rng(3)
    for V in (1, 7, 320, 4096, 4097):
        x = (rng.standard_normal(V)).astype(np.float32)
        for k in (1, 40, 5000):
            got = op_sample(x, None, 0, k=k, seed=V, draw=k)
            want = so.sample(x, None, 0, k=k, seed=V, draw=k)
            assert got[:3] == want[:3] and got[3].tolist() == want[3].tolist(), (V, k)
            same_bits(got[4], want[4], f"V={V} k={k}")


def test_op_sample_nan_is_a_sampler_failure():
    x = np.zeros(32000, np.float32)
    x[31999] = np.nan
    assert op_sample(x, None, 0)[0] == -6
    assert op_sample(np.zeros(32000, np.float32), None, 0)[0] == 0       # the next call is not affected


def test_op_sample_refusals():
    x = np.zeros(100, np.float32)
    for bad in (dict(k=0), dict(t=0.0), dict(penalty=0.0), dict(last_n=-1), dict(p=float("nan"))):
        assert op_sample(x, None, 0, **bad)[0] == -2, bad


# ---- generation against the reference --------------------------------------------------------------------------------------------------------
def step(s, params, rng):
    """one infer_next_token; an end-of-text token (a model loaded from a file has a vocabulary) is returned like any other"""
    try:
        return s.infer_next_token(params, rng)
    except llm_b200.EndOfText as e:
        return e.token


def f16(t, w):
    return np.ascontiguousarray(w, np.float32).astype(np.float16)


def llama_case(ref, orc, tmp_path, name, n_ctx):
    """(native session, reference model, hp, kv compare)"""
    from oracle import kv32
    cfg, wtype = {"mha": ("tiny8", B.Q4_0), "gqa": ("gqa8", B.Q5_1), "f16": ("tiny8", B.F16), "kv32": ("tiny8", B.Q4_0)}[name]
    hp, tens = synth.make_llama(dict(synth.CONFIGS[cfg], n_ctx=n_ctx), wtype, f16 if wtype == B.F16 else orc.quantize)
    if name == "f16":
        from llm_b200.loader import load, write_llama
        path = str(tmp_path / "f16.bin")
        write_llama(path, hp, tens, synth.tensor_shapes(hp))
        m = load(path, llm_b200.ModelParameters(context_size=n_ctx))
    else:
        m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=n_ctx), tens)
    if name == "kv32":
        if not kv32.have_ref():
            pytest.skip("oracle/_ref/*_kv32.so not built")
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64, memory_k_type=KV.Float32, memory_v_type=KV.Float32))
        cpu = kv32.ref_lib().llama(hp, tens, n_threads=16, n_batch=64)
        kv = lambda which: kv32.kv_f32(cpu, which)
    else:
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64))
        cpu = ref.llama(hp, tens, n_threads=16, n_batch=64)
        kv = cpu.kv

    def kv_equal():
        for which in (0, 1):
            a = s.kv(which)
            assert np.array_equal(a.view(np.uint8), kv(which)[:a.size].view(np.uint8)), which
    return m, s, cpu, hp, kv_equal


def neox_case(ref, orc, name, n_ctx):
    from llm_b200.neox import Bloom, Gpt2, GptJ, GptNeoX, Mpt
    q = orc.quantize
    if name == "neox":
        hp, tens = synth.make_neox(dict(synth.NEOX_CONFIGS["neox-tiny"], n_ctx=n_ctx), B.Q4_0, q)
        m, cpu, v_by_pos = GptNeoX(hp, tens), B.RefLib("ref").neox(hp, tens, n_threads=8, n_batch=64), False
    elif name == "gpt2":
        hp, tens = synth.make_gpt2(dict(synth.GPT2_CONFIGS["gpt2-tiny"], n_ctx=n_ctx), B.Q8_0, q)
        m, cpu, v_by_pos = Gpt2(hp, tens), B.RefLib("ref").gpt2(hp, tens, n_threads=8, n_batch=64), True
    elif name in ("mpt", "bloom"):
        from oracle import alibi as A
        if not A.have_ref():
            pytest.skip("oracle/_ref/libggml_alibi.so not built")
        arch, cls, make, cfg = (A.MPT, Mpt, A.make_mpt, A.MPT_CONFIGS["mpt-tiny"]) if name == "mpt" else (A.BLOOM, Bloom, A.make_bloom, A.BLOOM_CONFIGS["bloom-tiny"])
        hp, tens = make(dict(cfg, n_ctx=n_ctx), B.Q5_0, q)
        m, cpu, v_by_pos = cls(hp, tens), A.RefAlibi(hp, tens, arch, n_threads=8, n_batch=64), True
    else:
        from oracle import gptj as J
        if not J.have_ref():
            pytest.skip("oracle/_ref/libggml_gptj.so not built")
        hp, tens = J.make_gptj(dict(J.GPTJ_CONFIGS["gptj-hd64"], n_ctx=n_ctx), B.Q4_1, q)
        m, cpu, v_by_pos = GptJ(hp, tens), J.RefGptJ(hp, tens, n_threads=8, n_batch=64), False
    s = m.start_session(64)

    def kv_equal():
        nl, e = hp["n_layer"], hp["n_embd"]
        assert np.array_equal(s.kv(0), cpu.kv(0)), "K"
        v = cpu.kv(1)
        if v_by_pos:
            v = v.reshape(nl, n_ctx, e).transpose(0, 2, 1).ravel()
        assert np.array_equal(s.kv(1), v), "V"
    return m, s, cpu, hp, kv_equal


def ref_rows(cpu, toks):
    """the reference's rows of toks, fed in batches of its n_batch (64)"""
    rows = [np.asarray(cpu.eval(np.asarray(toks[i:i + 64], np.int32)), np.float32).reshape(len(toks[i:i + 64]), -1) for i in range(0, len(toks), 64)]
    return np.concatenate(rows, 0)


CASES = ["llama-mha", "llama-gqa", "llama-f16", "llama-kv32", "neox", "gpt2", "mpt", "bloom", "gptj"]


def make_case(ref, orc, tmp_path, name, n_ctx=512):
    if name.startswith("llama-"):
        return llama_case(ref, orc, tmp_path, name[6:], n_ctx)
    return neox_case(ref, orc, name, n_ctx)


@pytest.mark.parametrize("name", CASES)
def test_greedy_matches_reference(ref, orc, tmp_path, name):
    """k = 1, no penalty: each id is the argmax (first on ties) of the reference's row, across the 256-position graph bucket"""
    m, s, cpu, hp, kv_equal = make_case(ref, orc, tmp_path, name)
    prompt = synth.make_tokens(hp, 250, seed=0x6E)
    want = ref_rows(cpu, prompt)[-1]
    if name.startswith("llama"):
        for i in range(0, prompt.size, 64):
            s.evaluate(prompt[i:i + 64])
    else:
        s.feed_prompt(prompt)
    rng = llm_b200.Rng(1)
    ids = []
    for i in range(14):                              # positions 250 .. 263
        tok = step(s, GREEDY, rng)
        assert tok == int(np.argmax(want)), (name, i, tok, int(np.argmax(want)))
        ids.append(tok)
        want = ref_rows(cpu, [tok])[-1]
    assert s.n_past == 264 and rng.draw == 14
    same_bits(s.last_logits, want, f"{name} last_logits")
    kv_equal()
    assert s.tokens().tolist() == prompt.tolist() + ids
    s.close(); m.close(); cpu.close()


@pytest.mark.parametrize("seed", [0, 7, 2**64 - 1])
def test_default_chain_matches_restatement(ref, orc, tmp_path, so, seed):
    """the reference defaults (penalty 1.3 over 64, k 40, p 0.95, T 0.8) for 64 steps: each id is the C restatement on the reference's row"""
    m, s, cpu, hp, _ = make_case(ref, orc, tmp_path, "llama-mha", n_ctx=256)
    prompt = synth.make_tokens(hp, 30, seed=seed & 0xFFFF)
    s.evaluate(prompt)
    row = ref_rows(cpu, prompt)[-1]
    hist = list(prompt)
    rng = llm_b200.Rng(seed)
    params = llm_b200.InferenceParameters()
    for i in range(64):
        rc, want, *_ = so.sample(row, np.array(hist, np.int32), len(hist), seed=rng.seed, draw=rng.draw)
        assert rc == 0
        tok = s.infer_next_token(params, rng)
        assert tok == want, (seed, i, tok, want)
        hist.append(tok)
        row = ref_rows(cpu, [tok])[-1]
    assert s.tokens().tolist() == hist
    same_bits(s.last_logits, row, "last_logits")
    s.close(); m.close(); cpu.close()


# ---- stopping --------------------------------------------------------------------------------------------------------------------------------
def small_llama(orc, n_ctx=128, vocabulary=None, flags=0):
    hp, tens = synth.make_llama(dict(synth.CONFIGS["tiny8"], n_ctx=n_ctx), B.Q4_0, orc.quantize)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=n_ctx), tens, vocabulary=vocabulary)
    return hp, m, m.start_session(llm_b200.InferenceSessionConfig(n_batch=32, flags=flags))


def test_infer_stops_at_end_of_text(orc):
    hp, m, s = small_llama(orc)
    prompt = synth.make_tokens(hp, 10)
    s.evaluate(prompt)
    rng = llm_b200.Rng(5)
    first = [s.infer_next_token(None, rng) for _ in range(6)]
    s.close(); m.close()
    eot = first[3]                                        # a token the model emits at step 4
    vocab = [b"t%d" % i for i in range(hp["n_vocab"])]
    vocab[eot] = b"</s>"
    hp, m, s = small_llama(orc, vocabulary=vocab)
    assert m.eot_token_id() == eot
    seen = []
    stats = s.infer(llm_b200.InferenceRequest(prompt), llm_b200.Rng(5), seen.append)
    stop = first.index(eot)
    assert seen == first[:stop], "the end-of-text token is not passed to the callback"
    assert s.n_past == 10 + stop + 1, "the end-of-text token has been evaluated"
    assert (stats.prompt_tokens, stats.predict_tokens) == (10, s.n_past)
    s.close(); m.close()
    _, m, _ = small_llama(orc, vocabulary=[b"x"] * hp["n_vocab"])
    assert m.eot_token_id() == 2                          # no "</s>": the reference's fallback
    m.close()


def test_infer_maximum_token_count_and_halt(orc):
    hp, m, s = small_llama(orc)
    prompt = synth.make_tokens(hp, 12)
    rng = llm_b200.Rng(9)
    seen = []
    s.infer(llm_b200.InferenceRequest(prompt, maximum_token_count=5), rng, seen.append)
    assert len(seen) == 5 and s.n_past == 17 and rng.draw == 5
    halt = []

    def cb(tok):
        halt.append(tok)
        return llm_b200.InferenceFeedback.Halt if len(halt) == 3 else llm_b200.InferenceFeedback.Continue
    s.infer(llm_b200.InferenceRequest([]), rng, cb)
    assert len(halt) == 3 and s.n_past == 20 and rng.draw == 8
    assert s.tokens().tolist() == prompt.tolist() + seen + halt
    s.close(); m.close()


def test_context_full_changes_nothing(orc):
    hp, m, s = small_llama(orc, n_ctx=128)
    toks = synth.make_tokens(hp, 127)
    for i in range(0, 127, 32):
        s.evaluate(toks[i:i + 32])
    assert s.n_past == 127
    before = s.last_logits.copy()
    rng = llm_b200.Rng(1)
    with pytest.raises(llm_b200.ContextFull):
        s.infer_next_token(None, rng)
    assert s.n_past == 127 and rng.draw == 0 and s.tokens().tolist() == toks.tolist()
    same_bits(s.last_logits, before, "last_logits")
    s.rewind(126)
    s.infer_next_token(None, rng)                          # 126 + 1 < 128 runs
    assert s.n_past == 127 and rng.draw == 1
    with pytest.raises(llm_b200.ContextFull):
        s.infer_next_token(None, rng)
    assert s.n_past == 127 and rng.draw == 1
    with pytest.raises(llm_b200.ContextFull):
        s.infer(llm_b200.InferenceRequest([]), rng)
    s.close(); m.close()


# ---- rewind --------------------------------------------------------------------------------------------------------------------------------
def test_rewind_replays_the_same_draws(orc):
    hp, m, s = small_llama(orc, n_ctx=256)
    prompt = synth.make_tokens(hp, 20)
    s.evaluate(prompt)
    rng = llm_b200.Rng(42)
    params = llm_b200.InferenceParameters()
    ids = [s.infer_next_token(params, rng) for _ in range(30)]
    r = 12
    every = prompt.tolist() + ids                          # 50 positions
    # rewind past the r tokens and one more, and evaluate that one again: last_logits is the row the first of the r tokens was drawn from
    s.rewind(len(every) - r - 1)
    s.evaluate(np.array(every[len(every) - r - 1:len(every) - r], np.int32))
    rng.draw -= r
    again = [s.infer_next_token(params, rng) for _ in range(r)]
    assert again == ids[-r:]
    assert s.tokens().tolist() == every
    fresh = m.start_session(llm_b200.InferenceSessionConfig(n_batch=32))
    prefix = np.array(prompt.tolist() + ids[:-r], np.int32)
    for i in range(0, prefix.size, 32):
        fresh.evaluate(prefix[i:i + 32])
    rng2 = llm_b200.Rng(42)
    rng2.draw = 30 - r
    assert [fresh.infer_next_token(params, rng2) for _ in range(r)] == ids[-r:]
    same_bits(fresh.last_logits, s.last_logits, "last_logits")
    fresh.close(); s.close(); m.close()


# ---- other sessions ---------------------------------------------------------------------------------------------------------------------------
def test_fast_session_generates(orc):
    hp, m, s = small_llama(orc, flags=4)
    s.evaluate(synth.make_tokens(hp, 10))
    rng = llm_b200.Rng(3)
    ids = [s.infer_next_token(None, rng) for _ in range(20)]
    assert all(0 <= t < hp["n_vocab"] for t in ids) and s.n_past == 30
    assert s.tokens()[10:].tolist() == ids
    s.close(); m.close()


def test_infer_before_evaluate_and_refusals(orc):
    hp, m, s = small_llama(orc)
    with pytest.raises(RuntimeError):
        s.infer_next_token(None, llm_b200.Rng(0))           # no row evaluated yet
    s.evaluate(synth.make_tokens(hp, 4))
    with pytest.raises(RuntimeError):
        s.infer_next_token(llm_b200.InferenceParameters(llm_b200.Sampler(top_k=0)), llm_b200.Rng(0))
    assert s.n_past == 4
    L = lib()
    tok = C.c_int32(0)
    sp = _lib.SamplerParams(1.3, 64, 40, 0.95, 0.8, 0, 0)
    assert L.b200_session_infer_next_token(None, C.byref(sp), C.byref(tok)) == -2
    assert L.b200_session_infer_next_token(s._s, None, C.byref(tok)) == -2
    assert L.b200_session_infer_next_token(s._s, C.byref(sp), None) == -2
    assert s.n_past == 4
    s.close(); m.close()


def test_tensor_parallel_refused(orc):
    from llm_b200.tp import TpLlama
    L = lib()
    hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], B.Q4_0, orc.quantize)
    m = TpLlama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens, rank=0, world=2, device=0)
    cfg = _lib.SessionConfig(n_batch=8, flags=0)
    sp_ = L.b200_model_start_session(m._m, C.byref(cfg))
    assert sp_
    sp = _lib.SamplerParams(1.3, 64, 40, 0.95, 0.8, 0, 0)
    tok = C.c_int32(0)
    assert L.b200_session_infer_next_token(sp_, C.byref(sp), C.byref(tok)) == -2
    L.b200_session_free(sp_)
    m.close()
