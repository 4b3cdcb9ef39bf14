"""Batched decode across the sessions of one LLaMA model (b200_model_evaluate_sessions / b200_model_infer_next_tokens): one step advances n
sessions, and every session must be bit-identical to a twin -- a second session of the same model, fed the same prompt and stepped alone with
evaluate([tok]) (the single-session paths the other tests hold to the reference).  Equal means equal bit patterns.

  parity          tiny8 / gqa8 in Q4_0 at n = 1 .. 64 (both sides of the exact mat-mul's 16-row switch and of the K-quant kernels' 32-row
                  switch); Q5_1, Q8_0, F16 and a Q4_K_M mix on f16 and f32 caches; every session at its own n_past; after every step the
                  logits row, both caches, n_past and tokens() of each session equal its twin's
  oracle          three sessions against the C oracle's own graphs, logits and caches
  7B geometry     the 7b-2l shapes at n = 2, 16, 17
  long context    sessions at n_past 0, 3071, 3072, 3500 and 4094 of a 4096-position context, up to its last slot, f16 and f32 caches
  interleaving    batched step, a graph step on one session, a rewind of another, a batched step, snapshots
  generation      greedy infer_next_tokens over 32 steps; the default chain with a seed per session against infer_next_token and or_sample;
                  a NaN row fails its own session only
  refusals        every refusal of the contract leaves every session unchanged
  launches        the launch count of a batched step does not depend on n"""
import numpy as np
import pytest

import llm_b200
from llm_b200 import ModelKVMemoryType as KV
from oracle import bindings as B
from oracle import kquant as KQ
from oracle import synth

pytestmark = pytest.mark.gpu

F16 = 1
NS = [1, 2, 5, 15, 16, 17, 31, 32, 33, 64]
GREEDY = llm_b200.InferenceParameters(llm_b200.Sampler(repetition_penalty=1.0, top_k=1))


def same_bits(got, want, what):
    g, w = np.asarray(got), np.asarray(want)
    assert g.shape == w.shape and g.dtype == w.dtype, (what, g.shape, w.shape, g.dtype, w.dtype)
    bad = g.view(np.uint8).reshape(g.shape + (-1,)) != w.view(np.uint8).reshape(w.shape + (-1,))
    assert not bad.any(), (what, int(bad.any(axis=-1).sum()))


def make_model(cfg, wtype, n_ctx=None, mix=None, seed=0x5EED0001):
    """a model of synth.CONFIGS[cfg] with weights synthesised on the device; mix: a K-quant mix's type per tensor (n_vocab raised to 512 and,
    for GQA, 4 KV heads, so that every matrix takes whole super-blocks both ways, as the mix's quantizer requires)"""
    hp = dict(synth.CONFIGS[cfg])
    hp["wtype"] = wtype
    types = None
    if mix:
        hp["n_vocab"] = 512
        if hp["n_head_kv"] != hp["n_head"]:
            hp["n_head_kv"] = hp["n_head"] // 2
        types = KQ.mix_types(hp, mix)
        hp["wtype"] = KQ.MIXES[mix][0]
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=n_ctx or hp["n_ctx"]), tensor_types=types)
    m.synthesize(seed)
    return m


def start(m, kv32=False, n_batch=512, flags=0):
    t = KV.Float32 if kv32 else KV.Float16
    return m.start_session(llm_b200.InferenceSessionConfig(n_batch=n_batch, flags=flags, memory_k_type=t, memory_v_type=t))


def pairs(m, n, prompt_lens, kv32=False, seed=1):
    """n (batched, twin) session pairs, pair i fed the same prompt of prompt_lens[i] ids (0: nothing)"""
    rng = np.random.default_rng(seed)
    V = m.hyperparameters["n_vocab"]
    out = []
    for i in range(n):
        a, b = start(m, kv32), start(m, kv32)
        p = rng.integers(0, V, prompt_lens[i]).astype(np.int32)
        if p.size:
            a.feed_prompt(p)
            b.feed_prompt(p)
        out.append((a, b))
    return out


def check_pair(a, b, what, logits=None, kv=True):
    assert a.n_past == b.n_past, (what, a.n_past, b.n_past)
    if logits is not None:
        same_bits(logits, b.last_logits, what + " logits")
    same_bits(a.last_logits, b.last_logits, what + " last_logits")
    same_bits(a.tokens(), b.tokens(), what + " tokens")
    if kv:
        for w in (0, 1):
            same_bits(a.kv(w), b.kv(w), f"{what} kv{w}")


def state(s):
    """n_past, tokens(), the last row as the device holds it, both caches"""
    s._last_logits = None
    return (s.n_past, s.tokens(), s.last_logits.copy(), s.kv(0), s.kv(1))


def run_parity(m, n, kv32, steps=8, kv_every_step=True):
    n_ctx = m.context_size()
    lens = [(1 + 7 * i) % max(2, n_ctx - steps - 2) for i in range(n)]
    ps = pairs(m, n, lens, kv32)
    V = m.hyperparameters["n_vocab"]
    rng = np.random.default_rng(n)
    for step in range(steps):
        toks = rng.integers(0, V, n).astype(np.int32)
        got = m.evaluate_sessions([a for a, _ in ps], toks)
        assert got.shape == (n, V)
        for i, (a, b) in enumerate(ps):
            b.evaluate(toks[i:i + 1])
            check_pair(a, b, f"n={n} step {step} session {i}", logits=got[i], kv=kv_every_step or step == steps - 1)
    return ps


@pytest.mark.parametrize("cfg", ["tiny8", "gqa8"])
@pytest.mark.parametrize("n", NS)
def test_parity_q4_0(cfg, n):
    m = make_model(cfg, B.Q4_0)
    run_parity(m, n, kv32=False)


@pytest.mark.parametrize("cfg", ["tiny8", "gqa8"])
@pytest.mark.parametrize("wt", ["q4_0", "q5_1", "q8_0", "f16", "q4_K_M"])
@pytest.mark.parametrize("kv32", [False, True])
@pytest.mark.parametrize("n", [2, 17, 33])
def test_parity_types(cfg, wt, kv32, n):
    if wt == "q4_K_M":
        m = make_model(cfg, None, mix="q4_K_M")
    else:
        m = make_model(cfg, F16 if wt == "f16" else B.QUANT_TYPES[wt])
    run_parity(m, n, kv32, steps=4)


@pytest.mark.parametrize("kv32", [False, True])
def test_q4_k_m_all_batch_sizes(kv32):
    m = make_model("tiny8", None, mix="q4_K_M")
    for n in NS:
        run_parity(m, n, kv32, steps=2, kv_every_step=False)


def test_against_oracle(orc):
    """three sessions at different positions, each checked against the C oracle's graph on its own cache"""
    hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], B.Q4_0, orc.quantize)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tensors=tens)
    toks = synth.make_tokens(hp, 60)
    lens = [1, 9, 23]
    ss = [start(m) for _ in lens]
    mos = [orc.llama(hp, tens) for _ in lens]
    V = hp["n_vocab"]
    for s, mo, k in zip(ss, mos, lens):
        same_bits(s.feed_prompt(toks[:k]), np.asarray(mo.eval(toks[:k]), np.float32).reshape(-1, V)[-1], "prompt")
    for step in range(6):
        ids = np.array([toks[k + step] for k in lens], np.int32)
        got = m.evaluate_sessions(ss, ids)
        for i, (s, mo) in enumerate(zip(ss, mos)):
            same_bits(got[i], np.asarray(mo.eval(ids[i:i + 1]), np.float32).reshape(-1, V)[-1], f"step {step} session {i}")
    for s, mo in zip(ss, mos):
        for w in (0, 1):
            assert np.array_equal(s.kv(w), mo.kv(w)), w


@pytest.mark.parametrize("n", [2, 16, 17])
def test_7b_geometry(n):
    m = make_model("7b-2l", B.Q4_0)
    ps = pairs(m, n, [3 + 11 * i for i in range(n)])
    rng = np.random.default_rng(7)
    for step in range(3):
        toks = rng.integers(0, 32000, n).astype(np.int32)
        got = m.evaluate_sessions([a for a, _ in ps], toks)
        for i, (a, b) in enumerate(ps):
            b.evaluate(toks[i:i + 1])
            check_pair(a, b, f"7b n={n} step {step} session {i}", logits=got[i], kv=step == 2)


@pytest.mark.parametrize("kv32", [False, True])
def test_long_context(kv32):
    m = make_model("tiny8", B.Q4_0, n_ctx=4096)
    ps = pairs(m, 5, [0, 3071, 3072, 3500, 4094], kv32)
    rng = np.random.default_rng(4096)
    for step in range(2):                                       # 4094 -> 4095: the last slot
        toks = rng.integers(0, 320, 5).astype(np.int32)
        got = m.evaluate_sessions([a for a, _ in ps], toks)
        for i, (a, b) in enumerate(ps):
            b.evaluate(toks[i:i + 1])
            check_pair(a, b, f"long step {step} session {i}", logits=got[i])
    assert ps[4][0].n_past == 4096
    with pytest.raises(llm_b200.ContextFull):
        m.evaluate_sessions([a for a, _ in ps], np.zeros(5, np.int32))


def test_interleaving():
    """the graph's device n_past is stale after a batched step, as after a rewind: a graph step on one session must see the new n_past"""
    m = make_model("gqa8", B.Q4_0)
    ps = pairs(m, 4, [5, 12, 30, 7])
    A = [a for a, _ in ps]
    m.evaluate_sessions(A, np.array([1, 2, 3, 4], np.int32))
    for i, (a, b) in enumerate(ps):
        b.evaluate([i + 1])
    ps[0][0].evaluate([9]); ps[0][1].evaluate([9])              # a single graph step on one session
    ps[1][0].rewind(8); ps[1][1].rewind(8)                      # a rewind of another
    m.evaluate_sessions(A, np.array([11, 12, 13, 14], np.int32))
    for i, (a, b) in enumerate(ps):
        b.evaluate([11 + i])
    ps[2][0].evaluate([21]); ps[2][1].evaluate([21])            # and a graph step after it
    for i, (a, b) in enumerate(ps):
        check_pair(a, b, f"interleaved session {i}")
        sa, sb = a.get_snapshot(), b.get_snapshot()
        assert sa.npast == sb.npast
        for f in ("tokens", "last_logits", "memory_k", "memory_v"):
            same_bits(getattr(sa, f), getattr(sb, f), f"snapshot {f} {i}")


def test_greedy_generation():
    m = make_model("tiny8", B.Q5_1)
    ps = pairs(m, 6, [1, 4, 9, 16, 25, 36])
    A = [a for a, _ in ps]
    ra, rb = [llm_b200.Rng(i) for i in range(6)], [llm_b200.Rng(i) for i in range(6)]
    for step in range(32):
        ids = m.infer_next_tokens(A, GREEDY, ra)
        for i, (a, b) in enumerate(ps):
            assert ids[i] == b.infer_next_token(GREEDY, rb[i]), (step, i)
            assert ra[i].draw == rb[i].draw == step + 1
    for i, (a, b) in enumerate(ps):
        check_pair(a, b, f"greedy session {i}")


def test_default_chain_generation():
    from oracle.sampler import SamplerOracle
    so = SamplerOracle()
    m = make_model("gqa8", B.Q4_0)
    ps = pairs(m, 5, [2, 8, 20, 40, 70])
    A = [a for a, _ in ps]
    params = [llm_b200.InferenceParameters(llm_b200.Sampler(top_k=k)) for k in (40, 40, 1024, 5, 40)]
    ra, rb = [llm_b200.Rng(1000 + 17 * i) for i in range(5)], [llm_b200.Rng(1000 + 17 * i) for i in range(5)]
    for step in range(24):
        rows = [b.last_logits.copy() for _, b in ps]
        hists = [b.tokens() for _, b in ps]
        ids = m.infer_next_tokens(A, params, ra)
        for i, (a, b) in enumerate(ps):
            sp = params[i].sampler
            rc, want, _, _, _ = so.sample(rows[i], hists[i], len(hists[i]), sp.repetition_penalty, sp.repetition_last_n, sp.top_k, sp.top_p,
                                          sp.temperature, rb[i].seed, rb[i].draw)
            assert rc == 0 and ids[i] == want, (step, i, ids[i], want)
            assert ids[i] == b.infer_next_token(params[i], rb[i]), (step, i)
    for i, (a, b) in enumerate(ps):
        check_pair(a, b, f"chain session {i}")


def test_sampler_failure_is_per_session():
    m = make_model("tiny8", B.Q4_0)
    ps = pairs(m, 3, [3, 6, 9])
    snap = ps[1][0].get_snapshot()
    snap.last_logits = snap.last_logits.copy()
    snap.last_logits[17] = np.nan
    bad = llm_b200.InferenceSession.from_snapshot(snap, m)
    before = state(bad)
    A = [ps[0][0], bad, ps[2][0]]
    ra = [llm_b200.Rng(i) for i in range(3)]
    rb = [llm_b200.Rng(i) for i in range(3)]
    with pytest.raises(llm_b200.SamplerFailure) as ei:
        m.infer_next_tokens(A, GREEDY, ra)
    assert ei.value.sessions == [1] and ei.value.tokens[1] == -1
    assert ra[1].draw == 0 and ra[0].draw == ra[2].draw == 1
    after = state(bad)
    assert before[0] == after[0]
    for x, y, f in zip(before[1:], after[1:], ("tokens", "last_logits", "kv0", "kv1")):
        same_bits(y, x, "failed session " + f)
    for i in (0, 2):
        assert ei.value.tokens[i] == ps[i][1].infer_next_token(GREEDY, rb[i])
        check_pair(ps[i][0], ps[i][1], f"survivor {i}")


def test_refusals():
    m = make_model("tiny8", B.Q4_0)
    other = make_model("tiny8", B.Q4_0)
    ss = [start(m) for _ in range(3)]
    for i, s in enumerate(ss):
        s.feed_prompt([1 + i, 2, 3])
    fast = start(m, flags=4)                          # B200_SESSION_FAST
    fast.feed_prompt([1])
    f32 = start(m, kv32=True)
    f32.feed_prompt([1])
    foreign = start(other)
    foreign.feed_prompt([1])
    full = start(m)
    full.feed_prompt(np.arange(m.context_size(), dtype=np.int32) % 320)
    snapshot = [state(s) for s in ss]
    L = m.L
    ok = np.array([1, 2, 3], np.int32)

    def refused(sessions, toks, code):
        h = m._session_handles(sessions)
        toks = np.ascontiguousarray(toks, np.int32)
        assert L.b200_model_evaluate_sessions(m._m, h, len(sessions), toks.ctypes.data, None) == code
        sp = (llm_b200._lib.SamplerParams * max(1, len(sessions)))(*[llm_b200._lib.SamplerParams(1.0, 64, 1, 0.95, 0.8, 0, 0)] * len(sessions))
        out, st = np.zeros(max(1, len(sessions)), np.int32), np.zeros(max(1, len(sessions)), np.int32)
        if code == -2 and len(toks) and toks.min() >= 0 and toks.max() < 320 or code == -1:
            assert L.b200_model_infer_next_tokens(m._m, h, len(sessions), sp, out.ctypes.data, st.ctypes.data) == code
        for s, want in zip(ss, snapshot):
            got = state(s)
            assert got[0] == want[0]
            for g, w in zip(got[1:], want[1:]):
                same_bits(g, w, "refused")

    refused(ss[:2] + [foreign], ok, -2)                # another model's session
    refused([ss[0], ss[1], ss[0]], ok, -2)             # a duplicate
    refused(ss[:2] + [fast], ok, -2)                   # a FAST session
    refused(ss[:2] + [f32], ok, -2)                    # mixed KV types
    refused(ss[:2] + [full], ok, -1)                   # one full session among free ones
    refused([], np.zeros(0, np.int32), -2)             # n = 0
    many = [start(m) for _ in range(65)]
    for s in many:
        s.feed_prompt([1])
    refused(many, np.ones(65, np.int32), -2)           # n = 65
    refused(ss, np.array([1, 320, 2], np.int32), -2)   # an id outside the vocabulary
    refused(ss, np.array([1, -1, 2], np.int32), -2)
    bad = (llm_b200._lib.SamplerParams * 3)(*[llm_b200._lib.SamplerParams(1.0, 64, 0, 0.95, 0.8, 0, 0)] * 3)   # top_k 0
    out, st = np.zeros(3, np.int32), np.zeros(3, np.int32)
    assert L.b200_model_infer_next_tokens(m._m, m._session_handles(ss), 3, bad, out.ctypes.data, st.ctypes.data) == -2
    nearly = start(m)                                  # infer's rule is one slot stricter: n_past + 1 >= n_ctx
    nearly.feed_prompt(np.arange(m.context_size() - 1, dtype=np.int32) % 320)
    with pytest.raises(llm_b200.ContextFull):
        m.infer_next_tokens(ss[:2] + [nearly], GREEDY, [llm_b200.Rng(0) for _ in range(3)])
    for s, want in zip(ss, snapshot):
        assert state(s)[0] == want[0]


def test_launch_count_does_not_depend_on_n():
    m = make_model("gqa8", B.Q4_0)
    counts = {}
    for n in (2, 64):
        ss = [start(m) for _ in range(n)]
        for s in ss:
            s.feed_prompt([1, 2])
        m.evaluate_sessions(ss, np.full(n, 3, np.int32))
        counts[n] = {s.last_launches for s in ss}
    assert len(counts[2]) == 1 and counts[2] == counts[64], counts
