"""Ragged batched evaluation (b200_model_evaluate_ragged / b200_neox_evaluate_ragged): one step feeds n sessions of one model a chunk of
tokens each, and every session must be bit-identical to a twin -- a second session of the same model, fed the same prompt and stepped alone
with evaluate(chunk, all_logits) (the single-session paths the other tests hold to the reference).  Equal means equal bit patterns.

  chunks          tiny8 / gqa8: chunks of 1, 7, 8, 9 (the warp / tiled attention bound), 31, 32, 33 (tile edges), 64, 96 and 512 rows beside
                  one-token rows in the same step, every session at its own n_past, with and without all_logits; after every step the logits,
                  both caches, n_past, tokens() and last_logits of each session equal its twin's
  types           Q4_0, Q5_1, Q8_0, F16 and a Q4_K_M mix on f16 and F32 caches
  GEMM forms      8 x 16 rows (the step on the wgmma GEMM, each twin on mma.sync); the 7b-2l shapes at 8 x 64 rows
  edges           chunks ending on the last slot of a 4096-position context (both caches); a step of exactly B200_MAX_BATCH_ROWS rows
  oracle          ragged steps against the C oracle's own graphs, logits and caches
  GPT-NeoX family every architecture's small configs on f16 and F32 caches, GPT-2 up to its last wpe row, a mixed-type MPT file
  decode          all-ones ragged steps give evaluate_sessions' bits and launch counts; a mixed step adds exactly its tiled and gather launches
  feed_prompts    against feed_prompt alone: prompts longer than n_batch, different n_batch per session, an empty prompt, a split at the row cap
  afterwards      generation, snapshots, a rewind and a single-session graph step after ragged steps
  refusals        every refusal of the contract leaves every session unchanged"""
import functools

import numpy as np
import pytest

import llm_b200
from llm_b200 import ModelKVMemoryType as KV
from llm_b200 import neox
from oracle import alibi as A
from oracle import bindings as B
from oracle import gptj as J
from oracle import kquant as KQ
from oracle import neox_kquant as NK
from oracle import synth

pytestmark = pytest.mark.gpu

F16 = 1
MAX_ROWS = 4096
GREEDY = llm_b200.InferenceParameters(llm_b200.Sampler(repetition_penalty=1.0, top_k=1))


def same_bits(got, want, what):
    g, w = np.asarray(got), np.asarray(want)
    assert g.shape == w.shape and g.dtype == w.dtype, (what, g.shape, w.shape, g.dtype, w.dtype)
    if g.size == 0:
        return
    bad = g.view(np.uint8).reshape(g.shape + (-1,)) != w.view(np.uint8).reshape(w.shape + (-1,))
    assert not bad.any(), (what, int(bad.any(axis=-1).sum()))


# ---- LLaMA models and sessions ------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def make_model(cfg, wtype, n_ctx=None, mix=None, seed=0x5EED0001):
    """a model of synth.CONFIGS[cfg] with weights synthesised on the device (mix: a K-quant mix, as in test_gpu_batch_decode.py)"""
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
    if isinstance(m, neox.GptNeoX):
        return m.start_session(n_batch, t, t)
    return m.start_session(llm_b200.InferenceSessionConfig(n_batch=n_batch, flags=flags, memory_k_type=t, memory_v_type=t))


def pairs(m, prompt_lens, kv32=False, n_batch=512, seed=1):
    """(ragged, twin) session pairs, pair i fed the same prompt of prompt_lens[i] ids (0: nothing)"""
    rng = np.random.default_rng(seed)
    V = m.hyperparameters["n_vocab"]
    out = []
    for k in prompt_lens:
        a, b = start(m, kv32, n_batch), start(m, kv32, n_batch)
        p = rng.integers(0, V, k).astype(np.int32)
        if p.size:
            a.feed_prompt(p)
            b.feed_prompt(p)
        out.append((a, b))
    return out


def check_pair(a, b, what, kv=True):
    assert a.n_past == b.n_past, (what, a.n_past, b.n_past)
    same_bits(a.last_logits, b.last_logits, what + " last_logits")
    same_bits(a.tokens(), b.tokens(), what + " tokens")
    if kv:
        for w in (0, 1):
            same_bits(a.kv(w), b.kv(w), f"{what} kv{w}")


def state(s):
    """n_past, tokens(), the last row as the device holds it, both caches"""
    s._last_logits = None
    return (s.n_past, s.tokens(), s.last_logits.copy(), s.kv(0), s.kv(1))


def run_steps(m, ps, plan, all_logits=False, kv_every_step=True, seed=3):
    """plan: one list of chunk lengths per step, one length per pair (0: the pair sits the step out).  Every step is checked against the twins."""
    V = m.hyperparameters["n_vocab"]
    rng = np.random.default_rng(seed)
    for step, lens in enumerate(plan):
        idx = [i for i, c in enumerate(lens) if c]
        chunks = [rng.integers(0, V, lens[i]).astype(np.int32) for i in idx]
        got = m.evaluate_ragged([ps[i][0] for i in idx], chunks, all_logits=all_logits)
        assert len(got) == len(idx)
        for k, i in enumerate(idx):
            a, b = ps[i]
            want = b.evaluate(chunks[k], all_logits=all_logits)
            what = f"step {step} session {i} ({lens[i]} rows)"
            assert got[k].shape == ((lens[i], V) if all_logits else (V,)), (what, got[k].shape)
            same_bits(got[k], want, what + " logits")
            check_pair(a, b, what, kv=kv_every_step or step == len(plan) - 1)


# chunk lengths: across the warp / tiled bound (7, 8, 9), the tile edges (31, 32, 33), several tiles, beside one-token rows
LENS = [1, 7, 8, 9, 31, 32, 33, 64, 96, 1, 1]
PLAN = [LENS, LENS[3:] + LENS[:3], [1] * len(LENS), LENS[::-1], [0, 1, 0, 8, 0, 33, 0, 1, 7, 0, 9]]
PROMPTS = [0, 3, 17, 40, 1, 64, 5, 100, 0, 9, 2]


@pytest.mark.parametrize("cfg", ["tiny8", "gqa8"])
@pytest.mark.parametrize("all_logits", [False, True])
def test_chunks(cfg, all_logits):
    m = make_model(cfg, B.Q4_0, n_ctx=1024)
    run_steps(m, pairs(m, PROMPTS), PLAN, all_logits)


@pytest.mark.parametrize("cfg", ["tiny8", "gqa8"])
def test_n_batch_chunk(cfg):
    """a full 512-row chunk beside a tiled and a one-token chunk, then 64 sessions in one step"""
    m = make_model(cfg, B.Q4_0, n_ctx=1024)
    run_steps(m, pairs(m, [0, 11, 200]), [[512, 40, 1], [1, 512, 9]])
    ps = pairs(m, [(5 * i) % 70 for i in range(64)])
    run_steps(m, ps, [[(1, 8, 33, 2)[i % 4] for i in range(64)], [(9, 1, 1, 32)[i % 4] for i in range(64)]], kv_every_step=False)


@pytest.mark.parametrize("cfg", ["tiny8", "gqa8"])
@pytest.mark.parametrize("wt", ["q4_0", "q5_1", "q8_0", "f16", "q4_K_M"])
@pytest.mark.parametrize("kv32", [False, True])
def test_types(cfg, wt, kv32):
    if wt == "q4_K_M":
        m = make_model(cfg, None, n_ctx=512, mix="q4_K_M")
    else:
        m = make_model(cfg, F16 if wt == "f16" else B.QUANT_TYPES[wt], n_ctx=512)
    ps = pairs(m, [0, 7, 30, 2, 50], kv32)
    run_steps(m, ps, [[9, 1, 33, 8, 64], [1, 32, 1, 7, 1], [96, 8, 1, 31, 1]], all_logits=kv32)


def test_wgmma_step_against_mma_twins():
    """8 x 16 = 128 rows: the step's mat-muls run the wgmma GEMM while each twin's 16 rows run the mma.sync kernel"""
    m = make_model("tiny8", B.Q4_0, n_ctx=512)
    ps = pairs(m, [3 * i for i in range(8)])
    run_steps(m, ps, [[16] * 8, [16] * 8], all_logits=True)


def test_7b_geometry():
    m = make_model("7b-2l", B.Q4_0)
    ps = pairs(m, [2 + 13 * i for i in range(8)], n_batch=64)
    run_steps(m, ps, [[64] * 8, [1, 64, 1, 64, 8, 1, 33, 1]], kv_every_step=False)


@pytest.mark.parametrize("kv32", [False, True])
def test_last_slot_of_4096(kv32):
    m = make_model("tiny8", B.Q4_0, n_ctx=4096)
    ps = pairs(m, [4096 - 33, 4096 - 8, 4096 - 96 - 7, 4096 - 1, 3000], kv32)
    run_steps(m, ps, [[33, 8, 96, 1, 9], [0, 0, 7, 0, 32]])
    assert [a.n_past for a, _ in ps] == [4096, 4096, 4096, 4096, 3041]
    with pytest.raises(llm_b200.ContextFull):
        m.evaluate_ragged([ps[4][0], ps[0][0]], [[1], [2]])


def test_max_batch_rows():
    m = make_model("tiny8", B.Q4_0, n_ctx=1024)
    ps = pairs(m, [i for i in range(8)])
    run_steps(m, ps, [[512] * 8], kv_every_step=True)                     # exactly B200_MAX_BATCH_ROWS
    assert sum(a.n_past for a, _ in ps) - sum(range(8)) == MAX_ROWS
    before = [state(a) for a, _ in ps]
    extra = start(m)
    with pytest.raises(RuntimeError):
        m.evaluate_ragged([a for a, _ in ps] + [extra], [np.ones(512, np.int32)] * 8 + [[1]])
    for (a, _), want in zip(ps, before):
        got = state(a)
        assert got[0] == want[0]
        for g, w in zip(got[1:], want[1:]):
            same_bits(g, w, "refused")


def test_against_oracle(orc):
    """sessions at different positions, each ragged step checked against the C oracle's graph on its own cache"""
    hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], B.Q4_0, orc.quantize)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tensors=tens)
    toks = synth.make_tokens(hp, 120)
    lens = [1, 9, 23, 0]
    ss = [start(m, n_batch=64) for _ in lens]
    mos = [orc.llama(hp, tens) for _ in lens]
    V = hp["n_vocab"]
    for s, mo, k in zip(ss, mos, lens):
        if k:
            same_bits(s.feed_prompt(toks[:k]), np.asarray(mo.eval(toks[:k]), np.float32).reshape(-1, V)[-1], "prompt")
    pos = list(lens)
    for step, counts in enumerate([[8, 1, 33, 9], [1, 32, 7, 1], [31, 1, 1, 40]]):
        chunks = [toks[p:p + c] for p, c in zip(pos, counts)]
        got = m.evaluate_ragged(ss, chunks, all_logits=True)
        for i, (mo, ch) in enumerate(zip(mos, chunks)):
            same_bits(got[i], np.asarray(mo.eval(ch), np.float32).reshape(-1, V), f"step {step} session {i}")
        pos = [p + c for p, c in zip(pos, counts)]
    for s, mo in zip(ss, mos):
        for w in (0, 1):
            assert np.array_equal(s.kv(w), mo.kv(w)), w


# ---- the GPT-NeoX family ----------------------------------------------------------------------------------------------------------------------
CLASS = {"gptneox": neox.GptNeoX, "gpt2": neox.Gpt2, "mpt": neox.Mpt, "bloom": neox.Bloom, "gptj": neox.GptJ}
CFGS = {
    "neox-tiny": ("gptneox", synth.NEOX_CONFIGS["neox-tiny"], False),
    "gpt2-tiny": ("gpt2", synth.GPT2_CONFIGS["gpt2-tiny"], False),
    "gpt2-tiny-lm_head": ("gpt2", synth.GPT2_CONFIGS["gpt2-tiny"], True),
    "mpt-tiny": ("mpt", A.MPT_CONFIGS["mpt-tiny"], False),
    "bloom-12h": ("bloom", A.BLOOM_CONFIGS["bloom-12h"], False),
    "gptj-tiny": ("gptj", J.GPTJ_CONFIGS["gptj-tiny"], False),                  # 256-wide heads
    "gptj-hd64": ("gptj", J.GPTJ_CONFIGS["gptj-hd64"], False),
}


@functools.lru_cache(maxsize=None)
def cfg_model(name):
    arch, hp, lm_head = CFGS[name]
    q = B.Oracle().quantize
    if arch == "gptneox":
        hp, tens = synth.make_neox(hp, B.Q4_0, q)
    elif arch == "gpt2":
        hp, tens = synth.make_gpt2(hp, B.Q4_0, q, lm_head=lm_head)
    elif arch == "mpt":
        hp, tens = A.make_mpt(hp, B.Q4_0, q)
    elif arch == "bloom":
        hp, tens = A.make_bloom(hp, B.Q4_0, q)
    else:
        hp, tens = J.make_gptj(hp, B.Q4_0, q)
    return CLASS[arch](hp, tens, context_size=hp["n_ctx"])


def neox_plan(n_ctx):
    """prompts and steps that fit n_ctx and end one chunk on its last slot (GPT-2: the last wpe row)"""
    prompts = [0, 5, 12, n_ctx - 41, 2]
    return prompts, [[9, 1, 33, 8, 1], [1, 8, 1, 32, 7], [0, 0, 1, 1, 0]]


@pytest.mark.parametrize("cfg", list(CFGS))
@pytest.mark.parametrize("kv32", [False, True])
def test_neox_family(cfg, kv32):
    m = cfg_model(cfg)
    prompts, plan = neox_plan(m.context_size)
    ps = pairs(m, prompts, kv32, n_batch=64)
    run_steps(m, ps, plan, all_logits=kv32)
    assert ps[3][0].n_past == m.context_size


def test_neox_mixed_file():
    if not NK.have_ref():
        pytest.skip("oracle/_ref/*_kq.so not built (the reference's quantizers draw the typed models)")
    hp0 = dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2, alibi_bias_max=8.0)
    names = NK.matrices("mpt", dict(hp0, wtype=0))
    types = {}
    for name in names:
        layer = next((int(t) for t in name.split(".") if t.isdigit()), None)
        types[name] = B.Q6_K if layer is None else B.Q4_K if layer == 0 else B.Q5_0
    hp, tens, types = NK.make_typed("mpt", hp0, types[names[-1]], NK.ref_lib(), types=types)
    m = neox.Mpt(hp, tens, context_size=hp["n_ctx"], tensor_types=types)
    for kv32 in (False, True):
        ps = pairs(m, [0, 4, 20, 50], kv32, n_batch=64)
        run_steps(m, ps, [[8, 1, 33, 9], [1, 31, 1, 7]])


# ---- decode steps are the all-ones case ---------------------------------------------------------------------------------------------------------
def decode_twins(m, n, kv32=False):
    ps = pairs(m, [(3 + 5 * i) % 60 for i in range(n)], kv32)
    return [a for a, _ in ps], [b for _, b in ps]


@pytest.mark.parametrize("model", ["llama", "mpt-tiny", "gptj-hd64"])
def test_all_ones_is_evaluate_sessions(model):
    m = make_model("gqa8", B.Q4_0) if model == "llama" else cfg_model(model)
    A_, B_ = decode_twins(m, 17)
    V = m.hyperparameters["n_vocab"]
    rng = np.random.default_rng(5)
    for step in range(3):
        toks = rng.integers(0, V, len(A_)).astype(np.int32)
        got = m.evaluate_ragged(A_, [toks[i:i + 1] for i in range(len(A_))])
        want = m.evaluate_sessions(B_, toks)
        for i, (a, b) in enumerate(zip(A_, B_)):
            same_bits(got[i], want[i], f"step {step} session {i}")
            check_pair(a, b, f"step {step} session {i}", kv=step == 2)
            assert a.last_launches == b.last_launches, (a.last_launches, b.last_launches)


@pytest.mark.parametrize("model", ["llama", "bloom-12h"])
def test_mixed_step_launches(model):
    """a step with tiled chunks launches both attention forms per layer, and one gather before the final norm"""
    m = make_model("gqa8", B.Q4_0) if model == "llama" else cfg_model(model)
    n_layer = m.hyperparameters["n_layer"]
    s = [start(m) for _ in range(3)]
    m.evaluate_ragged(s, [[1], [2], [3]])
    ones = s[0].last_launches
    m.evaluate_ragged(s, [[1], np.arange(9) % 50, [4]])
    assert s[0].last_launches == ones + 2 * n_layer + 1, (s[0].last_launches, ones)
    m.evaluate_ragged(s, [np.arange(8) % 50, np.arange(9) % 50, np.arange(33) % 50], all_logits=True)
    assert s[0].last_launches == ones, (s[0].last_launches, ones)                      # tiled only, no gather
    m.evaluate_ragged(s, [[1], [2], np.arange(3) % 50])
    assert s[0].last_launches == ones + 1                                                # warp only, with the gather


# ---- feed_prompts -------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["llama", "gpt2-tiny"])
def test_feed_prompts(model):
    m = make_model("tiny8", B.Q4_0, n_ctx=1024) if model == "llama" else cfg_model(model)
    n_ctx = m.context_size() if model == "llama" else m.context_size
    V = m.hyperparameters["n_vocab"]
    rng = np.random.default_rng(11)
    n_batches = [8, 32, 7, 64, 16, 9]
    lens = [min(n_ctx - 6, x) for x in (50, 100, 0, 130, 3, 77)]           # longer than n_batch, an empty prompt
    A_ = [start(m, n_batch=nb) for nb in n_batches]
    B_ = [start(m, n_batch=nb) for nb in n_batches]
    for a, b in zip(A_[:2], B_[:2]):                                     # two sessions that already hold tokens
        p = rng.integers(0, V, 5).astype(np.int32)
        a.feed_prompt(p)
        b.feed_prompt(p)
    prompts = [rng.integers(0, V, k).astype(np.int32) for k in lens]
    got = m.feed_prompts(A_, prompts)
    for i, (a, b, p) in enumerate(zip(A_, B_, prompts)):
        want = b.feed_prompt(p)
        same_bits(got[i], want, f"session {i}")
        check_pair(a, b, f"session {i}")
    assert A_[2].n_past == 0


def test_feed_prompts_split_at_row_cap():
    """ten sessions of n_batch 512: the first chunk step holds 5120 rows and is split across two ragged steps"""
    m = make_model("tiny8", B.Q4_0, n_ctx=1024)
    V = m.hyperparameters["n_vocab"]
    rng = np.random.default_rng(12)
    prompts = [rng.integers(0, V, 600 + 7 * i).astype(np.int32) for i in range(10)]
    A_ = [start(m) for _ in range(10)]
    B_ = [start(m) for _ in range(10)]
    got = m.feed_prompts(A_, prompts)
    for i, (a, b, p) in enumerate(zip(A_, B_, prompts)):
        same_bits(got[i], b.feed_prompt(p), f"session {i}")
        check_pair(a, b, f"session {i}")
    full = start(m)
    full.feed_prompt(np.zeros(1000, np.int32))
    before = state(A_[0])[0]
    with pytest.raises(llm_b200.ContextFull):
        m.feed_prompts([A_[0], full], [[1, 2], np.zeros(30, np.int32)])
    assert A_[0].n_past == before


# ---- after a ragged step -------------------------------------------------------------------------------------------------------------------------
def test_after_ragged_steps():
    m = make_model("gqa8", B.Q4_0)
    ps = pairs(m, [5, 0, 30, 12])
    run_steps(m, ps, [[9, 33, 1, 8]])
    ra, rb = [llm_b200.Rng(i) for i in range(4)], [llm_b200.Rng(i) for i in range(4)]
    ids = m.infer_next_tokens([a for a, _ in ps], GREEDY, ra)                     # greedy after a ragged step
    for i, (a, b) in enumerate(ps):
        assert ids[i] == b.infer_next_token(GREEDY, rb[i]), i
    run_steps(m, ps, [[1, 8, 32, 7]], seed=4)
    chain = llm_b200.InferenceParameters(llm_b200.Sampler(top_k=40))             # the default chain, one session at a time
    for i, (a, b) in enumerate(ps):
        assert a.infer_next_token(chain, llm_b200.Rng(100 + i)) == b.infer_next_token(chain, llm_b200.Rng(100 + i)), i
    run_steps(m, ps, [[16, 1, 9, 1]], seed=5)
    ps[0][0].evaluate([9]); ps[0][1].evaluate([9])                                # a single-session graph step must see the new n_past
    ps[1][0].rewind(20); ps[1][1].rewind(20)                                      # a rewind
    run_steps(m, ps, [[8, 9, 1, 1]], seed=6)
    ps[2][0].evaluate([21]); ps[2][1].evaluate([21])
    for i, (a, b) in enumerate(ps):
        check_pair(a, b, f"session {i}")
        sa, sb = a.get_snapshot(), b.get_snapshot()
        assert sa.npast == sb.npast
        for f in ("tokens", "last_logits", "memory_k", "memory_v"):
            same_bits(getattr(sa, f), getattr(sb, f), f"snapshot {f} {i}")
    restored = [(llm_b200.InferenceSession.from_snapshot(a.get_snapshot(), m), b) for a, b in ps]
    run_steps(m, restored, [[1, 12, 8, 1]], seed=7)


# ---- refusals ------------------------------------------------------------------------------------------------------------------------------------
def test_refusals():
    m = make_model("tiny8", B.Q4_0)
    other = make_model("tiny8", B.Q4_0, seed=0x5EED0002)
    ss = [start(m, n_batch=16) for _ in range(3)]
    for i, s in enumerate(ss):
        s.feed_prompt([1 + i, 2, 3])
    fast = start(m, flags=4)                          # B200_SESSION_FAST
    fast.feed_prompt([1])
    f32 = start(m, kv32=True)
    f32.feed_prompt([1])
    foreign = start(other)
    foreign.feed_prompt([1])
    nearly = start(m)
    nearly.feed_prompt(np.arange(m.context_size() - 4, dtype=np.int32) % 320)
    snapshot = [state(s) for s in ss + [nearly]]
    L = m.L

    def refused(sessions, counts, code, toks=None, null=None):
        h = m._session_handles(sessions)
        counts = np.ascontiguousarray(counts, np.int32)
        toks = np.ascontiguousarray(np.arange(max(1, int(counts.sum()))) % 320 if toks is None else toks, np.int32)
        args = [counts.ctypes.data, toks.ctypes.data]
        if null is not None:
            args[null] = None
        assert L.b200_model_evaluate_ragged(m._m, h, len(sessions), args[0], args[1], None, 0) == code
        for s, want in zip(ss + [nearly], snapshot):
            got = state(s)
            assert got[0] == want[0]
            for g, w in zip(got[1:], want[1:]):
                same_bits(g, w, "refused")

    refused(ss[:2] + [foreign], [1, 2, 3], -2)        # another model's session
    refused([ss[0], ss[1], ss[0]], [1, 2, 3], -2)     # a duplicate
    refused(ss[:2] + [fast], [1, 2, 3], -2)           # a FAST session
    refused(ss[:2] + [f32], [1, 2, 3], -2)            # mixed KV types
    refused([], [], -2)                               # n = 0
    refused(ss, [1, 0, 3], -2)                        # an empty chunk
    refused(ss, [1, -2, 3], -2)
    refused(ss, [1, 17, 3], -2)                       # above the session's n_batch
    refused(ss, [1, 2, 3], -2, toks=[1, 2, 320, 4, 5, 6])     # an id outside the vocabulary
    refused(ss, [1, 2, 3], -2, toks=[1, 2, 3, -1, 5, 6])
    refused(ss, [1, 2, 3], -2, null=0)                # null counts
    refused(ss, [1, 2, 3], -2, null=1)                # null tokens
    refused(ss + [nearly], [1, 2, 3, 5], -1)          # a chunk that does not fit
    big = [start(m, n_batch=512) for _ in range(9)]
    refused(big, [512] * 8 + [1], -2)                 # more than B200_MAX_BATCH_ROWS rows
    with pytest.raises(llm_b200.ContextFull):
        m.evaluate_ragged(ss + [nearly], [[1], [2], [3], [4, 5, 6, 7, 8]])
    with pytest.raises(RuntimeError):
        m.evaluate_ragged(ss, [[1], [], [3]])
    with pytest.raises(ValueError):
        m.evaluate_ragged(ss, [[1], [2]])
    with pytest.raises(RuntimeError):
        m.evaluate_ragged(ss[:2] + [foreign], [[1], [2], [3]])
    nx = cfg_model("mpt-tiny")
    with pytest.raises(TypeError):
        m.evaluate_ragged([ss[0], start(nx)], [[1], [2]])
    with pytest.raises(TypeError):
        nx.feed_prompts([ss[0]], [[1]])
    for s, want in zip(ss + [nearly], snapshot):
        assert state(s)[0] == want[0]
