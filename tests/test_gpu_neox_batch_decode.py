"""Batched decode across the sessions of one GPT-NeoX, GPT-2, MPT, BLOOM or GPT-J model (b200_neox_evaluate_sessions /
b200_neox_infer_next_tokens): one step advances n sessions, and every session must be bit-identical to a twin -- a second session of the same
model, fed the same prompt and stepped alone with evaluate([tok]) (the single-session paths the other tests hold to the reference).  Equal means
equal bit patterns.

  parity          every architecture's small configs in Q4_0 at n = 1 .. 64, every session at its own n_past; after every step the logits
                  row, both caches, n_past and tokens() of each session equal its twin's
  layouts         the other classic formats, F16, pure Q4_K / Q6_K, a mixed file, GPT-J's v_proj of its own type and RoPE overrides, on f16
                  and F32 caches
  reference       three sessions per architecture against the reference graphs, logits and caches (and one F32-cache case)
  long context    MPT to the last slot of 4096 positions, GPT-J with 256-wide heads at 2048, GPT-2 up to its last wpe row
  geometry        two-layer MPT-7B, GPT-J-6B and NeoX-20B shapes
  interleaving    batched step, a graph step on one session, a rewind of another, a batched step, a snapshot restored between steps
  generation      greedy infer_next_tokens over 32 steps; the default chain against infer_next_token and or_sample; a NaN row fails alone
  refusals        every refusal of the contract leaves every session unchanged; TypeError / RuntimeError for foreign sessions in Python
  launches        the launch count of a step is the same at n = 2 and 64 and equals DESIGN.md §6's formula"""
import ctypes as C
import functools

import numpy as np
import pytest

import llm_b200
from llm_b200 import ModelKVMemoryType as KV
from llm_b200 import neox
from oracle import alibi as A
from oracle import bindings as B
from oracle import gptj as J
from oracle import kv32 as K32
from oracle import neox_kquant as NK
from oracle import synth

pytestmark = pytest.mark.gpu

F16 = 1
NS = [1, 2, 5, 15, 16, 17, 31, 32, 33, 64]
GREEDY = llm_b200.InferenceParameters(llm_b200.Sampler(repetition_penalty=1.0, top_k=1))
CLASS = {"gptneox": neox.GptNeoX, "gpt2": neox.Gpt2, "mpt": neox.Mpt, "bloom": neox.Bloom, "gptj": neox.GptJ}
# name: (architecture, hyperparameters, GPT-2 with its own model/lm_head)
CFGS = {
    "neox-tiny": ("gptneox", synth.NEOX_CONFIGS["neox-tiny"], False),           # parallel residual, n_rot 8 of 32
    "neox-tiny-seq": ("gptneox", synth.NEOX_CONFIGS["neox-tiny-seq"], False),
    "gpt2-tiny": ("gpt2", synth.GPT2_CONFIGS["gpt2-tiny"], False),              # output tied to wte
    "gpt2-tiny-lm_head": ("gpt2", synth.GPT2_CONFIGS["gpt2-tiny"], True),
    "mpt-tiny": ("mpt", A.MPT_CONFIGS["mpt-tiny"], False),
    "mpt-24h": ("mpt", A.MPT_CONFIGS["mpt-24h"], False),                        # heads 16..23 on ALiBi's m1 branch
    "bloom-12h": ("bloom", A.BLOOM_CONFIGS["bloom-12h"], False),
    "gptj-tiny": ("gptj", J.GPTJ_CONFIGS["gptj-tiny"], False),                  # 256-wide heads
    "gptj-hd192": ("gptj", J.GPTJ_CONFIGS["gptj-hd192"], False),
    "gptj-hd64": ("gptj", J.GPTJ_CONFIGS["gptj-hd64"], False),
}
# one small config per architecture for the layout, reference and feature cases (K = 256: whole K-quant super-blocks)
GEOM = dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2)
ARCH_HP = {"gptneox": dict(GEOM, n_rot=16, use_parallel_residual=1), "gpt2": GEOM, "mpt": dict(GEOM, alibi_bias_max=8.0), "bloom": GEOM,
           "gptj": dict(GEOM, n_rot=16)}


def same_bits(got, want, what):
    g, w = np.asarray(got), np.asarray(want)
    assert g.shape == w.shape and g.dtype == w.dtype, (what, g.shape, w.shape, g.dtype, w.dtype)
    bad = g.view(np.uint8).reshape(g.shape + (-1,)) != w.view(np.uint8).reshape(w.shape + (-1,))
    assert not bad.any(), (what, int(bad.any(axis=-1).sum()))


def draw(arch, hp, wtype, quantize, lm_head=False):
    """(hp with wtype, tensors): the architecture's synthetic model, its 2-D weights quantized with `quantize`"""
    if arch == "gptneox":
        return synth.make_neox(hp, wtype, quantize)
    if arch == "gpt2":
        return synth.make_gpt2(hp, wtype, quantize, lm_head=lm_head)
    if arch == "mpt":
        return A.make_mpt(hp, wtype, quantize)
    if arch == "bloom":
        return A.make_bloom(hp, wtype, quantize)
    return J.make_gptj(hp, wtype, quantize)


@functools.lru_cache(maxsize=None)
def cfg_model(name, wtype, n_ctx=None):
    """a model of CFGS[name] (context n_ctx) with weights quantized by the C oracle's quantizer; cached across the cases that share it"""
    arch, hp, lm_head = CFGS[name]
    hp = dict(hp, **({"n_ctx": n_ctx} if n_ctx else {}))
    hp, tens = draw(arch, hp, wtype, B.Oracle().quantize, lm_head)
    return CLASS[arch](hp, tens, context_size=hp["n_ctx"])


def start(m, kv32=False, n_batch=128):
    t = KV.Float32 if kv32 else KV.Float16
    return m.start_session(n_batch, t, t)


def feed(s, p):
    if len(p):
        s.feed_prompt(p)


def pairs(m, n, prompt_lens, kv32=False, seed=1):
    """n (batched, twin) session pairs, pair i fed the same prompt of prompt_lens[i] ids (0: nothing)"""
    rng = np.random.default_rng(seed)
    V = m.hyperparameters["n_vocab"]
    out = []
    for i in range(n):
        a, b = start(m, kv32), start(m, kv32)
        p = rng.integers(0, V, prompt_lens[i]).astype(np.int32)
        feed(a, p)
        feed(b, p)
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


def step_and_check(m, ps, toks, what, kv=True):
    got = m.evaluate_sessions([a for a, _ in ps], toks)
    assert got.shape == (len(ps), m.hyperparameters["n_vocab"])
    for i, (a, b) in enumerate(ps):
        b.evaluate(toks[i:i + 1])
        check_pair(a, b, f"{what} session {i}", logits=got[i], kv=kv)


def run_parity(m, n, kv32, steps=6, kv_every_step=True):
    n_ctx = m.context_size
    lens = [(1 + 7 * i) % max(2, n_ctx - steps - 2) for i in range(n)]
    ps = pairs(m, n, lens, kv32)
    V = m.hyperparameters["n_vocab"]
    rng = np.random.default_rng(n)
    for step in range(steps):
        step_and_check(m, ps, rng.integers(0, V, n).astype(np.int32), f"n={n} step {step}", kv=kv_every_step or step == steps - 1)
    closing(ps)


def closing(ps):
    for a, b in ps:
        a.close(); b.close()


# ---- parity, every architecture -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", list(CFGS))
@pytest.mark.parametrize("n", NS)
def test_parity_q4_0(cfg, n):
    run_parity(cfg_model(cfg, B.Q4_0), n, kv32=False)


# ---- weight layouts and caches --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nk():
    if not NK.have_ref():
        pytest.skip("oracle/_ref/*_kq.so not built (the reference's quantizers draw the typed models)")
    return NK.ref_lib()


def mixed(arch, hp):
    """Q4_K layer 0, Q5_0 layer 1, a Q6_K output (GPT-2 and MPT: the tied wte) beside a Q8_0 wte where the model has both"""
    names = NK.matrices(arch, dict(hp, wtype=0))
    t = {}
    for name in names:
        layer = next((int(tok) for tok in name.replace("/h", ".").replace("/", ".").split(".") if tok.isdigit()), None)
        t[name] = B.Q6_K if layer is None else B.Q4_K if layer == 0 else B.Q5_0
    if arch in ("gptneox", "bloom", "gptj"):
        t[names[0]] = B.Q8_0
    return t


@functools.lru_cache(maxsize=None)
def layout_model(arch, kind):
    """ARCH_HP[arch] in weight layout `kind`: a classic format or f16 throughout, q4_K / q6_K throughout, "mixed", "vproj" (GPT-J Q4_K with layer
    0's v_proj Q8_0, its own matrix), "rope" (Q4_0 with rope_freq_base 20000, rope_freq_scale 0.5)"""
    hp0 = ARCH_HP[arch]
    names = NK.matrices(arch, dict(hp0, wtype=0))
    kw = {}
    if kind == "mixed":
        types = mixed(arch, hp0)
    elif kind == "vproj":
        types = dict({n: B.Q4_K for n in names}, **{"transformer.h.0.attn.v_proj.weight": B.Q8_0})
    else:
        t = {"f16": F16, "q4_K": B.Q4_K, "q6_K": B.Q6_K, "rope": B.Q4_0}.get(kind) or B.QUANT_TYPES[kind]
        types = {n: t for n in names}
        if kind == "rope":
            kw = dict(rope_freq_base=20000.0, rope_freq_scale=0.5)
    base = types[names[-1]]
    hp, tens, types = NK.make_typed(arch, hp0, base, NK.ref_lib(), types=types)
    return CLASS[arch](hp, tens, context_size=hp["n_ctx"], tensor_types=types, **kw)


LAYOUTS = [(a, k) for a in ARCH_HP for k in ("q4_1", "q5_0", "q5_1", "q8_0", "f16", "q4_K", "q6_K", "mixed")]
LAYOUTS += [("gptj", "vproj"), ("gptneox", "rope"), ("gptj", "rope")]


@pytest.mark.parametrize("arch,kind", LAYOUTS)
@pytest.mark.parametrize("kv32", [False, True])
@pytest.mark.parametrize("n", [2, 17, 33])
def test_parity_layouts(nk, arch, kind, kv32, n):
    run_parity(layout_model(arch, kind), n, kv32, steps=3, kv_every_step=False)


# ---- the reference directly -------------------------------------------------------------------------------------------------------------------
def reference(arch, hp, tens, kv32):
    """(reference model, V kept by position in it)"""
    if arch in ("gptneox", "gpt2"):
        if not B.have_ref("ref_kv32" if kv32 else "ref"):
            pytest.skip("oracle/_ref not built")
        lib = K32.ref_lib() if kv32 else B.RefLib("ref")
        return (lib.neox if arch == "gptneox" else lib.gpt2)(hp, tens, n_threads=8, n_batch=64), arch == "gpt2"
    if arch in ("mpt", "bloom"):
        if not (K32.have_ref() if kv32 else A.have_ref()):
            pytest.skip("oracle/_ref alibi libraries not built")
        a = A.MPT if arch == "mpt" else A.BLOOM
        return (K32.RefAlibiKV32 if kv32 else A.RefAlibi)(hp, tens, a, n_threads=8, n_batch=64), True
    if not (K32.have_ref() if kv32 else J.have_ref()):
        pytest.skip("oracle/_ref GPT-J libraries not built")
    return (K32.RefGptJKV32 if kv32 else J.RefGptJ)(hp, tens, n_threads=8, n_batch=64), False


def ref_kv(cpu, which, kv32, v_by_position, hp, n_ctx):
    got = K32.kv_f32(cpu, which) if kv32 else cpu.kv(which)
    if which and v_by_position:                 # the native cache keeps V by channel
        got = got.reshape(hp["n_layer"], n_ctx, hp["n_embd"]).transpose(0, 2, 1).ravel()
    return np.ascontiguousarray(got)


@pytest.mark.parametrize("arch,kv32", [(a, False) for a in ARCH_HP] + [("mpt", True)])
def test_against_reference(orc, arch, kv32):
    """three sessions at different positions, each against the reference graph on its own cache"""
    hp, tens = draw(arch, ARCH_HP[arch], B.Q4_0, orc.quantize)
    m = CLASS[arch](hp, tens, context_size=hp["n_ctx"])
    toks = synth.make_tokens(hp, 60)
    lens = [1, 9, 23]
    ss = [start(m, kv32) for _ in lens]
    cpus = [reference(arch, hp, tens, kv32) for _ in lens]
    V = hp["n_vocab"]
    for s, (cpu, _), k in zip(ss, cpus, lens):
        same_bits(s.feed_prompt(toks[:k]), np.asarray(cpu.eval(toks[:k]), np.float32).reshape(-1, V)[-1], "prompt")
    for step in range(6):
        ids = np.array([toks[k + step] for k in lens], np.int32)
        got = m.evaluate_sessions(ss, ids)
        for i, (cpu, _) in enumerate(cpus):
            same_bits(got[i], np.asarray(cpu.eval(ids[i:i + 1]), np.float32).reshape(-1, V)[-1], f"step {step} session {i}")
    for s, (cpu, vpos) in zip(ss, cpus):
        for w in (0, 1):
            want = ref_kv(cpu, w, kv32, vpos, hp, m.context_size)
            got = s.kv(w)
            same_bits(got.view(np.uint8), want[:got.size].view(np.uint8), f"kv{w}")
        s.close(); cpu.close()


# ---- long context ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.slow
def test_mpt_long_context():
    m = cfg_model("mpt-tiny", B.Q4_0, 4096)
    ps = pairs(m, 4, [0, 3071, 3072, 4094])
    rng = np.random.default_rng(4096)
    for step in range(2):                                       # 4094 -> 4096: the last slot
        step_and_check(m, ps, rng.integers(0, 320, 4).astype(np.int32), f"mpt long step {step}")
    assert ps[3][0].n_past == 4096
    with pytest.raises(llm_b200.ContextFull):
        m.evaluate_sessions([a for a, _ in ps], np.zeros(4, np.int32))
    closing(ps)


@pytest.mark.slow
def test_gptj_hd256_long_context():
    m = cfg_model("gptj-tiny", B.Q4_0, 2048)
    ps = pairs(m, 3, [0, 1500, 2045])
    rng = np.random.default_rng(2048)
    for step in range(3):
        step_and_check(m, ps, rng.integers(0, 320, 3).astype(np.int32), f"gptj long step {step}")
    assert ps[2][0].n_past == 2048
    closing(ps)


def test_gpt2_last_position_row():
    """GPT-2's context is wpe's rows: every session's position picks its own row, up to the last one"""
    m = cfg_model("gpt2-tiny", B.Q4_0)
    n_ctx = m.context_size
    ps = pairs(m, 4, [0, 17, n_ctx - 3, n_ctx - 2])
    rng = np.random.default_rng(64)
    for step in range(2):
        step_and_check(m, ps, rng.integers(0, 320, 4).astype(np.int32), f"gpt2 wpe step {step}")
    assert ps[3][0].n_past == n_ctx
    with pytest.raises(llm_b200.ContextFull):
        m.evaluate_sessions([a for a, _ in ps], np.zeros(4, np.int32))
    closing(ps)


# ---- published geometry --------------------------------------------------------------------------------------------------------------------------
GEOMETRY = {
    "mpt-7b": ("mpt", dict(A.MPT_CONFIGS["mpt-7b"], n_layer=2, n_ctx=256)),
    "gptj-6b": ("gptj", dict(J.GPTJ_CONFIGS["gptj-6b"], n_layer=2, n_ctx=256)),
    "neox-20b": ("gptneox", dict(synth.NEOX_CONFIGS["neox-20b"], n_layer=2, n_ctx=256)),
}


@functools.lru_cache(maxsize=None)
def geometry_model(name):
    arch, hp = GEOMETRY[name]
    m = CLASS[arch](dict(hp, wtype=B.Q4_0), context_size=hp["n_ctx"])
    m.synthesize(0x6E0)
    return m


@pytest.mark.slow
@pytest.mark.parametrize("name", list(GEOMETRY))
@pytest.mark.parametrize("n", [2, 17])
def test_published_geometry(name, n):
    m = geometry_model(name)
    ps = pairs(m, n, [3 + 11 * i for i in range(n)])
    rng = np.random.default_rng(7)
    V = m.hyperparameters["n_vocab"]
    for step in range(3):
        step_and_check(m, ps, rng.integers(0, V, n).astype(np.int32), f"{name} n={n} step {step}", kv=step == 2)
    closing(ps)


# ---- interleaving -------------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def arch_model(arch):
    """ARCH_HP[arch] in Q4_0: a model whose single-session steps run the decode graph"""
    hp, tens = draw(arch, ARCH_HP[arch], B.Q4_0, B.Oracle().quantize)
    return CLASS[arch](hp, tens, context_size=hp["n_ctx"])


@pytest.mark.parametrize("arch", list(ARCH_HP))
def test_interleaving(arch):
    """the graph's device n_past is stale after a batched step, as after a rewind: a graph step on one session must see the new n_past"""
    m = arch_model(arch)
    ps = pairs(m, 4, [5, 12, 30, 7])
    A_ = [a for a, _ in ps]
    step_and_check(m, ps, np.array([1, 2, 3, 4], np.int32), "first batched step")
    ps[0][0].evaluate([9]); ps[0][1].evaluate([9])              # a single graph step on one session
    assert ps[0][0].last_launches < 12 * m.hyperparameters["n_layer"]
    ps[1][0].rewind(8); ps[1][1].rewind(8)                      # a rewind of another
    step_and_check(m, ps, np.array([11, 12, 13, 14], np.int32), "after a graph step and a rewind")
    snap = ps[2][0].get_snapshot()                              # a snapshot restored between batched steps
    ps[2][0].close()
    ps[2] = (neox.NeoxSession.from_snapshot(snap, m), ps[2][1])
    A_ = [a for a, _ in ps]
    got = m.evaluate_sessions(A_, np.array([21, 22, 23, 24], np.int32))
    for i, (a, b) in enumerate(ps):
        b.evaluate([21 + i])
        check_pair(a, b, f"after a restored snapshot, session {i}", logits=got[i])
    ps[3][0].evaluate([31]); ps[3][1].evaluate([31])            # and a graph step after it
    for i, (a, b) in enumerate(ps):
        check_pair(a, b, f"interleaved session {i}")
        sa, sb = a.get_snapshot(), b.get_snapshot()
        assert sa.npast == sb.npast
        for f in ("tokens", "last_logits", "memory_k", "memory_v"):
            same_bits(getattr(sa, f), getattr(sb, f), f"snapshot {f} {i}")
    closing(ps)


# ---- generation ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", ["neox-tiny", "gpt2-tiny-lm_head", "mpt-tiny", "bloom-12h", "gptj-hd64"])
def test_greedy_generation(cfg):
    m = cfg_model(cfg, B.Q5_1)
    ps = pairs(m, 6, [1, 4, 9, 16, 25, 30])                    # + 32 steps: within the 64 positions of the smallest context
    A_ = [a for a, _ in ps]
    ra, rb = [llm_b200.Rng(i) for i in range(6)], [llm_b200.Rng(i) for i in range(6)]
    for step in range(32):
        ids = m.infer_next_tokens(A_, GREEDY, ra)
        for i, (a, b) in enumerate(ps):
            assert ids[i] == b.infer_next_token(GREEDY, rb[i]), (step, i)
            assert ra[i].draw == rb[i].draw == step + 1
    for i, (a, b) in enumerate(ps):
        check_pair(a, b, f"greedy session {i}")
    closing(ps)


@pytest.mark.parametrize("cfg", ["neox-tiny-seq", "mpt-24h", "gptj-hd192"])
def test_default_chain_generation(cfg):
    from oracle.sampler import SamplerOracle
    so = SamplerOracle()
    m = cfg_model(cfg, B.Q4_0)
    ps = pairs(m, 5, [2, 8, 20, 40, 50])
    A_ = [a for a, _ in ps]
    params = [llm_b200.InferenceParameters(llm_b200.Sampler(top_k=k)) for k in (40, 40, 1024, 5, 40)]
    ra, rb = [llm_b200.Rng(1000 + 17 * i) for i in range(5)], [llm_b200.Rng(1000 + 17 * i) for i in range(5)]
    for step in range(12):
        rows = [b.last_logits.copy() for _, b in ps]
        hists = [b.tokens() for _, b in ps]
        ids = m.infer_next_tokens(A_, params, ra)
        for i, (a, b) in enumerate(ps):
            sp = params[i].sampler
            rc, want, _, _, _ = so.sample(rows[i], hists[i], len(hists[i]), sp.repetition_penalty, sp.repetition_last_n, sp.top_k, sp.top_p,
                                          sp.temperature, rb[i].seed, rb[i].draw)
            assert rc == 0 and ids[i] == want, (step, i, ids[i], want)
            assert ids[i] == b.infer_next_token(params[i], rb[i]), (step, i)
    for i, (a, b) in enumerate(ps):
        check_pair(a, b, f"chain session {i}")
    closing(ps)


def test_sampler_failure_is_per_session():
    m = cfg_model("bloom-12h", B.Q4_0)
    ps = pairs(m, 3, [3, 6, 9])
    snap = ps[1][0].get_snapshot()
    snap.last_logits = snap.last_logits.copy()
    snap.last_logits[17] = np.nan
    bad = neox.NeoxSession.from_snapshot(snap, m)
    before = state(bad)
    A_ = [ps[0][0], bad, ps[2][0]]
    ra = [llm_b200.Rng(i) for i in range(3)]
    rb = [llm_b200.Rng(i) for i in range(3)]
    with pytest.raises(llm_b200.SamplerFailure) as ei:
        m.infer_next_tokens(A_, GREEDY, ra)
    assert ei.value.sessions == [1] and ei.value.tokens[1] == -1
    assert ra[1].draw == 0 and ra[0].draw == ra[2].draw == 1
    after = state(bad)
    assert before[0] == after[0]
    for x, y, f in zip(before[1:], after[1:], ("tokens", "last_logits", "kv0", "kv1")):
        same_bits(y, x, "failed session " + f)
    for i in (0, 2):
        assert ei.value.tokens[i] == ps[i][1].infer_next_token(GREEDY, rb[i])
        check_pair(ps[i][0], ps[i][1], f"survivor {i}")
    bad.close()
    closing(ps)


# ---- refusals -----------------------------------------------------------------------------------------------------------------------------------
def test_refusals():
    m = cfg_model("gptj-hd64", B.Q4_0)
    other = cfg_model("gptj-hd64", B.Q8_0)
    V, n_ctx = m.hyperparameters["n_vocab"], m.context_size
    ss = [start(m) for _ in range(3)]
    for i, s in enumerate(ss):
        s.feed_prompt([1 + i, 2, 3])
    f32 = start(m, kv32=True)
    f32.feed_prompt([1])
    foreign = start(other)
    foreign.feed_prompt([1])
    full = start(m)
    full.feed_prompt(np.arange(n_ctx, dtype=np.int32) % V)
    fresh = start(m)                                   # no evaluated row: infer refuses it
    snapshot = [state(s) for s in ss]
    L = m.L

    def unchanged():
        for s, want in zip(ss, snapshot):
            got = state(s)
            assert got[0] == want[0]
            for g, w in zip(got[1:], want[1:]):
                same_bits(g, w, "refused")

    def refused(sessions, toks, code, infer=True):
        h = m._session_handles(sessions)
        toks = np.ascontiguousarray(toks, np.int32)
        assert L.b200_neox_evaluate_sessions(m._m, h, len(sessions), toks.ctypes.data, None) == code
        sp = (llm_b200._lib.SamplerParams * max(1, len(sessions)))(*[llm_b200._lib.SamplerParams(1.0, 64, 1, 0.95, 0.8, 0, 0)] * len(sessions))
        out, st = np.zeros(max(1, len(sessions)), np.int32), np.zeros(max(1, len(sessions)), np.int32)
        if infer:
            assert L.b200_neox_infer_next_tokens(m._m, h, len(sessions), sp, out.ctypes.data, st.ctypes.data) == code
        unchanged()

    refused(ss[:2] + [foreign], [1, 2, 3], -2)         # another model's session
    refused([ss[0], ss[1], ss[0]], [1, 2, 3], -2)      # a duplicate
    refused(ss[:2] + [f32], [1, 2, 3], -2)             # mixed KV types
    refused(ss[:2] + [full], [1, 2, 3], -1)            # one full session among free ones
    refused([], np.zeros(0, np.int32), -2)             # n = 0
    many = [start(m, n_batch=1) for _ in range(65)]
    for s in many:
        s.feed_prompt([1])
    refused(many, np.ones(65, np.int32), -2)           # n = 65
    refused(ss, [1, V, 2], -2, infer=False)            # an id outside the vocabulary
    refused(ss, [1, -1, 2], -2, infer=False)
    h = (C.c_void_p * 3)(ss[0]._s, ss[1]._s, None)     # a null entry
    assert L.b200_neox_evaluate_sessions(m._m, h, 3, np.array([1, 2, 3], np.int32).ctypes.data, None) == -2
    bad = (llm_b200._lib.SamplerParams * 3)(*[llm_b200._lib.SamplerParams(1.0, 64, 0, 0.95, 0.8, 0, 0)] * 3)   # top_k 0
    out, st = np.zeros(3, np.int32), np.zeros(3, np.int32)
    assert L.b200_neox_infer_next_tokens(m._m, m._session_handles(ss), 3, bad, out.ctypes.data, st.ctypes.data) == -2
    with pytest.raises(RuntimeError):
        m.infer_next_tokens(ss[:2] + [fresh], GREEDY, [llm_b200.Rng(0) for _ in range(3)])
    nearly = start(m)                                  # infer's rule is one slot stricter: n_past + 1 >= n_ctx
    nearly.feed_prompt(np.arange(n_ctx - 1, dtype=np.int32) % V)
    with pytest.raises(llm_b200.ContextFull):
        m.infer_next_tokens(ss[:2] + [nearly], GREEDY, [llm_b200.Rng(0) for _ in range(3)])
    # in Python: a session of another runtime, and one of another model, are refused before the library sees them
    lm = llm_b200.Llama(synth.CONFIGS["tiny8"] | {"wtype": B.Q4_0}, llm_b200.ModelParameters(context_size=64))
    lm.synthesize(1)
    ls = lm.start_session(llm_b200.InferenceSessionConfig(n_batch=8))
    ls.feed_prompt([1])
    with pytest.raises(TypeError):
        m.evaluate_sessions(ss[:2] + [ls], [1, 2, 3])
    with pytest.raises(TypeError):
        lm.evaluate_sessions([ls, ss[0]], [1, 2])
    with pytest.raises(TypeError):
        m.infer_next_tokens(ss[:2] + [ls], GREEDY, [llm_b200.Rng(0) for _ in range(3)])
    with pytest.raises(RuntimeError):
        m.evaluate_sessions(ss[:2] + [foreign], [1, 2, 3])
    with pytest.raises(RuntimeError):
        m.infer_next_tokens(ss[:2] + [foreign], GREEDY, [llm_b200.Rng(0) for _ in range(3)])
    unchanged()
    ls.close(); lm.close()
    for s in ss + many + [f32, foreign, full, fresh, nearly]:
        s.close()


# ---- launches ----------------------------------------------------------------------------------------------------------------------------------
def launch_formula(arch, n_layer, own_v_proj_layers=0):
    """DESIGN.md §6: the embedding gather (+ BLOOM's LayerNorm, + GPT-2's positions), per layer 21 launches with biases (17 for MPT; GPT-J 18,
    + 2 for a v_proj of its own type), then the final LayerNorm, the lm_head (+ GPT-J's bias) and the commit; every mat-mul is two launches"""
    head = 1 + (arch == "bloom") + (arch == "gpt2")
    per_layer = {"mpt": 17, "gptj": 18}.get(arch, 21)
    return head + per_layer * n_layer + 2 * own_v_proj_layers + 4 + (arch == "gptj")


@pytest.mark.parametrize("cfg", ["neox-tiny", "neox-tiny-seq", "gpt2-tiny", "mpt-tiny", "bloom-12h", "gptj-hd64"])
def test_launch_count_does_not_depend_on_n(cfg):
    m = cfg_model(cfg, B.Q4_0)
    counts = {}
    for n in (2, 64):
        ss = [start(m, n_batch=8) for _ in range(n)]
        for s in ss:
            s.feed_prompt([1, 2])
        m.evaluate_sessions(ss, np.full(n, 3, np.int32))
        counts[n] = {s.last_launches for s in ss}
        for s in ss:
            s.close()
    want = launch_formula(CFGS[cfg][0], m.hyperparameters["n_layer"])
    assert counts[2] == counts[64] == {want}, (counts, want)


def test_launch_count_gptj_own_v_proj(nk):
    m = layout_model("gptj", "vproj")
    ss = [start(m) for _ in range(2)]
    for s in ss:
        s.feed_prompt([1, 2])
    m.evaluate_sessions(ss, np.array([3, 4], np.int32))
    assert {s.last_launches for s in ss} == {launch_formula("gptj", m.hyperparameters["n_layer"], 1)}
    for s in ss:
        s.close()
