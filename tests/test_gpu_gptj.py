"""GPT-J on the native GPT-NeoX / GPT-2 runtime: logits and both KV caches bit-identical to the reference's own ggml.c running the restated graph
(oracle/ref_gptj.c).

Every case runs: a 20-token prefill, 10 decode steps on the graph schedule (6 launches per layer + 3), a 17-token batch, one more decode step, a batch
whose last row only comes back, then both caches.  Head sizes: 256 (GPT-J 6B's; the wide cluster attention with 8 CTAs per head), 192 (clusters of 6,
not a power of two) and 64 (the attention kernel of heads up to 128 wide)."""
import numpy as np
import pytest

from oracle import bindings as B
from oracle import gptj as J

pytestmark = pytest.mark.gpu

FORMATS = ["q4_0", "q4_1", "q5_0", "q5_1", "q8_0"]
CHUNK = 512


def check(g, c, what):
    c = np.asarray(c, np.float32).reshape(np.shape(g))
    assert np.array_equal(np.asarray(g, np.float32).view(np.uint32), c.view(np.uint32)), (what, float(np.abs(g - c).max() / np.abs(c).max()), int((g != c).sum()))


def ref_or_skip():
    if not J.have_ref():
        pytest.skip("oracle/_ref/libggml_gptj.so not built (the GPT-J CPU model is the reference graph on the reference's ggml)")


def native(hp, tens):
    from llm_b200 import GptJ
    m = GptJ(hp, tens)
    return m, m.start_session(CHUNK)


def kv_equal(s, cpu):
    """both caches in the reference's own layout: K [n_layer][n_ctx][n_embd], V [n_layer][n_embd][n_ctx]"""
    assert np.array_equal(s.kv(0), cpu.kv(0)), "K"
    assert np.array_equal(s.kv(1), cpu.kv(1)), "V"


def graph_launches(hp):
    return 6 * hp["n_layer"] + 3


def run_sequence(hp, tens):
    graph = graph_launches(hp)
    cpu = J.RefGptJ(hp, tens, n_threads=8, n_batch=CHUNK)
    m, s = native(hp, tens)
    toks = np.random.default_rng(0x6D71).integers(0, hp["n_vocab"], size=64, dtype=np.int32)
    check(s.evaluate(toks[:20], all_logits=True), cpu.eval(toks[:20]), "prefill 20")
    for i in range(20, 30):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        assert s.last_launches == graph, ("graph schedule", i, s.last_launches, graph)
    check(s.evaluate(toks[30:47], all_logits=True), cpu.eval(toks[30:47]), "batch of 17")
    check(s.evaluate(toks[47:48], all_logits=True), cpu.eval(toks[47:48]), "decode after the batch")
    assert s.last_launches == graph
    check(s.evaluate(toks[48:53]), cpu.eval(toks[48:53])[-1], "last row only")
    assert s.n_past == 53
    kv_equal(s, cpu)
    s.close(); m.close(); cpu.close()


@pytest.mark.parametrize("qname", FORMATS)
@pytest.mark.parametrize("cfg", ["gptj-tiny", "gptj-hd192", "gptj-hd64"])
def test_gptj_matches_reference(orc, cfg, qname):
    ref_or_skip()
    hp, tens = J.make_gptj(J.GPTJ_CONFIGS[cfg], B.QUANT_TYPES[qname], orc.quantize)
    run_sequence(hp, tens)


def _long_context(orc, n_ctx, seed, plan, per_op_from):
    import llm_b200
    ref_or_skip()
    hp, tens = J.make_gptj(dict(J.GPTJ_CONFIGS["gptj-tiny"], n_ctx=n_ctx), B.Q4_0, orc.quantize)
    graph = graph_launches(hp)
    toks = np.random.default_rng(seed).integers(0, hp["n_vocab"], size=n_ctx, dtype=np.int32)
    cpu = J.RefGptJ(hp, tens, n_threads=16, n_batch=CHUNK)
    m, s = native(hp, tens)
    for kind, a, b in plan:
        if kind == "prefill":
            for i in range(a, b, CHUNK):
                j = min(i + CHUNK, b)
                check(s.evaluate(toks[i:j]), cpu.eval(toks[i:j])[-1], f"prefill {i}..{j}")
        else:
            for i in range(a, b):
                check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
                if i < per_op_from:
                    assert s.last_launches == graph, ("graph schedule", i, s.last_launches)
                else:
                    assert s.last_launches > graph, ("per-op schedule", i, s.last_launches)
    with pytest.raises(llm_b200.ContextFull):
        s.evaluate(toks[:1])
    assert s.n_past == n_ctx
    kv_equal(s, cpu)
    s.close(); m.close(); cpu.close()


@pytest.mark.slow
def test_gptj_long_context_hd256(orc):
    """n_ctx 2048 at hd 256: past 1024 positions the wide kernel's second KQ pass (128 positions per CTA per pass) and second soft_max pass, on the
    graph schedule up to the last slot, then ContextFull"""
    _long_context(orc, 2048, 0x6D72, [("prefill", 0, 1020), ("decode", 1020, 1030), ("prefill", 1030, 2040), ("decode", 2040, 2048)], per_op_from=2048)


@pytest.mark.slow
def test_gptj_context_4096(orc):
    """n_ctx 4096 at hd 256: the graph schedule up to n_past 3071, the per-op schedule from 3072 (the 3328-position bucket does not fit the cluster
    attention's shared memory), the last slot, then ContextFull"""
    _long_context(orc, 4096, 0x6D73, [("prefill", 0, 3068), ("decode", 3068, 3076), ("prefill", 3076, 4090), ("decode", 4090, 4096)], per_op_from=3072)


@pytest.mark.slow
def test_gptj_6b_geometry(orc):
    """GPT-J 6B layer geometry with 2 layers, Q4_0: a 130-token prefill (the wgmma GEMM serves batches >= 96), decode across the 256-position bucket edge,
    the 50400-row lm_head with its bias"""
    ref_or_skip()
    hp, tens = J.make_gptj(dict(J.GPTJ_CONFIGS["gptj-6b"], n_layer=2, n_ctx=512), B.Q4_0, orc.quantize)
    graph = graph_launches(hp)
    toks = np.random.default_rng(0x6D74).integers(0, hp["n_vocab"], size=262, dtype=np.int32)
    cpu = J.RefGptJ(hp, tens, n_threads=16, n_batch=CHUNK)
    m, s = native(hp, tens)
    check(s.evaluate(toks[:130]), cpu.eval(toks[:130])[-1], "prefill 130")
    check(s.evaluate(toks[130:250]), cpu.eval(toks[130:250])[-1], "second prefill")
    for i in range(250, 262):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        assert s.last_launches == graph, (i, s.last_launches)
    kv_equal(s, cpu)
    s.close(); m.close(); cpu.close()


def test_gptj_constructor_rules(orc):
    """arch 4 needs an even n_rot in (0, head size]; b200_neox_new_alibi refuses arch 4"""
    import ctypes as C

    from llm_b200 import _lib
    from llm_b200.neox import NeoxHparams, _bind
    L = _bind(_lib.lib())
    assert L.b200_init(0) == 0

    def hp(n_rot):
        return NeoxHparams(n_vocab=320, n_embd=512, n_head=2, n_layer=2, n_rot=n_rot, use_parallel_residual=1, wtype=B.Q4_0, context_size=128, arch=4, has_lm_head=0)

    for n_rot in (63, 0, -2, 258):
        assert not L.b200_neox_new(C.byref(hp(n_rot))), n_rot
    for n_rot in (2, 64, 256):
        h = L.b200_neox_new(C.byref(hp(n_rot)))
        assert h, n_rot
        L.b200_neox_free(h)
    assert not L.b200_neox_new_alibi(C.byref(hp(64)), 8.0)


def test_gptj_model_file_loads_like_tensors(orc, tmp_path):
    """a GPT-J file written by write_model("gptj") and loaded into GptJ gives the logits of the same tensors loaded directly"""
    from llm_b200 import GptJ, loader
    hp, tens = J.make_gptj(J.GPTJ_CONFIGS["gptj-tiny"], B.Q5_0, orc.quantize)
    path = str(tmp_path / "gptj.bin")
    loader.write_model(path, "gptj", dict(hp, file_type=8), tens, J.gptj_tensor_shapes(hp), B.Q5_0)
    f = loader.GgmlFile(path, "gptj")
    words = f.hyperparameters()
    from_file = {t["name"]: f.tensor_bytes(i).view(np.float32) if t["type"] == 0 else f.tensor_bytes(i).reshape(t["ne"][1], -1) for i, t in enumerate(f.tensors())}
    f.close()
    fhp = dict(n_vocab=words["n_vocab"], n_ctx=words["n_ctx"], n_embd=words["n_embd"], n_head=words["n_head"], n_layer=words["n_layer"], n_rot=words["n_rot"],
               wtype=B.Q5_0)
    assert fhp == dict(hp, wtype=B.Q5_0)
    toks = np.arange(9, dtype=np.int32) * 7 % hp["n_vocab"]
    outs = []
    for tensors, h in ((tens, hp), (from_file, fhp)):
        m = GptJ(h, tensors)
        s = m.start_session(16)
        outs.append(s.evaluate(toks, all_logits=True))
        s.close(); m.close()
    check(outs[1], outs[0], "file vs tensors")
