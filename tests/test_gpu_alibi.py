"""MPT and BLOOM (ALiBi attention) on the native GPT-NeoX / GPT-2 runtime: logits and both KV caches bit-identical to the reference's own ggml.c
running the restated graphs (oracle/ref_alibi.c).

Every case runs: a 20-token prefill, 10 decode steps on the graph schedule (8 launches per layer, + 3 for MPT and + 4 for BLOOM, whose embedding row
goes through a LayerNorm), a 17-token batch, one more decode step, a batch whose last row only comes back, then both caches.  The 24-head MPT config
(not a power of two) puts heads 16..23 on ggml_alibi's m1 branch, the 12-head BLOOM one heads 8..11."""
import numpy as np
import pytest

from oracle import alibi as A
from oracle import bindings as B

pytestmark = pytest.mark.gpu

FORMATS = ["q4_0", "q4_1", "q5_0", "q5_1", "q8_0"]
CHUNK = 512


def check(g, c, what):
    c = np.asarray(c, np.float32).reshape(np.shape(g))
    assert np.array_equal(np.asarray(g, np.float32).view(np.uint32), c.view(np.uint32)), (what, float(np.abs(g - c).max() / np.abs(c).max()), int((g != c).sum()))


def ref_or_skip():
    if not A.have_ref():
        pytest.skip("oracle/_ref/libggml_alibi.so not built (the MPT / BLOOM CPU model is the reference graph on the reference's ggml)")


def native(arch, hp, tens):
    from llm_b200.neox import Bloom, Mpt
    m = (Mpt if arch == A.MPT else Bloom)(hp, tens)
    return m, m.start_session(CHUNK)


def kv_equal(s, cpu, hp):
    """the native cache keeps V by channel ([n_layer][n_embd][n_ctx]), the reference by position"""
    nl, n_ctx, e = hp["n_layer"], hp["n_ctx"], hp["n_embd"]
    assert np.array_equal(s.kv(0), cpu.kv(0)), "K"
    assert np.array_equal(s.kv(1), cpu.kv(1).reshape(nl, n_ctx, e).transpose(0, 2, 1).ravel()), "V"


def run_sequence(arch, hp, tens):
    nl = hp["n_layer"]
    graph = 8 * nl + (3 if arch == A.MPT else 4)
    cpu = A.RefAlibi(hp, tens, arch, n_threads=8, n_batch=CHUNK)
    m, s = native(arch, hp, tens)
    toks = np.random.default_rng(0xA11B1).integers(0, hp["n_vocab"], size=64, dtype=np.int32)
    check(s.evaluate(toks[:20], all_logits=True), cpu.eval(toks[:20]), "prefill 20")
    for i in range(20, 30):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        assert s.last_launches == graph, ("graph schedule", i, s.last_launches, graph)
    check(s.evaluate(toks[30:47], all_logits=True), cpu.eval(toks[30:47]), "batch of 17")
    check(s.evaluate(toks[47:48], all_logits=True), cpu.eval(toks[47:48]), "decode after the batch")
    assert s.last_launches == graph
    check(s.evaluate(toks[48:53]), cpu.eval(toks[48:53])[-1], "last row only")
    assert s.n_past == 53
    kv_equal(s, cpu, hp)
    s.close(); m.close(); cpu.close()


@pytest.mark.parametrize("qname", FORMATS)
@pytest.mark.parametrize("cfg", ["mpt-tiny", "mpt-24h"])
def test_mpt_matches_reference(orc, cfg, qname):
    ref_or_skip()
    hp, tens = A.make_mpt(A.MPT_CONFIGS[cfg], B.QUANT_TYPES[qname], orc.quantize)
    run_sequence(A.MPT, hp, tens)


@pytest.mark.parametrize("cfg,qname", [("mpt-tiny", "q4_0"), ("mpt-24h", "q5_1")])
def test_mpt_alibi_bias_max_5(orc, cfg, qname):
    ref_or_skip()
    hp, tens = A.make_mpt(dict(A.MPT_CONFIGS[cfg], alibi_bias_max=5.0), B.QUANT_TYPES[qname], orc.quantize)
    run_sequence(A.MPT, hp, tens)


@pytest.mark.parametrize("qname", FORMATS)
@pytest.mark.parametrize("cfg", ["bloom-tiny", "bloom-12h"])
def test_bloom_matches_reference(orc, cfg, qname):
    ref_or_skip()
    hp, tens = A.make_bloom(A.BLOOM_CONFIGS[cfg], B.QUANT_TYPES[qname], orc.quantize)
    run_sequence(A.BLOOM, hp, tens)


@pytest.mark.slow
def test_mpt_long_context(orc):
    """n_ctx 4096: the fused attention's second KQ pass (n_kv > 512 at hd 64) and second soft_max pass (n_kv > 1024) on the graph, the per-op
    schedule (soft_max_alibi_kernel at key positions past 3072) from n_past 3072, the last slot, then ContextFull"""
    import llm_b200
    ref_or_skip()
    hp, tens = A.make_mpt(dict(A.MPT_CONFIGS["mpt-tiny"], n_ctx=4096), B.Q4_0, orc.quantize)
    n_ctx, nl = hp["n_ctx"], hp["n_layer"]
    toks = np.random.default_rng(0xA11B2).integers(0, hp["n_vocab"], size=n_ctx, dtype=np.int32)
    cpu = A.RefAlibi(hp, tens, A.MPT, n_threads=16, n_batch=CHUNK)
    m, s = native(A.MPT, hp, tens)

    def prefill(a, b):
        for i in range(a, b, CHUNK):
            j = min(i + CHUNK, b)
            check(s.evaluate(toks[i:j]), cpu.eval(toks[i:j])[-1], f"prefill {i}..{j}")

    def decode(a, b):
        for i in range(a, b):
            check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
            if i < 3072:
                assert s.last_launches == 8 * nl + 3, ("graph schedule", i, s.last_launches)
            else:
                assert s.last_launches > 8 * nl + 4, ("per-op schedule", i, s.last_launches)

    prefill(0, 1020)
    decode(1020, 1030)
    prefill(1030, 3068)
    decode(3068, 3076)
    prefill(3076, 4090)
    decode(4090, n_ctx)
    with pytest.raises(llm_b200.ContextFull):
        s.evaluate(toks[:1])
    assert s.n_past == n_ctx
    kv_equal(s, cpu, hp)
    s.close(); m.close(); cpu.close()


@pytest.mark.slow
@pytest.mark.parametrize("arch,cfg,n_prefill,n_decode", [(A.MPT, "mpt-7b", 130, (250, 262)), (A.BLOOM, "bloom-560m", 100, (100, 104))])
def test_geometry(orc, arch, cfg, n_prefill, n_decode):
    """MPT-7B and BLOOM-560m layer geometry with 2 layers.  MPT: a 130-token prefill (the wgmma GEMM serves batches >= 96), then decode across the
    256-position bucket edge; BLOOM: the 250880-row lm_head"""
    ref_or_skip()
    base = dict((A.MPT_CONFIGS if arch == A.MPT else A.BLOOM_CONFIGS)[cfg], n_layer=2, n_ctx=512)
    hp, tens = (A.make_mpt if arch == A.MPT else A.make_bloom)(base, B.Q4_0, orc.quantize)
    nl = hp["n_layer"]
    graph = 8 * nl + (3 if arch == A.MPT else 4)
    toks = np.random.default_rng(0xA11B3).integers(0, hp["n_vocab"], size=n_decode[1], dtype=np.int32)
    cpu = A.RefAlibi(hp, tens, arch, n_threads=16, n_batch=CHUNK)
    m, s = native(arch, hp, tens)
    check(s.evaluate(toks[:n_prefill]), cpu.eval(toks[:n_prefill])[-1], "prefill")
    if n_decode[0] > n_prefill:
        check(s.evaluate(toks[n_prefill:n_decode[0]]), cpu.eval(toks[n_prefill:n_decode[0]])[-1], "second prefill")
    for i in range(*n_decode):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        assert s.last_launches == graph, (i, s.last_launches)
    kv_equal(s, cpu, hp)
    s.close(); m.close(); cpu.close()


def test_constructor_rejects_other_archs(orc):
    """b200_neox_new still refuses arch 2 / 3, b200_neox_new_alibi refuses 0 / 1"""
    import ctypes as C

    from llm_b200 import _lib
    from llm_b200.neox import NeoxHparams, _bind
    L = _bind(_lib.lib())
    assert L.b200_init(0) == 0
    for arch in range(4):
        hp = NeoxHparams(n_vocab=320, n_embd=256, n_head=4, n_layer=2, n_rot=16, use_parallel_residual=1, wtype=B.Q4_0, context_size=128, arch=arch, has_lm_head=0)
        old, new = L.b200_neox_new(C.byref(hp)), L.b200_neox_new_alibi(C.byref(hp), 8.0)
        assert bool(old) == (arch < 2) and bool(new) == (arch >= 2), arch
        for h in (old, new):
            if h:
                L.b200_neox_free(h)


def test_model_files_load_like_tensors(orc, tmp_path):
    """an MPT and a BLOOM file written by write_model and loaded into Mpt / Bloom give the logits of the same tensors loaded directly"""
    from llm_b200 import loader
    from llm_b200.neox import Bloom, Mpt
    for arch, cls, make, cfg in ((A.MPT, Mpt, A.make_mpt, "mpt-tiny"), (A.BLOOM, Bloom, A.make_bloom, "bloom-tiny")):
        hp, tens = make(dict(A.MPT_CONFIGS[cfg], alibi_bias_max=6.0) if arch == A.MPT else A.BLOOM_CONFIGS[cfg], B.Q5_0, orc.quantize)
        shapes = (A.mpt_tensor_shapes if arch == A.MPT else A.bloom_tensor_shapes)(hp)
        name = "mpt" if arch == A.MPT else "bloom"
        header = dict(hp, max_seq_len=hp["n_ctx"], clip_kqv=-1.0, n_mult=1, file_type=2) if arch == A.MPT else dict(hp, n_mult=1, file_type=2)
        path = str(tmp_path / f"{name}.bin")
        loader.write_model(path, name, header, tens, shapes, B.Q5_0)
        f = loader.GgmlFile(path, name)
        words = f.hyperparameters()
        from_file = {t["name"]: f.tensor_bytes(i).view(np.float32) if t["type"] == 0 else f.tensor_bytes(i).reshape(t["ne"][1], -1) for i, t in enumerate(f.tensors())}
        f.close()
        fhp = dict(n_vocab=words["n_vocab"], n_ctx=hp["n_ctx"], n_embd=words["n_embd"], n_head=words["n_head"], n_layer=words["n_layer"], wtype=B.Q5_0)
        if arch == A.MPT:
            fhp["alibi_bias_max"] = words["alibi_bias_max"]
            assert fhp["alibi_bias_max"] == 6.0
        toks = np.arange(9, dtype=np.int32) * 7 % hp["n_vocab"]
        outs = []
        for tensors, h in ((tens, hp), (from_file, fhp)):
            m = cls(h, tensors)
            s = m.start_session(16)
            outs.append(s.evaluate(toks, all_logits=True))
            s.close(); m.close()
        check(outs[1], outs[0], f"{name}: file vs tensors")
