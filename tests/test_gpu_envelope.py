"""Bit-exact tests at the edges of the geometries the decode schedules accept: logits and both KV caches identical to the CPU model (the reference's
own ggml.c running the reference graph, oracle/_ref), at points of the envelope no other test reaches.

Three predicates define that envelope:
  - neox_decode_fits (decode_ops.cu): GPT-NeoX, MPT, GPT-J decode on the graph schedule for hd % 32 == 0, hd <= 128 (GPT-J: 256), n_embd % 128 == 0,
    n_embd <= 8192, n_ctx % 8 == 0, a context bucket attn_fused_fits admits, and rows of n_embd and 4 n_embd mmv_exact_stream_supported accepts;
  - graph_ok (session.cu): LLaMA decodes on the graph for hd 64 or 128 and n_embd <= 6144; wider models decode per op;
  - mmv_exact_stream_supported (exact_stream.cu): K with nb = K / 32 a multiple of 8 whose activation records fit the kernel's shared memory.
Every decode step asserts its launch count, so each case proves which schedule ran."""
import numpy as np
import pytest

from oracle import alibi as A
from oracle import bindings as B
from oracle import gptj as J
from oracle import synth

pytestmark = pytest.mark.gpu

FORMATS = ["q4_0", "q4_1", "q5_0", "q5_1", "q8_0"]
CHUNK = 512


def check(g, c, what):
    c = np.asarray(c, np.float32).reshape(np.shape(g))
    assert np.array_equal(np.asarray(g, np.float32).view(np.uint32), c.view(np.uint32)), (what, float(np.abs(g - c).max() / np.abs(c).max()), int((g != c).sum()))


def rng_tokens(hp, n, seed):
    return np.random.default_rng(seed).integers(0, hp["n_vocab"], size=n, dtype=np.int32)


def prefill(s, cpu, toks, a, b):
    """positions [a, b) in chunks of CHUNK; the last row of each chunk compared"""
    assert s.n_past == a
    for i in range(a, b, CHUNK):
        j = min(i + CHUNK, b)
        check(s.evaluate(toks[i:j]), cpu.eval(toks[i:j])[-1], f"prefill {i}..{j}")


def decode(s, cpu, toks, a, b, want):
    """one token per step at n_past = a .. b-1; want(launches) is True for the schedule the step must run"""
    for i in range(a, b):
        assert s.n_past == i
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        assert want(s.last_launches), ("schedule", i, s.last_launches)


def graph(n):
    return lambda launches: launches == n


def per_op(graph_launches):
    return lambda launches: launches > graph_launches


def neox_kv_equal(s, cpu, hp, v_by_position):
    """K [n_layer][n_ctx][n_embd]; the native V is by channel, the reference MPT graph keeps it by position"""
    nl, n_ctx, e = hp["n_layer"], hp["n_ctx"], hp["n_embd"]
    assert np.array_equal(s.kv(0), cpu.kv(0)), "K"
    v = cpu.kv(1)
    if v_by_position:
        v = v.reshape(nl, n_ctx, e).transpose(0, 2, 1).ravel()
    assert np.array_equal(s.kv(1), v), "V"


def gptj_cpu(hp, tens):
    if not J.have_ref():
        pytest.skip("oracle/_ref/libggml_gptj.so not built (the GPT-J CPU model is the reference graph on the reference's ggml)")
    return J.RefGptJ(hp, tens, n_threads=16, n_batch=CHUNK)


def neox_cpu(hp, tens):
    if not B.have_ref("ref"):
        pytest.skip("oracle/_ref/libggml_ref.so not built (the GPT-NeoX CPU model is the reference graph on the reference's ggml)")
    return B.RefLib("ref").neox(hp, tens, n_threads=16, n_batch=CHUNK)


def mpt_cpu(hp, tens):
    if not A.have_ref():
        pytest.skip("oracle/_ref/libggml_alibi.so not built (the MPT CPU model is the reference graph on the reference's ggml)")
    return A.RefAlibi(hp, tens, A.MPT, n_threads=16, n_batch=CHUNK)


def llama_cpu(orc, hp, tens):
    """the reference's own compiled ggml.c when oracle/_ref is present, else the plain-C port"""
    if B.have_ref("ref"):
        return B.RefLib("ref").llama(hp, tens, n_threads=16, n_batch=CHUNK)
    return orc.llama(hp, tens)


def short_sequence(s, cpu, hp, want, seed):
    """seven single tokens from an empty cache (fewer positions than CTAs in a cluster: some CTAs own no KQ positions), a 20-token batch, ten decode
    steps, a 17-token batch, one more step, a batch whose last row only comes back"""
    toks = rng_tokens(hp, 64, seed)
    decode(s, cpu, toks, 0, 7, want)
    check(s.evaluate(toks[7:27], all_logits=True), cpu.eval(toks[7:27]), "batch of 20")
    decode(s, cpu, toks, 27, 37, want)
    check(s.evaluate(toks[37:54], all_logits=True), cpu.eval(toks[37:54]), "batch of 17")
    decode(s, cpu, toks, 54, 55, want)
    check(s.evaluate(toks[55:60]), cpu.eval(toks[55:60])[-1], "last row only")
    assert s.n_past == 60


# ---- 1. the cluster attention at every cluster size --------------------------------------------------------------------------------------------
# attn_fused_kernel runs one cluster of hd / 32 CTAs per head.  GPT-J's wide form (hd > 128, NV = 8) covers clusters of 5..8: thread u of a quad
# feeds the scores to CTA u and, where u + 4 < hd / 32, to CTA u + 4 -- clusters of 5 and 7 send from only one or three of the four threads.
# 8 heads keep n_embd a multiple of 256: with 4 heads of 160 (n_embd 640, nb 20) mmv_exact_stream_supported refuses the rows and the model
# decodes per op, which the launch counts would catch.
GPTJ_CLUSTERS = {
    "hd160": dict(n_vocab=320, n_ctx=128, n_embd=1280, n_head=8, n_layer=2, n_rot=64),     # clusters of 5
    "hd224": dict(n_vocab=320, n_ctx=128, n_embd=1792, n_head=8, n_layer=2, n_rot=96),     # clusters of 7
    "hd128": dict(n_vocab=320, n_ctx=128, n_embd=512, n_head=4, n_layer=2, n_rot=32),      # the kernel of hd <= 128 under RoPE mode 0, n_rot < hd
}


def gptj_graph(hp):
    return 6 * hp["n_layer"] + 3


@pytest.mark.parametrize("qname", FORMATS)
@pytest.mark.parametrize("cfg", list(GPTJ_CLUSTERS))
def test_gptj_cluster_sizes(orc, cfg, qname):
    """GPT-J at clusters of 5, 7 and 4 CTAs per head, on the graph schedule at every step (neox_decode_fits: hd % 32 == 0, hd <= 256)"""
    from llm_b200 import GptJ
    hp, tens = J.make_gptj(GPTJ_CLUSTERS[cfg], B.QUANT_TYPES[qname], orc.quantize)
    cpu = gptj_cpu(hp, tens)
    m = GptJ(hp, tens)
    s = m.start_session(CHUNK)
    short_sequence(s, cpu, hp, graph(gptj_graph(hp)), 0xC1A5)
    neox_kv_equal(s, cpu, hp, False)
    s.close(); m.close(); cpu.close()


def second_kq_pass(hd):
    """the first n_past at which attn_fused_kernel (f16 cache) makes a second KQ pass: each of the hd / 32 CTAs takes per = ceil(n_kv / (hd / 32)) positions
    and one pass covers PU * ATH / 4 of them (PU = 16 / NV; NV = 8 for hd > 128, else 4; ATH = 256): 128 or 256 positions per CTA per pass"""
    per_pass = (16 // (8 if hd > 128 else 4)) * 256 // 4
    return per_pass * (hd // 32)            # n_kv > per_pass * hd / 32, i.e. n_past >= that


SOFT_MAX_SECOND_PASS = 4 * 256              # SB * ATH table look-ups per pass over the row: a second pass from n_kv 1025, n_past 1024


@pytest.mark.slow
@pytest.mark.parametrize("cfg,qname", [("hd160", "q5_1"), ("hd224", "q4_0"), ("hd128", "q8_0")])
def test_gptj_cluster_sizes_long_context(orc, cfg, qname):
    """n_ctx 2048, every step on the graph schedule (neox_decode_fits: attn_fused_fits admits every bucket up to 2048 at these head sizes): decode
    across the second KQ pass (n_past 640 at hd 160, 896 at hd 224, 1024 at hd 128), across the soft_max's second pass (n_past 1024), into the last
    slot; then ContextFull and both caches"""
    import llm_b200
    from llm_b200 import GptJ
    hp, tens = J.make_gptj(dict(GPTJ_CLUSTERS[cfg], n_ctx=2048), B.QUANT_TYPES[qname], orc.quantize)
    hd = hp["n_embd"] // hp["n_head"]
    kq2 = second_kq_pass(hd)
    assert kq2 == {"hd160": 640, "hd224": 896, "hd128": 1024}[cfg]
    toks = rng_tokens(hp, 2048, 0xC1A6)
    cpu = gptj_cpu(hp, tens)
    m = GptJ(hp, tens)
    s = m.start_session(CHUNK)
    want = graph(gptj_graph(hp))
    for a in sorted({kq2, SOFT_MAX_SECOND_PASS}):
        prefill(s, cpu, toks, s.n_past, a - 3)
        decode(s, cpu, toks, a - 3, a + 3, want)
    prefill(s, cpu, toks, s.n_past, 2042)
    decode(s, cpu, toks, 2042, 2048, want)
    with pytest.raises(llm_b200.ContextFull):
        s.evaluate(toks[:1])
    assert s.n_past == 2048
    neox_kv_equal(s, cpu, hp, False)
    s.close(); m.close(); cpu.close()


@pytest.mark.parametrize("qname", FORMATS)
def test_neox_hd128_sequential_residual(orc, qname):
    """GPT-NeoX with 128-wide heads (clusters of 4, the most the kernel of hd <= 128 takes) and the sequential residual, on the graph schedule"""
    from llm_b200.neox import GptNeoX
    hp, tens = synth.make_neox(dict(n_vocab=384, n_ctx=128, n_embd=512, n_head=4, n_layer=2, n_rot=32, use_parallel_residual=0), B.QUANT_TYPES[qname],
                               orc.quantize)
    cpu = neox_cpu(hp, tens)
    m = GptNeoX(hp, tens)
    s = m.start_session(CHUNK)
    short_sequence(s, cpu, hp, graph(8 * hp["n_layer"] + 3), 0xC1A7)
    neox_kv_equal(s, cpu, hp, False)
    s.close(); m.close(); cpu.close()


# ---- 2. n_embd 8192, the widest row the GPT-NeoX-family graph takes, and 8448, the first it refuses -------------------------------------------
# ln_pack_body holds the row in float4 v[MAXV], MAXV = 8: 8 x 256 threads x 4 = 8192 values, exactly full.

def wide_sequence(s, cpu, hp, want, seed):
    """a 100-token prefill (the wgmma GEMM serves batches of 96 tokens and more), then four decode steps"""
    toks = rng_tokens(hp, 104, seed)
    check(s.evaluate(toks[:100], all_logits=True), cpu.eval(toks[:100]), "prefill 100")
    decode(s, cpu, toks, 100, 104, want)


@pytest.mark.slow
def test_neox_width_8192(orc):
    """GPT-NeoX, 64 heads of 128, n_embd 8192 (neox_decode_fits: n_embd <= 8192; fc_out rows of 32768 = 1024 blocks), parallel residual: graph"""
    from llm_b200.neox import GptNeoX
    hp, tens = synth.make_neox(dict(n_vocab=384, n_ctx=256, n_embd=8192, n_head=64, n_layer=2, n_rot=32, use_parallel_residual=1), B.Q4_0, orc.quantize)
    cpu = neox_cpu(hp, tens)
    m = GptNeoX(hp, tens)
    s = m.start_session(CHUNK)
    wide_sequence(s, cpu, hp, graph(8 * hp["n_layer"] + 3), 0x8192)
    neox_kv_equal(s, cpu, hp, False)
    s.close(); m.close(); cpu.close()


@pytest.mark.slow
def test_mpt_width_8192(orc):
    """MPT, 64 heads of 128 (ALiBi: the attention kernel of hd <= 128), n_embd 8192, no biases (ln_pack_nobias_kernel): graph"""
    from llm_b200.neox import Mpt
    hp, tens = A.make_mpt(dict(n_vocab=320, n_ctx=256, n_embd=8192, n_head=64, n_layer=2, alibi_bias_max=8.0), B.Q5_0, orc.quantize)
    cpu = mpt_cpu(hp, tens)
    m = Mpt(hp, tens)
    s = m.start_session(CHUNK)
    wide_sequence(s, cpu, hp, graph(8 * hp["n_layer"] + 3), 0x8193)
    neox_kv_equal(s, cpu, hp, True)
    s.close(); m.close(); cpu.close()


@pytest.mark.slow
def test_gptj_width_8192(orc):
    """GPT-J, 32 heads of 256 (clusters of 8), n_embd 8192, Q8_0 (the largest ring stage beside 1024 activation records): graph"""
    from llm_b200 import GptJ
    hp, tens = J.make_gptj(dict(n_vocab=320, n_ctx=256, n_embd=8192, n_head=32, n_layer=2, n_rot=64), B.Q8_0, orc.quantize)
    cpu = gptj_cpu(hp, tens)
    m = GptJ(hp, tens)
    s = m.start_session(CHUNK)
    wide_sequence(s, cpu, hp, graph(gptj_graph(hp)), 0x8194)
    neox_kv_equal(s, cpu, hp, False)
    s.close(); m.close(); cpu.close()


@pytest.mark.slow
def test_neox_width_8448_per_op(orc):
    """GPT-NeoX at n_embd 8448 (66 heads of 128), one layer: neox_decode_fits refuses n_embd > 8192, so every step decodes per op, still exact"""
    from llm_b200.neox import GptNeoX
    hp, tens = synth.make_neox(dict(n_vocab=384, n_ctx=256, n_embd=8448, n_head=66, n_layer=1, n_rot=32, use_parallel_residual=0), B.Q4_1, orc.quantize)
    cpu = neox_cpu(hp, tens)
    m = GptNeoX(hp, tens)
    s = m.start_session(CHUNK)
    wide_sequence(s, cpu, hp, per_op(8 * hp["n_layer"] + 4), 0x8448)
    neox_kv_equal(s, cpu, hp, False)
    s.close(); m.close(); cpu.close()


# ---- 3. LLaMA wider than the graph's 6144 ------------------------------------------------------------------------------------------------------
LLAMA_WIDE = {
    "65b": (dict(n_vocab=512, n_embd=8192, n_head=64, n_head_kv=64, n_layer=2, n_ff=22016, n_rot=128, n_ctx=256), B.Q4_0),   # LLaMA-65B layers
    "70b": (dict(n_vocab=512, n_embd=8192, n_head=64, n_head_kv=8, n_layer=2, n_ff=28672, n_rot=128, n_ctx=256), B.Q5_1),    # LLaMA-2-70B: GQA 8
}


@pytest.mark.slow
@pytest.mark.parametrize("cfg", list(LLAMA_WIDE))
def test_llama_wider_than_graph(orc, cfg):
    """LLaMA-65B and LLaMA-2-70B layer geometry, 2 layers: graph_ok refuses n_embd > 6144, so decode runs per op -- the streaming mat-vec at
    K = 8192 and at K = n_ff (22016 / 28672: 688 / 896 blocks).  Prefill 95 tokens (the mma.sync GEMM) and 97 more (the wgmma GEMM, from 96), then
    four per-op decode steps and both caches."""
    import llm_b200
    base, t = LLAMA_WIDE[cfg]
    hp, tens = synth.make_llama(base, t, orc.quantize)
    nl = hp["n_layer"]
    toks = synth.make_tokens(hp, 196)
    cpu = llama_cpu(orc, hp, tens)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=CHUNK))
    check(s.evaluate(toks[:95], all_logits=True), cpu.eval(toks[:95]), "prefill 95")
    check(s.evaluate(toks[95:192], all_logits=True), cpu.eval(toks[95:192]), "prefill 97")
    decode(s, cpu, toks, 192, 196, per_op(8 * nl + 4))
    for which in (0, 1):          # the CPU model sizes its cache by n_embd; with GQA only the first n_layer * n_ctx * n_embd_gqa values are used
        a = s.kv(which)
        assert np.array_equal(a, cpu.kv(which)[:a.size]), which
    s.close(); m.close(); cpu.close()


# ---- 4. the exact mat-mul dispatch and the streaming mat-vec's limit ---------------------------------------------------------------------------
MM_AUTO, MM_EXACT_STREAM = 0, 5          # B200_MM_AUTO, B200_MM_EXACT_STREAM (include/llm_b200.h)
ERR_BAD_ARG = -2                         # B200_ERR_BAD_ARG


@pytest.fixture(scope="module")
def L():
    from llm_b200 import _lib
    lib = _lib.lib()
    assert lib.b200_init(0) == 0
    return lib


def mul_mat_case(orc, t, K, N, Bn, seed):
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    x = (rng.standard_normal((Bn, K)) * rng.uniform(0.05, 8, (Bn, 1))).astype(np.float32)
    x[Bn // 2, :32] = 0.0
    wq = orc.quantize(t, w)
    return wq, x, orc.mul_mat(t, wq, x)


@pytest.mark.parametrize("name", FORMATS)
@pytest.mark.parametrize("K", [4096, 704])
@pytest.mark.parametrize("Bn", [1, 15, 16, 95, 96, 97])
def test_mul_mat_auto_dispatch_edges(L, orc, name, K, Bn):
    """impl AUTO is mul_mat_exact_auto (mul_mat.cu), the dispatch of every session: the streaming mat-vec at B == 1 (K 4096; K 704 has 22 blocks,
    not a multiple of 8, so exact.cu), exact.cu below 16, the mma.sync GEMM below 96, the wgmma GEMM from 96.  N = 197 is ragged against every tile
    width (32-row mat-vec tiles, 64- and 128-wide GEMM tiles)"""
    t = B.QUANT_TYPES[name]
    N = 197
    wq, x, want = mul_mat_case(orc, t, K, N, Bn, K * 19 + Bn + t)
    got = np.empty((Bn, N), np.float32)
    assert L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, got.ctypes.data, MM_AUTO) == 0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, K, Bn, int((got != want).sum()))


def stream_max_k():
    """the largest K mmv_exact_stream_supported accepts, from its own formula: nb % 8 == 0 and nb * 64 + 256 + St<T_Q8_0>::RING_BYTES <= 227 KB, where
    RING_BYTES = SST (4) stages of SR (32) rows x SCB (16) blocks: Q8_0 quants (32 B per block) and scales (2 B), each row padded by 16 B (stream_core.cuh)"""
    SR, SCB, SST = 32, 16, 4
    ring = SST * (SR * (SCB * 32 + 16) + SR * (SCB * 2 + 16))
    nb = (227 * 1024 - 256 - ring) // 64 // 8 * 8
    return nb * 32


@pytest.mark.parametrize("name", FORMATS)
def test_mul_mat_stream_largest_k(L, orc, name):
    """impl EXACT_STREAM at the largest K it accepts (79104 = 2472 blocks), bit-exact; at the next multiple of 256 (79360) it returns B200_ERR_BAD_ARG"""
    t = B.QUANT_TYPES[name]
    K, N = stream_max_k(), 45
    assert K == 79104
    wq, x, want = mul_mat_case(orc, t, K, N, 1, 0x57EA + t)
    got = np.empty((1, N), np.float32)
    assert L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, 1, got.ctypes.data, MM_EXACT_STREAM) == 0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, K, int((got != want).sum()))
    K2 = K + 256
    wq2, x2, _ = mul_mat_case(orc, t, K2, 8, 1, 0x57EB + t)
    out = np.empty((1, 8), np.float32)
    assert L.b200_op_mul_mat(t, wq2.ctypes.data, K2, 8, x2.ctypes.data, 1, out.ctypes.data, MM_EXACT_STREAM) == ERR_BAD_ARG
