"""K-quant and mixed-type sessions across the decode envelope, bit for bit against the reference graphs on the same per-tensor types
(oracle/kquant.mk, oracle/neox_kquant.mk; on an F32 KV cache oracle/kquant_kv32.mk).

Every decode step compares its logits with the reference and asserts its launch count, which proves the schedule it ran; both KV caches are
compared at the end.  Prompts go in as chunks of 512 (n_batch 512), as in test_gpu_long_context.py.
  a. LLaMA, Q4_0 layers and the Q6_K output.weight the reference's quantizer writes, f16 cache, n_ctx 4096 (hd 128, and hd 64 with GQA 4): the
     graph across two bucket captures (256, 512), across n_kv 1024, across n_past 3072 (7 launches per layer + 4 below, 8 + 4 from there: the
     K-quant lm_head follows the two-kernel attention), into the last slot and ContextFull, then a rewind to 3000 that replays a lower bucket's
     graph after two-kernel steps.  The hd-128 model also runs in lockstep with a B200_SESSION_NO_GRAPH session: the same bits and counts.
  b. the same models on an F32 cache, n_ctx 2048: across the f32 cluster attention's bound (buckets up to 1536 fuse), the last slots; a
     B200_SESSION_UNFUSED session in lockstep decodes per op with the same bits.
  c. the per-op mixes at long context: Q4_K_M and Q3_K_M on an f16 cache (n_ctx 4096), Q5_K_M and Q2_K on an F32 cache (n_ctx 2048), at the hd-128
     geometry and at 8 heads of 128 over 2 K/V heads.
  d. prompt batches at the K-quant kernels' edges inside one session (31 / 32 / 33 / 63 / 64 / 65 / 96 / 512 tokens: the warp kernel, the tiled
     GEMM's full and ragged token tiles, the fused residual addend of wo and w2 on both), with n_ff 2816 (11 super-blocks per w2 row).
  e. the LLaMA-7B geometry: the real LLaMA-7B "Q4_0" file's types (Q6_K output) on the decode graph at n_past 512, and Q4_K_M per op.
  f. GPT-NeoX, GPT-2, MPT, BLOOM and GPT-J K-quant and mixed files at n_ctx 2048 (per op): across n_kv 1024, the last slots, a rewind; MPT and GPT-J
     again on an F32 cache.
  g. session features at n_past 3500 on a Q4_K_M model: from_snapshot, a session file round trip, embeddings on a decode step past 3072."""
import numpy as np
import pytest

import llm_b200
from llm_b200 import ModelKVMemoryType as KV
from oracle import bindings as B
from oracle import kquant as KQ
from oracle import neox_kquant as NK
from oracle import synth
from test_gpu_kquant_sessions import GQA, per_op_launches, write_and_load
from test_gpu_long_context import CHUNK, LLAMA_LONG, PER_OP, check, context_full, decode, prefill, ref_rewind
from test_gpu_neox_files import HP, KCASES, mixed_types, write

pytestmark = pytest.mark.gpu

F32CFG = dict(memory_k_type=KV.Float32, memory_v_type=KV.Float32)
NO_GRAPH, UNFUSED = 1, 2
HD128 = LLAMA_LONG["hd128_q4_0"][0]
HD64_GQA = LLAMA_LONG["hd64_gqa_q5_1"][0]


@pytest.fixture(scope="module")
def rkq():
    if not KQ.have_ref_kq():
        pytest.skip("oracle/_ref/libggml_ref_kq.so not built")
    return KQ.RefKq()


@pytest.fixture(scope="module")
def rkq32():
    if not KQ.have_ref_kq(kv32=True):
        pytest.skip("oracle/_ref/libggml_ref_kq_kv32.so not built")
    return KQ.RefKq(kv32=True)


@pytest.fixture(scope="module")
def nxkq():
    if not (NK.have_ref() and NK.have_ref(kv32=True)):
        pytest.skip("oracle/_ref/*_kq.so / *_kq_kv32.so not built")
    return NK.ref_lib()


def kv_equal(s, cpu):
    """both caches byte for byte, f16 or f32 (the reference sizes its cache by n_embd: with GQA only its first part is used)"""
    for which in (0, 1):
        got = np.ascontiguousarray(s.kv(which)).view(np.uint8)
        want = np.ascontiguousarray(cpu.kv(which)).view(np.uint8)[:got.size]
        assert np.array_equal(got, want), ("cache", which)


def neox_kv_equal(s, cpu):
    """both caches whole, f16 or f32; GPT-2, MPT and BLOOM keep V by position in the reference, the native cache by channel"""
    hp = s.model.hyperparameters
    for which in (0, 1):
        got = s.kv(which)
        want = np.ascontiguousarray(cpu.kv(which)).view(got.dtype)[:got.size]
        if which and cpu.arch in ("gpt2", "mpt", "bloom"):
            want = want.reshape(hp["n_layer"], s.model.context_size, hp["n_embd"]).transpose(0, 2, 1).ravel()
        assert np.array_equal(got.view(np.uint8), np.ascontiguousarray(want).view(np.uint8)), ("cache", which)


def prefill_all(ss, cpu, toks, a, b):
    """test_gpu_long_context.prefill for sessions fed the same tokens (the reference runs once)"""
    for i in range(a, b, CHUNK):
        j = min(i + CHUNK, b)
        want = cpu.eval(toks[i:j])[-1:]
        for s in ss:
            assert s.n_past == i
            check(np.asarray(s.evaluate(toks[i:j])).reshape(1, -1), want, f"prefill {i}..{j}")


def decode_all(ss, cpu, toks, a, b, wants, n_layer):
    """test_gpu_long_context.decode for sessions fed the same tokens: wants[k](n_past) is session k's launch count, or PER_OP"""
    for i in range(a, b):
        want = cpu.eval(toks[i:i + 1])
        for s, w in zip(ss, wants):
            assert s.n_past == i
            check(s.evaluate(toks[i:i + 1], all_logits=True), want, f"decode at n_past {i}")
            n = w(i)
            if n == PER_OP:
                assert s.last_launches > 8 * n_layer + 4, ("per-op schedule expected", i, s.last_launches)
            else:
                assert s.last_launches == n, ("schedule", i, s.last_launches, n)


def llama_case(ref, tmp_path, base, mix, n_ctx, flags=(0,), f32=False, model=None):
    """(hp, types, model loaded from its file, sessions with `flags`, reference on the same types); model: (hp, tensors, types) already drawn"""
    hp, tens, types = model or KQ.make_llama_mixed(dict(base, n_ctx=n_ctx), mix, ref)
    m = write_and_load(tmp_path, hp, tens, types, mix)
    ss = [m.start_session(llm_b200.InferenceSessionConfig(n_batch=CHUNK, flags=f, **(F32CFG if f32 else {}))) for f in flags]
    cpu = ref.llama_typed(hp, tens, types, n_threads=8, n_batch=CHUNK)
    return hp, types, m, ss, cpu


def close(m, ss, cpu):
    for s in ss:
        s.close()
    m.close(); cpu.close()


# ---- a. Q4_0 layers + Q6_K output on the decode graph, f16 cache, n_ctx 4096 ----------------------------------------------------------------

@pytest.mark.slow
@pytest.mark.parametrize("geom", ["hd128", "hd64_gqa"])
def test_q6_k_output_graph_long_context(rkq, tmp_path, geom):
    base = HD128 if geom == "hd128" else HD64_GQA
    flags = (0, NO_GRAPH) if geom == "hd128" else (0,)
    hp, types, m, ss, cpu = llama_case(rkq, tmp_path, base, "q4_0", 4096, flags)
    assert types["output.weight"] == B.Q6_K and all(t == B.Q4_0 for k, t in types.items() if k != "output.weight")
    nl, n_ctx = hp["n_layer"], hp["n_ctx"]
    graph = lambda i: 7 * nl + 4 if i < 3072 else 8 * nl + 4      # from n_past 3072: attn_kq + attn_sv, then quantize_row_q8_K + the Q6_K mat-vec
    wants = [graph] * len(ss)
    toks = synth.make_tokens(hp, n_ctx)
    for a, b in ((250, 260), (510, 515), (1020, 1030), (3068, 3076), (4090, n_ctx)):
        prefill_all(ss, cpu, toks, ss[0].n_past, a)
        decode_all(ss, cpu, toks, a, b, wants, nl)
    for s in ss:
        context_full(s, toks)
        kv_equal(s, cpu)
    for s in ss:
        s.rewind(3000)
    cpu.set_n_past(3000)
    other = synth.make_tokens(hp, 3003, seed=7)                    # new tokens: positions 3000..3002 are written afresh
    decode_all(ss, cpu, other, 3000, 3003, wants, nl)
    for s in ss:
        kv_equal(s, cpu)
    close(m, ss, cpu)


# ---- b. the same on an F32 cache, n_ctx 2048 ------------------------------------------------------------------------------------------------

def fused_f32(nl):
    return lambda i: 7 * nl + 4 if i + 1 <= 1536 else 8 * nl + 4       # the f32 cluster attention fuses buckets up to 1536 positions


@pytest.mark.parametrize("geom", ["hd128", "hd64_gqa"])
def test_q6_k_output_graph_f32_cache(rkq32, tmp_path, geom):
    hp, types, m, ss, cpu = llama_case(rkq32, tmp_path, HD128 if geom == "hd128" else HD64_GQA, "q4_0", 2048, (0, UNFUSED), f32=True)
    assert types["output.weight"] == B.Q6_K
    nl, n_ctx = hp["n_layer"], hp["n_ctx"]
    wants = [fused_f32(nl), lambda i: PER_OP]
    toks = synth.make_tokens(hp, n_ctx)
    for a, b in ((1530, 1545), (n_ctx - 6, n_ctx)):
        prefill_all(ss, cpu, toks, ss[0].n_past, a)
        decode_all(ss, cpu, toks, a, b, wants, nl)
    for s in ss:
        context_full(s, toks)
        kv_equal(s, cpu)
    close(m, ss, cpu)


# ---- c. the per-op mixes at long context ------------------------------------------------------------------------------------------------------

GEOMS = {"hd128": HD128, "gqa": GQA}


@pytest.mark.slow
@pytest.mark.parametrize("mix", ["q4_K_M", "q3_K_M"])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_per_op_mix_long_context(rkq, tmp_path, mix, geom):
    hp, types, m, ss, cpu = llama_case(rkq, tmp_path, GEOMS[geom], mix, 4096)
    nl, n_ctx = hp["n_layer"], hp["n_ctx"]
    want = per_op_launches(hp, types)
    toks = synth.make_tokens(hp, n_ctx, seed=hp["n_embd"] + hp["wtype"])
    for a, b in ((1020, 1030), (3068, 3076), (n_ctx - 6, n_ctx)):
        prefill(ss[0], cpu, toks, ss[0].n_past, a)
        decode(ss[0], cpu, toks, a, b, lambda i: want, nl)
    context_full(ss[0], toks)
    kv_equal(ss[0], cpu)
    close(m, ss, cpu)


@pytest.mark.parametrize("mix", ["q5_K_M", "q2_K"])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_per_op_mix_f32_cache(rkq32, tmp_path, mix, geom):
    hp, types, m, ss, cpu = llama_case(rkq32, tmp_path, GEOMS[geom], mix, 2048, f32=True)
    nl, n_ctx = hp["n_layer"], hp["n_ctx"]
    want = per_op_launches(hp, types)
    toks = synth.make_tokens(hp, n_ctx, seed=hp["n_embd"] + hp["wtype"])
    for a, b in ((1530, 1545), (n_ctx - 6, n_ctx)):
        prefill(ss[0], cpu, toks, ss[0].n_past, a)
        decode(ss[0], cpu, toks, a, b, lambda i: want, nl)
    context_full(ss[0], toks)
    kv_equal(ss[0], cpu)
    close(m, ss, cpu)


# ---- d. prompt batches at the K-quant kernels' edges -----------------------------------------------------------------------------------------

def test_prompt_batches_at_kernel_edges(rkq, tmp_path):
    """Q4_K_M, 8 heads of 128 over 2 K/V heads, n_embd 1024, n_ff 2816 (w2 rows of 11 super-blocks): batches below, at and past the tiled GEMM's
    32-token tile, each compared row by row and followed by one decode step"""
    hp, types, m, ss, cpu = llama_case(rkq, tmp_path, dict(GQA, n_ff=2816), "q4_K_M", 1024)
    s, nl = ss[0], hp["n_layer"]
    assert types["layers.0.feed_forward.w2.weight"] == B.Q4_K and types["layers.1.feed_forward.w2.weight"] == B.Q6_K
    want = per_op_launches(hp, types)
    toks = synth.make_tokens(hp, hp["n_ctx"], seed=0xED6E)
    for n in (31, 32, 33, 63, 64, 65, 96, 512):
        at = s.n_past
        check(s.evaluate(toks[at:at + n], all_logits=True), cpu.eval(toks[at:at + n]), f"prompt batch of {n} at {at}")
        decode(s, cpu, toks, at + n, at + n + 1, lambda i: want, nl)
    kv_equal(s, cpu)
    close(m, ss, cpu)


# ---- e. the LLaMA-7B geometry ----------------------------------------------------------------------------------------------------------------

MIXES_7B = ("q4_0", "q4_K_M")


@pytest.fixture(scope="module")
def llama_7b(rkq):
    """{mix: (hp, tensors, types)} of one synthetic 7b-2l model in both mixes.  A 7B-wide layer is too large for make_llama_mixed's float64 draws
    and one-thread quantizing to stay cheap (about a minute per mix), so each tensor is drawn here in float32 (N(0, 1/K), gains 1 + 0.1 N(0, 1), a
    generator per tensor) and quantized by the reference's own quantizers on threads; every tensor is quantized for both mixes from one
    draw and its f32 values are dropped at once."""
    from concurrent.futures import ThreadPoolExecutor
    hp = dict(synth.CONFIGS["7b-2l"])
    types = {mix: KQ.mix_types(hp, mix) for mix in MIXES_7B}
    KQ.quantize_as(rkq, B.Q4_0, np.zeros((1, 32), np.float32))             # the reference initialises its tables once, before the threads

    def quantize(t, w):                                                   # rows are independent: the largest matrices in 8 row blocks
        return np.concatenate(list(rows.map(lambda r: KQ.quantize_as(rkq, t, r), np.array_split(w, 8))))

    def draw(item):
        idx, (name, shp) = item
        rng = np.random.default_rng(0x7B000000 + idx)
        if len(shp) == 1:
            a = (1.0 + 0.1 * rng.standard_normal(shp)).astype(np.float32)
            return name, {mix: a for mix in MIXES_7B}
        w = rng.standard_normal(shp, dtype=np.float32) * np.float32(1.0 / np.sqrt(shp[1]))
        return name, {mix: quantize(types[mix][name], w) for mix in MIXES_7B}

    with ThreadPoolExecutor(8) as ex, ThreadPoolExecutor(8) as rows:
        drawn = dict(ex.map(draw, enumerate(synth.tensor_shapes(hp).items())))
    return {mix: (dict(hp, wtype=KQ.MIXES[mix][0]), {n: d[mix] for n, d in drawn.items()}, types[mix]) for mix in MIXES_7B}


@pytest.mark.parametrize("mix", MIXES_7B)
def test_llama_7b_geometry(rkq, llama_7b, tmp_path, mix):
    """q4_0: the types of the real LLaMA-7B Q4_0 file (Q6_K output.weight) on the decode graph, the step bench.py measures; q4_K_M per op"""
    hp, types, m, ss, cpu = llama_case(rkq, tmp_path, None, mix, None, model=llama_7b[mix])
    s, nl = ss[0], hp["n_layer"]
    assert hp["n_embd"] == 4096 and hp["n_ff"] == 11008 and hp["n_vocab"] == 32000 and hp["n_ctx"] == 1024
    assert types["output.weight"] == B.Q6_K
    want = 7 * nl + 4 if mix == "q4_0" else per_op_launches(hp, types)
    toks = synth.make_tokens(hp, 516, seed=0x7B)
    prefill(s, cpu, toks, 0, 512)
    decode(s, cpu, toks, 512, 516, lambda i: want, nl)
    kv_equal(s, cpu)
    close(m, ss, cpu)


# ---- f. the GPT-NeoX family from files at n_ctx 2048 --------------------------------------------------------------------------------------------

NEOX_RUNS = [(name, False) for name in KCASES] + [(name, True) for name, (arch, _) in KCASES.items() if arch in ("mpt", "gptj")]


@pytest.mark.parametrize("name,f32", NEOX_RUNS, ids=[f"{n}-{'f32' if f else 'f16'}" for n, f in NEOX_RUNS])
def test_neox_family_files_long_context(nxkq, tmp_path, name, f32):
    arch, kind = KCASES[name]
    hp0 = dict(HP[arch], n_ctx=2048)
    types = mixed_types(arch, dict(hp0, wtype=0), kind)
    base = types[NK.matrices(arch, dict(hp0, wtype=0))[-1]]
    hp, tens, types = NK.make_typed(arch, hp0, base, nxkq, types=types)
    if arch == "gpt2":
        assert tens["model/wpe"].shape[0] == 2048
    path = write(tmp_path, name, arch, hp, tens, types)
    m = llm_b200.load_dynamic(arch, path, llm_b200.ModelParameters(context_size=hp["n_ctx"]))
    assert m.context_size == 2048
    s = m.start_session(CHUNK, **(F32CFG if f32 else {}))
    cpu = NK.RefTyped(arch, hp, tens, types, n_threads=8, n_batch=CHUNK, kv32=f32)
    nl, n_ctx = hp["n_layer"], hp["n_ctx"]
    per_op = lambda i: PER_OP
    toks = np.random.default_rng(0x2048).integers(4, hp["n_vocab"], n_ctx).astype(np.int32)
    for a, b in ((1020, 1030), (n_ctx - 6, n_ctx)):
        prefill(s, cpu, toks, s.n_past, a)
        decode(s, cpu, toks, a, b, per_op, nl)
    context_full(s, toks)
    neox_kv_equal(s, cpu)
    s.rewind(1000)
    ref_rewind(cpu, toks, 1000)
    other = np.random.default_rng(7).integers(4, hp["n_vocab"], 1003).astype(np.int32)
    decode(s, cpu, other, 1000, 1003, per_op, nl)
    neox_kv_equal(s, cpu)
    s.close(); m.close(); cpu.close()


# ---- g. session features at long context -----------------------------------------------------------------------------------------------------

@pytest.mark.slow
def test_session_features_at_long_context(rkq, tmp_path):
    """Q4_K_M, f16 cache, n_ctx 4096, at n_past 3500: from_snapshot and a session file round trip each decode three steps bit for bit with the
    reference and end with its caches; embeddings of a decode step past 3072 are the reference's final norm row"""
    from oracle import embd as E
    hp, types, m, ss, cpu = llama_case(rkq, tmp_path, HD128, "q4_K_M", 4096)
    s, nl = ss[0], hp["n_layer"]
    want = per_op_launches(hp, types)
    toks = synth.make_tokens(hp, 3510, seed=0x3500)
    prefill(s, cpu, toks, 0, 3500)
    snap = s.get_snapshot()
    path = str(tmp_path / "session.bin")
    s.write_snapshot(path)
    assert snap.npast == 3500
    for restore in (lambda: type(s).from_snapshot(snap, m), lambda: type(s).read_snapshot(path, m)):
        r = restore()
        assert r.n_past == 3500
        cpu.set_n_past(3500)
        decode(r, cpu, toks, 3500, 3503, lambda i: want, nl)
        kv_equal(r, cpu)
        r.close()
    cpu.set_n_past(3500)
    req = llm_b200.OutputRequest(embeddings=np.empty(0, np.float32))
    g = s.evaluate(toks[3500:3501], all_logits=True, output_request=req)
    want_l, want_e, _ = E.eval_embd(cpu, toks[3500:3501])
    check(g, want_l, "logits of the step with embeddings")
    check(req.embeddings.reshape(1, -1), want_e[-1:], "embeddings at n_past 3500")
    assert s.last_launches == want
    decode(s, cpu, toks, 3501, 3503, lambda i: want, nl)
    kv_equal(s, cpu)
    close(m, ss, cpu)
