"""Bit-exact tests at the ragged geometries of published checkpoints, against the reference's own ggml.c running the reference graphs (oracle/_ref):

  checkpoint          arch      n_embd  heads x hd  n_rot  n_ff    what it drives
  OpenLLaMA-3B        LLaMA     3200    32 x 100    100    8640    per-op decode below 6144 wide (graph_ok wants hd 64 / 128); K = 3200 (100 blocks)
                                                                   and 8640 (270) are not whole groups of 8 blocks, so B = 1 runs mm_exact_kernel; KQ
                                                                   dots of 100 = 3 x 32 + 4 leftovers; RoPE mode 0 over 50 pairs
  Pythia-2.8B         GPT-NeoX  2560    32 x 80     20     10240   per-op decode (neox_decode_fits wants hd % 32 == 0); KQ leftovers of 16; RoPE mode 2 on
                                                                   10 pairs of an 80-wide head
  RedPajama-3B        GPT-NeoX  2560    32 x 80     80     10240   the same with full rotary (40 pairs)
  GPT-2 XL            GPT-2     1600    25 x 64     -      6400    per-op decode (n_embd % 128 != 0); K = 1600 (50 blocks) is not stream-supported
  Vicuna-7B           LLaMA     4096    32 x 128    128    11008   the graph schedule with 32001 logits rows: a partial last tile in the logits mat-vec

Each session case prefills in three batches, one per exact weight GEMM (< 16 tokens: mm_exact_kernel, 16..95: the mma.sync GEMM, >= 96: the wgmma
GEMM), then decodes single tokens, comparing the logits of every step on uint32 views and both KV caches whole; every decode step asserts its launch
count.  The weight type rotates through the five block formats so that each meets a K the streaming mat-vec refuses.  Layers are cut to 1 or 2 and
the vocabulary to a few hundred rows (but for the 32001-row case) so that the CPU reference stays quick.

The second half tests the attention mat-muls (exact.cu: mul_mat_f16_exact / mul_mat_f32_exact) through b200_op_mul_mat_kv against numpy
restatements of ggml_vec_dot_f16 and ggml_vec_dot_f32, which are themselves checked against the plain-C oracle and the pinned f32 restatement."""
import numpy as np
import pytest

import llm_b200
from llm_b200 import ModelKVMemoryType as KV
from llm_b200 import OutputRequest
from oracle import bindings as B
from oracle import kv32
from oracle import synth

CHUNK = 128
PREFILL = (7, 40, 100)          # mm_exact_kernel (< 16), exact_mma (16..95), exact_tc5 (>= 96)
DECODE = 9


def check(g, c, what):
    g = np.asarray(g, np.float32)
    c = np.asarray(c, np.float32).reshape(g.shape)
    bad = g.view(np.uint32) != c.view(np.uint32)
    assert not bad.any(), (what, int(bad.sum()), g.size, int(np.argmax(bad.ravel())), float(np.abs(g - c).max()))


def f16(t, w):
    return np.ascontiguousarray(w, np.float32).astype(np.float16)


# ---- the session cases -------------------------------------------------------------------------------------------------------------------------
OPENLLAMA_3B = dict(n_vocab=320, n_embd=3200, n_head=32, n_head_kv=32, n_layer=1, n_ff=8640, n_rot=100, n_ctx=256)
PYTHIA_2_8B = dict(n_vocab=384, n_ctx=256, n_embd=2560, n_head=32, n_layer=2, n_rot=20, use_parallel_residual=1)
REDPAJAMA_3B = dict(PYTHIA_2_8B, n_rot=80)
GPT2_XL = dict(n_vocab=320, n_ctx=256, n_embd=1600, n_head=25, n_layer=2)
VICUNA_7B = dict(n_vocab=32001, n_embd=4096, n_head=32, n_head_kv=32, n_layer=1, n_ff=11008, n_rot=128, n_ctx=256)

# name: (architecture, geometry, weight type, f32 cache)
CASES = {
    "openllama3b-q4_0":      ("llama", OPENLLAMA_3B, B.Q4_0, False),
    "openllama3b-q4_1-kv32": ("llama", OPENLLAMA_3B, B.Q4_1, True),
    "openllama3b-gqa4-q5_0": ("llama", dict(OPENLLAMA_3B, n_head_kv=8), B.Q5_0, False),    # the per-op KQ broadcasts 4 heads per K head
    "gpt2xl-q5_1":           ("gpt2", GPT2_XL, B.Q5_1, False),
    "gpt2xl-q8_0-kv32":      ("gpt2", GPT2_XL, B.Q8_0, True),
    "pythia2.8b-q8_0":       ("neox", PYTHIA_2_8B, B.Q8_0, False),
    "pythia2.8b-q4_0-kv32":  ("neox", PYTHIA_2_8B, B.Q4_0, True),
    "redpajama3b-q5_1":      ("neox", REDPAJAMA_3B, B.Q5_1, False),
}


def graph_launches(arch, hp):
    return {"llama": 7, "neox": 8, "gpt2": 8}[arch] * hp["n_layer"] + (4 if arch == "gpt2" else 3)


def stream_supported(K):
    """mmv_exact_stream_supported (exact_stream.cu) at these widths: a whole number of 8-block groups"""
    return (K // 32) % 8 == 0


def need_ref(kv_f32):
    if not B.have_ref("ref") or (kv_f32 and not kv32.have_ref()):
        pytest.skip("oracle/_ref not built (the CPU model is the reference graph on the reference's ggml)")


class Case:
    """a native session and the reference on the same tensors and cache type"""

    def __init__(self, orc, arch, base, wtype, kv_f32, cpu=None):
        need_ref(kv_f32)
        quant = f16 if wtype == B.F16 else orc.quantize
        kv = KV.Float32 if kv_f32 else KV.Float16
        self.arch, self.kv_f32 = arch, kv_f32
        ref = kv32.ref_lib() if kv_f32 else B.RefLib("ref")
        if arch == "llama":
            self.hp, tens = synth.make_llama(base, wtype, quant)
            self.m = llm_b200.Llama(self.hp, llm_b200.ModelParameters(context_size=self.hp["n_ctx"]), tens)
            self.s = self.m.start_session(llm_b200.InferenceSessionConfig(n_batch=CHUNK, memory_k_type=kv, memory_v_type=kv))
            self.cpu = cpu(self.hp, tens) if cpu else ref.llama(self.hp, tens, n_threads=16, n_batch=CHUNK)
        else:
            from llm_b200.neox import Gpt2, GptNeoX
            make, cls = (synth.make_neox, GptNeoX) if arch == "neox" else (synth.make_gpt2, Gpt2)
            self.hp, tens = make(base, wtype, quant)
            self.m = cls(self.hp, tens)
            self.s = self.m.start_session(CHUNK, memory_k_type=kv, memory_v_type=kv)
            self.cpu = getattr(ref, arch)(self.hp, tens, n_threads=16, n_batch=CHUNK)
        self.toks = synth.make_tokens(self.hp, sum(PREFILL) + DECODE + 4, seed=self.hp["n_embd"] + wtype)

    def cpu_kv(self, which):
        return kv32.kv_f32(self.cpu, which) if self.kv_f32 else self.cpu.kv(which)

    def kv_equal(self, s=None):
        s = s or self.s
        hp = self.hp
        for which in (0, 1):
            got, want = s.kv(which), self.cpu_kv(which)
            if which == 1 and self.arch == "gpt2":      # the native V is by channel, the reference GPT-2 graph keeps it by position
                want = want.reshape(hp["n_layer"], hp["n_ctx"], hp["n_embd"]).transpose(0, 2, 1).ravel()
            want = want[:got.size]                      # LLaMA: the reference sizes its cache by n_embd; with GQA only n_embd_gqa of each row is used
            want = np.ascontiguousarray(want)
            assert got.nbytes == want.nbytes and np.array_equal(got.view(np.uint8), want.view(np.uint8)), ("cache", which)

    def prefill(self):
        at = 0
        for n in PREFILL:
            check(self.s.evaluate(self.toks[at:at + n], all_logits=True), self.cpu.eval(self.toks[at:at + n]), f"prefill of {n} at {at}")
            at += n
        return at

    def decode(self, a, b, want):
        for i in range(a, b):
            assert self.s.n_past == i
            check(self.s.evaluate(self.toks[i:i + 1], all_logits=True), self.cpu.eval(self.toks[i:i + 1]), f"decode at n_past {i}")
            assert want(self.s.last_launches), ("schedule", i, self.s.last_launches)

    def close(self):
        self.s.close(); self.m.close(); self.cpu.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_session_matches_reference(orc, name):
    """three prefill batches, then decode steps per op (every case here is outside its graph schedule), logits of every step and both caches"""
    arch, base, wtype, kv_f32 = CASES[name]
    c = Case(orc, arch, base, wtype, kv_f32)
    hp = c.hp
    ks = [hp["n_embd"], hp["n_ff"] if arch == "llama" else 4 * hp["n_embd"]]
    if arch != "neox":
        assert not stream_supported(ks[0]), "the case must put B = 1 on mm_exact_kernel"
    at = c.prefill()
    graph = graph_launches(arch, hp)
    c.decode(at, at + DECODE, lambda n: n > graph)
    c.kv_equal()
    if arch == "neox" and not kv_f32:
        # InferenceSession::get_snapshot / from_snapshot at this geometry, then one more step on the restored session
        snap = c.s.get_snapshot()
        r = type(c.s).from_snapshot(snap, c.m)
        i = at + DECODE
        check(r.evaluate(c.toks[i:i + 1], all_logits=True), c.cpu.eval(c.toks[i:i + 1]), "decode after from_snapshot")
        assert r.last_launches > graph
        c.kv_equal(r)
        r.close()
    c.close()


@pytest.mark.gpu
def test_openllama3b_f16_weights():
    """F16 weights at K = 3200 and 8640: the ordered-FMA GEMM for the prefill batches, and per-op decode on the streaming F16 mat-vec, which
    mmv_f16_supported (exact_f16.cu: K % 64 == 0 and the fp16 row within shared memory) accepts at both widths; the GEMM would serve a row it
    refused, with the same launch count"""
    c = Case(None, "llama", OPENLLAMA_3B, B.F16, False)
    assert all(K % 64 == 0 and 2 * K < 64 * 1024 for K in (3200, 8640))
    at = c.prefill()
    c.decode(at, at + DECODE, lambda n: n == 17 * c.hp["n_layer"] + 4)       # the per-op schedule of one token
    c.kv_equal()
    c.close()


@pytest.mark.gpu
def test_vicuna7b_odd_vocabulary(orc):
    """LLaMA-7B with a 32001-row lm_head on the graph schedule: the logits mat-vec ends in a tile of one row.  Embeddings on a prefill and a decode
    step, top_k and the default sampler chain on the resulting rows"""
    from oracle import embd as E
    from oracle.sampler import SamplerOracle
    if not E.have_ref():
        pytest.skip("oracle/_ref/*_embd.so not built")
    c = Case(orc, "llama", VICUNA_7B, B.Q4_1, False, cpu=lambda hp, t: E.model("llama", hp, t, n_threads=16, n_batch=CHUNK))
    hp, s, cpu, toks = c.hp, c.s, c.cpu, c.toks
    assert hp["n_vocab"] % 32 == 1
    graph = graph_launches("llama", hp)

    def with_embeddings(t, what):
        want_logits, want_embd = E.eval_embd(cpu, t)[:2]
        r = OutputRequest(embeddings=np.empty(0, np.float32))
        check(s.evaluate(t, all_logits=True, output_request=r), want_logits, f"{what}: logits")
        check(r.embeddings, want_embd[-1], f"{what}: embeddings")

    with_embeddings(toks[:PREFILL[0]], "prefill")
    at = PREFILL[0]
    for n in PREFILL[1:]:
        check(s.evaluate(toks[at:at + n], all_logits=True), cpu.eval(toks[at:at + n]), f"prefill of {n}")
        at += n
    with_embeddings(toks[at:at + 1], "decode")
    assert s.last_launches == graph, s.last_launches
    c.decode(at + 1, at + DECODE, lambda n: n == graph)
    c.kv_equal()
    at += DECODE

    so = SamplerOracle()
    row = np.asarray(cpu.eval(toks[at:at + 1]), np.float32).reshape(-1)
    check(s.evaluate(toks[at:at + 1], all_logits=True), row, "decode before sampling")
    at += 1
    for k in (40, 1024):                                    # descending, ties by ascending id
        order = np.lexsort((np.arange(row.size), -row.astype(np.float64)))[:k]
        ids, vals = s.top_k(k)
        assert np.array_equal(ids, order.astype(np.int32)), k
        check(vals, row[order], f"top_k {k}")
    hist = list(toks[:at])
    rng = llm_b200.Rng(0x7A11)
    params = llm_b200.InferenceParameters()
    for i in range(3):
        rc, want, *_ = so.sample(row, np.array(hist, np.int32), len(hist), seed=rng.seed, draw=rng.draw)
        assert rc == 0
        tok = s.infer_next_token(params, rng)
        assert tok == want, (i, tok, want)
        assert s.last_launches == graph
        hist.append(tok)
        row = np.asarray(cpu.eval(np.array([tok], np.int32)), np.float32).reshape(-1)
        check(s.last_logits, row, f"last_logits after sampled token {i}")
    c.kv_equal()
    c.close()


# ---- the attention mat-muls at op level -------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fmaf on float32 arrays: the product is exact in double; the sum is rounded to odd in double (TwoSum), whose rounding to float32 is then
    the correctly rounded a * b + c (finite operands)"""
    p = a.astype(np.float64) * b.astype(np.float64)
    c = np.broadcast_to(c, p.shape).astype(np.float64)
    s = p + c
    bp = s - p
    err = (p - (s - bp)) + (c - bp)
    even = (s.view(np.uint64) & 1) == 0
    nudge = (err != 0) & even & np.isfinite(s)
    s = np.where(nudge, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def reduce32(c):
    """GGML_F32x8_REDUCE over the last axis of 32 chains"""
    c = c[..., :16] + c[..., 16:]
    c = c[..., :8] + c[..., 8:]
    c = c[..., :4] + c[..., 4:]
    return (c[..., 0] + c[..., 1]) + (c[..., 2] + c[..., 3])


def dots_f16(a16, b32):
    """ggml_vec_dot_f16 of rows a16 (fp16) with rows b32 rounded to fp16, broadcast over the leading axes: 32 f32 FMA chains (fp16 products are
    exact in f32), the reduce tree, the leftovers added in double"""
    a = a16.astype(np.float32)
    b = b32.astype(np.float16).astype(np.float32)
    n = a.shape[-1]
    n32 = n & ~31
    shape = np.broadcast_shapes(a.shape[:-1], b.shape[:-1])
    c = np.zeros(shape + (32,), np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for k in range(0, n32, 32):
            c = c + a[..., k:k + 32] * b[..., k:k + 32]
        s = reduce32(c).astype(np.float64)
        for k in range(n32, n):
            s = s + (a[..., k] * b[..., k]).astype(np.float64)
        return s.astype(np.float32)


def dots_f32(a, b):
    """ggml_vec_dot_f32 (the rule of tests/test_kv_f32_oracle.py) broadcast over the leading axes"""
    n = a.shape[-1]
    n32 = n & ~31
    shape = np.broadcast_shapes(a.shape[:-1], b.shape[:-1])
    c = np.zeros(shape + (32,), np.float32)
    for k in range(0, n32, 32):
        c = fma32(a[..., k:k + 32], b[..., k:k + 32], c)
    s = reduce32(c)
    nv = (n - n32) & ~3
    for k in range(n32, n32 + nv):
        s = s + a[..., k] * b[..., k]
    for k in range(n32 + nv, n):
        s = fma32(a[..., k], b[..., k], s)
    return np.asarray(s, np.float32)


NE00 = [1, 3, 4, 7, 8, 12, 31, 33, 45, 64, 80, 100, 127, 128, 256, 513]


def operands(rng, n, rows, f16_edges):
    """rows x n values for either operand; with f16_edges some are fp16 rounding ties, fp16 subnormals and values that overflow fp16"""
    x = rng.standard_normal((rows, n)).astype(np.float32)
    if f16_edges:
        h = x.astype(np.float16)
        tie = ((h.astype(np.float32) + np.nextafter(h, np.float16(np.inf)).astype(np.float32)) * 0.5).astype(np.float32)
        m = rng.random(x.shape) < 0.25
        x[m] = tie[m]
        sub = rng.random(x.shape) < 0.05
        x[sub] = (rng.standard_normal(int(sub.sum())) * 3e-6).astype(np.float32)
    return x


@pytest.mark.parametrize("n", NE00)
def test_dot_restatements_match_oracles(orc, n):
    """the numpy restatements above against the plain-C ggml_vec_dot_f16 and the pinned ggml_vec_dot_f32 restatement, row by row (no GPU)"""
    from test_kv_f32_oracle import vec_dot_f32
    rng = np.random.default_rng(0xD07 + n)
    a = operands(rng, n, 6, True)
    b = operands(rng, n, 6, True)
    a16 = a.astype(np.float16)
    got16 = dots_f16(a16, b)
    got32 = dots_f32(a, b * 3)
    for r in range(6):
        want16 = orc.vec_dot_f16(a16[r].view(np.uint16), b[r].astype(np.float16).view(np.uint16))
        assert np.float32(got16[r]).view(np.uint32) == np.float32(want16).view(np.uint32), (n, r, got16[r], want16)
        want32 = vec_dot_f32(a[r], b[r] * 3)
        assert np.float32(got32[r]).view(np.uint32) == np.float32(want32).view(np.uint32), (n, r, got32[r], want32)


# (rows of src0 ne01, src1 rows ne11, src0 matrices ne02, broadcast ne12 / ne02, causal: n_past or -1, src1 row padding in floats)
KV_SHAPES = [
    (300, 1, 1, 8, -1, 0),          # decode KQ of one query row against 300 positions, 8 query heads per K head
    (33, 20, 2, 4, 13, 0),          # prefill KQ: 20 query rows after 13 positions, causal; the tiled kernel
    (1, 9, 3, 1, -1, 0),            # one source row
    (65, 16, 1, 1, -1, 1),          # src1 rows not 16-byte aligned: the one-warp-per-dot kernel for a batch
]
SENTINEL = np.float32(-12345.5)


def run_kv(L, src0_type, a, ne00, ne01, ne02, ne11, ne12, b, pad, causal):
    """the cache layouts of the sessions: src0 [ne01][ne02][ne00] (nb01 = ne02 * ne00 elements, nb02 = ne00), src1 [ne11][ne12 * ne00 + pad]
    (nb12 = ne00 floats), dst [ne12][ne11][ne01]"""
    es = a.itemsize
    ld1 = ne12 * ne00 + pad
    src1 = np.zeros((ne11, ld1), np.float32)
    src1[:, :ne12 * ne00] = b.reshape(ne11, ne12 * ne00)
    dst = np.full((ne12, ne11, ne01), SENTINEL, np.float32)
    rc = L.b200_op_mul_mat_kv(src0_type, a.ctypes.data, ne00, ne01, ne02, ne02 * ne00 * es, ne00 * es, src1.ctypes.data, ne11, ne12, ld1 * 4, ne00 * 4,
                              dst.ctypes.data, ne01 * 4, ne11 * ne01 * 4, causal)
    assert rc == 0, rc
    return dst


@pytest.fixture(scope="module")
def L():
    from llm_b200 import _lib
    lib = _lib.lib()
    assert lib.b200_init(0) == 0
    return lib


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["f16", "f32"])
@pytest.mark.parametrize("n", NE00)
def test_op_mul_mat_kv(L, form, n):
    """mul_mat_f16_exact / mul_mat_f32_exact at every leftover count and a few whole multiples of 32, with GQA broadcast, the causal skip (whose
    outputs keep the caller's values) and both kernels (tiled for aligned batches, one warp per dot otherwise)"""
    rng = np.random.default_rng(0x4B5 + n * 2 + (form == "f32"))
    for ne01, ne11, ne02, ratio, causal, pad in KV_SHAPES:
        ne12 = ne02 * ratio
        a = operands(rng, n, ne01 * ne02, form == "f16").reshape(ne01, ne02, n)
        b = operands(rng, n, ne11 * ne12, form == "f16").reshape(ne11, ne12, n)
        if form == "f16":
            a = a.astype(np.float16)
            a[:, :, 1::5] = (rng.standard_normal(a[:, :, 1::5].shape) * 2e-5).astype(np.float16)     # fp16 subnormal weights
            a = np.where(a == 0, np.float16(0.5), a)                                                  # no inf * 0 below
            if ne11 > 1:
                b[1, :, n // 2] = 70000.0 * (1 if n % 2 else -1)                                      # rounds to +-inf in fp16: row 1 is +-inf
            want = dots_f16(a.transpose(1, 0, 2)[np.arange(ne12) // ratio][:, None, :, :], b.transpose(1, 0, 2)[:, :, None, :])
        else:
            want = dots_f32(a.transpose(1, 0, 2)[np.arange(ne12) // ratio][:, None, :, :], b.transpose(1, 0, 2)[:, :, None, :])
        assert not np.isnan(want).any()
        got = run_kv(L, B.F16 if form == "f16" else B.F32, np.ascontiguousarray(a), n, ne01, ne02, ne11, ne12, b, pad, causal)
        if causal >= 0:
            skip = np.arange(ne01)[None, :] > causal + np.arange(ne11)[:, None]
            want = np.where(skip[None], SENTINEL, want)
            assert skip.any()
        check(got, want, f"{form} ne00={n} ne01={ne01} ne11={ne11} ne02={ne02} x{ratio} causal={causal} pad={pad}")


@pytest.mark.gpu
def test_op_mul_mat_kv_refusals(L):
    a = np.zeros(64, np.float32)
    out = np.zeros(64, np.float32)
    ok = dict(ne00=8, ne01=2, ne02=1, nb01=32, nb02=64, ne11=2, ne12=1, nb11=32, nb12=64, nbd1=8, nbd2=16, c=-1)

    def call(t=B.F32, **kw):
        p = dict(ok, **kw)
        return L.b200_op_mul_mat_kv(t, a.ctypes.data, p["ne00"], p["ne01"], p["ne02"], p["nb01"], p["nb02"], a.ctypes.data, p["ne11"], p["ne12"],
                                    p["nb11"], p["nb12"], out.ctypes.data, p["nbd1"], p["nbd2"], p["c"])
    assert call() == 0
    assert call(t=B.Q4_0) == -2
    assert call(ne00=0) == -2
    assert call(ne02=2, ne12=3) == -2                   # ne12 % ne02
    assert call(nb01=28) == -2                          # rows overlap
    assert call(ne11=65536) == -2
