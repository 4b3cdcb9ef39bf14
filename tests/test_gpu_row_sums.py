"""The norms' row sums are the reference's to the last bit, on rows where the order of the double additions shows.

ggml_compute_forward_rms_norm_f32 / _norm_f32 (LC/ggml.c:10063-10175) add a row in index order in a double and keep (float)(sum / n).  The
kernels add the same terms in a tree, and that changes the float on rows built for it: a large term whose in-order sum lands exactly on a float
rounding midpoint of sum / n, then a tail of terms each below half an ulp of the running sum -- in order each is absorbed and the tie rounds to
even; added to each other first they survive and round the other way.  Every such row is built here from a seed by a small search, and the CPU
tests below show that it does split the two orders and that the reference's own op takes the in-order side.

Softmax is the counter-case: its terms are fp16 table values in (0, 1], multiples of 2^-24, so any partial sum of up to 2^29 of them is exact
in a double and the order cannot show.  Its tests pin that, on rows whose exponentials span the whole fp16 range.

The GPU tests compare bit for bit against the reference's ggml.c: the seam's RMS_NORM / NORM / SOFT_MAX (and scale -> diag_mask_inf ->
soft_max) per op, and whole native sessions whose layer-0 norm sees an adversarial embedding row, in a prefill batch and as one decode step."""
import math

import numpy as np
import pytest

from oracle import bindings as B
from oracle import synth

F32 = np.float32
NORM_EPS = F32(1e-5)


# ---- the two orders, predicted in numpy (f32 arithmetic is IEEE round-to-nearest, as the reference's) ----------------------------------

def _dsum(t, exact):
    """the double sum of `t`: in index order (add.accumulate is one add after another) or exact (math.fsum)"""
    t = np.asarray(t, np.float64)
    return math.fsum(t) if exact else float(np.add.accumulate(t)[-1])


def rms_predict(x, eps, exact):
    """(mean, scale, rms_norm(x)) with the row sum added in order (the reference) or exactly (what a tree sum approaches)"""
    x = np.asarray(x, F32)
    mean = F32(_dsum(x * x, exact) / x.size)
    scale = F32(1.0) / np.sqrt(mean + F32(eps))
    return mean, scale, x * scale


def norm_predict(x, exact):
    """((mean, variance, scale), norm(x)) with both row sums in order or exact"""
    x = np.asarray(x, F32)
    mean = F32(_dsum(x, exact) / x.size)
    v = x - mean
    variance = F32(_dsum(v * v, exact) / x.size)
    scale = F32(1.0) / np.sqrt(variance + NORM_EPS)
    return (mean, variance, scale), v * scale


def _bits(a):
    return np.asarray(a, F32).view(np.uint32)


def splits(op, x, eps=5e-6):
    """the in-order and the exact sums give a different row"""
    a = rms_predict(x, eps, False)[2] if op == "rms" else norm_predict(x, False)[1]
    b = rms_predict(x, eps, True)[2] if op == "rms" else norm_predict(x, True)[1]
    return not np.array_equal(_bits(a), _bits(b))


# ---- adversarial rows -------------------------------------------------------------------------------------------------------------------

def _midpoint_heads(n, rng, square, draw):
    """(x0, c, k, t): x0 then x1 = c * k (c odd, k a power of two) make an in-order sum Q (of squares when `square`) with Q / n exactly a midpoint between two floats, and a tail
    term t (t * t when `square`) at most a quarter of an ulp of Q, so that in order every tail term is absorbed."""
    odd = n // (n & -n)
    while True:
        x0 = float(draw(rng))
        t0 = float(F32(x0) * F32(x0)) if square else x0
        p = math.frexp(t0)[1] - 1                                   # t0 in [2^p, 2^(p+1))
        for s in range(p - 28, p - 23):                             # the lowest set bit of Q: below t0's ulp, so Q / 2^s is odd
            if square and s % 2:
                continue
            for c in (1, 3, 5, 7):
                k = 2.0 ** (s // 2) if square else 2.0 ** s
                x1 = c * k
                Q = t0 + (x1 * x1 if square else x1)
                q = int(Q / 2.0 ** s)
                if q % 2 == 0 or q % odd or not (1 << 24) <= q // odd < (1 << 25):
                    continue                                        # Q / n = (q / odd) 2^(s - log2(n / odd)): a 25-bit odd mantissa, a midpoint
                ulp = 2.0 ** (math.frexp(Q)[1] - 53)
                t = 2.0 ** math.floor((math.log2(ulp) - 2) / 2) if square else ulp / 4
                yield x0, c, k, t


def f32_row(op, n, seed):
    """an adversarial f32 row of length n for rms_norm ("rms") or norm ("norm"): x0, x1, then n - 2 tail terms"""
    rng = np.random.default_rng(seed)
    for x0, c, k, t in _midpoint_heads(n, rng, op == "rms", lambda r: F32(r.uniform(2048.0, 8192.0))):
        x = np.full(n, t, F32)
        x[0], x[1] = x0, c * k
        if splits(op, x):
            return x
    raise AssertionError("unreachable")


def _q8_0_row(blocks):
    """[(d, q[32])] -> (GGML Q8_0 bytes, dequantized f32 values: q * f32(f16(d)), exact)"""
    raw, vals = [], []
    for d, q in blocks:
        q = np.asarray(q, np.int8)
        raw.append(np.concatenate([np.array([d], np.float16).view(np.uint8), q.view(np.uint8)]))
        vals.append(q.astype(F32) * F32(np.float16(d)))
    return np.concatenate(raw), np.concatenate(vals)


def _f16_ok(v):
    return 2.0 ** -24 <= abs(v) <= 65504.0 and float(np.float16(v)) == v


def q8_0_rms_row(n, seed):
    """an rms_norm-adversarial row that Q8_0 holds: block 0 = d0 * q0 then zeros, block 1 = 2^k * c then zeros, the rest blocks of 2^j * 1"""
    rng = np.random.default_rng(seed)
    draw = lambda r: float(np.float16(r.uniform(0.25, 1.0))) * int(r.integers(90, 128))
    for x0, c, k, t in _midpoint_heads(n, rng, True, draw):
        q0 = next(q for q in range(127, 0, -1) if _f16_ok(x0 / q))
        if not (_f16_ok(k) and _f16_ok(t)):
            continue
        z = np.zeros(32, np.int8)
        head = [(x0 / q0, np.r_[q0, z[1:]]), (k, np.r_[c, z[1:]])]
        raw, x = _q8_0_row(head + [(t, np.ones(32, np.int8))] * (n // 32 - 2))
        if splits("rms", x):
            return raw, x
    raise AssertionError("unreachable")


def f16_rms_row(n, seed):
    """an rms_norm-adversarial row of halves: x0, x1, then n - 2 tail terms"""
    rng = np.random.default_rng(seed)
    for x0, c, k, t in _midpoint_heads(n, rng, True, lambda r: float(np.float16(r.uniform(16.0, 128.0)))):
        if not (_f16_ok(c * k) and _f16_ok(t)):
            continue
        x = np.full(n, t, np.float16)
        x[0], x[1] = x0, c * k
        if splits("rms", x.astype(F32)):
            return x
    raise AssertionError("unreachable")


def q8_0_norm_row(n):
    """a norm-adversarial row that Q8_0 holds (n = 256).  Its values are multiples of 2^-24, so a double sum can only round once it passes
    2^29: five blocks of 127 * 65504 take it to Q ~ 1.33e9 (ulp 2^-22), 64 and -31 ulp bring it to 31 ulp below a midpoint B of Q / n, and
    the 32 tail terms are 0.75 ulp each.  In order each rounds up to a whole ulp and the sum ends at B + 1 ulp (the float above); exactly it
    ends at B - 7 ulp (the float below)."""
    assert n == 256
    big, z = np.full(32, 127, np.int8), np.zeros(32, np.int8)
    blocks = [(65504.0, big)] * 5 + [(1.0, np.r_[64, z[1:]]), (2.0 ** -22, np.r_[-31, z[1:]]), (2.0 ** -24, np.full(32, 3, np.int8))]
    raw, x = _q8_0_row(blocks)
    assert splits("norm", x)
    return raw, x


# ---- the row a weight format's activations carry: tune one gain so that the two orders also give different activations ------------------

def _act_bytes(act, ref, y):
    y = np.asarray(y, F32)
    return ref.from_float(B.Q8_0, y) if act == "q8_0" else y.astype(np.float16).view(np.uint8)


def tune_gain(ref, pre_a, pre_b, gain, bias, act, i0=0):
    """pre_a / pre_b: the normed row before its gain (in order / exact).  Returns a copy of `gain` whose element i0 (in [2, 4): the largest of
    its block) makes the activations the next mat-mul reads differ too -- Q8_0 records (an f16 scale per block) or f16 values -- so a 1-ulp
    difference in the norm cannot vanish in them."""
    cand = (np.float32(2.0).view(np.uint32) + np.arange(1 << 21, dtype=np.uint32)).view(F32)
    ya, yb = pre_a[i0] * cand, pre_b[i0] * cand
    if bias is not None:
        ya, yb = ya + bias[i0], yb + bias[i0]
    if act == "q8_0":
        ya, yb = np.abs(ya) / F32(127), np.abs(yb) / F32(127)
    for k in np.flatnonzero(ya.astype(np.float16) != yb.astype(np.float16))[:64]:
        g = gain.copy()
        g[i0] = cand[k]
        a, b = pre_a * g, pre_b * g
        if bias is not None:
            a, b = a + bias, b + bias
        if not np.array_equal(_act_bytes(act, ref, a), _act_bytes(act, ref, b)):
            return g
    raise AssertionError("no gain separates the activations")


# ---- CPU: the fixtures split the orders, and the reference takes the in-order side -------------------------------------------------------

SIZES = [256, 320, 4096, 5120, 8192]
RMS_EPS = [5e-6, 1e-6]


def ref_op(ref, op, x, eps=5e-6):
    x = np.ascontiguousarray(x, F32)
    rows, n = x.reshape(-1, x.shape[-1]).shape
    return ref.op(1 if op == "rms" else 2, 0, None, x, (n, rows, 1), fparams=(eps, 0), out_shape=x.shape)


@pytest.mark.parametrize("n", SIZES)
def test_fixture_rms_rows_split_and_reference_is_in_order(ref, orc, n):
    x = f32_row("rms", n, n)
    for eps in RMS_EPS:
        ma, sa, ya = rms_predict(x, eps, False)
        mb, sb, _ = rms_predict(x, eps, True)
        assert ma != mb and sa != sb, (n, eps, ma, mb, sa, sb)
        got = ref_op(ref, "rms", x[None], eps)[0]
        assert np.array_equal(_bits(got), _bits(ya)), (n, eps)
        assert np.array_equal(_bits(orc.rms_norm(x[None], eps)[0]), _bits(got)), (n, eps)


@pytest.mark.parametrize("n", SIZES)
def test_fixture_norm_rows_split_and_reference_is_in_order(ref, orc, n):
    x = f32_row("norm", n, n)
    sa, ya = norm_predict(x, False)
    sb, _ = norm_predict(x, True)
    assert sa[0] != sb[0], (n, sa, sb)
    got = ref_op(ref, "norm", x[None])[0]
    assert np.array_equal(_bits(got), _bits(ya)), n
    assert np.array_equal(_bits(orc.norm(x[None])[0]), _bits(got)), n


def test_fixture_embedding_rows_split_and_reference_is_in_order(ref, orc):
    """the rows the native-session tests put into an embedding table, and the activations their tuned gains produce"""
    rows = {"q8_0 rms": ("rms", q8_0_rms_row(256, 1)[1]), "f16 rms": ("rms", f16_rms_row(256, 2).astype(F32)),
            "q8_0 norm": ("norm", q8_0_norm_row(256)[1])}
    for what, (op, x) in rows.items():
        if op == "rms":
            (ma, sa, ya), (mb, sb, yb) = rms_predict(x, 5e-6, False), rms_predict(x, 5e-6, True)
            assert ma != mb and sa != sb, what
        else:
            (sa, ya), (sb, yb) = norm_predict(x, False), norm_predict(x, True)
            assert sa[0] != sb[0], what
        got = ref_op(ref, op, x[None])[0]
        assert np.array_equal(_bits(got), _bits(ya)), what
        want = orc.rms_norm(x[None])[0] if op == "rms" else orc.norm(x[None])[0]
        assert np.array_equal(_bits(want), _bits(got)), what
        act = "f16" if what.startswith("f16") else "q8_0"
        g = tune_gain(ref, ya, yb, np.ones_like(x), None, act)
        assert not np.array_equal(_act_bytes(act, ref, ya * g), _act_bytes(act, ref, yb * g)), what


def test_fixture_soft_max_sums_are_exact():
    """every fp16 exp-table value in (0, 1] is a multiple of 2^-24 (so sums of up to 2^29 of them are exact in a double)"""
    h = np.arange(1, 0x3C01, dtype=np.uint16).view(np.float16).astype(np.float64)      # +subnormals .. 1.0
    assert h.min() == 2.0 ** -24 and h.max() == 1.0
    assert np.all(np.mod(h, 2.0 ** -24) == 0)
    assert (2 ** 29) * 2 ** 24 <= 2 ** 53                                                  # 2^29 terms of at most 1 in units of 2^-24


# ---- GPU: the seam, per op ------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def ctx():
    from llm_b200 import ggml
    c = ggml.Context()
    yield c
    c.close()


def _seam(ctx, op, x, *args):
    t = ctx.transfer_to_gpu(ctx.from_numpy(x))
    r = getattr(ctx, op)(t, *args)
    assert ctx.compute(r)
    return np.asarray(ctx.host_array(r), F32).reshape(x.shape)


def _edge_rows(op, n, rng):
    """random rows around the adversarial one, and rows at the edges: zeros, a constant (variance 0), squares that overflow, float subnormals,
    and a sum of x that cancels"""
    rows = [(rng.standard_normal(n) * 3).astype(F32) for _ in range(3)]
    rows.append(f32_row(op, n, n + 17))
    rows += [(rng.standard_normal(n) * 0.01).astype(F32) for _ in range(2)]
    rows.append(np.zeros(n, F32))
    rows.append(np.full(n, 3.25, F32))
    big = (rng.standard_normal(n)).astype(F32)
    big[[3, n // 2]] = F32(2.0 ** 65), F32(-2.0 ** 70)                  # |x| > 2^64: x * x is inf in f32
    rows.append(big)
    rows.append((rng.standard_normal(n) * 1e-40).astype(F32))            # float subnormals: their squares are 0
    canc = rng.standard_normal(n).astype(F32)
    canc[[0, 1, n - 1]] = F32(3e15), F32(-3e15), F32(1e15)               # sum x cancels by 15 orders of magnitude
    rows.append(canc)
    return np.stack(rows)


@pytest.mark.gpu
@pytest.mark.parametrize("eps", RMS_EPS)
@pytest.mark.parametrize("n", SIZES)
def test_seam_rms_norm_bit_exact(ctx, ref, n, eps):
    x = _edge_rows("rms", n, np.random.default_rng(n))
    want = ref_op(ref, "rms", x, eps)
    got = _seam(ctx, "op_rms_norm", x, eps)
    bad = [i for i in range(x.shape[0]) if not np.array_equal(_bits(got[i]), _bits(want[i]))]
    assert not bad, (n, eps, "rows differing", bad)


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_seam_norm_bit_exact(ctx, ref, n):
    x = _edge_rows("norm", n, np.random.default_rng(n + 1))
    want = ref_op(ref, "norm", x)
    got = _seam(ctx, "op_norm", x)
    bad = [i for i in range(x.shape[0]) if not np.array_equal(_bits(got[i]), _bits(want[i]))]
    assert not bad, (n, "rows differing", bad)


def _soft_max_rows(n, rows, rng, spread=18.0):
    """row maxima at 0 and the rest down to -spread: exp-table values from 1 through the fp16 subnormals (exp(-16.6) ~ 2^-24) to 0; -inf entries"""
    x = -rng.uniform(0.0, spread, (rows, n)).astype(F32)
    x[np.arange(rows), rng.integers(0, n, rows)] = 0.0
    x[0] = -np.linspace(0.0, spread, n, dtype=F32)[rng.permutation(n)]
    x[1, rng.random(n) < 0.3] = -np.inf
    x[2, :] = -np.inf
    x[2, n // 3] = 5.0
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES + [16384])
def test_seam_soft_max_bit_exact(ctx, ref, n):
    x = _soft_max_rows(n, 6, np.random.default_rng(n + 2))
    want = ref.op(3, 0, None, x, (n, x.shape[0], 1), out_shape=x.shape)
    got = _seam(ctx, "op_soft_max", x)
    assert np.array_equal(_bits(got), _bits(want)), n


@pytest.mark.gpu
@pytest.mark.parametrize("nc,nr,nz", [(256, 5, 3), (4096, 4, 2), (16384, 3, 2)])
def test_seam_scale_mask_soft_max_bit_exact(ctx, ref, nc, nr, nz):
    scale, n_past = 0.125, nc - nr
    x = np.stack([_soft_max_rows(nc, nr, np.random.default_rng(nc + z)) for z in range(nz)]) / F32(scale)
    x = np.where(np.isinf(x), F32(-3e4), x).astype(F32)
    want = ref.op(7, 0, None, x, (nc, nr, nz), iparams=(n_past, 0, 0, 0), fparams=(scale, 0), out_shape=x.shape)
    a = ctx.transfer_to_gpu(ctx.from_numpy(x))
    s = ctx.op_scale(a, scale); ctx.offload_no_scratch(s); assert ctx.compute(s)
    m = ctx.op_diag_mask_inf(s, n_past); ctx.offload_no_scratch(m); assert ctx.compute(m)
    r = ctx.op_soft_max(m); assert ctx.compute(r)
    got = np.asarray(ctx.host_array(r), F32).reshape(x.shape)
    assert np.array_equal(_bits(got), _bits(want)), (nc, nr, nz)


# ---- GPU: native sessions whose layer-0 norm sees an adversarial embedding row --------------------------------------------------------

TOK = 5


def _bits_equal(g, c, what):
    c = np.asarray(c, F32).reshape(np.shape(g))
    g = np.asarray(g, F32)
    assert np.array_equal(g.view(np.uint32), c.view(np.uint32)), (what, int((g != c).sum()), g.size)


def _tokens(hp):
    t = synth.make_tokens(hp, 24)
    t[t == TOK] = TOK + 1
    t[7] = TOK                                                  # inside the prefill batch
    t[15] = TOK                                                 # one decode step of its own
    return t


def _run(s, cpu, toks, graph, what):
    _bits_equal(s.evaluate(toks[:12], all_logits=True), cpu.eval(toks[:12]), f"{what}: prefill with the row at 7")
    for i in range(12, 18):
        _bits_equal(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"{what}: decode {i}")
        assert s.last_launches == graph, (what, i, s.last_launches, graph)


@pytest.mark.gpu
@pytest.mark.parametrize("wname", ["q8_0", "f16"])
def test_llama_session_adversarial_embedding(ref, wname):
    """LLaMA tiny8: the prefill's rms_norm_kernel (with its gain) and the decode step's norm_pack_kernel (Q8_0; an F16 file decodes per op,
    so rms_norm_kernel again)"""
    import llm_b200
    if wname == "q8_0":
        hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], B.Q8_0, ref.quantize)
        raw, x = q8_0_rms_row(hp["n_embd"], 1)
        tens["tok_embeddings.weight"] = tens["tok_embeddings.weight"].copy()
        tens["tok_embeddings.weight"][TOK] = raw
        graph = 7 * hp["n_layer"] + 3
    else:
        hp, tens = synth.make_llama(synth.CONFIGS["tiny8"], B.F16, lambda t, w: np.ascontiguousarray(w, F32).astype(np.float16))
        row = f16_rms_row(hp["n_embd"], 2)
        tens["tok_embeddings.weight"] = tens["tok_embeddings.weight"].copy()
        tens["tok_embeddings.weight"][TOK] = row
        x = row.astype(F32)
        graph = 17 * hp["n_layer"] + 4
    _, sa, _ = rms_predict(x, 5e-6, False)
    _, sb, _ = rms_predict(x, 5e-6, True)
    g = tens["layers.0.attention_norm.weight"]
    tens["layers.0.attention_norm.weight"] = tune_gain(ref, x * sa, x * sb, g, None, wname)
    cpu = ref.llama(hp, tens, n_threads=8, n_batch=64)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64))
    _run(s, cpu, _tokens(hp), graph, f"llama {wname}")
    for which in (0, 1):
        assert np.array_equal(s.kv(which), cpu.kv(which)[:s.kv(which).size]), which
    s.close(); m.close(); cpu.close()


def _ln_tune(ref, x, tens, gname, bname):
    tens[gname] = tune_gain(ref, norm_predict(x, False)[1], norm_predict(x, True)[1], tens[gname], tens[bname] if bname else None, "q8_0")


@pytest.mark.gpu
def test_neox_session_adversarial_embedding(ref):
    """GPT-NeoX, parallel residual, Q8_0: the prefill's layer_norm_kernel and the decode step's ln_pack_kernel (with bias)"""
    from llm_b200.neox import GptNeoX
    cfg = dict(n_vocab=384, n_ctx=128, n_embd=256, n_head=4, n_layer=2, n_rot=16, use_parallel_residual=1)
    hp, tens = synth.make_neox(cfg, B.Q8_0, ref.quantize)
    raw, x = q8_0_norm_row(hp["n_embd"])
    tens["gpt_neox.embed_in.weight"] = tens["gpt_neox.embed_in.weight"].copy()
    tens["gpt_neox.embed_in.weight"][TOK] = raw
    _ln_tune(ref, x, tens, "gpt_neox.layers.0.input_layernorm.weight", "gpt_neox.layers.0.input_layernorm.bias")
    cpu = ref.neox(hp, tens, n_threads=8, n_batch=64)
    m = GptNeoX(hp, tens)
    s = m.start_session(64)
    _run(s, cpu, _tokens(hp), 8 * hp["n_layer"] + 3, "neox")
    for which in (0, 1):
        assert np.array_equal(s.kv(which), cpu.kv(which)), which
    s.close(); m.close(); cpu.close()


@pytest.mark.gpu
def test_mpt_session_adversarial_embedding(ref):
    """MPT, Q8_0: layer_norm_kernel without a bias in the prefill, ln_pack_nobias_kernel in the decode step"""
    from oracle import alibi as A
    from llm_b200.neox import Mpt
    if not A.have_ref():
        pytest.skip("oracle/_ref/libggml_alibi.so not built")
    hp, tens = A.make_mpt(A.MPT_CONFIGS["mpt-tiny"], B.Q8_0, ref.quantize)
    raw, x = q8_0_norm_row(hp["n_embd"])
    tens["transformer.wte.weight"] = tens["transformer.wte.weight"].copy()
    tens["transformer.wte.weight"][TOK] = raw
    _ln_tune(ref, x, tens, "transformer.blocks.0.norm_1.weight", None)
    cpu = A.RefAlibi(hp, tens, A.MPT, n_threads=8, n_batch=64)
    m = Mpt(hp, tens)
    s = m.start_session(64)
    _run(s, cpu, _tokens(hp), 8 * hp["n_layer"] + 3, "mpt")
    nl, n_ctx, e = hp["n_layer"], hp["n_ctx"], hp["n_embd"]
    assert np.array_equal(s.kv(0), cpu.kv(0)), "K"
    assert np.array_equal(s.kv(1), cpu.kv(1).reshape(nl, n_ctx, e).transpose(0, 2, 1).ravel()), "V"
    s.close(); m.close(); cpu.close()
