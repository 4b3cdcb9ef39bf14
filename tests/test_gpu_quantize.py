"""Model quantization on the GPU (b200_quantize_file, llm_b200.quantize) against the reference's `quantize` restated over its own
ggml_quantize_q* (oracle/quantize.py): every output file, callback report, total, histogram and progress event compared byte for byte / bit for
bit, for every target, both source types and every architecture; hard blocks; sizes across the chunk ring; both containers; and a quantized
file that loads and runs bit-identical with the reference graph."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import quantize as Q

pytestmark = pytest.mark.gpu

TARGETS = {"q4_0": Q.Q4_0, "q4_1": Q.Q4_1, "q5_0": Q.Q5_0, "q5_1": Q.Q5_1, "q8_0": Q.Q8_0}
SOURCES = {"f16": Q.F16, "f32": Q.F32}
CASES = {"llama": ("llama", "llama", False), "llama-gqa": ("llama", "llama-gqa", False), "gpt2-tied": ("gpt2", "gpt2", False),
         "gpt2-lm-head": ("gpt2", "gpt2", True), "gptneox": ("gptneox", "gptneox", False), "mpt": ("mpt", "mpt", False),
         "bloom": ("bloom", "bloom", False), "gptj": ("gptj", "gptj", False)}


@pytest.fixture(scope="module", autouse=True)
def need_ref():
    if not Q.have_ref():
        pytest.skip("oracle/_ref/libggml_ref.so not built (the reference's ggml_quantize_q* are the oracle)")
    from llm_b200 import _lib
    assert _lib.lib().b200_init(0) == 0


def run_c(src, dst, arch, target, container=0):
    """b200_quantize_file with a callback that keeps every report: (rc, reports, original_size, reduced_size, hist)"""
    from llm_b200 import _lib
    from llm_b200.loader import ARCH
    reports = []

    def on_tensor(_user, rp):
        r = rp.contents
        reports.append(dict(name=r.name.decode(), n_dims=r.n_dims, src_type=r.src_type, dst_type=r.dst_type, ne=(r.ne[0], r.ne[1]),
                            n_elements=r.n_elements, original_size=r.original_size, reduced_size=r.reduced_size, hist=np.array(r.hist[:], np.int64)))
    orig, red, hist = C.c_int64(), C.c_int64(), (C.c_int64 * 16)()
    rc = _lib.lib().b200_quantize_file(src.encode(), dst.encode(), ARCH[arch], target, container, _lib.QUANTIZE_CALLBACK(on_tensor), None,
                                       C.byref(orig), C.byref(red), C.byref(hist))
    return rc, reports, orig.value, red.value, np.array(hist[:], np.int64)


def as_tuple(e):
    """a QuantizeProgress event of llm_b200.quantize in the oracle's form"""
    kind = type(e).__name__
    if kind == "TensorLoading":
        return (kind, e.name, tuple(e.dims), e.element_type, e.n_elements)
    if kind == "TensorQuantized":
        return (kind, e.name, e.original_size, e.reduced_size, np.asarray(e.history, np.float32))
    if kind == "TensorQuantizing":
        return (kind, e.name)
    if kind == "TensorSkipped":
        return (kind, e.name, e.size)
    if kind == "Finished":
        return (kind, e.original_size, e.reduced_size, np.asarray(e.history, np.float32))
    return (kind,)


def same(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        if a.dtype == np.float32:
            return a.shape == b.shape and np.array_equal(a.view(np.uint32), np.asarray(b, np.float32).view(np.uint32))
        return np.array_equal(a, b)
    if isinstance(a, (tuple, list)):
        return isinstance(b, (tuple, list)) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    return a == b


def check_all(tmp_path, arch, words, vocab, tensors, target, container="ggjt-v3"):
    """quantize the source both through the C entry point and llm_b200.quantize; every output against the oracle"""
    import llm_b200
    src = str(tmp_path / "src.bin")
    open(src, "wb").write(Q.write_file(words, vocab, tensors))
    exp = Q.quantize(arch, words, vocab, tensors, target, container)
    dst = str(tmp_path / "c.bin")
    rc, reports, orig, red, hist = run_c(src, dst, arch, target, 0 if container == "ggjt-v3" else 1)
    assert rc == 0
    assert open(dst, "rb").read() == exp["file"]
    assert len(reports) == len(exp["reports"])
    for g, w in zip(reports, exp["reports"]):
        assert same(g, w), (g["name"], g, w)
    assert (orig, red) == (exp["original_size"], exp["reduced_size"])
    assert np.array_equal(hist, exp["hist"])
    events = []
    dst2 = str(tmp_path / "py.bin")
    llm_b200.quantize(src, dst2, arch, target, container, progress=events.append)
    assert open(dst2, "rb").read() == exp["file"]
    got = [as_tuple(e) for e in events]
    assert len(got) == len(exp["events"])
    for g, w in zip(got, exp["events"]):
        assert same(g, w), (g, w)
    return exp


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("src", list(SOURCES))
@pytest.mark.parametrize("target", list(TARGETS))
def test_every_case_matches_reference(tmp_path, case, src, target):
    arch, cfg, lm_head = CASES[case]
    hp, words, vocab, tensors = Q.model(arch, cfg, SOURCES[src], lm_head=lm_head)
    exp = check_all(tmp_path, arch, words, vocab, tensors, TARGETS[target])
    n_q = sum(r["dst_type"] != r["src_type"] for r in exp["reports"])
    assert 0 < n_q < len(tensors)                                              # some tensors quantized, some copied
    if arch == "gpt2":
        wpe = next(r for r in exp["reports"] if r["name"] == "model/wpe")
        assert wpe["dst_type"] == wpe["src_type"] == SOURCES[src]               # positional embeddings stay F32 / F16


def hard_rows():
    """32-element blocks at the edges of the reference's rules"""
    rows = []
    z = np.zeros(32, np.float32)
    rows.append(z)                                                             # all zeros: d = 0, id = 0
    pz = z.copy(); pz[1::2] = -0.0; rows.append(pz)                            # +0 / -0
    mix = np.where(np.arange(32) % 3 == 0, -0.0, 0.0).astype(np.float32); mix[5] = 1e-3; rows.append(mix)
    for s in (1.0, -1.0):                                                      # amax ties of opposite sign: the first one wins
        t = np.linspace(-1, 1, 32).astype(np.float32) * 0.5; t[3] = 3 * s; t[20] = -3 * s; rows.append(t)
    tie = np.full(32, -2.0, np.float32); tie[::2] = 2.0; rows.append(tie)
    sub = (np.arange(32) - 16).astype(np.float32) * np.float32(2 ** -24); rows.append(sub)    # F16 subnormals
    big = np.full(32, 65504.0, np.float32); big[::3] = -65504.0; big[7] = 0.0; rows.append(big)     # F16 extremes
    for m in (-8.0, 8.0, -16.0, 16.0, -127.0, 127.0):                         # x * id + 8.5 (16.5, 0.5) exactly on an integer
        h = (np.arange(32) % 17 - 8).astype(np.float32) + 0.5; h[0] = m; rows.append(h)
    q1 = (np.arange(32) / 2).astype(np.float32) * 15 / 15.5; rows.append(q1)   # Q4_1 / Q5_1: (x - min) * id + 0.5 near integers
    rng = np.random.default_rng(7)
    rows.append((rng.integers(-16, 16, 32) + 0.5).astype(np.float32))
    rows.append((rng.standard_normal(32) * 1e-30).astype(np.float32))          # F32: tiny scales (F16 source: all zeros)
    rows.append((rng.standard_normal(32) * 1e30).astype(np.float32))           # F32: huge scales (F16 source: +-inf, not part of parity)
    return rows


@pytest.mark.parametrize("src", list(SOURCES))
@pytest.mark.parametrize("target", list(TARGETS))
def test_hard_blocks(tmp_path, src, target):
    rows = hard_rows()
    if SOURCES[src] == Q.F16:
        rows = rows[:-1]                                                       # f16(1e30) = inf: non-finite values are outside the parity claim
    n = len(rows) + len(rows) % 2
    x = np.concatenate(rows + [rows[0]] * (n - len(rows))).reshape(n // 2, 64)  # two blocks per row (Q4 rows need ne0 % 64 == 0)
    hp, words, vocab, tensors = Q.model("llama", "llama", SOURCES[src])
    check_all(tmp_path, "llama", words, vocab, tensors[:2] + [Q.tensor("hard.weight", x, SOURCES[src])], TARGETS[target])


@pytest.mark.parametrize("target", list(TARGETS))
def test_sizes(tmp_path, target):
    t = TARGETS[target]
    w = 64 if t in (Q.Q4_0, Q.Q4_1) else 32
    rng = np.random.default_rng(11)
    hp, words, vocab, _ = Q.model("llama", "llama", Q.F16)
    tensors = [Q.tensor("one.weight", rng.standard_normal((1, w)), Q.F32),           # one block (two for Q4)
               Q.tensor("odd.weight", rng.standard_normal((5, 192)), Q.F16),         # 30 blocks: the tail CTA holds 6
               Q.tensor("vec.weight", rng.standard_normal(96), Q.F32),               # 1-D: copied
               Q.tensor("seven.weight", rng.standard_normal((7, 64)), Q.F32)]        # 14 blocks
    check_all(tmp_path, "llama", words, vocab, tensors, t)


@pytest.mark.parametrize("target", ["q4_0", "q5_1"])
def test_large_tensor_crosses_the_ring(tmp_path, target):
    """a 32000 x 4096 F16 tensor: 4 Mi blocks, 64 chunks through a ring of 4"""
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((32000, 4096), np.float32) * np.float32(1 / 64)).astype(np.float16)
    hp, words, vocab, tensors = Q.model("llama", "llama", Q.F16)
    big = dict(name="tok_embeddings.weight", n_dims=2, ne=(4096, 32000), type=Q.F16, data=x.tobytes())
    del x
    check_all(tmp_path, "llama", words, vocab, [big] + tensors[1:3], TARGETS[target])


def test_ggml_container(tmp_path):
    hp, words, vocab, tensors = Q.model("gptneox", "gptneox", Q.F16, scored=False)
    exp = check_all(tmp_path, "gptneox", words, vocab, tensors, Q.Q8_0, "ggml")
    assert exp["file"][:4] == (0x67676D6C).to_bytes(4, "little")


def test_quantized_llama_runs_bit_exact_with_reference(tmp_path):
    """F16 LLaMA file -> Q4_0 here -> llm_b200.loader.load: logits over a short prompt identical to the reference graph on that file's weights"""
    import llm_b200
    from llm_b200.loader import GgmlFile, load
    from oracle import bindings as B
    from oracle import synth
    hp, words, vocab, tensors = Q.model("llama", "llama", Q.F16)
    src, dst = str(tmp_path / "f16.bin"), str(tmp_path / "q4_0.bin")
    open(src, "wb").write(Q.write_file(words, vocab, tensors))
    llm_b200.quantize(src, dst, "llama", "q4_0")
    f = GgmlFile(dst)
    tens = {}
    for i, t in enumerate(f.tensors()):
        b = f.tensor_bytes(i)
        tens[t["name"]] = b.view(np.float32) if t["n_dims"] == 1 else b.reshape(t["ne"][1], -1)
    assert f.llama_hyperparameters()["wtype"] == Q.Q4_0 and f.llama_hyperparameters()["llama_ftype"] == 2
    f.close()
    hp = dict(hp, wtype=Q.Q4_0)
    mr = B.RefLib("ref").llama(hp, tens, n_threads=8)
    m = load(dst, llm_b200.ModelParameters(context_size=hp["n_ctx"]))
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64))
    toks = synth.make_tokens(hp, 24)
    for chunk in (toks[:20], toks[20:21], toks[21:22]):
        g = np.asarray(s.evaluate(chunk, all_logits=True), np.float32)
        c = np.asarray(mr.eval(chunk), np.float32).reshape(g.shape)
        assert np.array_equal(g.view(np.uint32), c.view(np.uint32)), chunk.size
    s.close(); m.close(); mr.close()
    os.remove(dst)
