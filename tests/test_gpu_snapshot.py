"""Session snapshots (InferenceSession::get_snapshot / from_snapshot and the CLI's session files) on every native session, against the reference's own
ggml.c running the same graphs (oracle/bindings.py, alibi.py, gptj.py, kv32.py).

  parity       LLaMA (MHA, GQA; Q4_0 and an F16 model), GPT-NeoX (parallel and sequential residual), GPT-2, MPT, BLOOM, GPT-J, f16 and f32 caches:
               a prefill, then graph decode steps to P = 150 in contexts of 256 (LLaMA) and 200 positions, neither a multiple of the 32 / 64 transpose
               tile; memory_k / memory_v are the oracle's cache bytes, whole (GQA: its used part, then zeros), npast / tokens / last_logits / config
  round trips  the snapshot restored in memory and from a session file into a second model of the same tensors, then 40 decode steps and a batch:
               logits, both caches and the first step's launch count equal the uninterrupted session's and the oracle's
  interchange  the GPU snapshot applied to a second oracle (the reference's from_snapshot: the bytes into its tensors, n_past) continues like the
               GPU; the oracle's bytes as a snapshot continue on the GPU like the oracle
  generation   greedy and sampled infer_next_token after a restore, play_back_previous_tokens
  file format  a restatement of bincode + the zstd frame; libzstd's ZSTD_decompress when present; RLE blocks, fields across block boundaries;
               compressed blocks, truncation, trailing bytes, a bad magic and a reserved bit refused
  refusals     MemorySizeMismatch, BAD_ARG, a FAST session"""
import ctypes as C
import struct

import numpy as np
import pytest

import llm_b200
from llm_b200 import ModelKVMemoryType as KV
from llm_b200.neox import Bloom, Gpt2, GptJ, GptNeoX, Mpt, NeoxSession
from oracle import alibi as A
from oracle import bindings as B
from oracle import gptj as J
from oracle import kv32, synth

pytestmark = pytest.mark.gpu

P = 150                     # snapshot position: not a multiple of the transpose tiles (32 f32, 64 f16)
BAD_ARG, SIZE_MISMATCH, FORMAT = -2, -18, -19
ZMAGIC = b"\x28\xb5\x2f\xfd"


def check(g, c, what):
    g = np.asarray(g, np.float32)
    c = np.asarray(c, np.float32).reshape(g.shape)
    bad = g.view(np.uint32) != c.view(np.uint32)
    assert not bad.any(), (what, int(bad.sum()), g.size)


def ref_or_skip():
    if not (kv32.have_ref() and B.have_ref("ref") and A.have_ref() and J.have_ref()):
        pytest.skip("oracle/_ref not built (the reference graphs on the reference's ggml)")


# ---- the cases: a native model factory, an oracle factory, the session class, where the oracle keeps its cache -----------------------------------
NEOX = {"neox-par": dict(n_vocab=384, n_ctx=200, n_embd=256, n_head=4, n_layer=2, n_rot=16, use_parallel_residual=1),
        "neox-seq": dict(n_vocab=384, n_ctx=200, n_embd=256, n_head=8, n_layer=2, n_rot=32, use_parallel_residual=0)}
LLAMA = {"mha": ("tiny8", B.Q4_0), "gqa": ("gqa8", B.Q4_0), "mha-f16": ("tiny8", B.F16)}


class Case:
    def __init__(self, orc, name, kv):
        ref_or_skip()
        self.name, self.kv, self.f32 = name, kv, kv == KV.Float32
        self.llama = name in LLAMA
        if self.llama:
            cfg, wtype = LLAMA[name]
            quant = (lambda t, w: np.ascontiguousarray(w, np.float32).astype(np.float16)) if wtype == B.F16 else orc.quantize
            self.hp, self.tens = synth.make_llama(dict(synth.CONFIGS[cfg], n_ctx=256), wtype, quant)
        elif name in NEOX:
            self.hp, self.tens = synth.make_neox(NEOX[name], B.Q4_0, orc.quantize)
        elif name == "gpt2":
            self.hp, self.tens = synth.make_gpt2(dict(n_vocab=320, n_ctx=200, n_embd=256, n_head=4, n_layer=2), B.Q4_0, orc.quantize)
        elif name in ("mpt", "bloom"):
            make, base = (A.make_mpt, A.MPT_CONFIGS["mpt-tiny"]) if name == "mpt" else (A.make_bloom, A.BLOOM_CONFIGS["bloom-tiny"])
            self.hp, self.tens = make(dict(base, n_ctx=200), B.Q4_0, orc.quantize)
        else:
            self.hp, self.tens = J.make_gptj(dict(J.GPTJ_CONFIGS["gptj-tiny"], n_ctx=200), B.Q4_0, orc.quantize)
        self.n_ctx = self.hp["n_ctx"]
        self.v_by_position = name in ("gpt2", "mpt", "bloom")
        self.cls = llm_b200.InferenceSession if self.llama else NeoxSession

    def model(self):
        if self.llama:
            return llm_b200.Llama(self.hp, llm_b200.ModelParameters(context_size=self.n_ctx), self.tens)
        cls = {"gpt2": Gpt2, "mpt": Mpt, "bloom": Bloom, "gptj": GptJ}.get(self.name, GptNeoX)
        return cls(self.hp, self.tens)

    def session(self, m, flags=0):
        if self.llama:
            return m.start_session(llm_b200.InferenceSessionConfig(n_batch=128, flags=flags, memory_k_type=self.kv, memory_v_type=self.kv))
        return m.start_session(128, memory_k_type=self.kv, memory_v_type=self.kv)

    def oracle(self):
        lib = kv32.ref_lib() if self.f32 else B.RefLib("ref")
        if self.llama:
            return lib.llama(self.hp, self.tens, n_threads=8, n_batch=128)
        if self.name in NEOX:
            return lib.neox(self.hp, self.tens, n_threads=8, n_batch=128)
        if self.name == "gpt2":
            return lib.gpt2(self.hp, self.tens, n_threads=8, n_batch=128)
        if self.name in ("mpt", "bloom"):
            arch = A.MPT if self.name == "mpt" else A.BLOOM
            return (kv32.RefAlibiKV32 if self.f32 else A.RefAlibi)(self.hp, self.tens, arch, n_threads=8, n_batch=128)
        return (kv32.RefGptJKV32 if self.f32 else J.RefGptJ)(self.hp, self.tens, n_threads=8, n_batch=128)

    @staticmethod
    def cache(cpu, which):
        """(address, bytes) of the oracle's memory_k (0) / memory_v (1) tensor"""
        if isinstance(cpu, B.RefLlama):
            return cpu.kv_ptr(which)
        if isinstance(cpu, B.RefGpt2):
            L = cpu.ref.lib
            t = getattr(B._RgHead.from_address(cpu.m), "memory_v" if which else "memory_k")
            return L.ggml_get_data(t), L.ggml_nbytes(t)
        nb = C.c_size_t(0)
        ptr = (cpu.L.ra_kv if isinstance(cpu, A.RefAlibi) else cpu.L.rj_kv)(cpu.m, which, C.byref(nb))
        return ptr, nb.value

    def cache_bytes(self, cpu, which):
        p, n = self.cache(cpu, which)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), (n,)).copy()

    def apply(self, cpu, snap):
        """the reference's from_snapshot on an oracle: n_past (set, or reached by evaluating other tokens), then the snapshot's bytes in its tensors"""
        if isinstance(cpu, B.RefLlama):
            cpu.set_n_past(snap.npast)
        else:
            cpu.reset()
            filler = (np.arange(snap.npast, dtype=np.int32) * 7 + 3) % self.hp["n_vocab"]
            for a in range(0, snap.npast, 128):
                cpu.eval(filler[a:a + 128])
        for which, mem in ((0, snap.memory_k), (1, snap.memory_v)):
            p, n = self.cache(cpu, which)
            assert n == mem.nbytes
            C.memmove(p, mem.ctypes.data, n)


def prefill_and_decode(case, s, cpu, toks):
    check(s.evaluate(toks[:100], all_logits=True), cpu.eval(toks[:100]), "prefill 100")
    for i in range(100, P):
        want = cpu.eval(toks[i:i + 1])
        check(s.evaluate(toks[i:i + 1], all_logits=True), want, f"decode at {i}")
    return want[-1]


def continue_all(sessions, cpus, toks, what):
    """40 decode steps and a batch of 7 on every session and oracle: identical logits everywhere, and the first step's launch counts"""
    launches = None
    for i, n in [(i, 1) for i in range(P, P + 40)] + [(P + 40, 7)]:
        outs = [s.evaluate(toks[i:i + n], all_logits=True) for s in sessions]
        if i == P:
            launches = [s.last_launches for s in sessions]
            assert len(set(launches)) == 1, (what, launches)
        for c in cpus:
            check(outs[0], c.eval(toks[i:i + n]), f"{what}: oracle at {i}")
        for o in outs[1:]:
            check(o, outs[0], f"{what}: restored session at {i}")
    return launches


# ---- a restatement of the session file: bincode 1.3.3 (default options) in one zstd frame of raw / RLE blocks ------------------------------------
def zstd_content(data: bytes) -> bytes:
    assert data[:4] == ZMAGIC
    fhd = data[4]
    single = fhd >> 5 & 1
    fcs_n = {0: single, 1: 2, 2: 4, 3: 8}[fhd >> 6]
    off = 5 + (0 if single else 1) + [0, 1, 2, 4][fhd & 3]
    fcs = int.from_bytes(data[off:off + fcs_n], "little") + (256 if fcs_n == 2 else 0)
    off += fcs_n
    out = bytearray()
    while True:
        h = int.from_bytes(data[off:off + 3], "little")
        off += 3
        typ, size = h >> 1 & 3, h >> 3
        assert typ in (0, 1)
        out += data[off:off + size] if typ == 0 else bytes([data[off]]) * size
        off += size if typ == 0 else 1
        if h & 1:
            break
    off += 4 if fhd & 4 else 0
    assert off == len(data) and (fcs_n == 0 or fcs == len(out))
    return bytes(out)


def bincode_fields(b: bytes) -> dict:
    o = 0

    def u(fmt):
        nonlocal o
        v = struct.unpack_from(fmt, b, o)[0]
        o += struct.calcsize(fmt)
        return v

    def seq(dtype, size):
        nonlocal o
        n = u("<Q")
        a = np.frombuffer(b, dtype, n, o)
        o += n * size
        return a

    f = dict(npast=u("<Q"), k_type=u("<I"), v_type=u("<I"), n_batch=u("<Q"), n_threads=u("<Q"))
    f.update(tokens=seq(np.uint32, 4), last_logits=seq(np.float32, 4), memory_k=seq(np.uint8, 1), memory_v=seq(np.uint8, 1))
    assert o == len(b)
    return f


def frame(content: bytes, blocks) -> bytes:
    """a zstd frame (header 0xC0 0x38, 8-byte content size) of the given blocks: (kind, size), kind 0 raw, 1 RLE (of the content's byte there), 2
    compressed (a raw payload typed as compressed)"""
    out = bytearray(ZMAGIC + bytes([0xC0, 0x38]) + len(content).to_bytes(8, "little"))
    at = 0
    for i, (kind, size) in enumerate(blocks):
        out += ((size << 3) | (kind << 1) | (i == len(blocks) - 1)).to_bytes(3, "little")
        out += content[at:at + 1] if kind == 1 else content[at:at + size]
        at += size
    assert at == len(content)
    return bytes(out)


def raw_blocks(n, size=128 << 10):
    return [(0, min(size, n - a)) for a in range(0, n, size)]


def snapshots_equal(a, b, what):
    assert a.npast == b.npast and a.config.n_batch == b.config.n_batch, what
    assert a.config.memory_k_type == b.config.memory_k_type and a.config.memory_v_type == b.config.memory_v_type, what
    assert np.array_equal(a.tokens, b.tokens), what
    check(a.last_logits, b.last_logits, what)
    assert np.array_equal(a.memory_k, b.memory_k) and np.array_equal(a.memory_v, b.memory_v), what


def file_matches(path, snap):
    f = bincode_fields(zstd_content(open(path, "rb").read()))
    assert f["npast"] == snap.npast and f["n_batch"] == snap.config.n_batch and f["n_threads"] == 8
    assert f["k_type"] == f["v_type"] == llm_b200.session.KV_VARIANT[snap.config.memory_k_type]
    assert np.array_equal(f["tokens"], snap.tokens)
    check(f["last_logits"], snap.last_logits, "file last_logits")
    assert np.array_equal(f["memory_k"], snap.memory_k) and np.array_equal(f["memory_v"], snap.memory_v)


# ---- parity, round trips and interchange -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kv", [KV.Float16, KV.Float32], ids=["f16", "f32"])
@pytest.mark.parametrize("name", list(LLAMA) + list(NEOX) + ["gpt2", "mpt", "bloom", "gptj"])
def test_snapshot_matches_reference(orc, tmp_path, name, kv):
    case = Case(orc, name, kv)
    hp = case.hp
    m, cpu = case.model(), case.oracle()
    s = case.session(m)
    toks = np.random.default_rng(0x5A9).integers(0, hp["n_vocab"], size=P + 50, dtype=np.int32)
    last = prefill_and_decode(case, s, cpu, toks)

    snap = s.get_snapshot()
    assert snap.npast == P and snap.n_threads == 8
    assert snap.config.n_batch == 128 and snap.config.memory_k_type == kv and snap.config.memory_v_type == kv
    assert snap.tokens.dtype == np.uint32 and np.array_equal(snap.tokens, toks[:P].astype(np.uint32))
    check(snap.last_logits, last, "last_logits")
    for which, mem in ((0, snap.memory_k), (1, snap.memory_v)):
        want = case.cache_bytes(cpu, which)
        assert mem.nbytes == want.nbytes == hp["n_layer"] * case.n_ctx * hp["n_embd"] * (4 if case.f32 else 2), which
        used = hp["n_layer"] * case.n_ctx * (hp["n_embd"] // (hp["n_head"] // hp.get("n_head_kv", hp["n_head"]))) * (4 if case.f32 else 2)
        assert np.array_equal(mem[:used], want[:used]), ("cache bytes", which)
        assert not mem[used:].any(), ("unused tail", which)

    path = tmp_path / "session.bin"
    s.write_snapshot(path)
    file_matches(path, snap)

    m2 = case.model()                       # a second model object from the same tensors
    r_mem = case.cls.from_snapshot(snap, m2)
    r_file = case.cls.read_snapshot(path, m2)
    assert r_mem.n_past == r_file.n_past == P
    assert np.array_equal(r_mem.tokens(), toks[:P]) and np.array_equal(r_file.tokens(), toks[:P])
    check(r_file.last_logits, last, "restored last_logits")
    snapshots_equal(r_file.get_snapshot(), snap, "snapshot of the restored session")
    cpu_apply = case.oracle()               # the reference's from_snapshot of the GPU's bytes
    case.apply(cpu_apply, snap)
    continue_all([s, r_mem, r_file], [cpu, cpu_apply], toks, name)
    for which in (0, 1):
        k = s.kv(which)
        assert np.array_equal(r_mem.kv(which), k) and np.array_equal(r_file.kv(which), k), which

    # the oracle's bytes as a snapshot into a GPU session: it continues as the oracle does
    cpu_src = case.oracle()
    for a in range(0, P, 128):
        cpu_src.eval(toks[a:min(a + 128, P)])
    row = cpu_src.eval(toks[P:P + 1])[-1]
    ref_snap = llm_b200.InferenceSnapshot(npast=P + 1, config=snap.config, n_threads=8, tokens=toks[:P + 1].astype(np.uint32), last_logits=row,
                                          memory_k=case.cache_bytes(cpu_src, 0), memory_v=case.cache_bytes(cpu_src, 1))
    g = case.cls.from_snapshot(ref_snap, m2)
    for i in range(P + 1, P + 11):
        check(g.evaluate(toks[i:i + 1], all_logits=True), cpu_src.eval(toks[i:i + 1]), f"oracle snapshot on the GPU at {i}")
    for x in (s, r_mem, r_file, g):
        x.close()
    for c in (cpu, cpu_apply, cpu_src):
        c.close()
    m.close(); m2.close()


# ---- generation after a restore ------------------------------------------------------------------------------------------------------------------
def test_generation_after_restore(orc, tmp_path):
    case = Case(orc, "gqa", KV.Float16)
    m = case.model()
    s = case.session(m)
    toks = synth.make_tokens(case.hp, 60)
    s.feed_prompt(toks)
    snap = s.get_snapshot()
    s.write_snapshot(tmp_path / "g.bin")
    greedy = llm_b200.InferenceParameters(sampler=llm_b200.Sampler(top_k=1))
    sampled = llm_b200.InferenceParameters()
    for params in (greedy, sampled):
        runs = []
        for make in (lambda: case.cls.from_snapshot(snap, m), lambda: case.cls.read_snapshot(tmp_path / "g.bin", m), None):
            if make is None:               # uninterrupted: the prompt fed again on a new session
                x = case.session(m)
                x.feed_prompt(toks)
            else:
                x = make()
            rng = llm_b200.Rng(0xC0FFEE)
            rng.draw = 5                   # the same draw index in every run
            runs.append([x.infer_next_token(params, rng) for _ in range(12)])
            x.close()
        assert runs[0] == runs[1] == runs[2], runs
    seen = []
    r = case.cls.from_snapshot(snap, m)
    r.infer(llm_b200.InferenceRequest(prompt=[], maximum_token_count=3, play_back_previous_tokens=True), llm_b200.Rng(1), seen.append)
    assert seen[:60] == [int(t) for t in toks] and len(seen) == 63
    r.close(); s.close(); m.close()


def test_restored_row_is_sampled(orc):
    """infer_next_token samples from the snapshot's last row, even from the reference's initial zeros"""
    case = Case(orc, "mha", KV.Float16)
    m = case.model()
    s = case.session(m)
    toks = synth.make_tokens(case.hp, 20)
    s.evaluate(toks)
    snap = s.get_snapshot()
    row = np.full(case.hp["n_vocab"], -1.0, np.float32)
    row[123] = 5.0
    snap.last_logits = row
    r = case.cls.from_snapshot(snap, m)
    greedy = llm_b200.InferenceParameters(sampler=llm_b200.Sampler(top_k=1, repetition_penalty=1.0))
    assert r.infer_next_token(greedy, llm_b200.Rng(0)) == 123
    snap.last_logits = np.zeros_like(row)
    z = case.cls.from_snapshot(snap, m)
    assert z.infer_next_token(greedy, llm_b200.Rng(0)) == 0          # all ties: the lowest id
    fresh = case.session(m).get_snapshot()
    assert fresh.npast == 0 and not fresh.last_logits.any() and fresh.tokens.size == 0
    for x in (r, z, s):
        x.close()
    m.close()


# ---- the file format -----------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small(orc, tmp_path_factory):
    case = Case(orc, "gqa", KV.Float16)
    m = case.model()
    s = case.session(m)
    s.feed_prompt(synth.make_tokens(case.hp, 37))
    path = tmp_path_factory.mktemp("snap") / "small.bin"
    s.write_snapshot(path)
    yield case, m, s, s.get_snapshot(), open(path, "rb").read()
    s.close(); m.close()


def read_code(m, path):
    err = C.c_int(0)
    h = m.L.b200_model_session_read_snapshot(m._m, str(path).encode(), 0, C.byref(err))
    if h:
        m.L.b200_session_free(h)
    return err.value


def test_libzstd_reads_the_file(small):
    case, m, s, snap, data = small
    try:
        z = C.CDLL("libzstd.so.1")
    except OSError:
        pytest.skip("libzstd.so.1 is not installed")
    z.ZSTD_decompress.restype = C.c_size_t
    z.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    z.ZSTD_isError.argtypes = [C.c_size_t]
    content = zstd_content(data)
    out = C.create_string_buffer(len(content) + 64)
    n = z.ZSTD_decompress(out, len(out), data, len(data))
    assert not z.ZSTD_isError(n) and out.raw[:n] == content


def test_hand_made_frames(small, tmp_path):
    case, m, s, snap, data = small
    content = zstd_content(data)
    variants = {}
    # fields across block boundaries: 7-byte blocks over the header, the tokens and the logits, then odd sizes
    head = 40 + 4 * snap.npast + 8 + 4 * snap.last_logits.size + 8 + 64
    variants["straddle"] = frame(content, [(0, 7)] * (head // 7) + raw_blocks(len(content) - head // 7 * 7, 100003))
    # an RLE block over the zeros of the unused GQA tail of memory_k
    mk0 = len(content) - 2 * snap.memory_k.nbytes - 8
    used = case.hp["n_layer"] * case.n_ctx * (case.hp["n_embd"] // 4) * 2
    z0 = mk0 + used
    assert not any(content[z0:z0 + 4096])
    variants["rle"] = frame(content, raw_blocks(z0) + [(1, 4096)] + raw_blocks(len(content) - z0 - 4096))
    for k, v in variants.items():
        p = tmp_path / f"{k}.bin"
        p.write_bytes(v)
        r = case.cls.read_snapshot(p, m)
        snapshots_equal(r.get_snapshot(), snap, k)
        r.close()
    bad = {"compressed": frame(content, raw_blocks(1000) + [(2, 1000)] + raw_blocks(len(content) - 2000)),
           "truncated": data[:-10], "trailing": data + b"\0", "magic": b"\x29" + data[1:], "reserved bit": data[:4] + bytes([0xC8]) + data[5:],
           "block over the window": frame(content, [(0, 1 << 17 | 8)] + raw_blocks(len(content) - (1 << 17 | 8)))}
    over = bytearray(content)
    over[32:40] = (1 << 40).to_bytes(8, "little")               # a tokens count that overruns the frame
    bad["overrun"] = frame(bytes(over), raw_blocks(len(over)))
    for k, v in bad.items():
        p = tmp_path / "bad.bin"
        p.write_bytes(v)
        assert read_code(m, p) == FORMAT, k
        with pytest.raises(llm_b200.SnapshotError):
            case.cls.read_snapshot(p, m)


def test_failed_write_leaves_no_file(small, tmp_path):
    case, m, s, snap, data = small
    target = tmp_path / "missing-dir" / "x.bin"
    assert s.L.b200_session_write_snapshot(s._s, str(target).encode()) == -10
    assert not target.exists()


# ---- refusals ------------------------------------------------------------------------------------------------------------------------------------
def test_refusals(orc, small, tmp_path):
    from llm_b200.tp import TpLlama
    case, m, s, snap, data = small
    # another context size, another geometry, another KV type: MemorySizeMismatch with both sizes
    other_ctx = llm_b200.Llama(case.hp, llm_b200.ModelParameters(context_size=128), case.tens)
    hp2, t2 = synth.make_llama(dict(synth.CONFIGS["tiny8"], n_ctx=256), B.Q4_0, orc.quantize)
    other_geo = llm_b200.Llama(hp2, llm_b200.ModelParameters(context_size=256), t2)
    for other in (other_ctx, other_geo):
        with pytest.raises(llm_b200.MemorySizeMismatch) as e:
            case.cls.from_snapshot(snap, other)
        assert e.value.input_size == snap.memory_k.nbytes
        assert e.value.self_size == other.hyperparameters["n_layer"] * other.params.context_size * other.hyperparameters["n_embd"] * 2
        with pytest.raises(llm_b200.MemorySizeMismatch):
            case.cls.read_snapshot(_write(tmp_path, data), other)
    as_f32 = llm_b200.InferenceSnapshot(**{**snap.__dict__, "config": llm_b200.InferenceSessionConfig(
        n_batch=snap.config.n_batch, memory_k_type=KV.Float32, memory_v_type=KV.Float32)})
    with pytest.raises(llm_b200.MemorySizeMismatch) as e:
        case.cls.from_snapshot(as_f32, m)
    assert e.value.self_size == 2 * snap.memory_k.nbytes and e.value.input_size == snap.memory_k.nbytes

    L = m.L

    def code(model, c, flags=0):
        err = C.c_int(0)
        h = L.b200_model_session_from_snapshot(model._m, C.byref(c), flags, C.byref(err))
        if h:
            L.b200_session_free(h)
        return err.value

    def variant(**kw):
        c, keep = llm_b200.session._snapshot_struct(snap)
        for k, v in kw.items():
            setattr(c, k, v)
        return c, keep

    c, keep = variant()
    assert code(m, c) == 0
    assert code(m, c, flags=8) == BAD_ARG                       # a KV bit the snapshot does not have
    bad_ids = snap.tokens.copy()
    bad_ids[3] = case.hp["n_vocab"]
    for kw in (dict(memory_v_type=1), dict(n_tokens=snap.npast - 1), dict(npast=snap.npast + 1), dict(n_logits=snap.last_logits.size - 1),
               dict(npast=case.n_ctx + 1, n_tokens=case.n_ctx + 1), dict(n_batch=0), dict(tokens=bad_ids.ctypes.data)):
        c, keep = variant(**kw)
        assert code(m, c) == BAD_ARG, kw
    mt = TpLlama(hp2, llm_b200.ModelParameters(context_size=256), t2, rank=0, world=2, device=0)   # refused before any size check
    c, keep = variant()
    assert code(mt, c) == BAD_ARG
    mt.close(); other_ctx.close(); other_geo.close()


def _write(tmp_path, data):
    p = tmp_path / "copy.bin"
    p.write_bytes(data)
    return p


def test_fast_session(orc, tmp_path):
    case = Case(orc, "gqa", KV.Float16)
    m = case.model()
    s = case.session(m, flags=4)                                # B200_SESSION_FAST
    toks = synth.make_tokens(case.hp, 80)
    s.feed_prompt(toks[:50])
    snap = s.get_snapshot()
    s.write_snapshot(tmp_path / "fast.bin")
    a = case.cls.from_snapshot(snap, m, flags=4)
    b = case.cls.read_snapshot(tmp_path / "fast.bin", m, flags=4)
    for i in range(50, 60):
        want = s.evaluate(toks[i:i + 1])
        check(a.evaluate(toks[i:i + 1]), want, "FAST restored in memory")
        check(b.evaluate(toks[i:i + 1]), want, "FAST restored from a file")
    for x in (a, b, s):
        x.close()
    m.close()
