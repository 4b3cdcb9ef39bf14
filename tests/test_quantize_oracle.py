"""CPU checks of model quantization: the Python restatement of the reference's `quantize` (oracle/quantize.py) against the reference's own
ggml_quantize_q* and the native file parser, the tensor selection of every architecture, and every refusal of b200_quantize_file -- all of
which happen before the destination is created and before any device work."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import quantize as Q

TARGET_NAMES = {"q4_0": Q.Q4_0, "q4_1": Q.Q4_1, "q5_0": Q.Q5_0, "q5_1": Q.Q5_1, "q8_0": Q.Q8_0}


@pytest.fixture(scope="module")
def need_ref():
    if not Q.have_ref():
        pytest.skip("oracle/_ref/libggml_ref.so not built (the reference's ggml_quantize_q* are the oracle)")


def recount(target, data):
    """the histogram of LC/ggml.c:18092-18202 recounted from GGML blocks with numpy"""
    blk = np.frombuffer(data, np.uint8).reshape(-1, Q.BLOCK_BYTES[target])
    if target == Q.Q8_0:
        q = blk[:, 2:].copy().view(np.int8).astype(np.int64)
        bins = np.sign(q) * (np.abs(q) // 16) + 8                                  # C's truncating q / 16
    else:
        off = 4 if target in (Q.Q4_1, Q.Q5_1) else 2
        if target in (Q.Q5_0, Q.Q5_1):
            qh = blk[:, off:off + 4].copy().view(np.uint32)[:, 0].astype(np.int64)
            off += 4
        qs = blk[:, off:off + 16].astype(np.int64)
        lo, hi = qs & 0xF, qs >> 4
        if target in (Q.Q5_0, Q.Q5_1):
            # the reference's loop j = 0, 2, .., 30 pairs qs[j / 2] with fifth bits j and j + 16 -- not the element's own -- and on x86 its shifts
            # past bit 31 take their count mod 32: (qh & 1 << (j + 16)) >> (j + 12) is bit j + 16, 0 (j = 16, 18) or bit j - 16 (j >= 20)
            j = 2 * np.arange(16)
            hi_bit = np.where(j <= 14, j + 16, np.where(j >= 20, j - 16, 32))
            lo = (lo | (((qh[:, None] >> j) & 1) << 4)) // 2
            hi = (hi | (((qh[:, None] >> hi_bit) & 1) << 4)) // 2
        bins = np.concatenate([lo, hi], 1)
    return np.bincount(bins.ravel(), minlength=16)


@pytest.mark.parametrize("target", list(TARGET_NAMES.values()), ids=list(TARGET_NAMES))
def test_histogram_recount_matches_reference(need_ref, target):
    rng = np.random.default_rng(target)
    x = (rng.standard_normal((40, 256)) * rng.uniform(1e-3, 20, (40, 1))).astype(np.float32)
    x[1, :32] = 0.0
    x[2, :32] = np.concatenate([[127.0], -np.arange(1, 32, dtype=np.float32) / 2])      # Q8_0: d = 1, q = -1 .. -15 (bin 8) and -16 (bin 7)
    x[3, 32:64] = np.concatenate([[-127.0], np.arange(1, 32, dtype=np.float32) * 4])     # Q8_0: positive quants into bins 8 .. 15
    data, hist = Q.ggml_quantize(target, x, 256)
    assert np.array_equal(recount(target, data), hist)
    assert hist.sum() == x.size
    if target == Q.Q8_0:
        assert hist[0] == 0 and hist[8] > 0                                            # bin 0 needs q <= -128; |q| <= 127
        q2 = np.frombuffer(data, np.uint8).reshape(40, 8, 34)[2, 0, 2:].copy().view(np.int8)
        assert q2[0] == 127 and set(q2[1:31].tolist()) >= set(range(-15, 0))


@pytest.mark.parametrize("arch", Q.ARCHS)
def test_tensor_selection(arch):
    hp = Q.CONFIGS[arch]
    names = list(Q.shapes(arch, hp, lm_head=True))
    got = {n for n, s in Q.shapes(arch, hp, lm_head=True).items() if Q.selected(arch, n, len(s))}
    if arch == "gpt2":
        want = {"model/wte", "model/lm_head"} | {f"model/h{i}/{w}" for i in range(hp["n_layer"])
                                                for w in ("attn/c_attn/w", "attn/c_proj/w", "mlp/c_fc/w", "mlp/c_proj/w")}
        assert "model/wpe" in names and "model/wpe" not in got                         # positional embeddings stay as they are
    else:
        want = {n for n, s in Q.shapes(arch, hp).items() if len(s) == 2}            # every 2-D ".*weight"; 1-D norms and biases are copied
        assert all(n.endswith("weight") for n in want)
    assert got == want


@pytest.mark.parametrize("container", ["ggjt-v3", "ggml"])
@pytest.mark.parametrize("arch,cfg", [("llama", "llama"), ("gpt2", "gpt2"), ("gptneox", "gptneox"), ("mpt", "mpt"), ("bloom", "bloom"), ("gptj", "gptj")])
def test_restatement_files_parse(need_ref, tmp_path, arch, cfg, container):
    from llm_b200.loader import GgmlFile
    hp, words, vocab, tensors = Q.model(arch, cfg, Q.F16, lm_head=True, scored=container == "ggjt-v3")
    exp = Q.quantize(arch, words, vocab, tensors, Q.Q5_1, container)
    path = str(tmp_path / "q.bin")
    open(path, "wb").write(exp["file"])
    f = GgmlFile(path, arch)
    assert f.container == (("ggjt", 3) if container == "ggjt-v3" else ("ggml", 0))
    want_words = list(words)
    want_words[Q.FILE_TYPE_WORD[arch]] = 2009
    w8 = (C.c_int32 * 8)()
    f.L.b200_ggml_hparams(f._f, None, C.byref(w8), None)
    assert list(w8)[:len(words)] == want_words
    assert f.vocabulary() == [(t, np.float32(s)) for t, s in vocab]
    table = f.tensors()
    assert [t["name"] for t in table] == [t["name"] for t in tensors]
    for i, (t, r) in enumerate(zip(table, exp["reports"])):
        assert (t["type"], t["n_dims"], t["ne"], t["nbytes"]) == (r["dst_type"], r["n_dims"], r["ne"], r["reduced_size"])
        if container == "ggjt-v3":
            assert t["offset"] % 32 == 0
    for i, r in enumerate(exp["reports"]):
        want = tensors[i]["data"] if r["dst_type"] == r["src_type"] else None          # copied tensors, byte for byte
        assert want is None or f.tensor_bytes(i).tobytes() == want, r["name"]
    f.close()
    assert exp["events"][0] == ("HyperparametersLoaded",) and exp["events"][-1][0] == "Finished"


# ---- refusals: every check runs before the destination is created --------------------------------------------------------------------------
def _write(path, words, vocab, tensors, container="ggjt-v3"):
    open(path, "wb").write(Q.write_file(words, vocab, tensors, container))
    return str(path)


def _c_quantize(src, dst, arch, target, container=0):
    from llm_b200 import _lib
    from llm_b200.loader import ARCH
    return _lib.lib().b200_quantize_file(src.encode(), dst.encode(), ARCH[arch], target, container, _lib.QUANTIZE_CALLBACK(), None, None, None, None)


def _one(name, x, src_type=Q.F32):
    return [Q.tensor(name, x, src_type)]


@pytest.fixture
def small(tmp_path):
    hp, words, vocab, tensors = Q.model("llama", "llama", Q.F16)
    return words, vocab, tensors


def test_refusals_leave_no_file(tmp_path, small):
    import llm_b200
    from llm_b200.quantize import QuantizeError
    words, vocab, tensors = small
    dst = str(tmp_path / "out.bin")
    src = _write(tmp_path / "src.bin", words, vocab, tensors)
    cases = [  # (source path, arch, target, container, C code, Python error kind)
        (src, "llama", 1, 0, -16, "InvalidQuantizationTarget"),                                         # F16 is no QuantizationTarget
        (src, "llama", 14, 0, -16, "InvalidQuantizationTarget"),                                        # nor are the K-quants
        (src, "llama", 9, 0, -16, "InvalidQuantizationTarget"),                                         # nor Q8_1
        (src, "llama", Q.Q4_0, 1, -17, "VocabularyScoringNotSupported"),                               # GGML container, scored vocabulary
    ]
    q8 = dict(name="x.weight", n_dims=2, ne=(64, 2), type=Q.Q8_0, data=bytes(4 * 34))
    cases.append((_write(tmp_path / "q8.bin", words, vocab, [q8]), "llama", Q.Q4_0, 0, -14, "UnsupportedElementType"))
    i32 = dict(name="x.weight", n_dims=2, ne=(64, 2), type=18, data=bytes(512))
    cases.append((_write(tmp_path / "i32.bin", words, vocab, [i32]), "llama", Q.Q8_0, 0, -14, "UnsupportedElementType"))
    r96 = _write(tmp_path / "r96.bin", words, vocab, tensors[:2] + _one("x.weight", np.ones((3, 96))))
    cases += [(r96, "llama", t, 0, -13, "InvariantBroken") for t in (Q.Q4_0, Q.Q4_1)]                  # Q4 rows need ne0 % 64 == 0
    r48 = _write(tmp_path / "r48.bin", words, vocab, _one("x.weight", np.ones((2, 48)), Q.F16))
    cases += [(r48, "llama", t, 0, -13, "InvariantBroken") for t in Q.TARGETS]                         # ne0 % 32 != 0
    gpt2 = _write(tmp_path / "gpt2.bin", Q.header_words("gpt2", Q.CONFIGS["gpt2"], 1), vocab[:320],
                  _one("model/h0/mlp/c_fc/w", np.ones((2, 40)), Q.F16))
    cases.append((gpt2, "gpt2", Q.Q8_0, 0, -13, "InvariantBroken"))
    for src_path, arch, target, container, code, kind in cases:
        assert _c_quantize(src_path, dst, arch, target, container) == code, (src_path, target)
        assert not os.path.exists(dst)
        with pytest.raises(QuantizeError) as e:
            llm_b200.quantize(src_path, dst, arch, target, "ggml" if container else "ggjt-v3")
        assert e.value.kind == kind
        assert not os.path.exists(dst)
    # a matrix that is not selected is copied whatever its shape: GPT-2's positional embeddings, 1-D tensors
    # (checked on the GPU in tests/test_gpu_quantize.py); the source's LoadError is QuantizeError::Load
    open(tmp_path / "junk.bin", "wb").write(b"nope" * 8)
    assert _c_quantize(str(tmp_path / "junk.bin"), dst, "llama", Q.Q4_0) == -11
    with pytest.raises(QuantizeError) as e:
        llm_b200.quantize(str(tmp_path / "junk.bin"), dst, "llama", Q.Q4_0)
    assert e.value.kind == "Load" and e.value.load_error.kind == "InvalidMagic"
    assert not os.path.exists(dst)


def test_refusals_bad_arguments(tmp_path, small):
    import llm_b200
    from llm_b200 import _lib
    words, vocab, tensors = small
    src = _write(tmp_path / "src.bin", words, vocab, tensors)
    dst = str(tmp_path / "out.bin")
    L = _lib.lib()
    assert L.b200_quantize_file(src.encode(), dst.encode(), 6, Q.Q4_0, 0, _lib.QUANTIZE_CALLBACK(), None, None, None, None) == -2   # LoRA
    assert L.b200_quantize_file(src.encode(), dst.encode(), 0, Q.Q4_0, 2, _lib.QUANTIZE_CALLBACK(), None, None, None, None) == -2   # container
    assert not os.path.exists(dst)
    before = open(src, "rb").read()
    link = str(tmp_path / "link.bin")
    os.symlink(src, link)
    for same in (src, link, str(tmp_path / "." / "src.bin")):                          # the source itself, by any name: it would be truncated
        assert _c_quantize(src, same, "llama", Q.Q8_0) == -2
        with pytest.raises(ValueError):
            llm_b200.quantize(src, same, "llama", "q8_0")
    assert open(src, "rb").read() == before
    with pytest.raises(ValueError):
        llm_b200.quantize(src, dst, "lora", "q4_0")
    assert not os.path.exists(dst)
