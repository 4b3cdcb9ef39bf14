"""MPT and BLOOM model-file headers (no GPU): 8 words with two f32 among them (mpt lib.rs:317-330; the vocabulary count is word 4) and 6 plain
words (BLOOM: n_vocab n_embd n_mult n_head n_layer file_type)."""
import struct

import numpy as np
import pytest

from oracle import alibi as A
from oracle import bindings as B


def _vocab(n):
    return [(f"t{i}".encode(), float(i) * 0.5) for i in range(n)]


def test_mpt_header_roundtrip(orc, tmp_path):
    from llm_b200 import loader
    hp, tens = A.make_mpt(dict(A.MPT_CONFIGS["mpt-tiny"], n_vocab=96, alibi_bias_max=8.0), B.Q4_1, orc.quantize)
    p = str(tmp_path / "mpt.ggjt")
    header = dict(hp, max_seq_len=2048, clip_kqv=-0.75, file_type=3)      # a negative clip_kqv is accepted: read_f32 takes any value
    loader.write_model(p, "mpt", header, tens, A.mpt_tensor_shapes(hp), hp["wtype"], vocabulary=_vocab(hp["n_vocab"]))
    f = loader.GgmlFile(p, "mpt")
    h = f.hyperparameters()
    assert h == dict(n_embd=256, max_seq_len=2048, n_head=4, n_layer=2, n_vocab=96, alibi_bias_max=8.0, clip_kqv=-0.75, file_type=3)
    assert isinstance(h["alibi_bias_max"], float) and isinstance(h["clip_kqv"], float) and isinstance(h["n_embd"], int)
    assert f.vocabulary() == [(t, s) for t, s in _vocab(96)]            # word 4 counts the tokens; word 0 (n_embd = 256) would misread the file
    t = f.tensors()
    assert [x["name"] for x in t] == list(tens.keys())
    wqkv = next(i for i, x in enumerate(t) if x["name"] == "transformer.blocks.1.attn.Wqkv.weight")
    assert np.array_equal(f.tensor_bytes(wqkv).reshape(3 * 256, -1), tens["transformer.blocks.1.attn.Wqkv.weight"])
    f.close()
    words = struct.unpack("<8i", open(p, "rb").read()[8:40])
    assert words[:5] == (256, 2048, 4, 2, 96) and words[7] == 3
    assert struct.unpack("<2f", struct.pack("<2i", *words[5:7])) == (8.0, -0.75)


def test_bloom_header_roundtrip(orc, tmp_path):
    from llm_b200 import loader
    hp, tens = A.make_bloom(dict(A.BLOOM_CONFIGS["bloom-tiny"], n_vocab=80), B.Q8_0, orc.quantize)
    p = str(tmp_path / "bloom.ggjt")
    loader.write_model(p, "bloom", dict(hp, n_mult=1, file_type=7), tens, A.bloom_tensor_shapes(hp), hp["wtype"], vocabulary=_vocab(hp["n_vocab"]))
    f = loader.GgmlFile(p, "bloom")
    assert f.hyperparameters() == dict(n_vocab=80, n_embd=256, n_mult=1, n_head=4, n_layer=2, file_type=7)
    assert len(f.vocabulary()) == 80 and [x["name"] for x in f.tensors()] == list(tens.keys())
    f.close()
    assert struct.unpack("<6i", open(p, "rb").read()[8:32]) == (80, 256, 1, 4, 2, 7)


@pytest.mark.parametrize("arch,n_words", [("mpt", 8), ("bloom", 6)])
def test_truncated_header_is_io(tmp_path, arch, n_words):
    from llm_b200 import loader
    p = str(tmp_path / f"{arch}.bin")
    with open(p, "wb") as fp:                                          # GGJT v3, one header word short
        fp.write(struct.pack(f"<II{n_words - 1}i", 0x67676a74, 3, *range(1, n_words)))
    with pytest.raises(loader.LoadError) as e:
        loader.GgmlFile(p, arch)
    assert e.value.kind == "Io"


def test_negative_integer_words_are_still_invariant_broken(tmp_path):
    """only MPT's two f32 words skip the usize check"""
    from llm_b200 import loader
    p = str(tmp_path / "neg.bin")
    with open(p, "wb") as fp:
        fp.write(struct.pack("<II8i", 0x67676a74, 3, 64, 128, -2, 1, 0, 0, 0, 2))
    with pytest.raises(loader.LoadError) as e:
        loader.GgmlFile(p, "mpt")
    assert e.value.kind == "InvariantBroken"
