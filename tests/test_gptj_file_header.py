"""GPT-J model-file headers (no GPU): 8 words, n_vocab n_ctx n_embd n_head n_layer n_rot file_type n_vocab (gptj lib.rs:366-401); the repeated
n_vocab must equal the first ("GPTJ model expected n_vocab ..." -> InvariantBroken)."""
import struct

import numpy as np
import pytest

from oracle import bindings as B
from oracle import gptj as J


def _vocab(n):
    return [(f"t{i}".encode(), float(i) * 0.25) for i in range(n)]


def test_gptj_header_roundtrip(orc, tmp_path):
    from llm_b200 import loader
    hp, tens = J.make_gptj(dict(J.GPTJ_CONFIGS["gptj-hd64"], n_vocab=96, n_layer=1), B.Q4_1, orc.quantize)
    p = str(tmp_path / "gptj.ggjt")
    loader.write_model(p, "gptj", dict(hp, file_type=3), tens, J.gptj_tensor_shapes(hp), hp["wtype"], vocabulary=_vocab(hp["n_vocab"]))
    f = loader.GgmlFile(p, "gptj")
    assert f.hyperparameters() == dict(n_vocab=96, n_ctx=128, n_embd=256, n_head=4, n_layer=1, n_rot=16, file_type=3, n_vocab_again=96)
    assert f.vocabulary() == [(t, s) for t, s in _vocab(96)]
    t = f.tensors()
    assert [x["name"] for x in t] == list(tens.keys())
    k = next(i for i, x in enumerate(t) if x["name"] == "transformer.h.0.attn.k_proj.weight")
    assert t[k]["ne"] == (256, 256)
    assert np.array_equal(f.tensor_bytes(k).reshape(256, -1), tens["transformer.h.0.attn.k_proj.weight"])
    b = next(i for i, x in enumerate(t) if x["name"] == "lm_head.bias")
    assert t[b]["type"] == 0 and np.array_equal(f.tensor_bytes(b).view(np.float32), tens["lm_head.bias"])
    f.close()
    assert struct.unpack("<8i", open(p, "rb").read()[8:40]) == (96, 128, 256, 4, 1, 16, 3, 96)


def test_gptj_repeated_n_vocab_must_match(tmp_path):
    from llm_b200 import loader
    p = str(tmp_path / "gptj.bin")
    with open(p, "wb") as fp:                                          # GGJT v3, the last word disagrees with the first
        fp.write(struct.pack("<II8i", 0x67676a74, 3, 96, 128, 256, 4, 1, 16, 2, 95))
    with pytest.raises(loader.LoadError) as e:
        loader.GgmlFile(p, "gptj")
    assert e.value.kind == "InvariantBroken"


def test_gptj_truncated_header_is_io(tmp_path):
    from llm_b200 import loader
    p = str(tmp_path / "gptj.bin")
    with open(p, "wb") as fp:                                          # GGJT v3, one header word short
        fp.write(struct.pack("<II7i", 0x67676a74, 3, 96, 128, 256, 4, 1, 16, 2))
    with pytest.raises(loader.LoadError) as e:
        loader.GgmlFile(p, "gptj")
    assert e.value.kind == "Io"
