"""LoRA adapters without a GPU: the GGLA container as the reference's loader reads it (LoraParameters: r, alpha, no vocabulary), and the plain-C
restatement of LoraAdapter::patch (oracle/lora_oracle.c) pinned bit for bit to the reference's own ggml.c running the patch graph (oracle/ref_lora.c)."""
import struct

import numpy as np
import pytest

from oracle import bindings as B
from oracle import lora as Lo

TARGETS = {"f32": B.F32, **B.QUANT_TYPES}
RANKS = [7, 8, 31, 32, 40, 64]        # leftovers only (7, 8, 31), whole 32-element steps (32, 64), steps and leftovers (40)


def _table(tmp_path, r=4, alpha=8, version=1):
    rng = np.random.default_rng(1)
    tens, fac = Lo.adapter_tensors({"layers.0.attention.wq.weight": (64, 32), "norm.weight": (64, 1)}, r, rng)
    path = str(tmp_path / "a.ggla")
    Lo.write_ggla(path, r, alpha, tens)
    if version != 1:
        with open(path, "r+b") as f:
            f.seek(4)
            f.write(struct.pack("<I", version))
    return path, tens


def test_ggla_header_and_tensor_table(tmp_path):
    from llm_b200.loader import GgmlFile
    path, tens = _table(tmp_path, r=4, alpha=8)
    f = GgmlFile(path, "lora")
    assert f.container == ("ggla", 1)
    assert f.hyperparameters() == {"r": 4, "alpha": 8}
    assert f.vocabulary() == []
    got = f.tensors()
    assert [t["name"] for t in got] == list(tens)
    for t, (typ, ne, data) in zip(got, tens.values()):
        assert t["type"] == typ and t["n_dims"] == 2 and t["ne"] == (ne[0], ne[1])
        assert t["offset"] % 32 == 0
        assert t["nbytes"] == np.asarray(data).nbytes
    assert np.array_equal(f.tensor_bytes(0), np.asarray(tens["layers.0.attention.wq.weight.loraA"][2]).view(np.uint8).ravel())
    f.close()


def test_ggla_negative_alpha_is_a_scaling(tmp_path):
    from llm_b200.loader import GgmlFile
    path, _ = _table(tmp_path, r=16, alpha=-8)
    f = GgmlFile(path, "lora")
    assert f.hyperparameters() == {"r": 16, "alpha": -8}
    f.close()


@pytest.mark.parametrize("version", [0, 2])
def test_ggla_bad_version(tmp_path, version):
    from llm_b200.loader import GgmlFile, LoadError
    path, _ = _table(tmp_path, version=version)
    with pytest.raises(LoadError) as e:
        GgmlFile(path, "lora")
    assert e.value.kind == "InvalidFormatVersion"


@pytest.mark.parametrize("r", [0, -3])
def test_ggla_rank_must_be_positive(tmp_path, r):
    from llm_b200.loader import GgmlFile, LoadError
    path = str(tmp_path / "r.ggla")
    Lo.write_ggla(path, r, 8, {})
    with pytest.raises(LoadError) as e:
        GgmlFile(path, "lora")
    assert e.value.kind == "InvariantBroken"


@pytest.fixture(scope="module")
def pair(orc):
    if not Lo.have_ref():
        pytest.skip("oracle/_ref/libggml_lora.so not built (the reference's ggml running the LoRA patch graph)")
    return Lo.RefLora(), Lo.OracleLora()


def target(orc, wtype, K, N, rng):
    w = (rng.standard_normal((N, K)) * 0.1).astype(np.float32)
    return w if wtype == B.F32 else orc.quantize(wtype, w)


@pytest.mark.parametrize("alpha", ["r", 3])
@pytest.mark.parametrize("r", RANKS)
@pytest.mark.parametrize("a_f16", [False, True], ids=["A_f32", "A_f16"])
@pytest.mark.parametrize("tname", list(TARGETS))
def test_oracle_patch_matches_reference(orc, pair, tname, a_f16, r, alpha):
    ref, ora = pair
    wtype = TARGETS[tname]
    alpha = r if alpha == "r" else alpha
    rng = np.random.default_rng(1000 * r + wtype + 7 * a_f16)
    K, N = 96, 1 if wtype == B.F32 else 9            # an F32 target is a vector (a norm gain or bias)
    w = target(orc, wtype, K, N, rng)
    a, b = Lo.factors(rng, K, N, r, a_f16)
    s = Lo.scaling(r, alpha)
    want = ref.patch(wtype, w, K, N, a, b, s)
    got = ora.patch(wtype, w, K, N, a, b, s)
    assert np.array_equal(np.asarray(got).view(np.uint8), np.asarray(want).view(np.uint8))
    assert not np.array_equal(np.asarray(want).view(np.uint8), np.asarray(w).view(np.uint8))


def test_oracle_patch_repeats_rows_of_ba_on_f32_matrices(orc, pair):
    """add_f32 repeats the rows of ba over W (ggml_can_repeat_rows): an F32 [K, N] target with a loraB of one row"""
    ref, ora = pair
    rng = np.random.default_rng(5)
    w = target(orc, B.F32, 64, 6, rng)
    a, b = Lo.factors(rng, 64, 1, 12)
    assert np.array_equal(ora.patch(B.F32, w, 64, 6, a, b, 0.5), ref.patch(B.F32, w, 64, 6, a, b, 0.5))
