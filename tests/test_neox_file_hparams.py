"""The GPT-NeoX-family view of a model file, through the parser alone (no GPU): each header's mapping to the runtime's hyperparameters, the
type table the loader builds from the tensor records, and the quantization-version rule, for GPT-NeoX, GPT-2, MPT, BLOOM and GPT-J files."""
import numpy as np
import pytest

from llm_b200 import loader
from oracle import neox_kquant as NK

F32, F16, Q4_0, Q5_1, Q8_0, Q4_K, Q6_K = 0, 1, 2, 7, 8, 12, 14
BLOCK = {F16: (1, 2), Q4_0: (32, 18), Q5_1: (32, 24), Q8_0: (32, 34), Q4_K: (256, 144), Q6_K: (256, 210)}
E, V, N_LAYER = 256, 40, 2


def tensors(arch, hp, types, lm_head=False):
    """zero tensors of the right byte counts: 2-D weights of their type, everything else f32"""
    out = {}
    for name, shp in NK.tensor_shapes(arch, hp, lm_head).items():
        if name in types:
            blk, nb = BLOCK[types[name]]
            out[name] = np.zeros(shp, np.float16) if types[name] == F16 else np.zeros((shp[0], shp[1] // blk * nb), np.uint8)
        else:
            out[name] = np.zeros(shp, np.float32)
    return out


def write(tmp_path, arch, header, types, lm_head=False, extra=None):
    hp = dict(n_vocab=V, n_embd=E, n_layer=N_LAYER, n_ctx=header.get("n_ctx", 2048))
    t = tensors(arch, hp, types, lm_head)
    t.update(extra or {})
    path = str(tmp_path / f"{arch}.bin")
    shapes = dict(NK.tensor_shapes(arch, hp, lm_head), **{k: v.shape for k, v in (extra or {}).items()})
    loader.write_model(path, arch, dict(header, n_vocab=V, n_embd=E, n_layer=N_LAYER), t, shapes, Q4_0, tensor_types=types)
    return loader.GgmlFile(path, arch)


def types_of(arch, hp, base, lm_head=False, **over):
    return dict({n: base for n in NK.matrices(arch, hp, lm_head)}, **over)


HP = dict(n_vocab=V, n_embd=E, n_layer=N_LAYER, n_ctx=64)


def test_gptneox_header(tmp_path):
    f = write(tmp_path, "gptneox", dict(n_ctx=4096, n_head=8, n_rot=24, use_parallel_residual=0, file_type=2002),
              types_of("gptneox", HP, Q4_0, **{"embed_out.weight": Q6_K}))
    hp = loader.neox_hyperparameters(f)
    assert (hp["arch"], hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["n_layer"], hp["n_rot"], hp["use_parallel_residual"]) == (0, V, E, 8, N_LAYER, 24, 0)
    assert hp["n_ctx"] == 2048 and hp["wtype"] == Q4_0 and hp["quantization_version"] == 2 and hp["alibi_bias_max"] == 0.0
    types = loader.weight_types(f)
    assert types == types_of("gptneox", HP, Q4_0, **{"embed_out.weight": Q6_K})
    assert list(types)[:2] == ["gpt_neox.embed_in.weight", "embed_out.weight"]          # file order


@pytest.mark.parametrize("lm_head", [False, True])
def test_gpt2_header(tmp_path, lm_head):
    hp_ = dict(HP, n_ctx=64)
    f = write(tmp_path, "gpt2", dict(n_ctx=64, n_head=4, file_type=2007), types_of("gpt2", hp_, Q5_1, lm_head), lm_head)
    hp = loader.neox_hyperparameters(f)
    assert (hp["arch"], hp["n_ctx"], hp["n_head"], hp["has_lm_head"], hp["wtype"]) == (1, 64, 4, int(lm_head), Q5_1)
    types = loader.weight_types(f)
    assert "model/wpe" not in types                         # 2-D, but the learned positions are not a matrix the loader types
    assert types == types_of("gpt2", hp_, Q5_1, lm_head)


def test_mpt_header(tmp_path):
    f = write(tmp_path, "mpt", dict(max_seq_len=2048, n_head=4, alibi_bias_max=6.5, clip_kqv=0.0, file_type=2015),
              types_of("mpt", HP, Q4_K, **{"transformer.wte.weight": Q6_K, "transformer.blocks.1.ffn.down_proj.weight": Q8_0}))
    hp = loader.neox_hyperparameters(f)
    assert (hp["arch"], hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["n_layer"], hp["alibi_bias_max"]) == (2, V, E, 4, N_LAYER, 6.5)
    assert hp["wtype"] == Q6_K and hp["n_ctx"] == 2048
    assert loader.weight_types(f)["transformer.blocks.1.ffn.down_proj.weight"] == Q8_0


def test_bloom_header(tmp_path):
    f = write(tmp_path, "bloom", dict(n_mult=1, n_head=16, file_type=1), types_of("bloom", HP, F16))
    hp = loader.neox_hyperparameters(f)
    assert (hp["arch"], hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["alibi_bias_max"], hp["wtype"]) == (3, V, E, 16, 8.0, F16)
    assert loader.weight_types(f) == types_of("bloom", HP, F16)


def test_gptj_header_and_unknown_tensors(tmp_path):
    t = types_of("gptj", HP, Q4_K, **{"transformer.h.0.attn.v_proj.weight": Q8_0})
    extra = {"transformer.h.0.attn.rotary.weight": np.zeros((4, E), np.float32), "transformer.h.5.attn.q_proj.weight": np.zeros((4, E), np.float32)}
    f = write(tmp_path, "gptj", dict(n_ctx=2048, n_head=4, n_rot=32, file_type=2015), t, extra=extra)
    hp = loader.neox_hyperparameters(f)
    assert (hp["arch"], hp["n_head"], hp["n_rot"], hp["wtype"]) == (4, 4, 32, Q4_K)
    assert loader.weight_types(f) == t                      # a name the model does not hold, and a layer past n_layer, are not in the table


def test_quantization_version_rule(tmp_path):
    f = write(tmp_path, "gptneox", dict(n_ctx=64, n_head=4, n_rot=16, use_parallel_residual=1, file_type=1002), types_of("gptneox", HP, Q4_0))
    with pytest.raises(loader.LoadError) as e:
        loader.neox_hyperparameters(f)
    assert e.value.kind == "QuantizationVersion"
    f = write(tmp_path, "gptneox", dict(n_ctx=64, n_head=4, n_rot=16, use_parallel_residual=1, file_type=1001), types_of("gptneox", HP, F16))
    assert loader.neox_hyperparameters(f)["quantization_version"] == 1          # F16 files take any version
