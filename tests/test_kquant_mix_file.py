"""Per-tensor weight types on the host (CPU only): the quantizer's mix rules as oracle/kquant.py restates them, tensor by tensor against the reference
quantizer's code (LC/llama.cpp:2938-2965), and files written with each mix: the type table the loader reads back from them."""
import numpy as np
import pytest

from oracle import bindings as B
from oracle import kquant as KQ
from oracle import synth

HP = dict(n_vocab=512, n_embd=256, n_head=4, n_head_kv=4, n_layer=8, n_ff=768, n_rot=64, n_ctx=256)


@pytest.mark.parametrize("mix", list(KQ.MIXES))
def test_mix_rules_tensor_by_tensor(mix):
    t = KQ.mix_types(HP, mix)
    base = KQ.MIXES[mix][0]
    more = [il for il in range(8) if KQ.use_more_bits(il, 8)]
    assert more == [0, 3, 6, 7]                             # n/8 = 1: layer 0, layers >= 7, and (i - 1) % 3 == 2
    for name, typ in t.items():
        il = int(name.split(".")[1]) if name.startswith("layers.") else -1
        if name == "output.weight":
            want = B.Q6_K                                   # 512 x 256: both multiples of 256, whatever the file type
        elif name.endswith(("attention.wv.weight", "feed_forward.w2.weight")):
            want = B.Q4_K if mix in ("q3_K_M", "q2_K") else B.Q6_K if mix in ("q4_K_M", "q5_K_M") and il in more else base
        elif name.endswith("attention.wo.weight"):
            want = B.Q4_K if mix in ("q3_K_M", "q2_K") else base
        else:
            want = base
        assert typ == want, (mix, name, typ, want)
    assert len(t) == 2 + 7 * HP["n_layer"]


def test_mix_fallbacks():
    """a vocabulary that is not a multiple of 256 keeps output.weight out of Q6_K; a K-quant choice on a 320-row lm_head falls back to F16, on a
    320-row embedding to Q4_0, and on a layer tensor the quantizer throws"""
    hp = dict(HP, n_vocab=320)
    assert KQ.mix_types(hp, "q4_0")["output.weight"] == B.Q4_0
    t = KQ.mix_types(hp, "q4_K_M")
    assert t["output.weight"] == B.F16 and t["tok_embeddings.weight"] == B.Q4_0
    with pytest.raises(ValueError):
        KQ.mix_types(dict(HP, n_ff=704), "q4_K_M")


@pytest.mark.parametrize("mix", ["q4_0", "q4_K_M", "q5_K_M", "q3_K_M", "q6_K"])
def test_file_type_table(tmp_path, mix):
    """write_llama with a mix's types, read back through the file parser: every 2-D tensor carries its own type and byte count, the header
    its file type and the base type (that of layers.0.attention.wq)"""
    from llm_b200 import loader
    hp = dict(HP, n_layer=2)
    types = KQ.mix_types(hp, mix)
    _, f32 = synth.make_llama(hp, B.Q4_0, lambda t, w: w)
    tensors = {}
    for name, a in f32.items():
        if name in types:
            n, k = a.shape
            tensors[name] = np.zeros((n, B.row_bytes(types[name], k)), np.uint8)
        else:
            tensors[name] = a
    hp["wtype"] = KQ.MIXES[mix][0]
    path = str(tmp_path / f"{mix}.ggjt")
    loader.write_llama(path, hp, tensors, synth.tensor_shapes(hp), tensor_types=types, llama_ftype=KQ.MIXES[mix][1])
    f = loader.GgmlFile(path)
    infos = {t["name"]: t for t in f.tensors()}
    for name, typ in types.items():
        assert infos[name]["type"] == typ, name
        assert infos[name]["nbytes"] == tensors[name].nbytes, name
    h = f.llama_hyperparameters()
    assert h["wtype"] == KQ.MIXES[mix][0] and h["llama_ftype"] == KQ.MIXES[mix][1] and h["quantization_version"] == 2
    f.close()


def test_k_quant_file_needs_quantization_version_2(tmp_path):
    """the reference's loader counts K-quant tensors as quantized (ggml_is_quantized; crates/llm-base/src/loader.rs:481-484): a file holding only
    K-quant weights and F32 norms must carry quantization version 2"""
    from llm_b200 import loader
    hp = dict(HP, n_layer=1)
    types = KQ.mix_types(hp, "q6_K")
    _, f32 = synth.make_llama(hp, B.Q4_0, lambda t, w: w)
    tensors = {name: (np.zeros((a.shape[0], B.row_bytes(types[name], a.shape[1])), np.uint8) if name in types else a) for name, a in f32.items()}
    hp["wtype"] = B.Q6_K
    for qv, ok in ((1, False), (2, True)):
        path = str(tmp_path / f"qv{qv}.ggjt")
        loader.write_llama(path, hp, tensors, synth.tensor_shapes(hp), tensor_types=types, quantization_version=qv)
        f = loader.GgmlFile(path)
        if ok:
            assert f.llama_hyperparameters()["quantization_version"] == 2
        else:
            with pytest.raises(loader.LoadError) as e:
                f.llama_hyperparameters()
            assert e.value.kind == "QuantizationVersion"
        f.close()
