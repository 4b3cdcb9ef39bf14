"""The reference graphs' embeddings (OutputRequest::embeddings, crates/llm-base/src/model/common.rs:40-59) as the oracle returns them, pinned on the
CPU before any GPU run (no GPU needed).

oracle/embd.mk links copies of the GPT-2 / GPT-NeoX, MPT / BLOOM and GPT-J harnesses that also hand out every row of the final norm's output and of
the residual stream that norm reads (oracle/embd.py).  Each row is recomputed here from that residual: the reference's own ggml_norm (rh_op op 2),
then the gain and the bias as numpy float32 multiplies and adds, each rounded once like ggml's mul and add nodes (MPT: no add node).  The row must
match bit for bit and must differ from the residual, and the logits must be those of the committed harness's library.  The copies of the
F32-cache harnesses (oracle/kv32.mk) are checked the same way."""
import numpy as np
import pytest

from oracle import alibi as A
from oracle import bindings as B
from oracle import embd as E
from oracle import gptj as J
from oracle import kv32, synth

# arch -> (final norm gain, bias or None)
FINAL_NORM = {"neox-par": ("gpt_neox.final_layer_norm.weight", "gpt_neox.final_layer_norm.bias"),
              "neox-seq": ("gpt_neox.final_layer_norm.weight", "gpt_neox.final_layer_norm.bias"),
              "gpt2": ("model/ln_f/g", "model/ln_f/b"),
              "mpt": ("transformer.norm_f.weight", None),
              "bloom": ("output_norm.weight", "output_norm.bias"),
              "gptj": ("transformer.ln_f.weight", "transformer.ln_f.bias")}


def model(ref, arch, f32):
    """(hp, tensors, the model on oracle/embd.mk's library, the same model on the committed harness's library)"""
    if not (E.have_ref() and kv32.have_ref() and A.have_ref() and J.have_ref()):
        pytest.skip("oracle/_ref/*_embd.so / *_kv32.so not built")
    lib = kv32.ref_lib() if f32 else ref
    kw = dict(n_threads=4, n_batch=32)
    if arch.startswith("neox"):
        hp, t = synth.make_neox(synth.NEOX_CONFIGS["neox-tiny" if arch == "neox-par" else "neox-tiny-seq"], B.Q4_0, ref.quantize)
        return hp, t, E.model("neox", hp, t, f32, **kw), lib.neox(hp, t, **kw)
    if arch == "gpt2":
        hp, t = synth.make_gpt2(synth.GPT2_CONFIGS["gpt2-tiny"], B.Q4_0, ref.quantize, lm_head=True)
        return hp, t, E.model("gpt2", hp, t, f32, **kw), lib.gpt2(hp, t, **kw)
    if arch in ("mpt", "bloom"):
        make, base, a = (A.make_mpt, A.MPT_CONFIGS["mpt-tiny"], A.MPT) if arch == "mpt" else (A.make_bloom, A.BLOOM_CONFIGS["bloom-tiny"], A.BLOOM)
        hp, t = make(base, B.Q4_0, ref.quantize)
        return hp, t, E.model("alibi", hp, t, f32, a, **kw), (kv32.RefAlibiKV32 if f32 else A.RefAlibi)(hp, t, a, **kw)
    hp, t = J.make_gptj(J.GPTJ_CONFIGS["gptj-tiny"], B.Q4_0, ref.quantize)
    return hp, t, E.model("gptj", hp, t, f32, **kw), (kv32.RefGptJKV32 if f32 else J.RefGptJ)(hp, t, **kw)


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


@pytest.mark.parametrize("f32", [False, True], ids=["kv16", "kv32"])
@pytest.mark.parametrize("arch", list(FINAL_NORM))
def test_eval_embd_returns_the_final_norm_rows(ref, arch, f32):
    hp, t, cpu, plain = model(ref, arch, f32)
    e = hp["n_embd"]
    toks = synth.make_tokens(hp, 19)
    for a, b in ((0, 12), (12, 13), (13, 19)):                   # a batch, one token, a batch after it
        logits, embd, resid = E.eval_embd(cpu, toks[a:b])
        n = b - a
        assert logits.shape == (n, hp["n_vocab"]) and embd.shape == resid.shape == (n, e)
        assert np.array_equal(bits(logits), bits(plain.eval(toks[a:b]))), (arch, a)
        g_name, b_name = FINAL_NORM[arch]
        want = ref.op(2, 0, None, resid, (e, n, 1), out_shape=(n, e)) * np.asarray(t[g_name], np.float32)
        if b_name is not None:
            want = want + np.asarray(t[b_name], np.float32)
        assert want.dtype == np.float32
        assert np.array_equal(bits(embd), bits(want)), (arch, a)
        assert not np.array_equal(bits(embd), bits(resid)), (arch, a)
    cpu.close(); plain.close()


def test_llama_eval_embd_returns_the_final_norm_rows(ref):
    """LLaMA (rh_llama_eval's embd_out): the reference's own lm_head mat-mul over the returned rows gives its logits bit for bit, so the rows
    are the tensor that mat-mul reads"""
    hp, t = synth.make_llama(synth.CONFIGS["tiny8"], B.Q4_0, ref.quantize)
    toks = synth.make_tokens(hp, 9)
    if not E.have_ref():
        pytest.skip("oracle/_ref/*_embd.so not built")
    cpu, plain = E.model("llama", hp, t, n_threads=4, n_batch=32), ref.llama(hp, t, n_threads=4, n_batch=32)
    logits, embd, _ = E.eval_embd(cpu, toks)
    assert embd.shape == (9, hp["n_embd"])
    assert np.array_equal(bits(logits), bits(plain.eval(toks)))
    # the lm_head applied to the returned rows is the logits: the rows are what the reference's output mat-mul reads
    assert np.array_equal(bits(ref.mul_mat(B.Q4_0, t["output.weight"], embd)), bits(logits))
    cpu.close(); plain.close()
