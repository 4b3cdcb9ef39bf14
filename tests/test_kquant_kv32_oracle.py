"""The typed reference graphs on an F32 KV cache (oracle/kquant_kv32.mk), pinned on the CPU before any GPU test relies on them (no GPU needed):

  * with every 2-D weight of one classic type (Q4_0), each _kq_kv32 library gives the logits of every step and both caches of the one-type F32-cache
    library (oracle/kv32.mk), bit for bit: LLaMA, GPT-NeoX, GPT-2, MPT and GPT-J;
  * the F16-cache typed libraries (oracle/kquant.mk, oracle/neox_kquant.mk) still give the one-type F16 reference's bits, so building the new
    recipe changed nothing it shares with them;
  * on a mixed-type model (Q4_K_M) the F32 cache is really F32 and the types really reach it: layer 0 of the cache rounded to fp16 is the F16
    typed reference's layer 0, and the logits differ."""
import numpy as np
import pytest

from oracle import alibi as A
from oracle import bindings as B
from oracle import gptj as J
from oracle import kquant as KQ
from oracle import kv32
from oracle import neox_kquant as NK
from oracle import synth

LLAMA = dict(n_vocab=512, n_embd=256, n_head=4, n_head_kv=4, n_layer=2, n_ff=768, n_rot=64, n_ctx=64)
NEOX = {"gptneox": dict(n_vocab=320, n_ctx=64, n_embd=256, n_head=4, n_layer=2, n_rot=16, use_parallel_residual=1),
        "gpt2": dict(n_vocab=320, n_ctx=64, n_embd=256, n_head=4, n_layer=2),
        "mpt": dict(n_vocab=320, n_ctx=64, n_embd=256, n_head=4, n_layer=2, alibi_bias_max=8.0),
        "gptj": dict(n_vocab=320, n_ctx=64, n_embd=256, n_head=4, n_layer=2, n_rot=16)}
STEPS = (24,) + (1,) * 16                  # a prompt, then 16 single tokens: 40 positions


@pytest.fixture(scope="module")
def libs():
    if not (KQ.have_ref_kq(kv32=True) and NK.have_ref(kv32=True) and kv32.have_ref() and KQ.have_ref_kq() and NK.have_ref()):
        pytest.skip("oracle/_ref/*_kq_kv32.so, *_kv32.so or *_kq.so not built")


def same_bits(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.nbytes == b.nbytes and a.nbytes > 0, (what, a.nbytes, b.nbytes)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), what


def run_both(x, y, toks):
    """the logits of every step of two models fed the same tokens, compared bit for bit"""
    at = 0
    for n in STEPS:
        same_bits(x.eval(toks[at:at + n]), y.eval(toks[at:at + n]), f"logits of {n} tokens at {at}")
        at += n


def llama_q4_0(ref):
    hp, tens = synth.make_llama(LLAMA, B.Q4_0, ref.quantize)
    types = {n: B.Q4_0 for n, shp in synth.tensor_shapes(hp).items() if len(shp) == 2}
    return hp, tens, types


def test_llama_q4_0_kq_kv32_is_the_kv32_reference(ref, libs):
    hp, tens, types = llama_q4_0(ref)
    toks = synth.make_tokens(hp, sum(STEPS), seed=5)
    typed = KQ.RefKq(kv32=True).llama_typed(hp, tens, types, n_threads=4, n_batch=32)
    plain = kv32.ref_lib().llama(hp, tens, n_threads=4, n_batch=32)
    run_both(typed, plain, toks)
    for which in (0, 1):
        same_bits(kv32.kv_f32(typed, which), kv32.kv_f32(plain, which), ("cache", which))
    typed.close(); plain.close()


def test_llama_q4_0_kq_is_the_f16_reference(ref, libs):
    hp, tens, types = llama_q4_0(ref)
    toks = synth.make_tokens(hp, sum(STEPS), seed=6)
    typed = KQ.RefKq().llama_typed(hp, tens, types, n_threads=4, n_batch=32)
    plain = ref.llama(hp, tens, n_threads=4, n_batch=32)
    run_both(typed, plain, toks)
    for which in (0, 1):
        same_bits(typed.kv(which), plain.kv(which), ("cache", which))
    typed.close(); plain.close()


def one_type_kv32(arch, hp, tens):
    if arch == "gptneox":
        return kv32.ref_lib().neox(hp, tens, n_threads=4, n_batch=32)
    if arch == "gpt2":
        return kv32.ref_lib().gpt2(hp, tens, n_threads=4, n_batch=32)
    if arch == "mpt":
        return kv32.RefAlibiKV32(hp, tens, A.MPT, n_threads=4, n_batch=32)
    return kv32.RefGptJKV32(hp, tens, n_threads=4, n_batch=32)


@pytest.mark.parametrize("arch", list(NEOX))
def test_neox_family_q4_0_kq_kv32_is_the_kv32_reference(ref, libs, arch):
    hp, tens, types = NK.make_typed(arch, NEOX[arch], B.Q4_0, NK.ref_lib())
    toks = np.random.default_rng(7).integers(4, hp["n_vocab"], sum(STEPS)).astype(np.int32)
    typed = NK.RefTyped(arch, hp, tens, types, n_threads=4, n_batch=32, kv32=True)
    plain = one_type_kv32(arch, hp, tens)
    run_both(typed, plain, toks)
    for which in (0, 1):
        same_bits(kv32.kv_f32(typed, which), kv32.kv_f32(plain, which), ("cache", which))
    typed.close(); plain.close()


def test_neox_q4_0_kq_is_the_f16_reference(ref, libs):
    arch = "gptneox"
    hp, tens, types = NK.make_typed(arch, NEOX[arch], B.Q4_0, NK.ref_lib())
    toks = np.random.default_rng(8).integers(4, hp["n_vocab"], sum(STEPS)).astype(np.int32)
    typed = NK.RefTyped(arch, hp, tens, types, n_threads=4, n_batch=32)
    plain = ref.neox(hp, tens, n_threads=4, n_batch=32)
    run_both(typed, plain, toks)
    for which in (0, 1):
        same_bits(typed.kv(which), plain.kv(which), ("cache", which))
    typed.close(); plain.close()


def test_mixed_types_reach_the_f32_cache(libs):
    """Q4_K_M (Q6_K output, Q6_K wv / w2 in layer 1): after one prompt, layer 0 of the F32 cache rounded to fp16 is the F16 typed reference's"""
    rkq = KQ.RefKq()
    hp, tens, types = KQ.make_llama_mixed(LLAMA, "q4_K_M", rkq)
    assert types["output.weight"] == B.Q6_K and types["layers.1.feed_forward.w2.weight"] == B.Q6_K
    toks = synth.make_tokens(hp, 24, seed=9)
    m16 = rkq.llama_typed(hp, tens, types, n_threads=4, n_batch=32)
    m32 = KQ.RefKq(kv32=True).llama_typed(hp, tens, types, n_threads=4, n_batch=32)
    l16, l32 = m16.eval(toks), m32.eval(toks)
    n0 = hp["n_ctx"] * hp["n_embd"]                    # layer 0 of [n_layer][n_ctx][n_embd]
    for which in (0, 1):
        k16, k32 = m16.kv(which), kv32.kv_f32(m32, which)
        assert k16.dtype == np.uint16 and k32.size == k16.size
        assert np.array_equal(k32[:n0].astype(np.float16).view(np.uint16), k16[:n0]), which
        assert np.count_nonzero(k32[:n0]) > 0
    assert not np.array_equal(l16, l32)
    assert np.abs(l16 - l32).max() < 0.1 * np.abs(l16).max()        # only the cache's rounding differs
    m16.close(); m32.close()
