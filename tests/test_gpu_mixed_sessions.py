"""Sessions of different weight types and architectures decoding in one process, interleaved step by step, each bit-identical to its own CPU model.

A kernel's dynamic shared-memory opt-in (cudaFuncAttributeMaxDynamicSharedMemorySize) belongs to the kernel, once per process, while the decode
schedules are templates with one instantiation per weight type.  Any record of the opt-in kept per instantiation lets a second session LOWER the
attribute under a first one, whose next launch that needs more is then refused.  These tests run such sequences; every decode step asserts its launch
count, so each case proves which schedule it ran."""
import numpy as np
import pytest

from oracle import bindings as B
from oracle import gptj as J
from oracle import synth

pytestmark = [pytest.mark.gpu, pytest.mark.slow]

CHUNK = 512


def check(g, c, what):
    c = np.asarray(c, np.float32).reshape(np.shape(g))
    assert np.array_equal(np.asarray(g, np.float32).view(np.uint32), c.view(np.uint32)), (what, float(np.abs(g - c).max() / np.abs(c).max()), int((g != c).sum()))


class Run:
    """one native session, its CPU model, its tokens and the launch count each position's step must show"""

    def __init__(self, name, s, cpu, toks, want, close):
        self.name, self.s, self.cpu, self.toks, self.want, self._close = name, s, cpu, toks, want, close

    def prefill(self, b):
        for i in range(self.s.n_past, b, CHUNK):
            j = min(i + CHUNK, b)
            check(self.s.evaluate(self.toks[i:j]), self.cpu.eval(self.toks[i:j])[-1], f"{self.name}: prefill {i}..{j}")

    def step(self):
        i = self.s.n_past
        check(self.s.evaluate(self.toks[i:i + 1], all_logits=True), self.cpu.eval(self.toks[i:i + 1]), f"{self.name}: decode at n_past {i}")
        assert self.want(i, self.s.last_launches), (self.name, "schedule", i, self.s.last_launches)

    def kv_equal(self):
        for which in (0, 1):      # the LLaMA CPU model sizes its cache by n_embd; with GQA only the first n_layer * n_ctx * n_embd_gqa values are used
            a = self.s.kv(which)
            assert np.array_equal(a, self.cpu.kv(which)[:a.size]), (self.name, which)

    def close(self):
        self._close()


def llama_run(orc, name, hp, t, seed):
    import llm_b200
    hp, tens = synth.make_llama(hp, t, orc.quantize)
    cpu = B.RefLib("ref").llama(hp, tens, n_threads=16, n_batch=CHUNK) if B.have_ref("ref") else orc.llama(hp, tens)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=CHUNK))
    nl = hp["n_layer"]
    # the fused attention while the context bucket (n_kv rounded up to 256) fits its shared memory -- up to 3072 at these head sizes --, attn_kq +
    # attn_sv from n_past 3072 (bucket 3328)
    want = lambda i, n: n == (7 * nl + 3 if i < 3072 else 8 * nl + 3)
    return Run(name, s, cpu, synth.make_tokens(hp, hp["n_ctx"], seed), want, lambda: (s.close(), m.close(), cpu.close()))


def test_two_weight_types_past_the_fused_attention(orc):
    """A Q4_0 LLaMA session with n_ctx 8192 and a Q5_1 one with n_ctx 6656, both graph_ok (hd 128 / 64, n_embd 512, n_ctx % 128 == 0).
    attn_sv_kernel takes n_ctx * 6 + 10240 bytes of dynamic shared memory: 59392 and 50176, both past the 48 KB default.  The first step of
    each session opts the kernel in for what that session needs.  Then the steps alternate and both sessions cross n_past 3072, where the 3328-position
    bucket no longer fits the fused attention and attn_sv runs: the Q4_0 session first, with 59392 bytes, after the Q5_1 session has run.  With one
    record of the opt-in per weight type, the Q5_1 session had set the attribute to 50176 and that launch was refused."""
    a = llama_run(orc, "q4_0/8192", dict(n_vocab=512, n_embd=512, n_head=4, n_head_kv=4, n_layer=2, n_ff=1536, n_rot=128, n_ctx=8192), B.Q4_0, 0x5E55A)
    b = llama_run(orc, "q5_1/6656", dict(n_vocab=512, n_embd=512, n_head=8, n_head_kv=2, n_layer=2, n_ff=1536, n_rot=64, n_ctx=6656), B.Q5_1, 0x5E55B)
    a.prefill(3066)
    a.step(); a.step()                     # n_past 3066, 3067: the fused attention; the first step sets attn_sv_kernel's attribute for 8192 positions
    b.prefill(3066)
    b.step(); b.step()                     # the same for 6656 positions
    for _ in range(12):                    # n_past 3068 .. 3079, alternating: from 3072 both run attn_kq + attn_sv
        a.step()
        b.step()
    a.kv_equal(); b.kv_equal()
    a.close(); b.close()


def test_llama_and_gptj_interleaved_at_long_context(orc):
    """A Q4_0 LLaMA session (hd 128, the fused attention) and a Q4_0 GPT-J one (hd 256, the wide cluster attention), both n_ctx 4096, decoding in
    turn across n_past 3072: the LLaMA graph switches to attn_kq + attn_sv there, GPT-J to the per-op schedule (neox_decode_fits: the 3328-position
    bucket does not fit attn_fused_fits).  Below 3072 both cluster kernels share one shared-memory opt-in for buckets of 3072 positions."""
    from llm_b200 import GptJ
    if not J.have_ref():
        pytest.skip("oracle/_ref/libggml_gptj.so not built (the GPT-J CPU model is the reference graph on the reference's ggml)")
    a = llama_run(orc, "llama", dict(n_vocab=512, n_embd=512, n_head=4, n_head_kv=4, n_layer=2, n_ff=1536, n_rot=128, n_ctx=4096), B.Q4_0, 0x5E55C)
    hp, tens = J.make_gptj(dict(J.GPTJ_CONFIGS["gptj-tiny"], n_ctx=4096), B.Q4_0, orc.quantize)
    cpu = J.RefGptJ(hp, tens, n_threads=16, n_batch=CHUNK)
    m = GptJ(hp, tens)
    s = m.start_session(CHUNK)
    graph = 6 * hp["n_layer"] + 3
    toks = np.random.default_rng(0x5E55D).integers(0, hp["n_vocab"], size=hp["n_ctx"], dtype=np.int32)
    g = Run("gptj", s, cpu, toks, lambda i, n: n == graph if i < 3072 else n > graph, lambda: (s.close(), m.close(), cpu.close()))
    a.prefill(3066)
    g.prefill(3066)
    for _ in range(10):                    # n_past 3066 .. 3075
        a.step()
        g.step()
    a.kv_equal(); g.kv_equal()
    a.close(); g.close()
