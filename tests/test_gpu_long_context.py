"""Long-context decode: logits bit-identical to the CPU model at every step up to the last slot of the context, and both KV caches at the end.

Where the decode schedules change what they run, by position:
  - attn_fused_kernel on an f16 cache with heads of up to 128 makes more than one KQ pass once a CTA's share of the positions is over 256 (n_kv > 256 * hd / 32), and its soft_max
    makes a second pass at n_kv > 1024;
  - a context bucket (n_kv rounded up to 256, at most n_ctx) past 3264 positions does not fit that kernel's shared memory: from n_past 3072
    on, LLaMA decodes with the two-kernel attention (attn_kq + attn_sv, 8 launches per layer instead of 7) and GPT-NeoX / GPT-2 per op;
  - the last bucket is clamped to n_ctx, and a NeoX context that is not a multiple of 64 gets a bucket wider than the cache;
  - a LLaMA context that is not a multiple of 128 decodes per op, and an odd one leaves the V rows only 2-byte aligned.
Every decode step asserts its launch count, so each case proves which schedule it ran.  Prompts go in as chunks of 512 (n_batch 512)."""
import numpy as np
import pytest

from oracle import bindings as B
from oracle import synth

pytestmark = pytest.mark.gpu

CHUNK = 512
PER_OP = 0        # want(n_past) for a step on the per-op schedule: more launches than any graph schedule makes


def check(g, c, what):
    c = np.asarray(c, np.float32).reshape(g.shape)
    assert np.array_equal(g.view(np.uint32), c.view(np.uint32)), (what, float(np.abs(g - c).max() / np.abs(c).max()), int((g != c).sum()), g.size)


def prefill(s, cpu, toks, a, b):
    """positions [a, b) in chunks of CHUNK; the last row of each chunk compared"""
    assert s.n_past == a
    for i in range(a, b, CHUNK):
        j = min(i + CHUNK, b)
        check(np.asarray(s.evaluate(toks[i:j])).reshape(1, -1), cpu.eval(toks[i:j])[-1:], f"prefill {i}..{j}")


def decode(s, cpu, toks, a, b, want, n_layer):
    """one token per step at n_past = a .. b-1; want(n_past) is the step's launch count, or PER_OP"""
    for i in range(a, b):
        assert s.n_past == i
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        w = want(i)
        if w == PER_OP:
            assert s.last_launches > 8 * n_layer + 4, ("per-op schedule expected", i, s.last_launches)
        else:
            assert s.last_launches == w, ("schedule", i, s.last_launches, w)


def context_full(s, toks):
    import llm_b200
    n = s.n_past
    with pytest.raises(llm_b200.ContextFull):
        s.evaluate(toks[:1])
    assert s.n_past == n


# ---- LLaMA --------------------------------------------------------------------------------------------------------------------------------

def llama_cpu(orc, hp, tens):
    """the reference's own compiled ggml.c when oracle/_ref is present, else the plain-C port"""
    if B.have_ref("ref"):
        return B.RefLib("ref").llama(hp, tens, n_threads=16, n_batch=CHUNK)
    return orc.llama(hp, tens)


def llama_native(hp, tens):
    import llm_b200
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens)
    return m, m.start_session(llm_b200.InferenceSessionConfig(n_batch=CHUNK))


def llama_kv_equal(s, cpu):
    for which in (0, 1):          # the CPU model sizes its cache by n_embd; with GQA only the first n_layer * n_ctx * n_embd_gqa values are used
        a = s.kv(which)
        assert np.array_equal(a, cpu.kv(which)[:a.size]), which


# graph-eligible: n_embd and n_ff multiples of 256, n_ctx a multiple of 128
LLAMA_LONG = {
    "hd128_q4_0": (dict(n_vocab=1024, n_embd=512, n_head=4, n_head_kv=4, n_layer=2, n_ff=1536, n_rot=128, n_ctx=4096), B.Q4_0),
    "hd64_gqa_q5_1": (dict(n_vocab=1024, n_embd=512, n_head=8, n_head_kv=2, n_layer=2, n_ff=1536, n_rot=64, n_ctx=4096), B.Q5_1),
}


@pytest.mark.slow
@pytest.mark.parametrize("cfg", list(LLAMA_LONG))
def test_llama_long_context(orc, cfg):
    """n_ctx 4096: decode across n_kv 1024 (second soft_max pass; at hd 128 also the second KQ pass), across n_past 3072 (the fused
    attention gives way to attn_kq + attn_sv exactly there), into the last slot; ContextFull after it; then a rewind to 3000 replays the
    lower buckets' graphs after the two-kernel steps"""
    base, t = LLAMA_LONG[cfg]
    hp, tens = synth.make_llama(base, t, orc.quantize)
    n_ctx, nl = hp["n_ctx"], hp["n_layer"]
    toks = synth.make_tokens(hp, n_ctx)
    cpu = llama_cpu(orc, hp, tens)
    m, s = llama_native(hp, tens)
    want = lambda i: 7 * nl + 3 if i < 3072 else 8 * nl + 3      # n_kv <= 3072: bucket 3072 (fits); from n_past 3072 the bucket is 3328
    prefill(s, cpu, toks, 0, 1020)
    decode(s, cpu, toks, 1020, 1030, want, nl)
    prefill(s, cpu, toks, 1030, 3068)
    decode(s, cpu, toks, 3068, 3076, want, nl)
    prefill(s, cpu, toks, 3076, 4090)
    decode(s, cpu, toks, 4090, n_ctx, want, nl)
    context_full(s, toks)
    llama_kv_equal(s, cpu)
    s.rewind(3000)
    cpu.set_n_past(3000)
    other = synth.make_tokens(hp, 3003, seed=7)                  # new tokens: positions 3000..3002 are written afresh
    decode(s, cpu, other, 3000, 3003, want, nl)
    llama_kv_equal(s, cpu)
    s.close(); m.close(); cpu.close()


@pytest.mark.parametrize("n_ctx,qname", [(384, "q4_0"), (320, "q5_1"), (333, "q8_0")])
def test_llama_context_end(orc, n_ctx, qname):
    """the last six slots of a short context: 384 decodes on the graph with its last bucket clamped to 384; 320 (not a multiple of 128)
    decodes per op; 333 (odd) decodes per op with V rows that are only 2-byte aligned (mul_mat_f16_exact's one-warp-per-dot kernel)"""
    hp, tens = synth.make_llama(dict(synth.CONFIGS["small"], n_ff=1536, n_ctx=n_ctx), B.QUANT_TYPES[qname], orc.quantize)
    nl = hp["n_layer"]
    toks = synth.make_tokens(hp, n_ctx)
    cpu = llama_cpu(orc, hp, tens)
    m, s = llama_native(hp, tens)
    graph = n_ctx % 128 == 0
    prefill(s, cpu, toks, 0, n_ctx - 6)
    decode(s, cpu, toks, n_ctx - 6, n_ctx, lambda i: 7 * nl + 3 if graph else PER_OP, nl)
    context_full(s, toks)
    llama_kv_equal(s, cpu)
    s.close(); m.close(); cpu.close()


# ---- GPT-NeoX / GPT-2 (the CPU model is the reference's graph on its own ggml: oracle/_ref) --------------------------------------------------

def ref_lib():
    if not B.have_ref("ref"):
        pytest.skip("oracle/_ref/libggml_ref.so not built (the GPT-NeoX / GPT-2 CPU model is the reference graph on the reference's ggml)")
    return B.RefLib("ref")


def ref_rewind(cpu, toks, n):
    """the reference GPT-2 / NeoX harness has no rewind: start over and feed toks[:n] again, which rewrites the same cache positions"""
    cpu.reset()
    for i in range(0, n, CHUNK):
        cpu.eval(toks[i:min(i + CHUNK, n)])


def neox_kv_equal(s, cpu, hp, gpt2):
    nl, n_ctx, e = hp["n_layer"], hp["n_ctx"], hp["n_embd"]
    assert np.array_equal(s.kv(0), cpu.kv(0)), "K"
    v = cpu.kv(1)
    if gpt2:                      # the reference's GPT-2 keeps V by position; the native cache keeps it by channel, as for GPT-NeoX
        v = v.reshape(nl, n_ctx, e).transpose(0, 2, 1).ravel()
    assert np.array_equal(s.kv(1), v), "V"


@pytest.mark.slow
def test_neox_long_context(orc):
    """GPT-NeoX, head size 128, n_ctx 4096: across n_kv 1024 on the graph, across n_past 3072 (graph below, per op from there), to the last
    slot, then a rewind below 3072 goes back to the graph (the device n_past word is re-uploaded) with the same bits"""
    from llm_b200.neox import GptNeoX
    ref = ref_lib()
    hp, tens = synth.make_neox(dict(n_vocab=384, n_ctx=4096, n_embd=256, n_head=2, n_layer=2, n_rot=32, use_parallel_residual=1), B.Q8_0, orc.quantize)
    n_ctx, nl = hp["n_ctx"], hp["n_layer"]
    toks = synth.make_tokens(hp, n_ctx)
    cpu = ref.neox(hp, tens, n_threads=8, n_batch=CHUNK)
    m = GptNeoX(hp, tens)
    s = m.start_session(CHUNK)
    want = lambda i: 8 * nl + 3 if i < 3072 else PER_OP
    prefill(s, cpu, toks, 0, 1020)
    decode(s, cpu, toks, 1020, 1030, want, nl)
    prefill(s, cpu, toks, 1030, 3068)
    decode(s, cpu, toks, 3068, 3076, want, nl)
    prefill(s, cpu, toks, 3076, 4090)
    decode(s, cpu, toks, 4090, n_ctx, want, nl)
    context_full(s, toks)
    neox_kv_equal(s, cpu, hp, False)
    s.rewind(3000)
    ref_rewind(cpu, toks, 3000)
    other = synth.make_tokens(hp, 3003, seed=7)
    decode(s, cpu, other, 3000, 3003, want, nl)
    neox_kv_equal(s, cpu, hp, False)
    s.close(); m.close(); cpu.close()


NEOX_ENDS = {   # (config, decode windows (a, b) with a prefill to a before each)
    # head size 96 (the NeoX-20B head), sequential residual: second KQ pass from n_kv 769, last bucket 1024
    "hd96_seq": (dict(n_vocab=384, n_ctx=1024, n_embd=768, n_head=8, n_layer=2, n_rot=24, use_parallel_residual=0), ((764, 772), (1018, 1024))),
    # head size 32: one CTA per head, second KQ pass from n_kv 257
    "hd32": (dict(n_vocab=384, n_ctx=512, n_embd=256, n_head=8, n_layer=2, n_rot=16, use_parallel_residual=1), ((254, 262), (506, 512))),
    # n_ctx 200: the last bucket is 200 positions, its shared-memory layout 256 (wider than the cache)
    "hd64_ctx200": (dict(n_vocab=384, n_ctx=200, n_embd=256, n_head=4, n_layer=2, n_rot=16, use_parallel_residual=1), ((194, 200),)),
    # n_ctx 100, not a multiple of 8: per op
    "hd64_ctx100": (dict(n_vocab=384, n_ctx=100, n_embd=256, n_head=4, n_layer=2, n_rot=64, use_parallel_residual=0), ((94, 100),)),
}


@pytest.mark.parametrize("cfg", list(NEOX_ENDS))
def test_neox_head_sizes_and_context_end(orc, cfg):
    from llm_b200.neox import GptNeoX
    ref = ref_lib()
    base, windows = NEOX_ENDS[cfg]
    hp, tens = synth.make_neox(base, B.Q5_1, orc.quantize)
    n_ctx, nl = hp["n_ctx"], hp["n_layer"]
    toks = synth.make_tokens(hp, n_ctx)
    cpu = ref.neox(hp, tens, n_threads=8, n_batch=CHUNK)
    m = GptNeoX(hp, tens)
    s = m.start_session(CHUNK)
    want = lambda i: 8 * nl + 3 if n_ctx % 8 == 0 else PER_OP     # the graph schedule needs n_ctx % 8 == 0
    for a, b in windows:
        prefill(s, cpu, toks, s.n_past, a)
        decode(s, cpu, toks, a, b, want, nl)
    assert s.n_past == n_ctx
    context_full(s, toks)
    neox_kv_equal(s, cpu, hp, False)
    s.close(); m.close(); cpu.close()


@pytest.mark.slow
def test_gpt2_long_context(orc):
    """GPT-2 with 4096 learned positions: across n_past 3072 (graph below, per op from there), to the last slot, a rewind back onto the graph"""
    from llm_b200.neox import Gpt2
    ref = ref_lib()
    hp, tens = synth.make_gpt2(dict(n_vocab=320, n_ctx=4096, n_embd=256, n_head=4, n_layer=2), B.Q4_0, orc.quantize)
    n_ctx, nl = hp["n_ctx"], hp["n_layer"]
    toks = synth.make_tokens(hp, n_ctx)
    cpu = ref.gpt2(hp, tens, n_threads=8, n_batch=CHUNK)
    m = Gpt2(hp, tens)
    s = m.start_session(CHUNK)
    want = lambda i: 8 * nl + 4 if i < 3072 else PER_OP
    prefill(s, cpu, toks, 0, 3068)
    decode(s, cpu, toks, 3068, 3076, want, nl)
    prefill(s, cpu, toks, 3076, 4090)
    decode(s, cpu, toks, 4090, n_ctx, want, nl)
    context_full(s, toks)
    neox_kv_equal(s, cpu, hp, True)
    s.rewind(3000)
    ref_rewind(cpu, toks, 3000)
    other = synth.make_tokens(hp, 3003, seed=7)
    decode(s, cpu, other, 3000, 3003, want, nl)
    neox_kv_equal(s, cpu, hp, True)
    s.close(); m.close(); cpu.close()
