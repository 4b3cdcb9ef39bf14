"""Native LLaMA sessions on mixed-type model files (per-tensor weight types), bit for bit against the reference's LLaMA graph on the same types
(oracle/kquant.mk: the reference's ggml.c + k_quants.c, a type per 2-D weight).

Each model is a synthetic LLaMA quantized by the reference quantizer's mix rules (oracle/kquant.py: mix_types), written as a GGJT v3 file and loaded
with b200_llama_load_file:
  q4_0     Q4_0 everywhere but a Q6_K output.weight: the decode graph, with quantize_row_q8_K + the K-quant mat-vec as its last two nodes
  q4_K_M   Q4_K, with wv / w2 Q6_K in the layers use_more_bits picks (layer 1 of 2) and Q4_K in the others; Q6_K output
  q5_K_M   the same on Q5_K
  q3_K_M   Q3_K, with wo / wv / w2 Q4_K in every layer
  q6_K     Q6_K everywhere (one type, a K-quant)
  q2_K     Q2_K, with wo / wv / w2 Q4_K: Q2_K token embeddings (get_rows through dequantize_row_q2_K)
  gqa      q4_K_M with 8 heads of 128 over 2 K/V heads
  q4_0-wv  Q4_0 with every wv Q8_0: [wq | wk] and wv as two classic matrices writing the same qkv rows (per op)
Each prefills in batches of 7 (the warp kernel), 40 and 100 tokens (the tiled GEMM: ragged token tiles), decodes single tokens comparing the logits of
every step and asserting its launch count, and compares both KV caches at the end.  Then: one mixed model's session features (embeddings, greedy
infer_next_token, one perplexity chunk, a snapshot round trip), the K-quant mat-mul at the 7B shapes and at ragged N, and the refusals."""
import ctypes as C

import numpy as np
import pytest

import llm_b200
from llm_b200 import _lib, loader
from oracle import bindings as B
from oracle import kquant as KQ
from oracle import synth

pytestmark = pytest.mark.gpu

PREFILL = (7, 40, 100)
DECODE = 5
TINY = dict(n_vocab=512, n_embd=256, n_head=4, n_head_kv=4, n_layer=2, n_ff=768, n_rot=64, n_ctx=256)
GQA = dict(n_vocab=512, n_embd=1024, n_head=8, n_head_kv=2, n_layer=2, n_ff=1024, n_rot=128, n_ctx=256)
CASES = {"q4_0": (TINY, "q4_0", None), "q4_K_M": (TINY, "q4_K_M", None), "q5_K_M": (TINY, "q5_K_M", None), "q3_K_M": (TINY, "q3_K_M", None),
         "q6_K": (TINY, "q6_K", None), "q2_K": (TINY, "q2_K", None), "gqa-q4_K_M": (GQA, "q4_K_M", None),
         "q4_0-wv-q8_0": (TINY, "q4_0", {f"layers.{i}.attention.wv.weight": B.Q8_0 for i in range(TINY["n_layer"])})}


def check(g, c, what):
    g = np.asarray(g, np.float32)
    c = np.asarray(c, np.float32).reshape(g.shape)
    bad = g.view(np.uint32) != c.view(np.uint32)
    assert not bad.any(), (what, int(bad.sum()), g.size, int(np.argmax(bad.ravel())), float(np.abs(g - c).max()))


@pytest.fixture(scope="module")
def rkq():
    if not KQ.have_ref_kq():
        pytest.skip("oracle/_ref/libggml_ref_kq.so not built")
    return KQ.RefKq()


def write_and_load(tmp_path, hp, tensors, types, mix):
    """the GGJT v3 file of the model, loaded by b200_llama_load_file (GQA: the _gqa form with ModelParameters::n_gqa)"""
    path = str(tmp_path / f"{mix}.ggjt")
    loader.write_llama(path, hp, tensors, synth.tensor_shapes(hp), tensor_types=types, llama_ftype=KQ.MIXES[mix][1])
    params = llm_b200.ModelParameters(context_size=hp["n_ctx"])
    n_gqa = hp["n_head"] // hp["n_head_kv"]
    if n_gqa == 1:
        return loader.load(path, params)
    L = _lib.lib()
    err = C.c_int(0)
    h = L.b200_llama_load_file_lora(path.encode(), hp["n_ctx"], 0.0, 0.0, n_gqa, None, 0, C.byref(err))
    assert h, err.value
    m = llm_b200.Llama.__new__(llm_b200.Llama)
    m.L, m.hyperparameters, m.params, m._m, m.vocabulary = L, dict(hp), params, h, None
    return m


def per_op_launches(hp, types):
    split = sum(types[f"layers.{i}.attention.wv.weight"] != types[f"layers.{i}.attention.wq.weight"] for i in range(hp["n_layer"]))
    return 17 * hp["n_layer"] + 4 + 2 * split


def kv_equal(s, cpu):
    for which in (0, 1):
        got = s.kv(which)
        want = np.ascontiguousarray(cpu.kv(which)[:got.size])
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), ("cache", which)


@pytest.mark.parametrize("name", list(CASES))
def test_mixed_file_session(rkq, tmp_path, name):
    base, mix, overrides = CASES[name]
    hp, tens, types = KQ.make_llama_mixed(base, mix, rkq, overrides=overrides)
    m = write_and_load(tmp_path, hp, tens, types, mix)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=128))
    cpu = rkq.llama_typed(hp, tens, types)
    toks = synth.make_tokens(hp, sum(PREFILL) + DECODE, seed=hp["n_embd"] + hp["wtype"])
    at = 0
    for n in PREFILL:
        check(s.evaluate(toks[at:at + n], all_logits=True), cpu.eval(toks[at:at + n]), f"prefill of {n} at {at}")
        at += n
    layers_classic = all(t == hp["wtype"] for k, t in types.items() if k.startswith("layers.")) and hp["wtype"] not in KQ.KQUANTS
    if layers_classic:                  # the decode graph: the one-type schedule (7 per layer + 3) and one more node for the K-quant lm_head
        assert types["output.weight"] == B.Q6_K
        want = 7 * hp["n_layer"] + 3 + 1
    else:
        want = per_op_launches(hp, types)
    for i in range(at, at + DECODE):
        check(s.evaluate(toks[i:i + 1], all_logits=True), cpu.eval(toks[i:i + 1]), f"decode at n_past {i}")
        assert s.last_launches == want, (i, s.last_launches, want)
    kv_equal(s, cpu)
    s.close(); m.close(); cpu.close()


def test_q6_k_output_graph_is_one_node_longer(rkq):
    """the same Q4_0 model with a Q4_0 and with a Q6_K output.weight: the graph step differs by exactly the one added launch"""
    hp, tens, types = KQ.make_llama_mixed(TINY, "q4_0", rkq)
    counts = {}
    for out_type in (B.Q4_0, B.Q6_K):
        t = dict(types, **{"output.weight": out_type})
        tn = dict(tens, **{"output.weight": KQ.quantize_as(rkq, out_type, synth.make_llama(TINY, B.Q4_0, lambda _, w: w)[1]["output.weight"])})
        m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tn, tensor_types=t)
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=8))
        s.evaluate(np.arange(3, dtype=np.int32))
        s.evaluate(np.array([5], np.int32)); s.evaluate(np.array([6], np.int32))      # the second step replays the captured graph
        counts[out_type] = s.last_launches
        s.close(); m.close()
    assert counts[B.Q4_0] == 7 * hp["n_layer"] + 3 and counts[B.Q6_K] == counts[B.Q4_0] + 1, counts


def test_mixed_session_features(rkq, tmp_path):
    """on a Q4_K_M file: embeddings, greedy infer_next_token, a snapshot round trip, one chunk of perplexity"""
    from oracle import embd as E
    from oracle.ppl import PplOracle
    hp, tens, types = KQ.make_llama_mixed(TINY, "q4_K_M", rkq)
    m = write_and_load(tmp_path, hp, tens, types, "q4_K_M")
    cpu = rkq.llama_typed(hp, tens, types)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64))
    toks = synth.make_tokens(hp, 40, seed=3)
    req = llm_b200.OutputRequest(embeddings=np.empty(0, np.float32))
    g = s.evaluate(toks[:33], all_logits=True, output_request=req)
    want_l, want_e, _ = E.eval_embd(cpu, toks[:33])
    check(g, want_l, "prefill logits"); check(req.embeddings, want_e[-1], "embeddings")
    greedy = llm_b200.InferenceParameters(llm_b200.Sampler(repetition_penalty=1.0, top_k=1))
    rng = llm_b200.Rng(1)
    last = want_l[-1]
    for step in range(3):                                  # top_k = 1: the first id of the largest logit
        tok = s.infer_next_token(greedy, rng)
        assert tok == int(np.argmax(last)), (step, tok)
        last = cpu.eval(np.array([tok], np.int32))[0]
        check(s.last_logits, last, f"infer_next_token step {step}")
    snap = s.get_snapshot()
    r = type(s).from_snapshot(snap, m)
    nxt = toks[33:34]
    check(r.evaluate(nxt, all_logits=True), cpu.eval(nxt), "decode after from_snapshot")
    kv_equal(r, cpu)
    r.close(); s.close()
    por = PplOracle()
    C_ = hp["n_ctx"]
    ptoks = synth.make_tokens(hp, C_ + 8, seed=9)
    sp = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64))
    got_ppl, got_terms = sp.perplexity(ptoks, return_terms=True, bos=1)
    cpu.reset()
    want_ppl, want_terms = por.perplexity(cpu.eval, cpu.reset, ptoks, C_, 64, 1)
    check(got_terms, want_terms, "perplexity terms"); check(got_ppl, want_ppl, "perplexity")
    sp.close()
    m.close(); cpu.close()


def kquantize(ref, t, w):
    return np.stack([ref.from_float(t, row) for row in np.ascontiguousarray(w, np.float32)])


def acts(rng, Bn, K):
    x = (rng.standard_normal((Bn, K)) * rng.uniform(0.05, 8, (Bn, 1))).astype(np.float32)
    if Bn > 2:
        x[1, :256] = 0.0                                   # an all-zero super-block
        x[2] = np.round(x[2] * 4) / 4                      # ties in |x|
        x[2, 5] = -x[2].max(); x[2, 9] = x[2].max()        # equal magnitudes of opposite sign
    return x


@pytest.mark.parametrize("name,t", list(B.KQUANT_TYPES.items()))
@pytest.mark.parametrize("K,N,Bn", [(4096, 4096, 1), (4096, 11008, 1), (11008, 4096, 1), (4096, 32000, 1), (4096, 517, 9), (11008, 259, 17),
                                    (4096, 4096, 2), (4096, 1031, 100), (11008, 259, 33), (4096, 4096, 32), (256, 262147, 1), (256, 262147, 3),
                                    (256, 262147, 40)])
def test_op_mul_mat_kquant_7b_shapes(rkq, name, t, K, N, Bn):
    """through b200_op_mul_mat: the warp kernel (B < 32: decode and short batches) and the tiled GEMM (B >= 32, tiles of 8 rows x 32 tokens:
    100 / 33 / 40 tokens and 1031 / 259 rows leave ragged tiles), at the 7B shapes and past 262140 rows"""
    L = _lib.lib()
    assert L.b200_init(0) == 0
    rng = np.random.default_rng(K + N + Bn + t)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    w[:, :16] *= 8.0
    wq = kquantize(rkq, t, w)
    x = acts(rng, Bn, K)
    want = rkq.mul_mat(t, wq, x, n_threads=16)
    got = np.empty((Bn, N), np.float32)
    assert L.b200_op_mul_mat(t, wq.ctypes.data, K, N, x.ctypes.data, Bn, got.ctypes.data, 0) == 0
    check(got, want, (name, K, N, Bn))


def new_typed(hp, types):
    L = _lib.lib()
    assert L.b200_init(0) == 0
    h = _lib.LlamaHparams(**{k: int(hp[k]) for k in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_rot", "n_ff", "wtype")},
                          context_size=hp["n_ctx"])
    keep = [n.encode() for n in types]
    tab = (_lib.TensorType * len(types))(*[_lib.TensorType(n, t) for n, t in zip(keep, types.values())])
    err = C.c_int(1)
    m = L.b200_llama_new_typed(C.byref(h), tab, len(types), C.byref(err))
    if m:
        L.b200_model_free(m)
    return bool(m), err.value


def test_fast_session_runs_the_exact_kquant_kernels(rkq):
    """B200_SESSION_FAST on a pure K-quant model with an f32 cache (whose attention is exact in FAST sessions too): the same bits and launch
    counts as the default session, prefill and decode"""
    hp, tens, types = KQ.make_llama_mixed(TINY, "q6_K", rkq)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens, tensor_types=types)
    toks = synth.make_tokens(hp, 45, seed=11)
    out = {}
    for flags in (0, 4):                                   # 4: B200_SESSION_FAST
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64, flags=flags, memory_k_type=llm_b200.ModelKVMemoryType.Float32,
                                                            memory_v_type=llm_b200.ModelKVMemoryType.Float32))
        rows = [s.evaluate(toks[:40], all_logits=True)]
        launches = []
        for i in range(40, 45):
            rows.append(s.evaluate(toks[i:i + 1], all_logits=True)); launches.append(s.last_launches)
        out[flags] = (np.concatenate(rows), launches)
        s.close()
    check(out[4][0], out[0][0], "FAST vs default")
    assert out[4][1] == out[0][1]
    m.close()


def test_refusals(rkq, tmp_path):
    L = _lib.lib()
    hp = dict(TINY, wtype=B.Q4_0)
    # nothing is allocated by a refusal: a 7B-wide model refused 8 times leaves the device's free memory where it was (each would take ~300 MB)
    big = dict(n_vocab=32000, n_embd=4096, n_head=32, n_head_kv=32, n_layer=2, n_ff=11008, n_rot=128, n_ctx=256, wtype=B.Q4_0)
    free0 = C.c_size_t(0)
    assert new_typed(big, {"output.weight": B.Q6_K}) == (True, 0)                          # warm: the runtime's own buffers exist
    L.b200_device_info(None, C.byref(free0), None)
    for _ in range(8):
        assert new_typed(big, {"layers.1.attention.wk.weight": B.Q6_K}) == (False, -14)
    free1 = C.c_size_t(0)
    L.b200_device_info(None, C.byref(free1), None)
    assert int(free0.value) - int(free1.value) < (256 << 20), (free0.value, free1.value)
    assert new_typed(hp, {"output.weight": B.Q6_K, "layers.1.feed_forward.w2.weight": B.Q5_K}) == (True, 0)
    assert new_typed(hp, {"layers.0.attention.wk.weight": B.Q4_K}) == (False, -14)        # wk of another type than wq
    assert new_typed(hp, {"layers.1.feed_forward.w3.weight": B.Q6_K}) == (False, -14)     # w3 of another type than w1
    assert new_typed(hp, {"output.weight": B.F32}) == (False, -14)                         # F32 2-D weights stay refused
    assert new_typed(hp, {"output.weight": B.F16}) == (False, -14)                         # F16 beside other types
    assert new_typed(hp, {"layers.2.attention.wq.weight": B.Q4_K}) == (False, -3)          # no layer 2
    assert new_typed(dict(hp, n_ff=704), {"layers.0.feed_forward.w2.weight": B.Q4_K}) == (False, -13)   # ne0 = 704: not whole super-blocks
    h = _lib.LlamaHparams(**{k: int(hp[k]) for k in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_rot", "n_ff")}, wtype=B.Q4_K,
                          context_size=hp["n_ctx"])
    assert not L.b200_llama_new_tp(C.byref(h), 0, 2)                                       # K-quants on tensor-parallel shards
    # the file loader: a LoRA adapter onto a K-quant tensor, refused before the model is created
    hp2, tens, types = KQ.make_llama_mixed(TINY, "q4_K_M", rkq)
    path = str(tmp_path / "m.ggjt")
    loader.write_llama(path, hp2, tens, synth.tensor_shapes(hp2), tensor_types=types, llama_ftype=15)
    from oracle import lora
    ad = str(tmp_path / "lora.ggla")
    table, _ = lora.adapter_tensors({"layers.0.attention.wq.weight": (256, 256)}, 4, np.random.default_rng(1))
    lora.write_ggla(ad, 4, 8, table)
    with pytest.raises(loader.LoadError) as e:
        loader.load(path, llm_b200.ModelParameters(context_size=hp2["n_ctx"], lora_adapters=[ad]))
    assert e.value.kind == "UnsupportedElementType"
