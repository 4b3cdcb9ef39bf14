"""Embeddings (OutputRequest::embeddings), measured on a LLaMA-7B-geometry Q4_0 model (n_embd 4096, 32 layers, n_vocab 32000) synthesized in HBM,
context 2048, f16 cache.  The card's name and power limit are read in the same run.

  decode_ms       the graph decode step from n_past 512: CUDA events around --steps steps (device-resident tokens and logits), best of --reps
  final_norm_us   the decode timeline (B200_DECODE_PROF=1, b200_session_decode_timeline) of single steps: the final norm node, which also stores the
  attn_norm_us    f32 row, beside the per-layer attention-norm nodes of the same steps, which have the same shape and store nothing (medians; a node
                  runs from its griddepcontrol.wait to its last CTA's end)
  feed_prompt_ms  feed_prompt of 512 tokens (one chunk of n_batch 512) from n_past 0, with and without embeddings requested, alternated; host clock
                  around the call, which ends in a device synchronise (min and median of --reps2 each)
Then the reference's embeddings example (crates/llm/examples/embeddings.rs) on a small synthetic model: a query and three comparands, each
evaluated on a fresh session with embeddings requested, ranked by cosine similarity (f32 sums in order, as the example's iterators add).
Usage: python tools/embeddings_bench.py [--steps 64] [--reps 5] [--reps2 10]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["B200_DECODE_PROF"] = "1"        # read when a session starts: only the timeline session below is made before it is cleared

N_LAYER = 32


def card():
    q = "name,power.limit"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), (v.strip() for v in out[0].split(",")))) if out else {}


def model():
    import llm_b200
    hp = dict(n_vocab=32000, n_embd=4096, n_head=32, n_head_kv=32, n_layer=N_LAYER, n_rot=128, n_ff=11008, wtype=llm_b200.Q4_0)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=2048))
    m.synthesize()
    return hp, m


def timeline(m, hp, steps):
    """median duration (us) of the final norm node and of the attention-norm nodes over `steps` single graph steps from n_past 512"""
    import llm_b200
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=512))
    os.environ.pop("B200_DECODE_PROF")
    toks = (np.arange(512 + steps, dtype=np.int32) * 37) % hp["n_vocab"]
    s.evaluate(toks[:512])
    n = 1 + 7 * N_LAYER + 2                                   # get_rows, 7 per layer, the final norm, the lm_head
    out = np.zeros(8 * n, np.uint64)
    p = out.ctypes.data_as(C.c_void_p)
    final, attn = [], []
    for i in range(512, 512 + steps):
        assert s.L.b200_session_decode_timeline(s._s, None, 0, 1) == 0
        s.evaluate(toks[i:i + 1])
        assert s.last_launches == n, s.last_launches
        assert s.L.b200_session_decode_timeline(s._s, p, n, 0) == 0
        dur = (out[n:2 * n].astype(np.int64) - out[:n].astype(np.int64)) / 1e3
        if i > 512:                                           # the first step runs eagerly, later ones replay the graph
            final.append(dur[1 + 7 * N_LAYER])
            attn.extend(dur[1 + 7 * il] for il in range(N_LAYER))
    s.close()
    return dict(final_norm_us=round(float(np.median(final)), 2), attn_norm_us=round(float(np.median(attn)), 2),
                final_norm_p90_us=round(float(np.percentile(final, 90)), 2), attn_norm_p90_us=round(float(np.percentile(attn, 90)), 2))


def decode(m, hp, steps, reps):
    import llm_b200
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=512))
    toks = (np.arange(512 + steps, dtype=np.int32) * 37) % hp["n_vocab"]
    s.evaluate(toks[:512])
    best = None
    for _ in range(reps + 1):                                     # the first pass captures the graphs
        s.rewind(512)
        s.L.b200_timing_begin()
        for _ in range(steps):                                    # the token staged by the last evaluate, read from HBM
            assert s.L.b200_session_evaluate_device(s._s, None, 1) == 0
        ms = s.L.b200_timing_end_ms() / steps
        best = ms if best is None else min(best, ms)
    s.close()
    return dict(decode_ms=round(best, 4), decode_n_past=512, steps=steps)


def feed_prompt(m, hp, reps):
    import llm_b200
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=512))
    toks = (np.arange(512, dtype=np.int32) * 37) % hp["n_vocab"]
    t = {True: [], False: []}
    for r in range(2 * reps + 2):
        want = r % 2 == 0
        s.rewind(0)
        req = llm_b200.OutputRequest(embeddings=np.empty(0, np.float32)) if want else None
        a = time.perf_counter()
        s.feed_prompt(toks, output_request=req)
        b = time.perf_counter()
        if r >= 2:                                                # one warm-up call of each
            t[want].append((b - a) * 1e3)
        if want:
            assert req.embeddings.shape == (hp["n_embd"],) and np.isfinite(req.embeddings).all()
    s.close()
    return {f"feed_prompt_ms_{k}": dict(min=round(min(v), 3), median=round(float(np.median(v)), 3)) for k, v in (("with", t[True]), ("without", t[False]))}


def cosine(a, b):
    """the example's cosine_similarity: dot and magnitudes as f32 sums in order"""
    dot = np.float32(0); ma = np.float32(0); mb = np.float32(0)
    for x, y in zip(a, b):
        dot = np.float32(dot + np.float32(x * y)); ma = np.float32(ma + np.float32(x * x)); mb = np.float32(mb + np.float32(y * y))
    return float(dot / np.float32(np.sqrt(ma) * np.sqrt(mb)))


def example():
    import llm_b200
    from oracle import bindings as B
    from oracle import synth
    orc = B.Oracle()
    hp, tens = synth.make_llama(synth.CONFIGS["gqa8"], B.Q4_0, orc.quantize)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens)
    rng = np.random.default_rng(5)
    query = rng.integers(0, hp["n_vocab"], 9, dtype=np.int32)
    comparands = {"same": query.copy(), "shared prefix": np.concatenate([query[:6], rng.integers(0, hp["n_vocab"], 3, dtype=np.int32)]),
                  "unrelated": rng.integers(0, hp["n_vocab"], 9, dtype=np.int32)}

    def embed(toks):
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64))
        r = llm_b200.OutputRequest(embeddings=np.empty(0, np.float32))
        s.evaluate(toks, output_request=r)
        s.close()
        return r.embeddings

    q = embed(query)
    sims = sorted(((name, cosine(q, embed(t))) for name, t in comparands.items()), key=lambda x: -x[1])
    m.close()
    return dict(n_embd=len(q), similarities=[dict(text=n, score=round(v, 6)) for n, v in sims])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--reps2", type=int, default=10)
    a = ap.parse_args()
    res = dict(card=card())
    hp, m = model()
    res.update(timeline(m, hp, a.steps))
    res.update(decode(m, hp, a.steps, a.reps))
    res.update(feed_prompt(m, hp, a.reps2))
    m.close()
    res["example"] = example()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
