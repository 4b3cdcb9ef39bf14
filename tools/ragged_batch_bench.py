"""Ragged batched evaluation (b200_model_evaluate_ragged) on a device-synthesised LLaMA-7B model, Q4_0, context 2048.  Each comparison runs both
sides in this process, alternating them REPS times after a warm-up of each; every time is one CUDA-event interval on the backend stream
(b200_timing_begin / end), the median is reported with the spread:

  prefill_16x32    16 sessions x 32-token prompts: feed_prompts (one ragged step of 512 rows, the wgmma GEMM) against 16 feed_prompt calls
                   (32 rows each, the mma.sync GEMM)
  prefill_8x512    8 sessions x 512-token prompts: feed_prompts (one step of 4096 rows) against 8 feed_prompt calls of 512 rows
  mixed            63 sessions at n_past 512 decoding one token and one session prefilling a 256-token chunk: one ragged step against
                   evaluate_sessions(63) followed by one evaluate of 256
  decode           n = 1, 8, 64 sessions at n_past 512: an all-ones ragged step against evaluate_sessions (with --decode-only: evaluate_sessions
                   alone, which runs on builds without the ragged step)

The card's name and power limit are read in the same run.  Usage: python tools/ragged_batch_bench.py [--decode-only] [n_layer]"""
import json
import subprocess
import sys

sys.path.insert(0, ".")
import numpy as np  # noqa: E402

import llm_b200  # noqa: E402
from oracle import synth  # noqa: E402

N_CTX, PAST, REPS = 2048, 512, 5


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}


def timed(L, fn):
    assert L.b200_timing_begin() == 0
    fn()
    return L.b200_timing_end_ms()


def compare(L, sides, reset, reps=REPS):
    """{name: median ms, name_range: [min, max]} of the sides (name -> fn), alternated reps times after one warm-up each; reset() before every run"""
    for fn in sides.values():
        reset()
        fn()
    t = {k: [] for k in sides}
    for _ in range(reps):
        for k, fn in sides.items():
            reset()
            t[k].append(timed(L, fn))
    out = {}
    for k, v in t.items():
        out[k + "_ms"] = round(float(np.median(v)), 3)
        out[k + "_range_ms"] = [round(min(v), 3), round(max(v), 3)]
    return out


def session(m, n_batch):
    return m.start_session(llm_b200.InferenceSessionConfig(n_batch=n_batch))


def prefill(m, n, length, V, seed):
    """n fresh sessions (n_batch = length) and their prompts: feed_prompts against feed_prompt, each from n_past 0"""
    rng = np.random.default_rng(seed)
    ss = [session(m, length) for _ in range(n)]
    prompts = [rng.integers(0, V, length).astype(np.int32) for _ in range(n)]

    def reset():
        for s in ss:
            s.rewind(0)

    def ragged():
        m.feed_prompts(ss, prompts)

    def single():
        for s, p in zip(ss, prompts):
            s.feed_prompt(p)
    r = compare(m.L, dict(ragged=ragged, single=single), reset)
    r["rows"] = n * length
    for s in ss:
        s.close()
    return r


def decode(m, ss, ns, ragged):
    out = []
    L = m.L
    for n in ns:
        sub = ss[:n]
        toks = np.full(n, 7, np.int32)
        chunks = [toks[i:i + 1] for i in range(n)]

        def reset():
            for s in sub:
                s.rewind(PAST)
        sides = dict(evaluate_sessions=lambda: m.evaluate_sessions(sub, toks))
        if ragged:
            sides["ragged"] = lambda: m.evaluate_ragged(sub, chunks)
        r = compare(L, sides, reset, reps=3 * REPS)
        r["n"] = n
        r["launches"] = sub[0].last_launches
        out.append(r)
        print(json.dumps(r), file=sys.stderr, flush=True)
    return out


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    decode_only = "--decode-only" in sys.argv
    n_layer = int(args[0]) if args else 32
    info = card()
    hp = dict(synth.CONFIGS["7b"], n_layer=n_layer, wtype=2)                      # Q4_0
    V = hp["n_vocab"]
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=N_CTX))
    m.synthesize(0x5EED)
    ragged = hasattr(m, "evaluate_ragged")
    prompt = synth.make_tokens(hp, PAST)
    res = dict(card=info.get("name"), power_limit=info.get("power.limit"), sm_clock_max=info.get("clocks.max.sm"), n_layer=n_layer,
               model="LLaMA-7B geometry, Q4_0, device-synthesised", context_size=N_CTX, reps=REPS, ragged_step=ragged)
    # 64 decode sessions at n_past 512 (1 GiB of f16 cache each; n_batch 64 keeps their own activations small): the decode and mixed comparisons
    ss = []
    for _ in range(64):
        s = session(m, 64)
        s.feed_prompt(prompt)
        ss.append(s)
    res["decode"] = decode(m, ss, [1, 8, 64], ragged)
    if ragged and not decode_only:
        pre = session(m, 256)
        chunk = synth.make_tokens(hp, 256)
        dec, toks = ss[:63], np.full(63, 7, np.int32)

        def reset():
            for s in dec:
                s.rewind(PAST)
            pre.rewind(0)

        def mixed():
            m.evaluate_ragged(dec + [pre], [toks[i:i + 1] for i in range(63)] + [chunk])

        def separate():
            m.evaluate_sessions(dec, toks)
            pre.evaluate(chunk)
        res["mixed_63x1_plus_256"] = compare(m.L, dict(ragged=mixed, separate=separate), reset)
        pre.close()
        for s in ss:
            s.close()
        ss = []
        print(json.dumps(res["mixed_63x1_plus_256"]), file=sys.stderr, flush=True)
        res["prefill_16x32"] = prefill(m, 16, 32, V, 1)
        print(json.dumps(res["prefill_16x32"]), file=sys.stderr, flush=True)
        res["prefill_8x512"] = prefill(m, 8, 512, V, 2)
        print(json.dumps(res["prefill_8x512"]), file=sys.stderr, flush=True)
    for s in ss:
        s.close()
    m.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
