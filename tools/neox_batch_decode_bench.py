"""Batched decode across sessions of one GPT-NeoX-family model (b200_neox_evaluate_sessions) on device-synthesised MPT-7B and GPT-J-6B geometry,
Q4_0, context 1024 -- tools/batch_decode_bench.py's runs for these runtimes:

  batched   n = 1, 2, 4, 8, 16, 32, 64 sessions, each prefilled to n_past 512; one batched step advances all n.  step_ms is the mean of 64 steps
            timed with CUDA events (after 8 warm-up steps, sessions rewound to 512), tokens_per_s = n / step, launches = last_launches, and
            gb_per_s = (weights + n x the KV bytes a step reads at n_past 512) / step, from shapes
  single    one session's graph decode (b200_neox_evaluate_device) over the same 64 positions, for comparison
  profile   device time per batched step by kernel at n = 8 and 64 (torch.profiler, runs of their own)

The card's name and power limit are read in the same run.  Usage: python tools/neox_batch_decode_bench.py [n_layer]"""
import json
import sys

sys.path.insert(0, ".")
sys.path.insert(0, "tools")
import numpy as np  # noqa: E402

from batch_decode_bench import N_CTX, NS, PAST, STEPS, WARM, card, timed  # noqa: E402
from llm_b200 import neox  # noqa: E402
from oracle import alibi as A  # noqa: E402
from oracle import gptj as J  # noqa: E402
from oracle import synth  # noqa: E402

MODELS = {"mpt-7b": (neox.Mpt, A.MPT_CONFIGS["mpt-7b"]), "gptj-6b": (neox.GptJ, J.GPTJ_CONFIGS["gptj-6b"])}


def kv_bytes_read(hp, n_kv):
    return 2 * hp["n_layer"] * n_kv * hp["n_embd"] * 2                         # K and V, f16


def step_profile(m, ss, n, steps=8):
    """device time per batched step of n sessions by kernel (us), from a torch.profiler CUDA trace of `steps` steps in a run of their own"""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
    except Exception as e:
        print(f"neox_batch_decode_bench: no profiler ({e})", file=sys.stderr)
        return None
    for s in ss[:n]:
        s.rewind(PAST)
    toks = np.full(n, 7, np.int32)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            m.evaluate_sessions(ss[:n], toks)
        ss[0].sync()
    rows = sorted(((e.key, getattr(e, "device_time_total", 0) / steps) for e in prof.key_averages()), key=lambda r: -r[1])
    return {k[:90]: round(us, 1) for k, us in rows[:12] if us > 0}


def bench_model(cls, hp, prompt):
    m = cls(hp, context_size=N_CTX)
    m.synthesize(0x5EED)
    L = m.L
    ss = []
    for _ in range(max(NS)):
        s = m.start_session(PAST)
        s.evaluate(prompt)
        ss.append(s)
    rows = []
    for n in NS:
        sub = ss[:n]
        h = m._session_handles(sub)
        toks = np.full(n, 7, np.int32)

        def step():
            assert L.b200_neox_evaluate_sessions(m._m, h, n, toks.ctypes.data, None) == 0
        for s in sub:
            s.rewind(PAST)
        timed(L, step, WARM)
        for s in sub:
            s.rewind(PAST)
        ms = timed(L, step, STEPS)
        nbytes = m.weight_bytes + n * kv_bytes_read(hp, PAST + STEPS // 2)
        rows.append(dict(n=n, step_ms=round(ms, 3), tokens_per_s=round(n / ms * 1e3, 1), launches=sub[0].last_launches,
                         gb_per_s=round(nbytes / ms / 1e6, 1)))
        print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    s = ss[0]

    def single():
        assert L.b200_neox_evaluate_device(s._s, 1) == 0
    s.rewind(PAST)
    timed(L, single, WARM)
    s.rewind(PAST)
    single_ms = timed(L, single, STEPS)
    single = dict(step_ms=round(single_ms, 3), tokens_per_s=round(1e3 / single_ms, 1), launches=s.last_launches)
    profiles = {n: step_profile(m, ss, n) for n in (8, 64)}
    for s in ss:
        s.close()
    m.close()
    return dict(batched=rows, single=single, step_profile_us=profiles)


def main():
    n_layer = int(sys.argv[1]) if len(sys.argv) > 1 else None
    info = card()
    out = dict(card=info.get("name"), power_limit=info.get("power.limit"), sm_clock_max=info.get("clocks.max.sm"), context_size=N_CTX, n_past=PAST,
               steps=STEPS, weights="Q4_0, device-synthesised")
    for name, (cls, cfg) in MODELS.items():
        hp = dict(cfg, wtype=2, n_layer=n_layer or cfg["n_layer"])
        out[name] = dict(n_layer=hp["n_layer"], **bench_model(cls, hp, synth.make_tokens(hp, PAST)))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
