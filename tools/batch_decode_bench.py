"""Batched decode across sessions of one model (b200_model_evaluate_sessions) on a device-synthesised LLaMA-7B-geometry model, context 1024:

  batched   n = 1, 2, 4, 8, 16, 32, 64 sessions, each prefilled to n_past 512; one batched step advances all n.  step_ms is the mean of 64 steps
            timed with CUDA events (after 8 warm-up steps, sessions rewound to 512), tokens_per_s = n / step, launches = last_launches, and
            gb_per_s = (weights + n x the KV bytes a step reads at n_past 512) / step, from shapes
  single    one session's graph decode (b200_session_evaluate_device) over the same 64 positions, for comparison: n x single_ms is what n
            sessions stepped in turn take
  q4_k_m    the same model as a Q4_K_M mix (Q6_K output) at n = 1 and 8
  profile   device time per batched step by kernel at n = 2, 8 and 64 (torch.profiler, runs of their own)
  sampler   the batched sampler's kernels (sample_*_rows) per call against n single-session samplers (sample_select / merge / tail), summed
            from torch.profiler CUDA traces of 16 calls each, in runs of their own

The card's name and power limit are read in the same run.  Usage: python tools/batch_decode_bench.py [n_layer]"""
import json
import subprocess
import sys

sys.path.insert(0, ".")
import numpy as np  # noqa: E402

import llm_b200  # noqa: E402
from oracle import kquant as KQ  # noqa: E402
from oracle import synth  # noqa: E402

N_CTX, PAST, STEPS, WARM = 1024, 512, 64, 8
NS = [1, 2, 4, 8, 16, 32, 64]


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}


def kv_bytes_read(hp, n_kv):
    gqa = hp["n_embd"] // (hp["n_head"] // hp["n_head_kv"])
    return 2 * hp["n_layer"] * n_kv * gqa * 2                                   # K and V, f16


def timed(L, fn, steps):
    assert L.b200_timing_begin() == 0
    for _ in range(steps):
        fn()
    return L.b200_timing_end_ms() / steps


def bench_model(hp, types, ns, prompt):
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=N_CTX), tensor_types=types)
    m.synthesize(0x5EED)
    L = m.L
    ss = []
    for _ in range(max(ns)):
        s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=PAST))
        s.evaluate(prompt)
        ss.append(s)
    rows = []
    for n in ns:
        sub = ss[:n]
        h = m._session_handles(sub)
        toks = np.full(n, 7, np.int32)

        def step():
            assert L.b200_model_evaluate_sessions(m._m, h, n, toks.ctypes.data, None) == 0
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
        assert L.b200_session_evaluate_device(s._s, None, 1) == 0
    s.rewind(PAST)
    timed(L, single, WARM)
    s.rewind(PAST)
    single_ms = timed(L, single, STEPS)
    single_launches = s.last_launches
    return m, ss, rows, dict(step_ms=round(single_ms, 3), tokens_per_s=round(1e3 / single_ms, 1), launches=single_launches)


def sampler_us(m, ss, n):
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
    except Exception as e:                                                        # the rates stand without it
        print(f"batch_decode_bench: no profiler ({e})", file=sys.stderr)
        return None
    params = llm_b200.InferenceParameters()
    out = {}
    for name in ("batched", "single"):
        for s in ss[:n]:
            s.rewind(PAST)
            s.evaluate([7])
        rngs = [llm_b200.Rng(i) for i in range(n)]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(16):
                if name == "batched":
                    m.infer_next_tokens(ss[:n], params, rngs)
                else:
                    for s, r in zip(ss[:n], rngs):
                        s.infer_next_token(params, r)
            ss[0].sync()
        ks = [e for e in prof.key_averages() if "sample_" in e.key]
        out[name] = round(sum(getattr(e, "device_time_total", 0) for e in ks) / 16, 1)
    return out


def step_profile(m, ss, n, steps=8):
    """device time per batched step of n sessions by kernel (us), from a torch.profiler CUDA trace of `steps` steps in a run of their own"""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
    except Exception as e:
        print(f"batch_decode_bench: no profiler ({e})", file=sys.stderr)
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


def main():
    n_layer = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    info = card()
    hp = dict(synth.CONFIGS["7b"], n_layer=n_layer, wtype=2)                     # Q4_0
    prompt = synth.make_tokens(hp, PAST)
    m, ss, rows, single = bench_model(hp, None, NS, prompt)
    sampler = {n: sampler_us(m, ss, n) for n in (8, 64)}
    profiles = {n: step_profile(m, ss, n) for n in (2, 8, 64)}
    for s in ss:
        s.close()
    m.close()
    hq = dict(hp)
    mk, ssk, rows_k, single_k = bench_model(hq, KQ.mix_types(hq, "q4_K_M"), [1, 8], prompt)
    for s in ssk:
        s.close()
    mk.close()
    print(json.dumps(dict(card=info.get("name"), power_limit=info.get("power.limit"), sm_clock_max=info.get("clocks.max.sm"), n_layer=n_layer,
                          model="LLaMA-7B geometry, Q4_0, device-synthesised", context_size=N_CTX, n_past=PAST, steps=STEPS, batched=rows,
                          single=single, q4_k_m=dict(batched=rows_k, single=single_k), sampler_us=sampler, step_profile_us=profiles)), flush=True)


if __name__ == "__main__":
    main()
