"""Text generation on a device-synthesised LLaMA-7B-geometry Q4_0 model: a 512-token prompt, then 128 generated tokens, in tokens per second:

  infer_default   InferenceSession.infer_next_token with the reference's default chain (penalty 1.3 over 64, k 40, p 0.95, T 0.8) on the device
  infer_greedy    the same with k = 1
  evaluate        one-token evaluate steps alone (ids and logits stay in HBM: b200_session_evaluate_device), no sampling
  host            what a user had to do before: evaluate with the last row copied to the host (128 KB), then the chain restated in numpy
  sampler_us      the sampler's own kernels per call (sample_select / sample_merge / sample_tail), summed from a torch.profiler CUDA trace
                  of 64 calls in a run of their own

Each rate is 128 steps from n_past 512 (rewound before each pass), timed with a host clock around work that ends in a stream synchronise,
after one warm-up pass.  The card's name and power limit are read in the same run.  Usage: python tools/generate_bench.py [n_layer]"""
import ctypes as C
import json
import subprocess
import sys
import time

sys.path.insert(0, ".")
import numpy as np  # noqa: E402

import llm_b200  # noqa: E402
from oracle import synth  # noqa: E402

PROMPT, STEPS = 512, 128


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}


def host_chain(row, hist, sp, u):
    """the default chain in numpy on a host row (the cost of the host path; not the device's bits: numpy's exp is not glibc's expf)"""
    x = row.copy()
    ids = np.unique(np.asarray(hist[-sp.repetition_last_n:], np.int64))
    v = x[ids]
    x[ids] = np.where(v <= 0, v * np.float32(sp.repetition_penalty), v / np.float32(sp.repetition_penalty))
    top = np.lexsort((np.arange(x.size), -x))[:sp.top_k]
    vals = x[top]
    e = np.exp(vals - vals[0])
    p = e / e.sum(dtype=np.float32)
    keep = int(np.searchsorted(np.cumsum(p, dtype=np.float32) >= np.float32(sp.top_p), True) + 1)
    t = vals[:keep] / np.float32(sp.temperature)
    w = np.exp(t - t[0])
    c = np.cumsum(w, dtype=np.float32)
    i = int(np.searchsorted(c, np.float32(u) * c[-1], side="right"))
    return int(top[min(i, keep - 1)])


def main():
    n_layer = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    hp = dict(synth.CONFIGS["7b"], n_layer=n_layer, wtype=2)                      # Q4_0
    info = card()
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=2048))
    m.synthesize(0x5EED)
    L = m.L
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=512))
    prompt = synth.make_tokens(hp, PROMPT)
    default = llm_b200.InferenceParameters()
    greedy = llm_b200.InferenceParameters(llm_b200.Sampler(top_k=1))

    def start():
        s.rewind(0)
        s.evaluate(prompt)
        s.sync()

    def infer(params):
        def run():
            rng = llm_b200.Rng(1)
            for _ in range(STEPS):
                s.infer_next_token(params, rng)
        return run

    def evaluate():
        for _ in range(STEPS):
            assert L.b200_session_evaluate_device(s._s, None, 1) == 0

    def host():
        hist = list(prompt)
        logits = np.empty(hp["n_vocab"], np.float32)
        tok = np.empty(1, np.int32)
        sp = default.sampler
        for i in range(STEPS):
            tok[0] = host_chain(s.last_logits if i == 0 else logits, hist, sp, (i * 0.618) % 1.0)
            assert L.b200_session_evaluate(s._s, tok.ctypes.data_as(C.c_void_p), 1, logits.ctypes.data_as(C.c_void_p), 0) == 0
            hist.append(int(tok[0]))

    rates = {}
    for name, fn in (("infer_default", infer(default)), ("infer_greedy", infer(greedy)), ("evaluate", evaluate), ("host", host)):
        best = []
        for rep in range(3):                                                     # the first pass is the warm-up
            start()
            t0 = time.perf_counter()
            fn()
            s.sync()
            if rep:
                best.append(time.perf_counter() - t0)
        rates[name] = round(STEPS / float(np.mean(best)), 2)
    sampler_us = None
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        start()
        rng = llm_b200.Rng(2)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(64):
                s.infer_next_token(default, rng)
            s.sync()
        ks = [e for e in prof.key_averages() if "sample_" in e.key]
        if ks:
            sampler_us = round(sum(getattr(e, "device_time_total", None) or e.cuda_time_total for e in ks) / 64, 2)
    except Exception as e:                                                       # the rates above stand without it
        print(f"generate_bench: no profiler trace ({e})", file=sys.stderr)
    step_us = {k: round(1e6 / v, 1) for k, v in rates.items()}
    print(json.dumps(dict(card=info.get("name"), power_limit=info.get("power.limit"), sm_clock_max=info.get("clocks.max.sm"), n_layer=n_layer,
                          model="LLaMA-7B geometry, Q4_0, device-synthesised", prompt=PROMPT, steps=STEPS, tokens_per_s=rates, step_us=step_us,
                          sampler_us=sampler_us)), flush=True)
    s.close(); m.close()


if __name__ == "__main__":
    main()
