"""Tensor-parallel decode on >= 2 GPUs (torchrun, one process per GPU; skipped on a single-GPU box): logits and the ranks' KV-cache slices are
bit-identical to the CPU oracle -- the row split keeps every dst element one complete vec_dot, and the exchange (peer stores + flags, tp.cuh) only
moves finished values."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

WORKER = textwrap.dedent('''
    import json, os, sys
    sys.path.insert(0, %r)
    import numpy as np
    from oracle import bindings as B
    from oracle import synth
    import llm_b200
    from llm_b200 import tp
    rank, local_rank, world, dist = tp.init_distributed()
    cfg_name, qname, n_steps = os.environ["TP_CFG"], os.environ["TP_QUANT"], int(os.environ["TP_STEPS"])
    orc = B.Oracle()
    base = dict(synth.CONFIGS[cfg_name]) if cfg_name in synth.CONFIGS else json.loads(cfg_name)
    hp, tens = synth.make_llama(base, B.QUANT_TYPES[qname], orc.quantize)
    if os.environ.get("TP_START_CTX"):            # session start only: which context sizes a tensor-parallel session accepts
        started = {}
        for n_ctx in json.loads(os.environ["TP_START_CTX"]):
            m = tp.TpLlama(hp, llm_b200.ModelParameters(context_size=n_ctx), tens, rank=rank, world=world, device=local_rank)
            try:
                m.start_session(llm_b200.InferenceSessionConfig(n_batch=8), dist).close()
                started[n_ctx] = True
            except RuntimeError:
                started[n_ctx] = False
            m.close()
        open(os.path.join(os.environ["RESULT_DIR"], "rank%%d.json" %% rank), "w").write(json.dumps({"rank": rank, "started": started}))
        dist.barrier()
        dist.destroy_process_group()
        sys.exit(0)
    toks = synth.make_tokens(hp, n_steps + 4)
    m = tp.TpLlama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens, rank=rank, world=world, device=local_rank)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=8), dist)
    mo = orc.llama(hp, tens)
    bad = []
    for i in range(n_steps):
        g = s.evaluate(toks[i:i + 1], all_logits=True)
        w = mo.eval(toks[i:i + 1])
        if not np.array_equal(g.view(np.uint32), w.view(np.uint32)):
            bad.append((i, float(np.abs(g - w).max())))
    # a short batch goes through the same token-by-token schedule
    g = s.evaluate(toks[n_steps:n_steps + 3], all_logits=True)
    w = mo.eval(toks[n_steps:n_steps + 3])
    if not np.array_equal(g.view(np.uint32), w.view(np.uint32)):
        bad.append(("batch", float(np.abs(g - w).max())))
    # this rank's slice of the f16 KV cache
    e, nl, n_ctx = hp["n_embd"], hp["n_layer"], hp["n_ctx"]
    gqa = e // (hp["n_head"] // hp["n_head_kv"]); gl = gqa // world
    K = mo.kv(0)[:nl * n_ctx * gqa].reshape(nl, n_ctx, gqa)[:, :, rank * gl:(rank + 1) * gl]
    V = mo.kv(1)[:nl * n_ctx * gqa].reshape(nl, gqa, n_ctx)[:, rank * gl:(rank + 1) * gl, :]
    kv_ok = bool(np.array_equal(s.kv(0).reshape(nl, n_ctx, gl), K) and np.array_equal(s.kv(1).reshape(nl, gl, n_ctx), V))
    out = {"rank": rank, "bad": bad, "kv_ok": kv_ok, "timeouts": s.timeouts, "launches": s.last_launches}
    open(os.path.join(os.environ["RESULT_DIR"], "rank%%d.json" %% rank), "w").write(json.dumps(out))
    dist.barrier()
    s.close(); m.close()
    dist.destroy_process_group()
''') % ROOT


def n_gpus():
    try:
        import ctypes
        n = ctypes.c_int(0)
        return n.value if ctypes.CDLL("libcudart.so").cudaGetDeviceCount(ctypes.byref(n)) else n.value
    except OSError:
        import torch
        return torch.cuda.device_count()


def run_tp(tmp_path, world, cfg, quant, steps, port, start_ctx=None):
    script = tmp_path / "tp_worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, OMP_NUM_THREADS="4", RESULT_DIR=str(tmp_path), TP_CFG=cfg, TP_QUANT=quant, TP_STEPS=str(steps))
    if start_ctx:
        env["TP_START_CTX"] = json.dumps(start_ctx)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                          "--master-port", str(port), str(script)], capture_output=True, text=True, timeout=900, env=env)
    if out.returncode != 0:                                        # keep the workers' own words (pytest truncates long assertion payloads)
        dump = os.path.join(ROOT, "gpurun_out")
        if os.path.isdir(dump):
            open(os.path.join(dump, f"tp_worker_w{world}_{quant}.stderr"), "w").write(out.stderr[-20000:])
    assert out.returncode == 0, out.stderr[-1500:]
    return [json.loads((tmp_path / f"rank{i}.json").read_text()) for i in range(world)]


# every K a multiple of 256 (the streaming mat-vec's granularity), whole heads and 32-row pieces per rank for 2 and 4 ranks; the second one is grouped-query
TP_CFGS = {"mha": dict(n_vocab=1024, n_embd=512, n_head=8, n_head_kv=8, n_layer=3, n_ff=1024, n_rot=64, n_ctx=256),
           "gqa": dict(n_vocab=1024, n_embd=512, n_head=8, n_head_kv=4, n_layer=2, n_ff=1024, n_rot=64, n_ctx=256)}


@pytest.mark.parametrize("world,cfg,quant", [(2, "mha", "q4_0"), (2, "gqa", "q5_1"), (4, "mha", "q8_0"), (8, "mha", "q4_1")])
def test_tensor_parallel_decode_bit_exact(tmp_path, world, cfg, quant):
    if n_gpus() < world:
        pytest.skip(f"needs {world} GPUs")
    res = run_tp(tmp_path, world, json.dumps(TP_CFGS[cfg]), quant, 40, 29530 + world)
    for r in res:
        assert r["bad"] == [] and r["kv_ok"] and r["timeouts"] == 0, r


def test_tensor_parallel_context_limit(tmp_path):
    """the exchange lives in the fused attention kernel, which holds a whole context bucket in shared memory (at most 3264 positions): a
    longer context_size is refused when the session starts instead of aborting the first decode step past n_past 3072"""
    if n_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    res = run_tp(tmp_path, 2, json.dumps(TP_CFGS["mha"]), "q4_0", 0, 29539, start_ctx=[4096, 3264])
    for r in res:
        assert r["started"] == {"4096": False, "3264": True}, r


@pytest.mark.slow
def test_tensor_parallel_13b_geometry_q5_1(tmp_path):
    """BASELINE.json configs[3]: LLaMA-13B geometry (5120 / 40 heads / 13824), Q5_1, 2 layers, 2 GPUs"""
    if n_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    from oracle import synth
    cfg = json.dumps(dict(synth.CONFIGS["13b"], n_layer=2, n_ctx=256))
    res = run_tp(tmp_path, 2, cfg, "q5_1", 12, 29537)
    for r in res:
        assert r["bad"] == [] and r["kv_ok"] and r["timeouts"] == 0, r
