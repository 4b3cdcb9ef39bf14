"""Model files of the GPT-NeoX-family runtime at 7B geometry (GPT-J 6B: 28 layers, n_embd 4096, 50400 logits; MPT-7B: 32 layers, n_embd 4096,
50432 logits):

  load time of llm_b200.load_dynamic for F16 and Q4_0 files, from the page cache (each file is loaded once untimed, then timed)
  decode@1 at n_past 512 and prefill@512 for Q4_0, pure Q4_K and pure Q6_K models (weights synthesised on the device), with launches per step

The files are written to a temporary directory (zero weights: loading does not depend on the values) and removed after their measurement.
The timed quantities end in a device synchronise.  Prints one JSON line per measurement and the GPU's name, power limit and SM clock, read in
the same run.  Usage: python tools/neox_files_bench.py [--layers N] [--steps 32] [--skip-load]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import llm_b200  # noqa: E402
from llm_b200 import loader, neox  # noqa: E402
from oracle import neox_kquant as NK  # noqa: E402
from oracle import synth  # noqa: E402
from tools.kquant_bench import gpu_info  # noqa: E402

GEOM = {"gptj": dict(n_vocab=50400, n_ctx=2048, n_embd=4096, n_head=16, n_layer=28, n_rot=64),
        "mpt": dict(n_vocab=50432, n_ctx=2048, n_embd=4096, n_head=32, n_layer=32, alibi_bias_max=8.0)}
BLOCK = {1: (1, 2), 2: (32, 18)}
CLASS = {"gptj": neox.GptJ, "mpt": neox.Mpt}


def write_zero_file(path, arch, hp, wtype):
    tensors = {}
    for name, shp in NK.tensor_shapes(arch, hp).items():
        if len(shp) == 2:
            blk, nb = BLOCK[wtype]
            tensors[name] = np.zeros(shp, np.float16) if wtype == 1 else np.zeros((shp[0], shp[1] // blk * nb), np.uint8)
        else:
            tensors[name] = np.ones(shp, np.float32)
    header = dict(hp, file_type=1 if wtype == 1 else 2002, max_seq_len=hp["n_ctx"], clip_kqv=0.0)
    loader.write_model(path, arch, header, tensors, NK.tensor_shapes(arch, hp), wtype)
    return os.path.getsize(path)


def load_time(arch, hp, wtype, tmp):
    path = os.path.join(tmp, f"{arch}-{wtype}.bin")
    size = write_zero_file(path, arch, hp, wtype)
    params = llm_b200.ModelParameters(context_size=1024)
    llm_b200.load_dynamic(arch, path, params).close()             # brings the file into the page cache
    t0 = time.perf_counter()
    m = llm_b200.load_dynamic(arch, path, params)
    dt = time.perf_counter() - t0
    m.close()
    os.remove(path)
    return size, dt


def time_session(arch, hp, wtype, steps):
    m = CLASS[arch](dict(hp, wtype=wtype), None, context_size=1024)
    m.synthesize(0x5EED)
    s = m.start_session(n_batch=512)
    toks = synth.make_tokens(dict(hp, n_vocab=hp["n_vocab"]), 512 + steps + 8)
    s.evaluate(toks[:512])                                          # warm-up of the prefill shapes
    s.rewind(0)
    t0 = time.perf_counter(); s.evaluate(toks[:512]); t_pre = time.perf_counter() - t0
    for i in range(4):                                              # warm-up: the first step runs eagerly, the next captures the graph
        s.evaluate(toks[512 + i:513 + i])
    s.rewind(512)
    t0 = time.perf_counter()
    for i in range(steps):
        s.evaluate(toks[512 + i:513 + i])
    t_dec = (time.perf_counter() - t0) / steps
    launches = s.last_launches
    s.close(); m.close()
    return t_pre, t_dec, launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=0, help="layers of both models (default: their own)")
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--skip-load", action="store_true")
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    geom = {arch: dict(GEOM[arch], **({"n_layer": a.layers} if a.layers else {})) for arch in GEOM}
    for arch, hp in geom.items():
        for wtype, tname in ((2, "Q4_0"), (12, "Q4_K"), (14, "Q6_K")):
            t_pre, t_dec, launches = time_session(arch, hp, wtype, a.steps)
            print(json.dumps({"arch": arch, "model": tname, "layers": hp["n_layer"], "prefill512_ms": round(t_pre * 1e3, 2),
                              "decode_at_512_ms": round(t_dec * 1e3, 3), "decode_launches": launches}), flush=True)
    for arch, hp in ({} if a.skip_load else geom).items():
        with tempfile.TemporaryDirectory() as tmp:
            for wtype, tname in ((1, "F16"), (2, "Q4_0")):
                size, dt = load_time(arch, hp, wtype, tmp)
                print(json.dumps({"arch": arch, "file": tname, "layers": hp["n_layer"], "bytes": size, "load_s": round(dt, 3),
                                  "GB_s": round(size / dt / 1e9, 2)}), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
