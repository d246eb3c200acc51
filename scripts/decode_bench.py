#!/usr/bin/env python
"""scripts/decode_bench.py -- the TinyLlama-1.1B-shaped decode step (2047 cached positions, fp16 blobs) on the GPU, set up as bench.py's
tinyllama_decode workload: resident weights, the KV cache pushed once and kept in HBM, one captured CUDA graph per step, only the logits
read back.  --f32: fp32 arithmetic (llm.cpp --no-fp16): the decode GEMVs read the fp16 weights in place and widen them in registers.

With --parent-lib (another build of libonnxstream_b200.so, e.g. the parent commit's), both builds run in one process, their timed windows
alternated, and the logits of the two builds on the same seeded inputs are compared.

Prints ONE JSON line: the card (name, power limit, max and current SM clock, read with an nvidia-smi query in this process), then per build
  tokens_per_s      : steps over the device time (CUDA events) of --steps graph replays, median over --rounds windows (min / max too)
  hbm_gb_s          : algorithmic bytes over the step time -- every weight blob once as stored (fp16) plus every graph input once at the
                      activation type (the KV cache of fp32 arithmetic is fp32), as bench.py counts a decode step
  weight_resident_bytes : the engine's HBM weight cache after the first run
and max_rel_logits_diff = max |logits_new - logits_parent| / max |logits_parent|.  Needs a CUDA device; the model goes to a temporary
directory.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onnxstream_b200 import emit  # noqa: E402
from onnxstream_b200.model import ENGINE_LIB, Model  # noqa: E402

UPCAST = ("layernorm", "/norm/")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, max_clock, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": max_clock, "sm_clock": clock}


def make_model(lib, d, f32):
    m = Model(lib, 0, "ram+nocache")
    for o in ("use_scaled_dp_attn_op",) + (() if f32 else ("use_fp16_arithmetic",)):
        m.set_option(o, True)
    for p in UPCAST:
        m.add_upcast_pattern(p)
    for key in ("b200_resident_weights", "b200_cuda_graph", "b200_keep_inputs", "b200_drop_unconverted_outputs"):
        m.lib.model_set_option(m.h, key.encode(), 1)
    m.lib.model_ext_add_output_convert(m.h, b"logits")
    m.read_file(d + "model.txt")
    return m


def step(m, inputs):
    m.clear_tensors()
    for k, v in inputs.items():
        m.add_tensor(k, v)
    m.run()
    return m.get_tensor("logits")


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--f32", action="store_true", help="fp32 arithmetic (no use_fp16_arithmetic)")
    ap.add_argument("--parent-lib", default=None, help="a second build of libonnxstream_b200.so to alternate with")
    ap.add_argument("--steps", type=int, default=200, help="graph replays per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="timed windows per build (alternated between the builds)")
    ap.add_argument("--warmup", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("decode_bench.py needs a CUDA device")
    cfg = emit.LlamaConfig()
    d = tempfile.mkdtemp(prefix="osb200_decode_") + "/"
    try:
        g = emit.emit_llama_decode(d, cfg, "float16")
        inputs = emit.llama_inputs(cfg)
        later = {k: v for k, v in inputs.items() if not k.startswith("pkv")}
        act = 4 if a.f32 else 2
        algo = g.weight_bytes + sum(int(v.size) * (act if v.dtype == np.float32 else v.itemsize) for v in inputs.values())
        libs = {"new": ENGINE_LIB}
        if a.parent_lib:
            libs["parent"] = os.path.abspath(a.parent_lib)
        models, logits, ms = {}, {}, {k: [] for k in libs}
        for tag, lib in libs.items():
            m = make_model(lib, d, a.f32)
            for _ in range(3):      # run 1 fills the weight cache and pushes the KV cache, run 2 warms scratch, run 3 captures
                step(m, inputs)
            for _ in range(3):      # the later input set (KV cache kept in HBM): re-captured once
                step(m, later)
            m.run_resident(a.warmup)
            models[tag] = m
        for _ in range(a.rounds):
            for tag, m in models.items():
                ms[tag].append(m.run_resident(a.steps) / a.steps)
        res = {"card": card(), "dtype": "float32" if a.f32 else "float16", "workload": "TinyLlama-1.1B-shaped decode, %d cached positions, fp16 blobs" % cfg.past,
               "steps": a.steps, "rounds": a.rounds, "algorithmic_bytes_per_step": int(algo)}
        for tag, m in models.items():
            logits[tag] = step(m, later)
            med = float(np.median(ms[tag]))
            res[tag] = {"ms_per_token": round(med, 4), "tokens_per_s": round(1e3 / med, 1), "tokens_per_s_min": round(1e3 / max(ms[tag]), 1),
                        "tokens_per_s_max": round(1e3 / min(ms[tag]), 1), "hbm_gb_s": round(algo / (med * 1e-3) / 1e9, 1),
                        "weight_resident_bytes": int(m.stats()["weight_resident_bytes"])}
        if "parent" in models:
            res["speedup_vs_parent"] = round(res["parent"]["ms_per_token"] / res["new"]["ms_per_token"], 3)
            ref = logits["parent"].astype(np.float64)
            res["max_rel_logits_diff"] = float(np.abs(logits["new"] - ref).max() / max(np.abs(ref).max(), 1e-12))
        for m in models.values():
            m.close()
        print(json.dumps(res))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
