#!/usr/bin/env python
"""scripts/prefill_f16w_bench.py -- fp32-arithmetic prefill on fp16 weights (llm.cpp --no-fp16 on fp16 blobs) on the GPU.

Kernel level: for the TinyLlama-1.1B and Mistral-7B prefill projections at M = 2048 and 128, the device time (CUDA events over --iters
launches) of osb_tc_gemm_f32x_f16w -- the split of A, the GEMM that splits the fp16 weight in shared memory, the fp32 reduce -- against the
route it replaces: the bf16x6 expansion of A and osb_tc_gemm_f32x on a weight expanded beforehand (a resident model caches that expansion).
Each with fp32-work TFLOP/s (2 M N K over the time).

Model level: a Llama-shaped prefill of --tokens tokens into an empty cache, fp16 blobs, fp32 arithmetic, resident weights, device time
(stats last_gpu_ms) per run, median / min / max over --reps runs; weight_resident_bytes and act_high_water_bytes from the engine's stats.
--model tinyllama (default) or mistral (32 / 8 heads, d 128, hidden 4096, mlp 14336, vocab 32000; --layers sets the depth).  With
--parent-lib (another build of libonnxstream_b200.so), both builds run in one process, their runs alternated, and the logits compared.
--decode N: after the prefill, N decode steps over the grown cache (kept in HBM), tokens/s from their device time.

Prints ONE JSON line, with the card (name, power limit, SM clocks) read in the same process.  Needs a CUDA device.
"""
import argparse
import ctypes
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
PROJ = [("q/o 2048", 2048, 2048), ("k/v 2048", 2048, 256), ("gate/up 2048", 2048, 5632), ("down 2048", 5632, 2048),
        ("q/o 4096", 4096, 4096), ("k/v 4096", 4096, 1024), ("gate/up 4096", 4096, 14336), ("down 4096", 14336, 4096)]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, max_clock, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": max_clock, "sm_clock": clock}


def kernel_level(iters, warmup):
    import torch
    lib = ctypes.CDLL(ENGINE_LIB)
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.osb_tc_gemm_f32x_f16w.argtypes = [vp, vp, i64, vp, vp, vp, i64, i64, i64, vp, vp]
    lib.osb_bf16x3_expand_cols.argtypes = [vp, vp, i64, i64, i64, ci, vp]
    lib.osb_bf16x3_expand_rows.argtypes = [vp, vp, i64, i64, ci, vp]
    lib.osb_tc_gemm_f32x.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, ci, vp]
    lib.osb_tc_gemm_f32x_ok.argtypes = [i64] * 3
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = []
    for M in (2048, 128):
        for name, Kd, N in PROJ:
            a = torch.randn(M, Kd, device="cuda")
            w = torch.randn(Kd, N, device="cuda").half()
            c_new = torch.empty(M, N, device="cuda"); c_old = torch.empty(M, N, device="cuda")
            planes = torch.empty(3 * M * Kd, device="cuda", dtype=torch.bfloat16)
            a6 = torch.empty(M, 6 * Kd, device="cuda", dtype=torch.bfloat16)
            b6 = torch.empty(6 * Kd, N, device="cuda", dtype=torch.bfloat16)
            assert lib.osb_bf16x3_expand_rows(w.float().data_ptr(), b6.data_ptr(), Kd, N, 1, st) == 0

            def new():
                assert lib.osb_tc_gemm_f32x_f16w(a.data_ptr(), w.data_ptr(), N, c_new.data_ptr(), None, None, M, N, Kd, planes.data_ptr(), st) == 0

            def old():
                assert lib.osb_bf16x3_expand_cols(a.data_ptr(), a6.data_ptr(), M, Kd, Kd, 0, st) == 0
                assert lib.osb_tc_gemm_f32x(a6.data_ptr(), b6.data_ptr(), c_old.data_ptr(), None, None, M, N, 6 * Kd, 0, st) == 0

            def timed(fn):
                for _ in range(warmup):
                    fn()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1) / iters

            row = {"shape": name, "M": M, "K": Kd, "N": N}
            if not lib.osb_tc_gemm_f32x_ok(M, N, Kd):
                # the fp32 partials of the expanded route exceed the split-K workspace: the engine ran the CUDA-core GEMM there
                row["parent_route"] = "not supported (M N fp32 partials exceed the workspace)"
                row["new"] = {"ms": round(timed(new), 4)}
                row["new"]["tflops_fp32_work"] = round(2.0 * M * N * Kd / (row["new"]["ms"] * 1e-3) / 1e12, 1)
                out.append(row)
                continue
            t = {"new": [], "parent_route": []}
            for _ in range(3):      # alternated windows
                t["new"].append(timed(new)); t["parent_route"].append(timed(old))
            flops = 2.0 * M * N * Kd
            for k, v in t.items():
                ms = float(np.median(v))
                row[k] = {"ms": round(ms, 4), "tflops_fp32_work": round(flops / (ms * 1e-3) / 1e12, 1)}
            row["speedup"] = round(row["parent_route"]["ms"] / row["new"]["ms"], 3)
            row["max_rel_diff"] = float((c_new.double() - c_old.double()).abs().max() / c_old.double().abs().max())
            # bound: the tensor-core work of the five bf16 products at 989 TFLOP/s against the bytes of A (fp32), B (fp16) and C (fp32) at 3.35 TB/s
            t_mma = 5 * flops / 989e12; t_mem = (4.0 * M * Kd + 2.0 * Kd * N + 4.0 * M * N) / 3.35e12
            row["bound"] = "tensor-core (bf16)" if t_mma > t_mem else "HBM"
            out.append(row)
    return out


def make_model(lib, d, decode=False):
    m = Model(lib, 0, "ram+nocache")
    for o in ("use_scaled_dp_attn_op",) + (() if decode else ("support_dynamic_shapes",)):
        m.set_option(o, True)
    for p in UPCAST:
        m.add_upcast_pattern(p)
    for key in ("b200_resident_weights", "b200_keep_inputs", "b200_drop_unconverted_outputs"):
        m.lib.model_set_option(m.h, key.encode(), 1)
    m.lib.model_ext_add_output_convert(m.h, b"logits")
    m.read_file(d + "model.txt")
    return m


def run(m, inputs):
    m.clear_tensors()
    for k, v in inputs.items():
        m.add_tensor(k, v)
    m.run()
    return m.get_tensor("logits"), float(m.stats()["last_gpu_ms"])


def model_level(a):
    if a.model == "mistral":
        cfg = emit.LlamaConfig(vocab=32000, hidden=4096, heads=32, kv_heads=8, head_dim=128, mlp=14336, layers=a.layers or 32, past=0, max_pos=a.tokens + a.decode + 1)
    else:
        cfg = emit.LlamaConfig(past=0, max_pos=max(2048, a.tokens + a.decode + 1), **({"layers": a.layers} if a.layers else {}))
    T = a.tokens
    d = tempfile.mkdtemp(prefix="osb200_pf16w_") + "/"
    res = {"model": a.model, "layers": cfg.layers, "tokens": T}
    try:
        emit.emit_llama_decode(d, cfg, "float16", new_tokens=T)
        inputs = emit.llama_inputs(cfg, new_tokens=T)
        libs = {"new": ENGINE_LIB}
        if a.parent_lib:
            libs["parent"] = os.path.abspath(a.parent_lib)
        models = {t: make_model(lib, d) for t, lib in libs.items()}
        ms = {t: [] for t in libs}
        logits = {}
        for i in range(2 + a.reps):
            for t, m in models.items():
                logits[t], g = run(m, inputs)
                if i >= 2:
                    ms[t].append(g)
        for t, m in models.items():
            med = float(np.median(ms[t]))
            st = m.stats()
            res[t] = {"gpu_ms": round(med, 3), "tokens_per_s": round(T / med * 1e3, 1), "tokens_per_s_min": round(T / max(ms[t]) * 1e3, 1),
                      "tokens_per_s_max": round(T / min(ms[t]) * 1e3, 1), "weight_resident_bytes": int(st["weight_resident_bytes"]),
                      "act_high_water_bytes": int(st["act_high_water_bytes"])}
        if "parent" in models:
            ref = logits["parent"].astype(np.float64)
            res["max_rel_logits_diff"] = float(np.abs(logits["new"] - ref).max() / max(np.abs(ref).max(), 1e-12))
            res["speedup_vs_parent"] = round(res["parent"]["gpu_ms"] / res["new"]["gpu_ms"], 3)
        for m in models.values():
            m.close()
        if a.decode:
            # decode steps over the prefilled cache, kept in HBM: the same weights, a single-token graph
            dcfg = emit.LlamaConfig(**{**cfg.__dict__, "past": T})
            dd = tempfile.mkdtemp(prefix="osb200_pf16w_dec_") + "/"
            try:
                emit.emit_llama_decode(dd, dcfg, "float16")
                dinp = emit.llama_inputs(dcfg)
                m = make_model(ENGINE_LIB, dd, decode=True)
                later = {k: v for k, v in dinp.items() if not k.startswith("pkv")}
                run(m, dinp)
                g = [run(m, later)[1] for _ in range(a.decode)]
                st = m.stats()
                res["decode"] = {"past": T, "steps": a.decode, "gpu_ms_median": round(float(np.median(g[1:] or g)), 3),
                                 "tokens_per_s": round(1e3 / float(np.median(g[1:] or g)), 1), "weight_resident_bytes": int(st["weight_resident_bytes"]),
                                 "act_high_water_bytes": int(st["act_high_water_bytes"])}
                m.close()
            finally:
                shutil.rmtree(dd, ignore_errors=True)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20, help="timed launches per kernel window")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-kernel", action="store_true")
    ap.add_argument("--skip-model", action="store_true")
    ap.add_argument("--model", choices=("tinyllama", "mistral"), default="tinyllama")
    ap.add_argument("--layers", type=int, default=0, help="model depth (0: the model's own)")
    ap.add_argument("--tokens", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5, help="timed prefill runs per build (alternated)")
    ap.add_argument("--decode", type=int, default=0, help="decode steps after the prefill (this build only)")
    ap.add_argument("--parent-lib", default=None, help="a second build of libonnxstream_b200.so to alternate with")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("prefill_f16w_bench.py needs a CUDA device")
    res = {"card": card()}
    if not a.skip_kernel:
        res["kernel"] = kernel_level(a.iters, a.warmup)
    if not a.skip_model:
        res["model"] = model_level(a)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
