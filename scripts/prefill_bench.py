#!/usr/bin/env python
"""scripts/prefill_bench.py -- prompt prefill on the GPU: the grouped-KV masked flash attention kernel (osb_sdpa_flash) against the
per-row kernel it replaces (osb_attention), and the TinyLlama-1.1B-shaped prefill step end to end with b200_flash_attention on and off.
--f32: the same for fp32 arithmetic -- osb_sdpa_flash_f32x (its three plane splits included) against osb_attention in fp32 (at Tq <= 128
with Tk >= 256 that is the split-KV decode kernel), with short chat turns (Tq 17..128 over Tk 2048) added, and the model step without
use_fp16_arithmetic.

Prints ONE JSON line: the card (name, power limit, max SM clock, read with an nvidia-smi query), then
  kernel: per shape, ms per launch (CUDA events over --iters launches after warm-up) for both kernels, TFLOP/s as 4*Hq*Tq*Tk*d / t
          (masked keys counted), and the max |difference| between the two outputs
  model : per (T, past), prompt tokens/s of one Model::run (device-event time of the run, and host wall time including the logits
          read-back) with the flash route on and off, alternated in one process, and the max relative logits difference
Shapes: TinyLlama (32 / 4 heads, d 64) and Mistral-7B (32 / 8 heads, d 128) at Tq = Tk in {512, 2048} and a chat turn (Tq 128,
Tk 2048), causal masks.  Model level: LlamaConfig() defaults, fp16 weights and arithmetic, resident weights, the KV cache pushed
once and kept in HBM.  Needs a CUDA device; everything it writes goes to a temporary directory.
"""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onnxstream_b200 import emit  # noqa: E402
from onnxstream_b200.model import ENGINE_LIB, Model  # noqa: E402

F16, F32 = 2, 3
KERNEL_SHAPES = [
    # name, Hq, Hkv, Tq, Tk, d
    ("tinyllama_512", 32, 4, 512, 512, 64),
    ("tinyllama_2048", 32, 4, 2048, 2048, 64),
    ("tinyllama_turn_128x2048", 32, 4, 128, 2048, 64),
    ("mistral_512", 32, 8, 512, 512, 128),
    ("mistral_2048", 32, 8, 2048, 2048, 128),
    ("mistral_turn_128x2048", 32, 8, 128, 2048, 128),
]
# fp32 only: short turns, where osb_attention takes its split-KV decode kernel
F32_TURN_SHAPES = [
    ("tinyllama_turn_17x2048", 32, 4, 17, 2048, 64),
    ("tinyllama_turn_32x2048", 32, 4, 32, 2048, 64),
    ("tinyllama_turn_64x2048", 32, 4, 64, 2048, 64),
    ("mistral_turn_17x2048", 32, 8, 17, 2048, 128),
    ("mistral_turn_64x2048", 32, 8, 64, 2048, 128),
]
MODEL_CASES = [(512, 0), (2048, 0), (128, 1920)]     # (new tokens, cached positions)
UPCAST = ("layernorm", "/norm/")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def kernel_level(iters, warmup, f32=False):
    import torch
    lib = ctypes.CDLL(ENGINE_LIB)
    vp, i64, cf, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int
    lib.osb_sdpa_flash.argtypes = [vp] * 5 + [i64] * 5 + [cf, vp]
    lib.osb_sdpa_flash_f32x.argtypes = [vp] * 5 + [i64] * 5 + [cf, vp, vp]
    lib.osb_attention.argtypes = [vp] * 5 + [i64] * 5 + [cf, ci, i64, ci, vp]
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    dt = torch.float32 if f32 else torch.half
    out = []
    for name, Hq, Hkv, Tq, Tk, d in KERNEL_SHAPES + (F32_TURN_SHAPES if f32 else []):
        g = torch.Generator(device="cuda").manual_seed(Hq * Tq + Tk + d)
        q = torch.randn(Hq, Tq, d, device="cuda", generator=g).to(dt)
        k = torch.randn(Hkv, Tk, d, device="cuda", generator=g).to(dt)
        v = torch.randn(Hkv, Tk, d, device="cuda", generator=g).to(dt)
        past = Tk - Tq
        keep = torch.arange(Tk, device="cuda")[None, :] <= past + torch.arange(Tq, device="cuda")[:, None]
        mask = torch.where(keep, 0.0, -65504.0).to(dt)
        scale = 1.0 / d ** 0.5
        o_new = torch.empty(Hq, Tq, d, device="cuda", dtype=dt)
        o_old = torch.empty_like(o_new)
        planes = torch.empty(3 * (Hq * Tq + 2 * Hkv * Tk) * d, device="cuda", dtype=torch.bfloat16) if f32 else None

        def new():
            if f32:
                assert lib.osb_sdpa_flash_f32x(q.data_ptr(), k.data_ptr(), v.data_ptr(), mask.data_ptr(), o_new.data_ptr(), Hq, Hkv, Tq, Tk, d, scale,
                                               planes.data_ptr(), stream) == 0
            else:
                assert lib.osb_sdpa_flash(q.data_ptr(), k.data_ptr(), v.data_ptr(), mask.data_ptr(), o_new.data_ptr(), Hq, Hkv, Tq, Tk, d, scale, stream) == 0

        def old():
            assert lib.osb_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), mask.data_ptr(), o_old.data_ptr(), Hq, Tq, Tk, d, d, scale, 0, Hq // Hkv,
                                     F32 if f32 else F16, stream) == 0

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

        t_new, t_old = timed(new), timed(old)
        flop = 4.0 * Hq * Tq * Tk * d
        out.append({"shape": name, "Hq": Hq, "Hkv": Hkv, "Tq": Tq, "Tk": Tk, "d": d,
                    "flash_ms": round(t_new, 4), "rows_kernel_ms": round(t_old, 4),
                    "flash_tflops": round(flop / t_new / 1e9, 2), "rows_kernel_tflops": round(flop / t_old / 1e9, 3),
                    "speedup": round(t_old / t_new, 1), "max_abs_diff": float((o_new.float() - o_old.float()).abs().max())})
        del q, k, v, mask, o_new, o_old, planes
        torch.cuda.empty_cache()
    return out


def model_level(reps, warmup, f32=False):
    out = []
    for T, past in MODEL_CASES:
        cfg = emit.LlamaConfig(past=past)
        d = tempfile.mkdtemp(prefix="osb200_prefill_") + "/"
        try:
            emit.emit_llama_decode(d, cfg, "float16", new_tokens=T)
            inputs = emit.llama_inputs(cfg, new_tokens=T)
            models = {}
            for flash in (1, 0):
                m = Model(ENGINE_LIB, 0, "ram+nocache")
                for o in ("use_scaled_dp_attn_op",) + (() if f32 else ("use_fp16_arithmetic",)) + (("support_dynamic_shapes",) if past == 0 else ()):
                    m.set_option(o, True)
                for p in UPCAST:
                    m.add_upcast_pattern(p)
                for key, val in (("b200_resident_weights", 1), ("b200_keep_inputs", 1), ("b200_drop_unconverted_outputs", 1), ("b200_flash_attention", flash)):
                    m.lib.model_set_option(m.h, key.encode(), val)
                m.lib.model_ext_add_output_convert(m.h, b"logits")
                m.read_file(d + "model.txt")
                models[flash] = m
            later = {k: v for k, v in inputs.items() if not k.startswith("pkv")}
            logits, gpu_ms, wall_ms = {}, {1: [], 0: []}, {1: [], 0: []}
            for i in range(warmup + reps):
                for flash in (1, 0):
                    m = models[flash]
                    m.clear_tensors()
                    for k, v in (inputs if i == 0 else later).items():
                        m.add_tensor(k, v)
                    t0 = time.perf_counter()
                    m.run()
                    lg = m.get_tensor("logits")
                    t1 = time.perf_counter()
                    if i >= warmup:
                        gpu_ms[flash].append(m.stats()["last_gpu_ms"])
                        wall_ms[flash].append((t1 - t0) * 1e3)
                    logits[flash] = lg
            diff = float(np.abs(logits[1].astype(np.float64) - logits[0]).max() / max(np.abs(logits[0]).max(), 1e-12))
            row = {"T": T, "past": past, "runs": reps}
            for flash, tag in ((1, "flash_on"), (0, "flash_off")):
                g, w = float(np.median(gpu_ms[flash])), float(np.median(wall_ms[flash]))
                row[tag] = {"gpu_ms": round(g, 3), "tokens_per_s_gpu": round(T / g * 1e3, 1), "wall_ms": round(w, 3), "tokens_per_s_wall": round(T / w * 1e3, 1),
                            "gpu_ms_min": round(min(gpu_ms[flash]), 3), "gpu_ms_max": round(max(gpu_ms[flash]), 3)}
            row["speedup_gpu"] = round(row["flash_off"]["gpu_ms"] / row["flash_on"]["gpu_ms"], 2)
            row["max_rel_logits_diff"] = diff
            out.append(row)
            for m in models.values():
                m.close()
        finally:
            shutil.rmtree(d, ignore_errors=True)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=50, help="timed launches per kernel and shape")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5, help="timed model runs per setting (alternated)")
    ap.add_argument("--skip-model", action="store_true")
    ap.add_argument("--f32", action="store_true", help="fp32 arithmetic: osb_sdpa_flash_f32x against osb_attention in fp32, short turns added")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("prefill_bench.py needs a CUDA device")
    res = {"card": card(), "dtype": "float32" if a.f32 else "float16", "kernel": kernel_level(a.iters, a.warmup, a.f32)}
    if not a.skip_model:
        res["model"] = model_level(a.reps, 2, a.f32)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
