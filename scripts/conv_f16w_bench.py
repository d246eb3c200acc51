#!/usr/bin/env python
"""scripts/conv_f16w_bench.py -- fp32-arithmetic convolution on fp16 weights (sd.cpp's fp32 VAE decode and --rpi UNet on fp16 blobs) on the GPU.

Kernel level: for every distinct Conv shape with Cin % 8 == 0 and Cin >= 16 of the SD VAE decoder at 64x64 and 128x128 latents and of the
SD 1.5 UNet at a 64x64 latent, the device
time (CUDA events over --iters launches, windows alternated) of osb_tc_conv_f32x_f16w -- the split of x, the conv that splits the fp16
filter in shared memory, the fp32 reduce when split -- against the route the engine took for that shape before: the bf16x6 expansion of x
and osb_tc_conv_f32x on a filter expanded beforehand where its fp32 output fits the split-K workspace, else the fp32 CUDA-core conv
(osb_conv2d, igemm).  Each with fp32-work TFLOP/s (2 Ho Wo Cout kh kw Cin over the time) and the largest difference of the two outputs.

Model level: the VAE decoder at 64x64 and 128x128 latents and an SD 1.5-shaped UNet (64x64 latent), fp16 blobs, fp32 arithmetic, resident
weights: device time (stats last_gpu_ms) per run, median / min / max over --reps runs, weight_resident_bytes and act_high_water_bytes.
With --parent-lib (another build of libonnxstream_b200.so) both builds run in one process, their runs alternated, and the outputs compared.

Prints ONE JSON line, with the card (name, power limit, SM clocks) read in the same process.  Needs a CUDA device.
"""
import argparse
import ctypes
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onnxstream_b200 import emit  # noqa: E402
from onnxstream_b200.model import ENGINE_LIB, Model  # noqa: E402

OSB_F32 = 3


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, max_clock, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": max_clock, "sm_clock": clock}


def conv_shapes(g):
    """(H, W, Cin, Cout, k, stride) of a graph's Convs with Cin % 8 == 0 and Cin >= 16, in graph order, without repeats (pad k // 2)."""
    out = []
    for line in g.lines:
        if ":Conv*" not in line:
            continue
        _, cin, h, w = (int(v) for v in re.search(r"\*input:[^(]*\(([0-9,]*)\)", line).group(1).split(","))
        cout, _, k, _ = (int(v) for v in re.search(r"\(float16:([0-9,]*)\)", line).group(1).split(","))
        s = int(re.search(r"strides:([0-9]+)", line).group(1))
        if cin % 8 == 0 and cin >= 16 and (h, w, cin, cout, k, s) not in out:
            out.append((h, w, cin, cout, k, s))
    return out


def bench_shapes():
    """("vae 64" / "vae 128" / "unet 64", shape): the VAE decoder at 64x64 and 128x128 latents, the SD 1.5 UNet at 64x64"""
    out = []
    for latent in (64, 128):
        out += [(f"vae {latent}", sh) for sh in conv_shapes(emit.emit_vae_decoder(None, emit.VAEConfig(latent=latent), "float16"))]
    out += [("unet 64", sh) for sh in conv_shapes(emit.emit_unet(None, emit.UNetConfig.sd15(64), "float16"))]
    return out


def kernel_level(iters, warmup):
    import torch
    lib = ctypes.CDLL(ENGINE_LIB)
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.osb_tc_conv_f32x_f16w.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, vp, vp]
    lib.osb_tc_conv_f32x.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, vp]
    lib.osb_tc_conv_f32x_ok.argtypes = [i64, i64, i64, i64, ci, ci, ci, i64, i64]
    lib.osb_bf16x3_expand_cols.argtypes = [vp, vp, i64, i64, i64, ci, vp]
    lib.osb_conv2d.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, ci, ci, vp]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = []
    for model, (H, W, Cin, Cout, k, s) in bench_shapes():
        if any(r["shape"] == [H, W, Cin, Cout, k, s] for r in out):
            continue
        p = k // 2
        Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        x = torch.randn(H, W, Cin, device="cuda")
        w = (torch.randn(Cout, k, k, Cin, device="cuda") * 0.05).half()
        bias = torch.randn(Cout, device="cuda")
        y_new = torch.empty(Ho, Wo, Cout, device="cuda"); y_old = torch.empty(Ho, Wo, Cout, device="cuda")
        planes = torch.empty(3 * H * W * Cin, device="cuda", dtype=torch.bfloat16)
        expanded = bool(lib.osb_tc_conv_f32x_ok(H, W, Cin, Cout, k, k, s, Ho, Wo))

        def new():
            assert lib.osb_tc_conv_f32x_f16w(x.data_ptr(), w.data_ptr(), bias.data_ptr(), None, y_new.data_ptr(), H, W, Cin, Cout, k, k, s, p, p, Ho, Wo,
                                             planes.data_ptr(), st) == 0
        if expanded:
            x6 = torch.empty(H * W, 6 * Cin, device="cuda", dtype=torch.bfloat16)
            w6 = torch.empty(Cout * k * k, 6 * Cin, device="cuda", dtype=torch.bfloat16)
            assert lib.osb_bf16x3_expand_cols(w.float().data_ptr(), w6.data_ptr(), Cout * k * k, Cin, Cin, 1, st) == 0

            def old():
                assert lib.osb_bf16x3_expand_cols(x.data_ptr(), x6.data_ptr(), H * W, Cin, Cin, 0, st) == 0
                assert lib.osb_tc_conv_f32x(x6.data_ptr(), w6.data_ptr(), bias.data_ptr(), None, y_old.data_ptr(), H, W, 6 * Cin, Cout, k, k, s, p, p, Ho, Wo, st) == 0
        else:
            wf = w.float()

            def old():
                assert lib.osb_conv2d(x.data_ptr(), wf.data_ptr(), bias.data_ptr(), None, y_old.data_ptr(), H, W, Cin, Cout, k, k, s, p, p, Ho, Wo, OSB_F32, 0, st) == 0

        flops = 2.0 * Ho * Wo * Cout * k * k * Cin
        n = max(2, min(iters, int(2e13 / flops)))       # about 0.5 s of the slower route per window

        def timed(fn):
            for _ in range(warmup):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / n

        t = {"new": [], "parent_route": []}
        for _ in range(3):      # alternated windows
            t["new"].append(timed(new)); t["parent_route"].append(timed(old))
        row = {"model": model, "shape": [H, W, Cin, Cout, k, s], "parent_route_kind": "bf16x6 tensor cores" if expanded else "fp32 CUDA cores (igemm)"}
        for key, v in t.items():
            ms = float(np.median(v))
            row[key] = {"ms": round(ms, 4), "tflops_fp32_work": round(flops / (ms * 1e-3) / 1e12, 1)}
        row["speedup"] = round(row["parent_route"]["ms"] / row["new"]["ms"], 3)
        row["max_rel_diff"] = float((y_new.double() - y_old.double()).abs().max() / y_old.double().abs().max())
        out.append(row)
        del x, w, y_new, y_old, planes
        if expanded:
            del x6, w6
        torch.cuda.empty_cache()
    return out


def make_model(lib, d):
    m = Model(lib, 0, "ram+nocache")
    m.lib.model_set_option(m.h, b"b200_resident_weights", 1)
    m.read_file(d + "model.txt")
    return m


def run(m, inputs, out_name):
    m.clear_tensors()
    for k, v in inputs.items():
        m.add_tensor(k, v)
    m.run()
    return m.get_tensor(out_name), float(m.stats()["last_gpu_ms"])


def model_level(name, emit_fn, inputs, out_name, parent_lib, reps):
    d = tempfile.mkdtemp(prefix="osb200_cf16w_") + "/"
    res = {"model": name}
    try:
        emit_fn(d)
        libs = {"new": ENGINE_LIB}
        if parent_lib:
            libs["parent"] = os.path.abspath(parent_lib)
        ms = {t: [] for t in libs}
        outs, stats = {}, {}
        models = {t: make_model(lib, d) for t, lib in libs.items()}
        for i in range(2 + reps):
            for t, m in models.items():
                outs[t], g = run(m, inputs, out_name)
                if i >= 2:
                    ms[t].append(g)
        for t, m in models.items():
            st = m.stats()
            stats[t] = {"weight_resident_bytes": int(st["weight_resident_bytes"]), "act_high_water_bytes": int(st["act_high_water_bytes"])}
            m.close()
        for t in libs:
            med = float(np.median(ms[t]))
            res[t] = {"gpu_ms": round(med, 2), "gpu_ms_min": round(min(ms[t]), 2), "gpu_ms_max": round(max(ms[t]), 2), **stats[t]}
        if "parent" in libs:
            ref = outs["parent"].astype(np.float64)
            res["max_abs_diff"] = float(np.abs(outs["new"] - ref).max())
            res["max_rel_diff"] = float(np.abs(outs["new"] - ref).max() / max(np.abs(ref).max(), 1e-12))
            res["speedup_vs_parent"] = round(res["parent"]["gpu_ms"] / res["new"]["gpu_ms"], 3)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20, help="timed launches per kernel window (fewer for the largest shapes)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-kernel", action="store_true")
    ap.add_argument("--skip-model", action="store_true")
    ap.add_argument("--skip-unet", action="store_true")
    ap.add_argument("--reps", type=int, default=5, help="timed runs per build (alternated)")
    ap.add_argument("--parent-lib", default=None, help="a second build of libonnxstream_b200.so to alternate with")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("conv_f16w_bench.py needs a CUDA device")
    res = {"card": card()}
    if not a.skip_kernel:
        res["kernel"] = kernel_level(a.iters, a.warmup)
    if not a.skip_model:
        res["model"] = []
        for L in (64, 128):
            cfg = emit.VAEConfig(latent=L)
            inputs = {"input_2E_1": np.random.default_rng(5).standard_normal((1, 4, L, L)).astype(np.float32)}
            res["model"].append(model_level(f"vae_decoder {L}x{L} -> {8 * L}x{8 * L}", lambda d, cfg=cfg: emit.emit_vae_decoder(d, cfg, "float16"), inputs,
                                            "outsample", a.parent_lib, a.reps))
        if not a.skip_unet:
            ucfg = emit.UNetConfig.sd15(64)
            res["model"].append(model_level("sd15_unet 64x64", lambda d: emit.emit_unet(d, ucfg, "float16", seed=0), emit.unet_inputs(ucfg), "out_5F_sample",
                                            a.parent_lib, a.reps))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
