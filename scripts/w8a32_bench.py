#!/usr/bin/env python
"""scripts/w8a32_bench.py -- fp32-arithmetic convolutions and MatMuls on uint8 weights (W8A32, the SDXL base UNet of BASELINE config[2]).

Kernel level: for every distinct uint8 Conv and MatMul shape of the SDXL UNet at a 128x128 latent (and the 64x64 one's), the device time
(CUDA events over --iters launches, windows alternated) of the new route -- the split of x into bf16 planes, the kernel that converts
q - z in shared memory, the fp32 reduce when split -- against the routes the engine took before, on the same fp32 weight (q - z) s:
  conv:   the bf16x6 expansion of x and osb_tc_conv_f32x on a filter expanded beforehand (what a resident model ran)
  MatMul: the bf16x6 expansion of a and osb_tc_gemm_f32x on a weight expanded beforehand, and osb_gemm (the fp32 CUDA-core GEMM the
          attention projections ran)
each with fp32-work TFLOP/s (2 M N K over the time) and the largest difference of the outputs relative to max |out|.

Model level: the SDXL UNet, uint8 weights, fp32 arithmetic, at 64x64 and 128x128 latents, streamed and resident: device time (stats
last_gpu_ms) per step, weight_resident_bytes, act_high_water_bytes and weight_bytes_streamed, the new route against OSB_W8A32_TC=0.  The
switch is read once per process, so each (route, mode) runs in a child process; the children of the two routes alternate, --rounds times,
and their outputs are compared.

Prints ONE JSON line, with the card (name, power limit, SM clocks) read in the same call.  Needs a CUDA device.
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


def emit_models(d):
    """The SDXL UNet with uint8 weights: d/64/model.txt with its weights, and d/128/model.txt, which links to the same weight files (the
    second emit only records the graph text and writes its own int64 shape constants)."""
    dts = {}
    orig = emit.GraphBuilder.const

    def recording(self, arr, name=None, conv_weight=False, quantizable=True, force_dtype=None):
        t = orig(self, arr, name, conv_weight, quantizable, force_dtype)
        dts[t.name] = t.wtype
        return t
    os.makedirs(d + "64"); os.makedirs(d + "128")
    emit.GraphBuilder.const = recording
    try:
        emit.emit_unet(d + "64/", emit.UNetConfig.sdxl(64), "uint8", seed=0)
    finally:
        emit.GraphBuilder.const = orig
    for name, dt in dts.items():
        if dt != "int64":
            f = name.replace("_nchw.bin", "_nhwc.bin")
            os.symlink(os.path.join(d, "64", f), os.path.join(d, "128", f))

    def replay(self, arr, name=None, conv_weight=False, quantizable=True, force_dtype=None):
        base = name or self._uid("w")
        if np.asarray(arr).dtype == np.int64:
            return orig(self, arr, base, conv_weight, quantizable, force_dtype)
        fn = base + ("_nchw.bin" if conv_weight else ".bin")
        return emit.T(fn, tuple(np.asarray(arr).shape), dts[fn])
    saved_randn = emit.GraphBuilder.randn
    emit.GraphBuilder.const, emit.GraphBuilder.randn = replay, lambda self, shape, std=1.0, mean=0.0: np.zeros(shape, np.float32)
    try:
        emit.emit_unet(d + "128/", emit.UNetConfig.sdxl(128), "uint8", seed=0)
    finally:
        emit.GraphBuilder.const, emit.GraphBuilder.randn = orig, saved_randn


def graph_only(latent):
    """The SDXL UNet's graph text alone, for its shapes: zero weights, every one a uint8 blob of scale 1 (nothing is written)."""
    saved = emit.GraphBuilder.randn, emit.quantize_uint8
    emit.GraphBuilder.randn = lambda self, shape, std=1.0, mean=0.0: np.zeros(shape, np.float32)
    emit.quantize_uint8 = lambda a, *args, **kw: (np.zeros(a.shape, np.uint8), 1.0, 0)
    try:
        return emit.emit_unet(None, emit.UNetConfig.sdxl(latent), "uint8", seed=0)
    finally:
        emit.GraphBuilder.randn, emit.quantize_uint8 = saved


def shapes(g):
    """("conv", H, W, Cin, Cout, k, stride) and ("matmul", rows, K, N) of a graph's uint8-weight nodes, without repeats."""
    out = []
    for line in g.lines:
        m = re.match(r"[^:]*:(\w+)\*input:([^*]*)\*", line)
        if not m or ";" not in m.group(2) or "(uint8[" not in m.group(2).split(";")[1]:
            continue
        ins = m.group(2).split(";")
        xs = [int(v) for v in re.search(r"\(([0-9,]*)\)", ins[0]).group(1).split(",")]
        ws = [int(v) for v in re.search(r"\]:([0-9,]*)\)", ins[1]).group(1).split(",") if v]
        if m.group(1) == "Conv":
            s = int(re.search(r"strides:([0-9]+)", line).group(1))
            key = ("conv", xs[2], xs[3], xs[1], ws[0], ws[2], s)
        elif m.group(1) in ("MatMul", "Gemm") and len(ws) == 2 and int(np.prod(xs[:-1])) > 2:
            key = ("matmul", int(np.prod(xs[:-1])), ws[0], ws[1])
        else:
            continue
        if key not in out:
            out.append(key)
    return out


def kernel_level(all_shapes, iters, warmup):
    import torch
    lib = ctypes.CDLL(ENGINE_LIB)
    vp, i64, ci, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    lib.osb_tc_conv_f32x_u8w.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, cf, ci, vp, vp]
    lib.osb_tc_gemm_f32x_u8w.argtypes = [vp, vp, i64, vp, vp, vp, i64, i64, i64, cf, ci, vp, vp]
    lib.osb_tc_conv_f32x_u8w_ok.argtypes = [i64, i64, i64, i64, ci, ci, ci, i64, i64, ci]
    lib.osb_tc_conv_f32x.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, vp]
    lib.osb_tc_conv_f32x_ok.argtypes = [i64, i64, i64, i64, ci, ci, ci, i64, i64]
    lib.osb_tc_gemm_f32x.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, ci, vp]
    lib.osb_tc_gemm_f32x_ok.argtypes = [i64, i64, i64]
    lib.osb_bf16x3_expand_cols.argtypes = [vp, vp, i64, i64, i64, ci, vp]
    lib.osb_bf16x3_expand_rows.argtypes = [vp, vp, i64, i64, ci, vp]
    lib.osb_gemm.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    z, s = 131, 0.0037

    def timed(fn, n):
        for _ in range(warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    out = []
    for sh in all_shapes:
        routes = {}
        if sh[0] == "conv":
            _, H, W, Cin, Cout, k, stv = sh
            p = k // 2
            Ho, Wo = (H + 2 * p - k) // stv + 1, (W + 2 * p - k) // stv + 1
            flops = 2.0 * Ho * Wo * Cout * k * k * Cin
            if not lib.osb_tc_conv_f32x_u8w_ok(H, W, Cin, Cout, k, k, stv, Ho, Wo, z):
                continue
            x = torch.randn(H, W, Cin, device="cuda")
            q = torch.randint(0, 256, (Cout, k, k, Cin), device="cuda", dtype=torch.uint8)
            wf = (q.float() - z) * s
            bias = torch.randn(Cout, device="cuda")
            ys = {r: torch.empty(Ho, Wo, Cout, device="cuda") for r in ("new", "expanded")}
            planes = torch.empty(3 * H * W * Cin, device="cuda", dtype=torch.bfloat16)
            routes["new"] = lambda: lib.osb_tc_conv_f32x_u8w(x.data_ptr(), q.data_ptr(), bias.data_ptr(), None, ys["new"].data_ptr(), H, W, Cin, Cout, k, k, stv,
                                                             p, p, Ho, Wo, s, z, planes.data_ptr(), st)
            if lib.osb_tc_conv_f32x_ok(H, W, Cin, Cout, k, k, stv, Ho, Wo):
                x6 = torch.empty(H * W, 6 * Cin, device="cuda", dtype=torch.bfloat16)
                w6 = torch.empty(Cout * k * k, 6 * Cin, device="cuda", dtype=torch.bfloat16)
                assert lib.osb_bf16x3_expand_cols(wf.data_ptr(), w6.data_ptr(), Cout * k * k, Cin, Cin, 1, st) == 0

                def expanded():
                    lib.osb_bf16x3_expand_cols(x.data_ptr(), x6.data_ptr(), H * W, Cin, Cin, 0, st)
                    return lib.osb_tc_conv_f32x(x6.data_ptr(), w6.data_ptr(), bias.data_ptr(), None, ys["expanded"].data_ptr(), H, W, 6 * Cin, Cout, k, k,
                                                stv, p, p, Ho, Wo, st)
                routes["expanded"] = expanded
        else:
            _, M, Kd, N = sh
            flops = 2.0 * M * N * Kd
            a = torch.randn(M, Kd, device="cuda")
            q = torch.randint(0, 256, (Kd, N), device="cuda", dtype=torch.uint8)
            wf = (q.float() - z) * s
            ys = {r: torch.empty(M, N, device="cuda") for r in ("new", "expanded", "cuda_cores")}
            planes = torch.empty(3 * M * Kd, device="cuda", dtype=torch.bfloat16)
            routes["new"] = lambda: lib.osb_tc_gemm_f32x_u8w(a.data_ptr(), q.data_ptr(), N, ys["new"].data_ptr(), None, None, M, N, Kd, s, z,
                                                             planes.data_ptr(), st)
            if lib.osb_tc_gemm_f32x_ok(M, N, Kd):
                a6 = torch.empty(M, 6 * Kd, device="cuda", dtype=torch.bfloat16)
                b6 = torch.empty(6 * Kd, N, device="cuda", dtype=torch.bfloat16)
                assert lib.osb_bf16x3_expand_rows(wf.data_ptr(), b6.data_ptr(), Kd, N, 1, st) == 0

                def expanded():
                    lib.osb_bf16x3_expand_cols(a.data_ptr(), a6.data_ptr(), M, Kd, Kd, 0, st)
                    return lib.osb_tc_gemm_f32x(a6.data_ptr(), b6.data_ptr(), ys["expanded"].data_ptr(), None, None, M, N, 6 * Kd, 0, st)
                routes["expanded"] = expanded
            routes["cuda_cores"] = lambda: lib.osb_gemm(a.data_ptr(), wf.data_ptr(), ys["cuda_cores"].data_ptr(), None, None, 1, M, N, Kd, 0, 0, 0, 0, OSB_F32,
                                                        0, st)
        for r, fn in routes.items():
            assert fn() == 0, (sh, r)
        torch.cuda.synchronize()
        n = max(3, min(iters, int(1e13 / flops)))
        t = {r: [] for r in routes}
        for _ in range(3):      # alternated windows
            for r, fn in routes.items():
                t[r].append(timed(fn, n))
        row = {"shape": list(sh)}
        ref = ys["expanded"] if "expanded" in routes else ys["cuda_cores"]
        for r in routes:
            ms = float(np.median(t[r]))
            row[r] = {"ms": round(ms, 4), "tflops_fp32_work": round(flops / (ms * 1e-3) / 1e12, 1)}
        for r in routes:
            if r != "new":
                row["speedup_vs_" + r] = round(row[r]["ms"] / row["new"]["ms"], 3)
        row["max_rel_diff"] = float((ys["new"].double() - ref.double()).abs().max() / ref.double().abs().max())
        out.append(row)
        del ys, planes
        torch.cuda.empty_cache()
    return out


def child(model_file, resident, steps):
    """One (route, mode) in this process: 2 warm-up steps, then `steps` timed ones; JSON on stdout, the output saved next to the model."""
    latent = int(os.path.basename(os.path.dirname(model_file)))
    cfg = emit.UNetConfig.sdxl(latent)
    inputs = emit.unet_inputs(cfg, seed=1)
    m = Model(ENGINE_LIB, 0, "ram+nocache")
    if resident:
        m.lib.model_set_option(m.h, b"b200_resident_weights", 1)
    m.read_file(model_file)
    ms = []
    for i in range(2 + steps):
        m.clear_tensors()
        for k, v in inputs.items():
            m.add_tensor(k, v)
        m.run()
        if i >= 2:
            ms.append(float(m.stats()["last_gpu_ms"]))
    out = m.get_tensor("out_5F_sample")
    st = m.stats()
    tag = os.environ.get("OSB_W8A32_TC", "1")
    np.save(f"{model_file}.{int(resident)}.{tag}.npy", out)
    print(json.dumps({"ms": ms, "weight_resident_bytes": int(st["weight_resident_bytes"]), "act_high_water_bytes": int(st["act_high_water_bytes"]),
                      "weight_bytes_streamed": int(st["weight_bytes_streamed"])}))
    m.close()


def model_level(d, rounds, steps, latents):
    res = []
    for latent in latents:
        mf = d + f"{latent}/model.txt"
        for resident in (False, True):
            runs = {"new": [], "old": []}
            stats = {}
            for _ in range(rounds):
                for route, env in (("new", "1"), ("old", "0")):
                    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", mf, "--resident", str(int(resident)), "--steps", str(steps)],
                                       capture_output=True, text=True, env=dict(os.environ, OSB_W8A32_TC=env))
                    if r.returncode != 0:
                        sys.stderr.write(f"{mf} resident={resident} OSB_W8A32_TC={env}:\n" + r.stdout[-2000:] + r.stderr[-4000:])
                        runs[route].append(float("nan"))
                        continue
                    j = json.loads(r.stdout.strip().splitlines()[-1])
                    runs[route] += j["ms"]
                    stats[route] = {k: v for k, v in j.items() if k != "ms"}
            row = {"model": f"sdxl_unet {latent}x{latent} W8A32", "mode": "resident" if resident else "streamed"}
            for route in runs:
                v = runs[route]
                row[route] = {"gpu_ms": round(float(np.median(v)), 1), "gpu_ms_min": round(min(v), 1), "gpu_ms_max": round(max(v), 1), **stats.get(route, {})}
            row["speedup"] = round(row["old"]["gpu_ms"] / row["new"]["gpu_ms"], 3)
            if not all(os.path.exists(f"{mf}.{int(resident)}.{t}.npy") for t in ("1", "0")):
                res.append(row)
                continue
            new, old = (np.load(f"{mf}.{int(resident)}.{t}.npy").astype(np.float64) for t in ("1", "0"))
            row["max_abs_diff"] = float(np.abs(new - old).max())
            row["max_rel_diff"] = float(np.abs(new - old).max() / max(np.abs(old).max(), 1e-12))
            res.append(row)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20, help="timed launches per kernel window (fewer for the largest shapes)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2, help="alternated child processes per route and mode")
    ap.add_argument("--steps", type=int, default=3, help="timed steps per child")
    ap.add_argument("--latents", default="64,128", help="model-level latent sizes")
    ap.add_argument("--skip-kernel", action="store_true")
    ap.add_argument("--skip-model", action="store_true")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--resident", type=int, default=0, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a.child, bool(a.resident), a.steps)
    import torch
    if not torch.cuda.is_available():
        sys.exit("w8a32_bench.py needs a CUDA device")
    res = {"card": card()}
    if not a.skip_kernel:
        res["kernel"] = kernel_level(list(dict.fromkeys(shapes(graph_only(128)) + shapes(graph_only(64)))), a.iters, a.warmup)
    if not a.skip_model:
        d = tempfile.mkdtemp(prefix="osb200_w8a32_") + "/"
        try:
            emit_models(d)
            res["model"] = model_level(d, a.rounds, a.steps, [int(v) for v in a.latents.split(",")])
        finally:
            shutil.rmtree(d, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
