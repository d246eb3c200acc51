#!/usr/bin/env python
"""scripts/tile_bench.py -- the tensor-core GEMM / conv tile shapes at the shapes of one SD 1.5 UNet step (512^2, batch 1, fp16).

Prints ONE JSON line (and, with --table, a readable table on stderr): the card (name, power limit, max SM clock, read with an nvidia-smi
query), then
  shapes   : every distinct tensor-core launch of one eager UNet step (osb_tc_profile_dump under the default rule: M N K taps batch conv
             and the B layout), how often the step runs it, and per candidate the ms per launch (CUDA events around one replay of a CUDA
             graph of --iters launches, after --warmup eager launches: device time, as the engine's graph replay sees it), TF/s
             (2*M*N*K*taps*batch / t) and the (bm, bn, split) the launch ran:
               old   : the previous rule (osb_tc_set_tile(-1, 0, 0): 128 x 128 tiles, split only below 100 tiles and from 32 k-blocks)
               rule  : the default rule (osb_tc_set_tile(0, 0, 0))
               BMxBN : that tile forced, the rule's split for it
             Replays run the shape on fresh Gaussian operands: a GEMM with bias (batch > 1: the grouped q/k/v launch), a conv with bias,
             stride 1, zero padding (kh - 1) / 2 on a square image (the dump does not record the stride: the three stride-2 downsamplers
             run as stride-1 convs of the same output size).
  breakdown: GPU time of one eager UNet step (resident weights, no CUDA graph) under the old rule and under the default rule, by kernel
             family from a torch.profiler trace: tc_gemm_kernel, splitk_reduce, flash attention, GroupNorm / eltwise, other.
OSB_ENGINE_LIB selects the engine library (build variants).  Needs a CUDA device; the model it emits goes to a temporary directory.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onnxstream_b200 import emit  # noqa: E402
from onnxstream_b200.model import ENGINE_LIB, Model  # noqa: E402

F16 = 2
# the instantiated tiles (gemm_wgmma.cu: TC_TILES_KMAJOR, TC_TILES_MNMAJOR)
TILES_KMAJOR = [(128, 128), (128, 64), (128, 80), (128, 160), (64, 64), (64, 128), (64, 160)]
TILES_MNMAJOR = [(128, 128), (128, 64), (64, 128)]
FAMILIES = [("tc_gemm_kernel", r"tc_gemm_kernel"), ("splitk_reduce", r"splitk_reduce"), ("flash", r"flash_attention|f32x_split"),
            ("groupnorm_eltwise", r"gn_|group_norm|layer_norm|unary|binary|geglu|eltwise|softmax|add|silu|copy|transpose|concat|upsample|resize"),
            ("other", r".")]
PROF_KEYS = ("M", "N", "K", "taps", "batch", "split", "conv", "ms", "gflop", "bm", "bn", "kmajor")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def load_lib():
    lib = ctypes.CDLL(ENGINE_LIB)
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.osb_gemm_ld.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_gemm_grouped.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(vp), ci, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_conv2d_ex.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, ci, ci, vp, vp, ci, ctypes.POINTER(ci)]
    lib.osb_tc_set_tile.argtypes = [ci, ci, ci]
    lib.osb_tc_set_tile.restype = None
    lib.osb_tc_profile.argtypes = [ci]
    lib.osb_tc_profile.restype = None
    lib.osb_tc_profile_dump.argtypes = [ctypes.c_char_p, ci]
    return lib


def profile_lines(lib, fn):
    import torch
    torch.cuda.synchronize()
    lib.osb_tc_profile(1)
    try:
        fn()
        torch.cuda.synchronize()
        buf = ctypes.create_string_buffer(1 << 20)
        n = lib.osb_tc_profile_dump(buf, len(buf))
        assert n >= 0
    finally:
        lib.osb_tc_profile(0)
    out = []
    for line in buf.value.decode().splitlines():
        f = line.split()
        out.append({k: (float(v) if k in ("ms", "gflop") else int(v)) for k, v in zip(PROF_KEYS, f)})
    return out


class UNetStep:
    def __init__(self):
        self.cfg = emit.UNetConfig.sd15(64)
        self.dir = tempfile.mkdtemp(prefix="osb200_tile_bench_") + "/"
        emit.emit_unet(self.dir, self.cfg, "float16", seed=0)
        self.inputs = emit.unet_inputs(self.cfg)
        self.m = Model(ENGINE_LIB, 0, "ram+nocache")
        for o in ("use_fp16_arithmetic", "fuse_ops_in_attention"):
            self.m.set_option(o, True)
        self.m.lib.model_set_option(self.m.h, b"b200_resident_weights", 1)
        self.m.lib.model_set_option(self.m.h, b"b200_cuda_graph", 0)
        self.m.read_file(self.dir + "model.txt")

    def step(self):
        self.m.clear_tensors()
        for k, v in self.inputs.items():
            self.m.add_tensor(k, v)
        self.m.run()

    def close(self):
        self.m.close()
        shutil.rmtree(self.dir, ignore_errors=True)


def breakdown(unet, lib, mode, trace_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile
    lib.osb_tc_set_tile(*mode)
    for _ in range(3):
        unet.step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        unet.step()
        torch.cuda.synchronize()
    st = unet.m.stats()
    path = os.path.join(trace_dir, "step_%s.pt.trace.json" % ("old" if mode[0] < 0 else "rule"))
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset")]
    fam = {name: 0.0 for name, _ in FAMILIES}
    count = {name: 0 for name, _ in FAMILIES}
    for e in ev:
        for name, rx in FAMILIES:
            if re.search(rx, e["name"]):
                fam[name] += e["dur"] * 1e-3
                count[name] += 1
                break
    total = sum(fam.values())
    lib.osb_tc_set_tile(0, 0, 0)
    return {"kernel_ms": total, "last_gpu_ms": st.get("last_gpu_ms"), "kernel_launches": int(st["kernel_launches"]),
            "families": {k: {"ms": fam[k], "share": fam[k] / total if total else None, "kernels": count[k]} for k in fam}}


def replay(lib, shape, g):
    """A closure that launches `shape` once on fresh operands."""
    import torch
    M, N, Kd, taps, batch, conv, kmajor = shape
    st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)   # noqa: E731  (the stream at call time: capture)
    h = lambda *s: (torch.randn(*s, device="cuda", generator=g) * 0.1).half()   # noqa: E731
    if conv:
        Ho = Wo = int(round(M ** 0.5))
        assert Ho * Wo == M, shape
        k = int(round(taps ** 0.5))
        x, w, b = h(Ho, Wo, Kd), h(N, k, k, Kd), h(N)
        y = torch.empty(Ho, Wo, N, device="cuda", dtype=torch.half)
        keep = (x, w, b, y)
        pad = (k - 1) // 2
        return lambda: lib.osb_conv2d_ex(x.data_ptr(), w.data_ptr(), b.data_ptr(), None, None, y.data_ptr(), Ho, Wo, Kd, N, k, k, 1, pad, pad, Ho, Wo, F16, 2,
                                         st(), None, 0, None), keep
    a = h(M, Kd)
    if batch > 1:
        ws = [h(N, Kd) if kmajor else h(Kd, N) for _ in range(batch)]
        cs = [torch.empty(M, N, device="cuda", dtype=torch.half) for _ in range(batch)]
        B = (ctypes.c_void_p * batch)(*[t.data_ptr() for t in ws]); C = (ctypes.c_void_p * batch)(*[t.data_ptr() for t in cs])
        return lambda: lib.osb_gemm_grouped(a.data_ptr(), B, C, batch, M, N, Kd, kmajor, F16, 2, st()), (a, ws, cs, B, C)
    w, b = (h(N, Kd) if kmajor else h(Kd, N)), h(N)
    c = torch.empty(M, N, device="cuda", dtype=torch.half)
    ldb = Kd if kmajor else N
    return lambda: lib.osb_gemm_ld(a.data_ptr(), Kd, w.data_ptr(), ldb, c.data_ptr(), N, b.data_ptr(), None, 1, M, N, Kd, 0, 0, 0, kmajor, F16, 2, st()), (a, w, b, c)


def time_launch(fn, iters, warmup, stream):
    """ms per launch on the device: `iters` launches captured into one CUDA graph (so the host's launch cost is not timed, as in the
    engine's graph replay), replayed after `warmup` eager launches and one warm-up replay."""
    import torch
    with torch.cuda.stream(stream):
        for _ in range(warmup):          # also gives the stream its split-K workspace before the capture
            assert fn() == 0
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        for _ in range(iters):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        e0.record()
        graph.replay()
        e1.record()
    torch.cuda.synchronize()
    del graph
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default="", help="also write the JSON result to this file")
    ap.add_argument("--trace-dir", default="", help="keep the torch.profiler traces here (default: a temporary directory)")
    ap.add_argument("--table", action="store_true", help="print a table of the shapes to stderr")
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    lib = load_lib()
    res = {"card": card()}
    unet = UNetStep()
    trace_dir = args.trace_dir or tempfile.mkdtemp(prefix="osb200_tile_trace_")
    os.makedirs(trace_dir, exist_ok=True)
    try:
        lib.osb_tc_set_tile(0, 0, 0)
        unet.step()
        launches = profile_lines(lib, unet.step)
        res["breakdown"] = {"old": breakdown(unet, lib, (-1, 0, 0), trace_dir), "rule": breakdown(unet, lib, (0, 0, 0), trace_dir)}
    finally:
        unet.close()
        if not args.trace_dir:
            shutil.rmtree(trace_dir, ignore_errors=True)
    shapes = {}
    for p in launches:
        key = (p["M"], p["N"], p["K"], p["taps"], p["batch"], p["conv"], p["kmajor"])
        shapes[key] = shapes.get(key, 0) + 1
    g = torch.Generator(device="cuda").manual_seed(0)
    stream = torch.cuda.Stream()
    rows = []
    for key, n in sorted(shapes.items(), key=lambda kv: -kv[0][0] * kv[0][1] * kv[0][2] * kv[0][3] * kv[0][4] * kv[1]):
        M, N, Kd, taps, batch, conv, kmajor = key
        fn, keep = replay(lib, key, g)
        flop = 2.0 * M * N * Kd * taps * batch
        cands = [("old", (-1, 0, 0)), ("rule", (0, 0, 0))] + [("%dx%d" % t, (t[0], t[1], 0)) for t in (TILES_KMAJOR if kmajor else TILES_MNMAJOR)]
        row = {"M": M, "N": N, "K": Kd, "taps": taps, "batch": batch, "conv": conv, "kmajor": kmajor, "per_step": n, "cand": {}}
        for name, mode in cands:
            lib.osb_tc_set_tile(*mode)
            with torch.cuda.stream(stream):
                ran = profile_lines(lib, fn)[0]
            ms = time_launch(fn, args.iters, args.warmup, stream)
            row["cand"][name] = {"ms": ms, "tflops": flop / (ms * 1e-3) / 1e12, "bm": ran["bm"], "bn": ran["bn"], "split": ran["split"]}
        lib.osb_tc_set_tile(0, 0, 0)
        forced = {k: v for k, v in row["cand"].items() if k not in ("old", "rule")}
        best = min(forced, key=lambda k: forced[k]["ms"])
        row["best"] = best
        row["rule_vs_best"] = row["cand"]["rule"]["ms"] / forced[best]["ms"]
        row["old_vs_rule"] = row["cand"]["old"]["ms"] / row["cand"]["rule"]["ms"]
        rows.append(row)
        del keep
    tot_old = sum(r["cand"]["old"]["ms"] * r["per_step"] for r in rows)
    tot_rule = sum(r["cand"]["rule"]["ms"] * r["per_step"] for r in rows)
    tot_best = sum(min(v["ms"] for k, v in r["cand"].items() if k not in ("old", "rule")) * r["per_step"] for r in rows)
    for r in rows:
        r["share_of_tc_time_old"] = r["cand"]["old"]["ms"] * r["per_step"] / tot_old
    res["shapes"] = rows
    res["step_tc_ms"] = {"old": tot_old, "rule": tot_rule, "best_forced": tot_best, "launches": len(launches)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if args.table:
        print("%-34s %5s %7s %7s %7s %-9s %7s %-9s %6s" % ("M x N x K (taps, batch, layout)", "n", "old ms", "rule ms", "best ms", "best", "rule/b",
                                                          "rule", "share"), file=sys.stderr)
        for r in rows:
            c = r["cand"]
            rule = "%dx%d/%d" % (c["rule"]["bm"], c["rule"]["bn"], c["rule"]["split"])
            print("%-34s %5d %7.4f %7.4f %7.4f %-9s %7.3f %-9s %6.3f" % (
                "%dx%dx%d (%d,%d,%s%s)" % (r["M"], r["N"], r["K"], r["taps"], r["batch"], "conv " if r["conv"] else "", "K" if r["kmajor"] else "MN"),
                r["per_step"], c["old"]["ms"], c["rule"]["ms"], c[r["best"]]["ms"], r["best"], r["rule_vs_best"], rule, r["share_of_tc_time_old"]),
                file=sys.stderr)
        print("tensor-core ms per step (sum of replays): old %.3f  rule %.3f  best forced %.3f" % (tot_old, tot_rule, tot_best), file=sys.stderr)


if __name__ == "__main__":
    main()
