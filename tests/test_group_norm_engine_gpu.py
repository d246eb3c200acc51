"""The GroupNorm the engine runs by default (fuse_nodes, keep_nhwc, batch 1, NHWC), end to end, against fp64.

In that configuration a GroupNorm reads its statistics from the current slot of a two-slot ring (engine_run.cpp: fused_groupnorm), filled
by the step before it -- the fp16 tensor-core conv epilogue, the split-K reduce kernel, the per-channel Add of a resnet's time embedding
(osb_channel_add_stats) -- or, when that producer declines, by an atomics pass of its own; then one apply pass (gn_apply_pre_kernel)
normalises and zeroes the other slot.  GroupNorms the ring cannot take run osb_group_norm, and a non-unit per-group affine runs the
unfused op sequence.  The graphs below chain those producers with large-mean inputs (explicit conv biases of mean M, a residual, a
per-channel addend) so that the ring slot changes hands several times in one run.

Each GroupNorm's input and output are extra outputs; the output is compared with fp64 GroupNorm(+SiLU) of the input the engine produced,
under _gn_tol (test_node_kernels_gpu.py).  The kernels of one eager run are read from a torch.profiler trace, so the test fails if the
routing changes instead of passing on another path."""
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from test_node_kernels_gpu import F16, F32, _assert_within, _gn_ref, _gn_tol
from util import run_model

pytestmark = pytest.mark.gpu

MEANS = [0.0, 64.0, 1024.0]     # the mean of the conv biases / addends that feed the GroupNorms (their input spread is O(1))


def _conv(g, x, cout, k, bias_mean, name):
    _, cin, h, w = x.shape
    wt = g.const(g.randn((cout, cin, k, k), std=1.0 / np.sqrt(cin * k * k)), conv_weight=True)
    b = g.const(g.randn((cout,), std=0.5, mean=bias_mean), quantizable=False)
    return g.node("Conv", [x, wt, b], [(1, cout, h, w)], [("dilations", "1,1"), ("group", "1"), ("kernel_shape", f"{k},{k}"),
                                                          ("pads", f"{k // 2},{k // 2},{k // 2},{k // 2}"), ("strides", "1,1")], out_names=[name])


def _group_norm(g, x, groups, silu, name, group_affine=None):
    """The diffusers export of GroupNorm (Reshape -> InstanceNormalization -> Reshape -> Mul -> Add [-> Sigmoid -> Mul]); `group_affine`:
    (scale, bias) of the InstanceNormalization, per group (unit by default).  Returns the output and the fp64 parameters."""
    _, c, h, w = x.shape
    gs, gb = group_affine if group_affine is not None else (np.ones(groups, np.float32), np.zeros(groups, np.float32))
    gamma, beta = g.randn((c, 1, 1), std=0.25, mean=1.0), g.randn((c, 1, 1), std=0.25)
    r = g.node("Reshape", [x, g.i64([0, groups, -1])], [(1, groups, c // groups * h * w)])
    n = g.node("InstanceNormalization", [r, g.const(gs, quantizable=False), g.const(gb, quantizable=False)], [r.shape], [("epsilon", "1e-05")])
    r2 = g.node("Reshape", [n, g.i64([1, c, h, w])], [(1, c, h, w)])
    m = g.node("Mul", [r2, g.const(gamma)], [(1, c, h, w)])
    out = g.node("Add", [m, g.const(beta)], [(1, c, h, w)], out_names=None if silu else [name])
    if silu:
        s = g.node("Sigmoid", [out], [out.shape])
        out = g.node("Mul", [out, s], [out.shape], out_names=[name])
    cast = (lambda a: a.astype(np.float16).astype(np.float64)) if g.wdtype == "float16" else (lambda a: a.astype(np.float64))
    return out, dict(G=groups, silu=silu, gamma=cast(gamma.reshape(-1)), beta=cast(beta.reshape(-1)), gs=cast(gs), gb=cast(gb))


def _graph_f16(d, M):
    """Branch A (96 x 96, 320 channels: enough tiles that no conv splits along K) then branch B (8 x 8, split-K sized convs); GroupNorms
    in execution order:
      gn1  conv (bias M) -> GroupNorm + SiLU                               statistics from the tile epilogue
      gn2  conv (bias M) + residual (conv_add, mean 2M) -> GroupNorm         the tile epilogue of the conv + residual
      gn3  conv -> Add t[1, C, 1, 1] (mean M) -> GroupNorm + SiLU            osb_channel_add_stats with the addend
      gn6  conv (bias M) -> GroupNorm with a non-unit group affine           unfused; the epilogue's statistics are dropped (memset)
      gn7  conv (bias M, Cout 256) -> GroupNorm (G 64, cpg 4) + SiLU         the tile epilogue, into the slot gn6 left
      gn4  8 x 8 x 640 -> 1280 conv (bias M) -> GroupNorm (cpg 40)           the split-K reduce kernel
      gn5  8 x 8 x 1280 -> 640 conv (bias M) -> GroupNorm (G 64, cpg 10)     split-K declines (cpg % 4 != 0): the GroupNorm's own pass
    gn5 gathers into the slot gn7 (G 64) used, which gn4 (G 32) cleared only as far as its own 32 groups: the engine zeroes the rest."""
    g = emit.GraphBuilder(d, "float16", seed=int(M) + 1)
    x, y = g.input("xa", (1, 320, 96, 96)), g.input("xb", (1, 640, 8, 8))
    p = {}
    c1 = _conv(g, x, 320, 3, M, "gnin1")
    a1, p["1"] = _group_norm(g, c1, 32, True, "gnout1")
    c2 = _conv(g, a1, 320, 3, M, "conv2")
    s2 = g.node("Add", [c2, c1], [c2.shape], out_names=["gnin2"])
    a2, p["2"] = _group_norm(g, s2, 32, False, "gnout2")
    c3 = _conv(g, a2, 320, 3, 0.0, "conv3")
    s3 = g.node("Add", [c3, g.const(g.randn((1, 320, 1, 1), std=0.5, mean=M))], [c3.shape], out_names=["gnin3"])
    a3, p["3"] = _group_norm(g, s3, 32, True, "gnout3")
    c6 = _conv(g, a3, 320, 3, M, "gnin6")
    aff = (g.randn((32,), std=0.2, mean=1.0), g.randn((32,), std=0.2))
    a6, p["6"] = _group_norm(g, c6, 32, True, "gnout6", group_affine=aff)
    c7 = _conv(g, a6, 256, 3, M, "gnin7")
    _, p["7"] = _group_norm(g, c7, 64, True, "gnout7")
    c4 = _conv(g, y, 1280, 3, M, "gnin4")
    a4, p["4"] = _group_norm(g, c4, 32, False, "gnout4")
    c5 = _conv(g, a4, 640, 3, M, "gnin5")
    _, p["5"] = _group_norm(g, c5, 64, False, "gnout5")
    g.finish()
    rng = np.random.default_rng(int(M) + 3)
    inputs = {"xa": rng.standard_normal((1, 320, 96, 96)).astype(np.float32), "xb": rng.standard_normal((1, 640, 8, 8)).astype(np.float32)}
    return inputs, p


def _graph_f32(d, M):
    """fp32 on both sides of osb_channel_add_stats' limit (C / 4 <= 256): the fp32 conv gathers no statistics, so
      gn1  C = 512:  the GroupNorm's own pass (gn_stats_nhwc_vec_kernel) into the ring slot, then gn_apply_pre_kernel
      gn2  C = 1280: osb_group_norm"""
    g = emit.GraphBuilder(d, "float32", seed=int(M) + 2)
    x = g.input("xa", (1, 512, 16, 16))
    p = {}
    c1 = _conv(g, x, 512, 3, M, "gnin1")
    a1, p["1"] = _group_norm(g, c1, 32, True, "gnout1")
    c2 = _conv(g, a1, 1280, 1, M, "gnin2")
    _, p["2"] = _group_norm(g, c2, 32, False, "gnout2")
    p["2"]["ring"] = False
    g.finish()
    rng = np.random.default_rng(int(M) + 4)
    return {"xa": rng.standard_normal((1, 512, 16, 16)).astype(np.float32)}, p


def _names(p):
    return [f"gnin{k}" for k in p] + [f"gnout{k}" for k in p]


def _check_outputs(out, p, dtype, what):
    """Every GroupNorm's output against fp64 GroupNorm(+SiLU) of the input the engine produced for it.  A group affine (gs, gb) folds into
    the per-channel one: gamma' = gs[g] gamma, beta' = gb[g] gamma + beta.  Bar: _gn_tol."""
    for k, q in p.items():
        xin = np.asarray(out[f"gnin{k}"], np.float64)
        got = np.asarray(out[f"gnout{k}"], np.float64).reshape(-1)
        _, C, H, W = xin.shape
        cpg = C // q["G"]
        gs, gb = np.repeat(q["gs"], cpg), np.repeat(q["gb"], cpg)
        ref, mean, rg = _gn_ref(xin.reshape(-1), 0, C, H * W, q["G"], gs * q["gamma"], gb * q["gamma"] + q["beta"], q["silu"])
        assert np.isfinite(got).all(), f"{what} gn{k}: non-finite output"
        _assert_within(got, ref, _gn_tol(ref, mean, rg, dtype), f"{what} gn{k} (input mean {float(xin.mean()):.4g})")


def _trace_kernels(lib, d, inputs, options, names):
    """Kernel names of one eager run (torch.profiler, CUDA activity), in launch order."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out, m = run_model(lib, d, inputs, options, extra_outputs=names)
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if e.device_type.name == "CUDA"]
    evs.sort(key=lambda e: e.time_range.start)
    return out, [e.name for e in evs]


def _count(kernels, key):
    return sum(1 for k in kernels if key in k)


FP16 = ("use_fp16_arithmetic",)


def _tc_profile(lib, fn):
    """tc launches of fn() as dicts (osb_tc_profile_dump: M N K taps batch split conv ms gflop bm bn kmajor)."""
    import ctypes
    K = ctypes.CDLL(lib)
    keys = ("M", "N", "K", "taps", "batch", "split", "conv", "ms", "gflop", "bm", "bn", "kmajor")
    K.osb_tc_profile(1)
    try:
        r = fn()
        buf = ctypes.create_string_buffer(1 << 16)
        assert K.osb_tc_profile_dump(buf, len(buf)) >= 0
    finally:
        K.osb_tc_profile(0)
    return r, [dict(zip(keys, (float(v) for v in line.split()))) for line in buf.value.decode().splitlines()]


@pytest.fixture(scope="module")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.mark.parametrize("M", MEANS)
def test_group_norm_ring_f16(engine_lib, cuda, M):
    """fp16 chain (_graph_f16), eager: outputs under _gn_tol.  The launch profile (one entry per conv, in graph order) shows branch A's
    convs unsplit and gn4's and gn5's split along K; the trace pins the paths -- six GroupNorms apply ring statistics (one
    gn_apply_pre_kernel each), gn_stats_nhwc_vec_kernel runs once for the time-embedding Add (gn3) and once for every split conv whose
    groups the reduce kernel cannot take (cpg % 4 != 0), a split-K reduce runs per split conv, and osb_group_norm's kernels do not."""
    with tempfile.TemporaryDirectory(prefix="osb200_gn_") as d:
        inputs, p = _graph_f16(d + "/", M)
        names = _names(p)
        (out, kernels), tc = _tc_profile(engine_lib, lambda: _trace_kernels(engine_lib, d, inputs, FP16, names))
        _check_outputs(out, p, F16, f"f16 eager M {M}")
        # the convs in graph order: (Cout, the groups of the GroupNorm whose statistics they may gather, or 0)
        convs = [(320, 32), (320, 32), (320, 0), (320, 0), (256, 64), (1280, 32), (640, 64)]
        assert [int(t["N"]) for t in tc] == [c for c, _ in convs], tc
        split = [int(t["split"]) > 1 for t in tc]
        assert split == [False] * 5 + [True, True], f"branch A unsplit, gn4 / gn5's convs split along K: {tc}"
        own_pass = sum(1 for (c, g), sp in zip(convs, split) if g and sp and (c // g) % 4)
        gn = [k for k in kernels if "gn_" in k]
        assert _count(kernels, "gn_apply_pre_kernel") == 6, gn
        assert _count(kernels, "gn_stats_nhwc_vec_kernel") == 1 + own_pass, gn
        assert _count(kernels, "splitk_reduce_kernel") == sum(split), kernels
        for k in ("gn_fused_nhwc_kernel", "gn_apply_kernel", "gn_stats_nhwc_kernel", "gn_stats_nchw_kernel"):
            assert _count(kernels, k) == 0, f"{k} ran: a GroupNorm left the ring path"


@pytest.mark.parametrize("M", MEANS)
def test_group_norm_ring_f32(engine_lib, cuda, M):
    """fp32 chain (_graph_f32), eager: outputs under _gn_tol; C = 512 takes the ring (one gn_stats_nhwc_vec_kernel + one
    gn_apply_pre_kernel), C = 1280 takes osb_group_norm."""
    with tempfile.TemporaryDirectory(prefix="osb200_gn_") as d:
        inputs, p = _graph_f32(d + "/", M)
        out, kernels = _trace_kernels(engine_lib, d, inputs, (), _names(p))
        _check_outputs(out, p, F32, f"f32 eager M {M}")
        assert _count(kernels, "gn_apply_pre_kernel") == 1, [k for k in kernels if "gn_" in k]
        assert _count(kernels, "gn_stats_nhwc_vec_kernel") == 1, [k for k in kernels if "gn_" in k]
        assert _count(kernels, "gn_fused_nhwc_kernel") + _count(kernels, "gn_apply_kernel") >= 1, [k for k in kernels if "gn_" in k]


@pytest.mark.parametrize("dtype", [F16, F32])
def test_group_norm_ring_graph_replays(engine_lib, cuda, dtype):
    """Resident weights + CUDA graph, five runs: every run is within the bar, and every ring-path GroupNorm (and every GroupNorm input)
    is bit-identical to the first run -- the ring is zeroed at the start of each run and every slot is left zero for the next producer.
    osb_group_norm's fp32 kernels fold channels with fp32 shared-memory atomics in any order, so their outputs are held to the bar only."""
    M = 1024.0
    with tempfile.TemporaryDirectory(prefix="osb200_gn_") as d:
        inputs, p = (_graph_f16 if dtype == F16 else _graph_f32)(d + "/", M)
        names = _names(p)
        from onnxstream_b200.model import Model
        m = Model(engine_lib, 4, "ram+nocache")
        if dtype == F16:
            m.set_option("use_fp16_arithmetic", True)
        m.lib.model_set_option(m.h, b"b200_resident_weights", 1)
        m.lib.model_set_option(m.h, b"b200_cuda_graph", 1)
        for n in names:
            m.add_extra_output(n)
        m.read_file(d + "/model.txt")
        runs = []
        for _ in range(5):
            m.clear_tensors()
            for k, v in inputs.items():
                m.add_tensor(k, v)
            m.run()
            runs.append({n: np.array(m.get_tensor(n)) for n in names})
        assert m.stats()["graph_replays"] >= 1
        for i, r in enumerate(runs):
            _check_outputs(r, p, dtype, f"graph run {i + 1}")
            if i:
                for n in names:
                    if n.startswith("gnout") and not p[n[5:]].get("ring", True):
                        continue
                    assert np.array_equal(r[n], runs[0][n]), f"run {i + 1}: {n} differs from the first run"


@pytest.mark.parametrize("dtype", [F16, F32])
def test_group_norm_unfused_agrees(engine_lib, cuda, dtype):
    """b200_fuse_nodes 0 (every GroupNorm as its op sequence, no ring) against fuse_nodes 1: each within the bar of its own inputs, and
    the two runs' GroupNorm inputs of the first producer (the same conv on the same input) identical."""
    M = 64.0
    with tempfile.TemporaryDirectory(prefix="osb200_gn_") as d:
        inputs, p = (_graph_f16 if dtype == F16 else _graph_f32)(d + "/", M)
        opts = FP16 if dtype == F16 else ()
        a, _ = run_model(engine_lib, d, inputs, opts, extra_outputs=_names(p), b200_options=(("b200_fuse_nodes", 1),))
        b, _ = run_model(engine_lib, d, inputs, opts, extra_outputs=_names(p), b200_options=(("b200_fuse_nodes", 0),))
        _check_outputs(a, p, dtype, "fuse_nodes 1")
        _check_outputs(b, p, dtype, "fuse_nodes 0")
        assert np.array_equal(a["gnin1"], b["gnin1"])
