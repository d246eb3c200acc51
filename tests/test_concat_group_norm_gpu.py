"""The skip-connection Concat of a UNet up block gathers the statistics of the GroupNorm that reads it (osb_concat2_stats).

The channel Concat of two NHWC images copies them and adds the per-group sums of what it stores into the GroupNorm's ring slot, so that
GroupNorm runs only its apply pass.  The graph puts two such Concats in a row: 640 + 320 channels into 32 groups (cpg 30, group 21
straddles the two sources), then 1280 + 1280 into 64 groups, i.e. a GroupNorm with more groups after one with fewer, with conv biases of
mean M in front.  Each GroupNorm's output is held to fp64 GroupNorm of the input the engine produced (test_group_norm_engine_gpu.py's
bar), and the trace shows no statistics pass of the GroupNorms' own."""
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from kernel_trace import trace_run
from test_group_norm_engine_gpu import FP16, MEANS, _check_outputs, _conv, _count, _group_norm, _names, cuda  # noqa: F401
from test_node_kernels_gpu import F16

pytestmark = pytest.mark.gpu


def _graph(d, M):
    g = emit.GraphBuilder(d, "float16", seed=int(M) + 11)
    xa, xb, xc = g.input("xa", (1, 64, 16, 16)), g.input("xb", (1, 32, 16, 16)), g.input("xc", (1, 64, 16, 16))
    p = {}
    a, b = _conv(g, xa, 640, 3, M, "ca"), _conv(g, xb, 320, 3, -M, "cb")
    c1 = g.node("Concat", [a, b], [(1, 960, 16, 16)], [("axis", "1")], out_names=["gnin1"])
    a1, p["1"] = _group_norm(g, c1, 32, True, "gnout1")
    c, e = _conv(g, a1, 1280, 1, M, "cc"), _conv(g, xc, 1280, 1, 2 * M, "ce")
    c2 = g.node("Concat", [c, e], [(1, 2560, 16, 16)], [("axis", "1")], out_names=["gnin2"])
    _, p["2"] = _group_norm(g, c2, 64, False, "gnout2")
    g.finish()
    rng = np.random.default_rng(int(M) + 5)
    inputs = {k: rng.standard_normal(s).astype(np.float32) for k, s in (("xa", (1, 64, 16, 16)), ("xb", (1, 32, 16, 16)), ("xc", (1, 64, 16, 16)))}
    return inputs, p


@pytest.mark.parametrize("M", MEANS)
def test_concat_group_norm_stats(engine_lib, cuda, M):
    with tempfile.TemporaryDirectory(prefix="osb200_cat_gn_") as d:
        inputs, p = _graph(d + "/", M)
        out, kernels = trace_run(engine_lib, d, inputs, FP16, extra_outputs=_names(p), keep=_names(p))
        _check_outputs(out, p, F16, f"concat M {M}")
        gn = [k for k in kernels if "gn_" in k]
        assert _count(kernels, "gn_apply_pre_kernel") == 2, gn
        # the two Concats gather (the stats kernel in its concatenating instantiation); no GroupNorm runs a statistics pass of its own
        assert _count(kernels, "gn_stats_nhwc_vec_kernel") == _count(kernels, "gn_stats_nhwc_vec_kernel<__half, 8, true>") == 2, gn
        for k in ("gn_fused_nhwc_kernel", "gn_apply_kernel", "gn_stats_nhwc_kernel", "gn_stats_nchw_kernel"):
            assert _count(kernels, k) == 0, f"{k} ran: {gn}"
