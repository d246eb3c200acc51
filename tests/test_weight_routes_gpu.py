"""Which kernel reads each static weight, and in what form: the engine's weight-route table, pinned per weight type and run configuration.

One small graph per weight type (float32, float16, uint8) holds every node shape the routes tell apart: MatMul + bias + residual at 1, 2, 4,
16 and 64 activation rows; two decode MatMuls sharing their input at 1 and 4 rows (the planner groups them into one GEMV step), and in the
float16 graph a group whose second weight is float32; a Gemm at 1 and 16 rows; a ragged-N (1003) decode MatMul, which takes the row-padded
copy with resident weights; a conv at a 16 x 16 and at a 128 x 128 output; and one self-attention block (q / k / v projections and the
output projection).  Each configuration runs it once, eagerly, and the kernel trace is reduced to per-family launch counts.  The expected
counts are written out as literal tables, so that a change of route shows up as a diff of a table."""
import os
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit

pytestmark = pytest.mark.gpu

K_IN = 256
N_OUT = 512
N_RAGGED = 1003


def _graph(d, wdtype):
    """The route graph in directory d: its inputs, seeded."""
    g = emit.GraphBuilder(d, wdtype, seed=11)
    rng = np.random.default_rng(12)
    inputs = {}

    def inp(name, shape):
        inputs[name] = rng.standard_normal(shape).astype(np.float32)
        return g.input(name, shape)

    def matmul(x, n, force=None):
        w = g.const(g.randn((x.shape[-1], n), std=1.0 / np.sqrt(x.shape[-1])), force_dtype=force)
        return g.node("MatMul", [x, w], [tuple(x.shape[:-1]) + (n,)])

    outs = []
    for rows in (1, 2, 4, 16, 64):
        x = inp(f"x{rows}", (1, rows, K_IN))
        y = g.linear(x, N_OUT, bias=True)
        outs.append(g.node("Add", [y, inp(f"r{rows}", (1, rows, N_OUT))], [y.shape]))
        if rows in (1, 4):
            outs += [matmul(x, N_OUT), matmul(x, N_OUT)]
    if wdtype == "float16":
        x = inp("xmix", (1, 1, K_IN))
        outs += [matmul(x, N_OUT), matmul(x, N_OUT, force="float32")]
    for rows in (1, 16):
        outs.append(g.gemm(inp(f"g{rows}", (rows, K_IN)), N_OUT))
    outs.append(matmul(inp("xr", (1, 1, K_IN)), N_RAGGED))
    outs.append(g.conv(inp("c16", (1, 16, 16, 16)), 32, 3))
    outs.append(g.conv(inp("c128", (1, 16, 128, 128)), 16, 3))
    xa = inp("xa", (1, 64, 128))
    outs.append(g.attention(xa, xa, heads=2))
    for o in outs:
        g.mark_output(o)
    g.finish()
    return inputs


# kernel family -> a test of the kernel name (torch.profiler's demangled name)
FAMILIES = {
    "f16w_gemm": lambda n: "tc_gemm_f16w_kernel<false>" in n,
    "f16w_conv": lambda n: "tc_gemm_f16w_kernel<true>" in n,
    "u8w_gemm": lambda n: "tc_gemm_u8w_kernel<false>" in n,
    "u8w_conv": lambda n: "tc_gemm_u8w_kernel<true>" in n,
    "gemv_w8": lambda n: "gemv_w8_panel" in n,
    "gemv_f16w": lambda n: "gemv_panel" in n and "<__half, float," in n,
    "gemv": lambda n: "gemv_panel" in n and "<__half, float," not in n,
    "bf16x3": lambda n: "bf16x3_expand" in n,
    "tc_f32x": lambda n: "tc_gemm_kernel" in n,
    "dequant": lambda n: "dequant_kernel" in n,
    "convert": lambda n: "convert_kernel" in n,
    "igemm": lambda n: "igemm_kernel" in n,
}

CONFIGS = {
    "f32": ((), (), {}),
    "f32_resident": ((), (("b200_resident_weights", 1),), {}),
    "f16": (("use_fp16_arithmetic",), (), {}),
    "f16_resident": (("use_fp16_arithmetic",), (("b200_resident_weights", 1),), {}),
    "f32_gemm_impl1": ((), (("b200_gemm_impl", 1),), {}),
    "f32_w8a32_tc_off": ((), (), {"OSB_W8A32_TC": "0"}),
}

RUNS = [(w, c) for w in ("float32", "float16", "uint8") for c in CONFIGS if c != "f32_w8a32_tc_off" or w == "uint8"]

# (weight type, configuration) -> expected launches per family; families not listed launch nothing
EXPECTED = {
    ("float32", "f32"): {"gemv": 6, "bf16x3": 8, "tc_f32x": 4, "igemm": 5},
    ("float32", "f32_resident"): {"gemv": 7, "bf16x3": 8, "tc_f32x": 4, "igemm": 5},
    ("float32", "f16"): {"gemv": 6, "tc_f32x": 5, "convert": 60, "igemm": 2},
    ("float32", "f16_resident"): {"gemv": 7, "tc_f32x": 5, "convert": 60, "igemm": 2},
    ("float32", "f32_gemm_impl1"): {"gemv": 6, "igemm": 11},
    ("float16", "f32"): {"f16w_gemm": 4, "f16w_conv": 1, "gemv_f16w": 5, "gemv": 2, "bf16x3": 2, "tc_f32x": 1, "convert": 18, "igemm": 3},
    ("float16", "f32_resident"): {"f16w_gemm": 4, "f16w_conv": 1, "gemv_f16w": 6, "gemv": 2, "bf16x3": 2, "tc_f32x": 1, "convert": 17, "igemm": 3},
    ("float16", "f16"): {"gemv": 7, "tc_f32x": 5, "convert": 35, "igemm": 2},
    ("float16", "f16_resident"): {"gemv": 8, "tc_f32x": 5, "convert": 35, "igemm": 2},
    ("float16", "f32_gemm_impl1"): {"gemv_f16w": 5, "gemv": 2, "convert": 23, "igemm": 11},
    ("uint8", "f32"): {"u8w_gemm": 10, "u8w_conv": 2, "gemv_w8": 3, "gemv": 1, "dequant": 11},
    ("uint8", "f32_resident"): {"u8w_gemm": 10, "u8w_conv": 2, "gemv_w8": 3, "gemv": 2, "dequant": 11},
    ("uint8", "f16"): {"gemv_w8": 3, "gemv": 4, "tc_f32x": 5, "dequant": 23, "convert": 33, "igemm": 2},
    ("uint8", "f16_resident"): {"gemv_w8": 3, "gemv": 5, "tc_f32x": 5, "dequant": 23, "convert": 33, "igemm": 2},
    ("uint8", "f32_gemm_impl1"): {"gemv_w8": 3, "gemv": 4, "dequant": 23, "igemm": 11},
    ("uint8", "f32_w8a32_tc_off"): {"gemv_w8": 3, "gemv": 4, "bf16x3": 8, "tc_f32x": 4, "dequant": 23, "igemm": 5},
}


def counts(names):
    """Per-family launch counts of a kernel trace (families with none left out)."""
    c = {f: sum(map(test, names)) for f, test in FAMILIES.items()}
    return {f: n for f, n in c.items() if n}


@pytest.fixture(scope="module")
def graphs():
    with tempfile.TemporaryDirectory(prefix="osb200_routes_") as root:
        out = {}
        for w in ("float32", "float16", "uint8"):
            d = os.path.join(root, w) + "/"
            os.makedirs(d)
            out[w] = (d, _graph(d, w))
        yield out


def trace(lib, graphs, wdtype, config):
    """The kernel names of one eager run of the route graph of `wdtype` under `config` (its environment switches already set)."""
    from kernel_trace import trace_run
    options, b200, _ = CONFIGS[config]
    d, inputs = graphs[wdtype]
    return trace_run(lib, d, inputs, options, wp="ram+nocache", b200_options=b200)[1]


@pytest.mark.parametrize("wdtype,config", RUNS)
def test_weight_routes(engine_lib, graphs, wdtype, config, monkeypatch):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    for k, v in CONFIGS[config][2].items():
        monkeypatch.setenv(k, v)
    got = counts(trace(engine_lib, graphs, wdtype, config))
    assert got == EXPECTED[(wdtype, config)], got
