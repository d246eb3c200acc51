"""The GEGLU feed-forward gate in the tensor-core GEMM epilogue (osb_tc_gemm_geglu): one launch for MatMul(x, W[K, 2 inner]) + bias and
value * gelu_erf(gate).

It must store exactly what the unfused chain stores -- the unsplit GEMM with its bias epilogue (rounded to fp16), then osb_geglu -- on
Gaussian operands at the SD 1.5 feed-forward shapes, ragged row counts and narrow inner widths, with and without a bias.  On integer
operands the pre-GELU halves are exact, so the result is also held to fp64 GELU at the bar of test_kernels_gpu.py::test_geglu.  In the
engine, the GEGLU step that absorbed the feed-forward MatMul + bias runs that one launch (no geglu_kernel in the trace) and agrees with
the op-by-op schedule, resident and streamed."""
import ctypes
import tempfile

import numpy as np
import pytest

from kernel_trace import trace_run
from onnxstream_b200 import emit
from test_kernels_gpu import F16, K, _stream  # noqa: F401  (K: the module fixture)
from util import run_model

pytestmark = pytest.mark.gpu

vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int

# M, inner, K: the SD 1.5 FF-in shapes at 64², 32², 16², 8², then ragged M and narrow inner
SHAPES = [(4096, 1280, 320), (1024, 2560, 640), (256, 5120, 1280), (64, 5120, 1280), (1000, 192, 320), (77, 64, 128), (33, 128, 64)]


def _bind(K):
    K.osb_tc_gemm_geglu.argtypes = [vp, vp, vp, vp, i64, i64, i64, vp]
    K.osb_geglu.argtypes = [vp, vp, ci, i64, i64, vp]
    K.osb_tc_set_tile.argtypes = [ci, ci, ci]
    K.osb_tc_set_tile.restype = None


def _fused(K, a, w, b, M, inner, Kd):
    import torch
    y = torch.full((M, inner), float("nan"), device="cuda", dtype=torch.half)
    assert K.osb_tc_gemm_geglu(a.data_ptr(), w.data_ptr(), y.data_ptr(), b.data_ptr() if b is not None else None, M, inner, Kd, _stream()) == 0
    return y


def _unfused(K, a, w, b, M, inner, Kd):
    """The chain the fused launch replaces: the 128 x 128 unsplit GEMM (forced) with its bias epilogue, then osb_geglu."""
    import torch
    x = torch.empty(M, 2 * inner, device="cuda", dtype=torch.half)
    y = torch.full((M, inner), float("nan"), device="cuda", dtype=torch.half)
    K.osb_tc_set_tile(128, 128, 1)
    try:
        assert K.osb_gemm(a.data_ptr(), w.data_ptr(), x.data_ptr(), b.data_ptr() if b is not None else None, None, 1, M, 2 * inner, Kd,
                          0, 0, 0, 0, F16, 2, _stream()) == 0
    finally:
        K.osb_tc_set_tile(0, 0, 0)
    assert K.osb_geglu(x.data_ptr(), y.data_ptr(), F16, M, inner, _stream()) == 0
    return y


@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("M,inner,Kd", SHAPES)
def test_gemm_geglu_bit_exact(K, M, inner, Kd, bias):
    import torch
    _bind(K)
    g = torch.Generator(device="cuda").manual_seed(M + inner + Kd)
    a = torch.randn(M, Kd, device="cuda", generator=g).half()
    w = (torch.randn(Kd, 2 * inner, device="cuda", generator=g) / Kd ** 0.5).half()
    b = torch.randn(2 * inner, device="cuda", generator=g).half() if bias else None
    got, want = _fused(K, a, w, b, M, inner, Kd), _unfused(K, a, w, b, M, inner, Kd)
    torch.cuda.synchronize()
    assert torch.isfinite(want).all()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"{int((got.view(torch.int16) != want.view(torch.int16)).sum())} elements differ"


@pytest.mark.parametrize("M,inner,Kd", [(4096, 1280, 320), (77, 192, 128)])
def test_gemm_geglu_integer_fp64(K, M, inner, Kd):
    """Integer operands: A . B + bias is exact in fp32 and in fp16 (|values| < 2048), so the result is value * gelu(gate) of exact halves."""
    import torch
    _bind(K)
    g = torch.Generator(device="cuda").manual_seed(7 + M)
    a = torch.randint(-2, 3, (M, Kd), device="cuda", generator=g).half()
    w = torch.randint(-2, 3, (Kd, 2 * inner), device="cuda", generator=g).half()
    b = torch.randint(-8, 9, (2 * inner,), device="cuda", generator=g).half()
    y = _fused(K, a, w, b, M, inner, Kd)
    torch.cuda.synchronize()
    x = a.double() @ w.double() + b.double()
    assert float(x.abs().max()) < 2048
    v, gate = x[:, :inner], x[:, inner:]
    ref = v * (0.5 * gate * (1.0 + torch.erf(gate / 2.0 ** 0.5)))
    tol = 2.0 ** -10 * (ref.abs() + (v * gate).abs() + 1.0)
    assert not ((y.double() - ref).abs() > tol).any()


def test_gemm_geglu_declines(K):
    """inner % 64 != 0 and unaligned operands are refused (cudaErrorNotSupported), nothing launched: the engine runs the two-step chain."""
    import torch
    _bind(K)
    a = torch.zeros(128, 64, device="cuda", dtype=torch.half)
    w = torch.zeros(64, 2 * 96, device="cuda", dtype=torch.half)
    y = torch.zeros(128, 96, device="cuda", dtype=torch.half)
    assert K.osb_tc_gemm_geglu(a.data_ptr(), w.data_ptr(), y.data_ptr(), None, 128, 96, 64, _stream()) == 801
    assert K.osb_tc_gemm_geglu(a.data_ptr() + 2, w.data_ptr(), y.data_ptr(), None, 128, 64, 64, _stream()) == 801


def _ff_graph(d, T, C):
    g = emit.GraphBuilder(d, "float16", seed=T + C)
    h = g.input("h", (1, T, C))
    ctx = g.input("ctx", (1, 77, C))
    out = g.transformer_block(h, ctx, heads=C // 64)
    g.finish()
    rng = np.random.default_rng(T)
    return {"h": rng.standard_normal((1, T, C)).astype(np.float32), "ctx": rng.standard_normal((1, 77, C)).astype(np.float32)}, out.name


@pytest.mark.parametrize("resident", [1, 0], ids=["resident", "streamed"])
def test_engine_transformer_block_geglu(engine_lib, K, resident):
    """A transformer block (emit) at T = 1024, C = 320: the fused GEGLU step runs osb_tc_gemm_geglu (no geglu_kernel in the trace) and
    the block's output agrees with the op-by-op schedule (b200_fuse_nodes 0) within the fp16 bar of the smoke run."""
    with tempfile.TemporaryDirectory(prefix="osb200_geglu_") as d:
        inputs, out = _ff_graph(d + "/", 1024, 320)
        wp = "ram+nocache" if resident else "nocache"
        opts = ("use_fp16_arithmetic", "fuse_ops_in_attention")
        a, names = trace_run(engine_lib, d, inputs, opts, keep=(out,), wp=wp, b200_options=(("b200_resident_weights", resident),))
        b, _ = run_model(engine_lib, d, inputs, opts, wp=wp, b200_options=(("b200_resident_weights", resident), ("b200_fuse_nodes", 0)))
        assert not any("geglu_kernel" in n for n in names), "the GEGLU step ran the two-step chain"
        assert any("tc_gemm_kernel<128, 128, false, 1, false, false, true>" in n for n in names), [n for n in names if "tc_gemm" in n]
        got, ref = np.asarray(a[out], np.float64), np.asarray(b[out], np.float64)
        assert np.isfinite(got).all()
        err, scale = float(np.abs(got - ref).max()), float(np.abs(ref).max())
        assert err <= 2e-2 * max(scale, 1.0), (err, scale)
