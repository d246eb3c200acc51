"""fp32-arithmetic decode on fp16 weights read in place: the panel GEMV with fp16 weights widened to fp32 in registers (osb_gemv_f16w, and
osb_gemv_grouped with wdtype OSB_F16 under dtype OSB_F32), and the engine routing that hands it the fp16 blob of a decode-shaped MatMul
instead of an fp32 copy (streamed: the ring slot; resident: the fp16 cache entry).

Kernel cases run in both regimes of tests/test_gemm_conv_paths_gpu.py: integer operands (the result is the fp64 result rounded once to
fp32, bit for bit) and Gaussian operands with rows of very different scale (|err| <= 1/2 ulp + 2^-16 S).  Each result is also held to the
same bar against the fp32 GEMV fed the widened weight, the route the engine took before."""
import ctypes
import os
import re
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from test_kernels_gpu import F16, F32, _operands, _verify
from util import reference_outputs, report, run_model

pytestmark = pytest.mark.gpu

REGIMES = ("exact", "gauss")
NOT_SUPPORTED = 801
TOL32 = 2e-4        # tests/test_models_gpu.py TOL["float32"]


@pytest.fixture(scope="module")
def K(engine_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = ctypes.CDLL(engine_lib)
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.osb_gemv_f16w.argtypes = [vp, vp, i64, vp, vp, vp, i64, i64, i64, vp]
    lib.osb_gemv_grouped.argtypes = [vp, vp, vp, vp, vp, vp, ci, i64, i64, ci, ci, vp]
    lib.osb_gemm_ld.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_launch_count.restype = ctypes.c_uint64
    lib.osb_launch_count_reset.restype = None
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _problem(regime, seed, M, N, Kd, has_bias, has_res):
    """fp32 x [M, K], fp16 W [K, N], fp32 bias [N] / residual [M, N]; the fp64 reference and S = sum |a_k w_k| + |bias| + |residual|."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, w, bias, res = _operands(regime, g, [(M, Kd), (Kd, N), (N,) if has_bias else None, (M, N) if has_res else None], torch.float32, lim=3, row_scaled=1)
    w = w.half()
    ref = a.double() @ w.double()
    absref = a.double().abs() @ w.double().abs()
    if has_bias:
        ref = ref + bias.double(); absref = absref + bias.double().abs()
    if has_res:
        ref = ref + res.double(); absref = absref + res.double().abs()
    return a, w, bias, res, ref, absref


def _widened_gemv(K, a, w, bias, res):
    """The fp32 GEMV (gemv_panel_kernel<float, float>) on the fp32 copy of w: the route an fp16 blob took under fp32 arithmetic."""
    import torch
    M, Kd = a.shape
    N = w.shape[1]
    out = torch.full((M, N), float("nan"), device="cuda")
    w32 = w.float()
    assert K.osb_gemm_ld(a.data_ptr(), Kd, w32.data_ptr(), N, out.data_ptr(), N, _ptr(bias), _ptr(res), 1, M, N, Kd, 0, 0, 0, 0, F32, 0, _stream()) == 0
    return out


def _counted(K, fn):
    K.osb_launch_count_reset()
    rc = fn()
    return rc, int(K.osb_launch_count())


# ---- osb_gemv_f16w --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("epi", ["none", "bias+res"])
@pytest.mark.parametrize("Kd", [64, 2048, 5632])
@pytest.mark.parametrize("N", [256, 264, 2048, 5632])
@pytest.mark.parametrize("M", [1, 2, 3, 8])
def test_gemv_f16w(K, M, N, Kd, epi, regime):
    import torch
    a, w, bias, res, ref, absref = _problem(regime, M * 7 + N + Kd, M, N, Kd, epi != "none", epi != "none")
    out = torch.full((M, N), float("nan"), device="cuda")
    rc, n = _counted(K, lambda: K.osb_gemv_f16w(a.data_ptr(), w.data_ptr(), N, out.data_ptr(), _ptr(bias), _ptr(res), M, N, Kd, _stream()))
    assert (rc, n) == (0, 1), "one launch of the fp16-weight panel kernel"
    torch.cuda.synchronize()
    what = f"gemv_f16w M={M} N={N} K={Kd} {epi} {regime}"
    _verify(regime, out, ref, absref, what)
    _verify(regime, out, _widened_gemv(K, a, w, bias, res).double(), absref, what + " vs fp32 GEMV on the widened weight")


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("M", [1, 3, 8])
def test_gemv_f16w_row_padded_vocabulary(K, M, regime):
    """A 32003-column weight stored 32008 wide (fp16 rows pad to a multiple of 8): the pad columns (7.0) never reach the output."""
    import torch
    N, ldb, Kd = 32003, 32008, 2048
    a, w, bias, res, ref, absref = _problem(regime, 11 + M, M, N, Kd, True, True)
    wp = torch.full((Kd, ldb), 7.0, device="cuda", dtype=torch.half)
    wp[:, :N] = w
    out = torch.full((M, N), float("nan"), device="cuda")
    rc, n = _counted(K, lambda: K.osb_gemv_f16w(a.data_ptr(), wp.data_ptr(), ldb, out.data_ptr(), _ptr(bias), _ptr(res), M, N, Kd, _stream()))
    assert (rc, n) == (0, 1)
    torch.cuda.synchronize()
    _verify(regime, out, ref, absref, f"gemv_f16w ldb={ldb} M={M} {regime}")


def test_gemv_f16w_refusals(K):
    """Shapes outside the panel kernel are refused with cudaErrorNotSupported and launch nothing: the caller converts the weight."""
    import torch
    a = torch.zeros(16, 4096, device="cuda")
    w = torch.zeros(4096 * 1024 + 8, device="cuda", dtype=torch.half)
    out = torch.zeros(16, 1024, device="cuda")
    p, pw, po = a.data_ptr(), w.data_ptr(), out.data_ptr()
    for what, args in [("M = 9", (pw, 512, po, None, None, 9, 512, 64)), ("M = 0", (pw, 512, po, None, None, 0, 512, 64)),
                       ("N < 256", (pw, 128, po, None, None, 1, 128, 64)), ("K < 64", (pw, 512, po, None, None, 1, 512, 32)),
                       ("ldb % 8", (pw, 516, po, None, None, 1, 516, 64)), ("ldb < N", (pw, 256, po, None, None, 1, 512, 64)),
                       ("unaligned W", (pw + 2, 512, po, None, None, 1, 512, 64))]:
        rc, n = _counted(K, lambda: K.osb_gemv_f16w(p, *args, _stream()))
        assert (rc, n) == (NOT_SUPPORTED, 0), what


# ---- osb_gemv_grouped, wdtype OSB_F16 / dtype OSB_F32 ---------------------------------------------------------------------------------

GROUPED = [
    # M, K, N per group
    (1, 2048, (2048, 256, 256)),         # TinyLlama q / k / v
    (1, 2048, (5632, 5632)),             # TinyLlama gate / up
    (2, 64, (264, 256)),
    (3, 5632, (256, 2048, 264)),
    (8, 2048, (2048, 5632)),
    (8, 64, (256, 264, 2048)),
]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("M,Kd,Ns", GROUPED)
def test_gemv_grouped_f16w(K, M, Kd, Ns, regime):
    import torch
    g = torch.Generator(device="cuda").manual_seed(M + Kd + sum(Ns))
    a, = _operands(regime, g, [(M, Kd)], torch.float32, lim=3, row_scaled=1)
    ws = [_operands(regime, g, [(Kd, n)], torch.float32, lim=3)[0].half() for n in Ns]
    outs = [torch.full((M, n), float("nan"), device="cuda") for n in Ns]
    n = len(Ns)
    B = (ctypes.c_void_p * 3)(*[w.data_ptr() for w in ws])
    C = (ctypes.c_void_p * 3)(*[o.data_ptr() for o in outs])
    Nv = (ctypes.c_int64 * 3)(*Ns)
    sc = (ctypes.c_float * 3)(0.0, 0.0, 0.0); zp = (ctypes.c_int * 3)(0, 0, 0)
    rc, launches = _counted(K, lambda: K.osb_gemv_grouped(a.data_ptr(), B, C, Nv, sc, zp, n, M, Kd, F16, F32, _stream()))
    assert (rc, launches) == (0, 1), "the groups share one launch"
    torch.cuda.synchronize()
    for i, (w, o) in enumerate(zip(ws, outs)):
        ref, absref = a.double() @ w.double(), a.double().abs() @ w.double().abs()
        what = f"gemv_grouped_f16w M={M} K={Kd} group {i} of {Ns} {regime}"
        _verify(regime, o, ref, absref, what)
        _verify(regime, o, _widened_gemv(K, a, w, None, None).double(), absref, what + " vs fp32 GEMV on the widened weight")


def test_gemv_grouped_f16w_refusals(K):
    """fp16 weights under fp32 activations only (not under fp16 ones, nor fp32 weights under fp16 activations), and the grouped shape range."""
    import torch
    a = torch.zeros(16, 256, device="cuda")
    w = torch.zeros(256 * 512, device="cuda", dtype=torch.half)
    o = torch.zeros(16 * 512, device="cuda")
    B = (ctypes.c_void_p * 3)(w.data_ptr(), w.data_ptr(), w.data_ptr())
    C = (ctypes.c_void_p * 3)(o.data_ptr(), o.data_ptr(), o.data_ptr())
    sc = (ctypes.c_float * 3)(0.0, 0.0, 0.0); zp = (ctypes.c_int * 3)(0, 0, 0)
    for what, Ns, M, Kd, wdt, dt in [("fp32 weights, fp16 activations", (256, 256), 1, 256, F32, F16), ("M = 9", (256, 256), 9, 256, F16, F32),
                                     ("N < 256", (256, 128), 1, 256, F16, F32), ("N % 8", (256, 260), 1, 256, F16, F32),
                                     ("K < 64", (256, 256), 1, 32, F16, F32)]:
        Nv = (ctypes.c_int64 * 3)(*(Ns + (0,) * (3 - len(Ns))))
        rc, n = _counted(K, lambda: K.osb_gemv_grouped(a.data_ptr(), B, C, Nv, sc, zp, len(Ns), M, Kd, wdt, dt, _stream()))
        assert (rc, n) == (NOT_SUPPORTED, 0), what


# ---- the engine: fp32-arithmetic Llama decode on fp16 blobs ----------------------------------------------------------------------------

OPTS = ("use_scaled_dp_attn_op",)        # fp32 arithmetic
EXTRA = ("opkv0", "opkv3")
# every decode MatMul of this shape is in the kernels' range in the streamed mode too: q / k / v 256 wide, gate / up 512, vocabulary 264
ROUTE_CFG = dict(vocab=264, hidden=256, heads=4, kv_heads=4, head_dim=64, mlp=512, layers=2, past=300, max_pos=512)


@pytest.fixture(scope="module")
def workdir():
    with tempfile.TemporaryDirectory(prefix="osb200_f16w_") as d:
        yield d


def _emit(workdir, tag, cfg, wdtype):
    d = os.path.join(workdir, f"{tag}_{wdtype}") + "/"
    emit.emit_llama_decode(d, cfg, wdtype)
    return d


def _decode_matmul_weights(d):
    """(K, N) of every MatMul with a static 2-D weight in model.txt (the decode MatMuls of these single-token graphs) and the number of
    fp16 weight references outside them."""
    mm, other = [], 0
    for line in open(d + "model.txt").read().splitlines():
        refs = re.findall(r"\(float16:([0-9,]*)\)", line)
        if ":MatMul*" in line:
            for s in refs:
                dims = [int(x) for x in s.split(",") if x]
                if len(dims) == 2:
                    mm.append(tuple(dims))
        else:
            other += len(refs)
    return mm, other


def test_llama_decode_f32_on_f16_weights(engine_lib, oracle_lib, workdir):
    """The mid-size decode step of tests/test_models_gpu.py::test_llama_decode_midsize_fused_paths with fp16 blobs under fp32 arithmetic:
    streamed, resident and graph-replay runs match the reference's fp32 run (the same reference call that test makes), and the plan keeps
    its grouped-GEMV, SwiGLU and Linear steps."""
    from onnxstream_b200.model import plan_summary
    cfg = emit.LlamaConfig(vocab=259, hidden=256, heads=4, kv_heads=2, head_dim=64, mlp=512, layers=2, past=300, max_pos=512)
    d = _emit(workdir, "llama_mid", cfg, "float16")
    inputs = emit.llama_inputs(cfg)
    mask = np.ones((1, cfg.past + 1), np.int64); mask[0, 5:40] = 0
    inputs["attention_5F_mask"] = mask
    last = plan_summary(open(d + "model.txt").read(), fp16_arithmetic=False, use_scaled_dp_attn_op=True, library_path=engine_lib).splitlines()[-1]
    for kind in ("GEMV_GROUP=", "SWIGLU=2", "LINEAR="):
        assert kind in last, last
    ref = reference_outputs(oracle_lib, d, inputs, OPTS, extra_outputs=EXTRA)
    for b200 in ((), (("b200_resident_weights", 1),), (("b200_resident_weights", 1), ("b200_cuda_graph", 1))):
        got, m = run_model(engine_lib, d, inputs, OPTS, extra_outputs=EXTRA, wp="ram+nocache", b200_options=b200, runs=4 if b200 else 1)
        for n in ("logits",) + EXTRA:
            assert got[n].shape == ref[n].shape
            assert report(got[n], ref[n])["rel_to_max"] <= TOL32, (n, b200, report(got[n], ref[n]))
        if len(b200) == 2:
            assert m.stats()["graph_replays"] >= 1
        m.close()


def test_llama_decode_f32_route_reads_f16_weights(engine_lib, workdir):
    """One streamed fp32 decode step launches the fp16-weight GEMV instantiations for every decode MatMul (grouped q / k / v and gate / up,
    single o / down / vocabulary projections) and no fp32 GEMV; the fp16 -> fp32 conversions left are those of the other fp16 weights
    (embedding, norms, rotary tables, constants), none for a MatMul weight."""
    from kernel_trace import trace_run
    cfg = emit.LlamaConfig(**ROUTE_CFG)
    d = _emit(workdir, "llama_route", cfg, "float16")
    _, names = trace_run(engine_lib, d, emit.llama_inputs(cfg), OPTS, wp="ram+nocache")
    mm, other = _decode_matmul_weights(d)
    single = sum("gemv_panel_kernel<__half, float," in n for n in names)
    grouped = sum("gemv_panel_grouped_kernel<__half, float," in n for n in names)
    assert grouped == 2 * cfg.layers, names            # q / k / v and gate / up of every layer
    assert single == 2 * cfg.layers + 1, names         # o and down of every layer, the vocabulary projection
    assert not [n for n in names if re.search(r"gemv_panel(_grouped)?_kernel<float, float|skinny_gemm_kernel<float", n)], names
    converts = sum("convert_kernel<__half, float>" in n for n in names)
    assert converts <= other, (converts, other, len(mm))


def test_llama_decode_f32_resident_bytes(engine_lib, workdir):
    """Resident weights: the decode MatMul weights are cached as their fp16 blobs (a vocabulary whose N is not a multiple of 8 adds one
    row-padded fp16 copy).  The same graph with fp32 blobs caches every weight in fp32 (with a padded fp32 copy of the vocabulary, rows a
    multiple of 4) -- which is what the fp16 graph cached when its blobs were converted at load."""
    cfg = emit.LlamaConfig(**dict(ROUTE_CFG, vocab=259))
    inputs = emit.llama_inputs(cfg)
    resident = {}
    for wdtype in ("float16", "float32"):
        d = _emit(workdir, "llama_bytes", cfg, wdtype)
        _, m = run_model(engine_lib, d, inputs, OPTS, wp="ram+nocache", b200_options=(("b200_resident_weights", 1),), runs=2)
        resident[wdtype] = int(m.stats()["weight_resident_bytes"])
        m.close()
    mm, _ = _decode_matmul_weights(d.replace("float32", "float16"))
    params = sum(k * n for k, n in mm)
    pad16 = cfg.hidden * ((cfg.vocab + 7) // 8 * 8)
    pad32 = cfg.hidden * ((cfg.vocab + 3) // 4 * 4)
    assert resident["float16"] == resident["float32"] - 4 * params - 4 * pad32 + 2 * params + 2 * pad16, resident
