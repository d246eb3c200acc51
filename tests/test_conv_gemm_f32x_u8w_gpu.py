"""fp32-arithmetic convolutions and MatMuls on uint8 weights read in place (W8A32): the tensor-core kernel that multiplies the bf16 planes of
x by the integer q - z converted in shared memory and applies the per-tensor scale in its epilogue (osb_tc_conv_f32x_u8w,
osb_tc_gemm_f32x_u8w), and the engine routing that hands it the uint8 blob instead of an fp32 copy and its bf16x6 expansion.

The reference of every kernel case is the fp64 result with the weight (q - z) s.  Exact regime: integer activations, power-of-two scales and
partial sums below 2^24, so each of the three products (x_l, x_m, x_h times q - z) and their sum is exact in fp32 and the result is the fp64
result rounded once, bit for bit.  Two operand sets cover it: "wide" x entries of 18 significant bits (nonzero m and l planes) against
|q - z| <= 7, and x in [-3, 3] against q - z over the whole range of the zero point, +-255 included.  Gaussian regime: within 1e-5 of
sum |x w| (plus half an fp32 ulp)."""
import ctypes
import os
import re
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from test_kernels_gpu import _check, _check_exact
from util import reference_outputs, report, run_model

pytestmark = pytest.mark.gpu

NOT_SUPPORTED = 801
BAR = 1e-5
CONV_KERNEL = "tc_gemm_u8w_kernel<true>"
GEMM_KERNEL = "tc_gemm_u8w_kernel<false>"


@pytest.fixture(scope="module")
def K(engine_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = ctypes.CDLL(engine_lib)
    vp, i64, ci, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    lib.osb_tc_conv_f32x_u8w_ok.argtypes = [i64, i64, i64, i64, ci, ci, ci, i64, i64, ci]
    lib.osb_tc_conv_f32x_u8w.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, cf, ci, vp, vp]
    lib.osb_tc_gemm_f32x_u8w_ok.argtypes = [i64, i64, i64, i64, ci]
    lib.osb_tc_gemm_f32x_u8w.argtypes = [vp, vp, i64, vp, vp, vp, i64, i64, i64, cf, ci, vp, vp]
    lib.osb_tc_set_tile.argtypes = [ci, ci, ci]
    lib.osb_tc_set_tile.restype = None
    lib.osb_launch_count.restype = ctypes.c_uint64
    lib.osb_launch_count_reset.restype = None
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _conv(K, x, q, s, z, bias, res, st, pt, pl, Ho, Wo):
    """osb_tc_conv_f32x_u8w on x [H, W, Cin] fp32 and q [Cout, kh, kw, Cin] uint8: (rc, launches, y [Ho, Wo, Cout])."""
    import torch
    H, W, Cin = x.shape
    Cout, kh, kw, _ = q.shape
    y = torch.full((Ho, Wo, Cout), float("nan"), device="cuda")
    planes = torch.empty(3 * H * W * Cin, device="cuda", dtype=torch.bfloat16)
    K.osb_launch_count_reset()
    rc = K.osb_tc_conv_f32x_u8w(x.data_ptr(), q.data_ptr(), _ptr(bias), _ptr(res), y.data_ptr(), H, W, Cin, Cout, kh, kw, st, pt, pl, Ho, Wo, s, z,
                                planes.data_ptr(), _stream())
    n = int(K.osb_launch_count())
    torch.cuda.synchronize()
    return rc, n, y


def _gemm(K, a, q, s, z, bias, res):
    """osb_tc_gemm_f32x_u8w on a [M, K] fp32 and q [K, N] uint8: (rc, launches, c [M, N])."""
    import torch
    M, Kd = a.shape
    N = q.shape[1]
    c = torch.full((M, N), float("nan"), device="cuda")
    planes = torch.empty(3 * M * Kd, device="cuda", dtype=torch.bfloat16)
    K.osb_launch_count_reset()
    rc = K.osb_tc_gemm_f32x_u8w(a.data_ptr(), q.data_ptr(), N, c.data_ptr(), _ptr(bias), _ptr(res), M, N, Kd, s, z, planes.data_ptr(), _stream())
    n = int(K.osb_launch_count())
    torch.cuda.synchronize()
    return rc, n, c


def _conv64(x, w, st, pt, pl, Ho, Wo):
    import torch.nn.functional as Fn
    H, W, _ = x.shape
    _, kh, kw, _ = w.shape
    pb, pr = (Ho - 1) * st + kh - H - pt, (Wo - 1) * st + kw - W - pl
    xn = Fn.pad(x.double().permute(2, 0, 1)[None], (pl, pr, pt, pb))
    return Fn.conv2d(xn, w.double().permute(0, 3, 1, 2), None, stride=st)[0].permute(1, 2, 0)


def _epilogue(ref, absref, bias, res):
    if bias is not None:
        ref = ref + bias.double(); absref = absref + bias.double().abs()
    if res is not None:
        ref = ref + res.double(); absref = absref + res.double().abs()
    return ref, absref


def _weights(g, shape, z, case):
    """uint8 weights: "wide": q - z in [-7, 7]; "full" / "gauss": q over [0, 255] with both ends present (q - z = +-255 at z = 0 / 255)."""
    import torch
    if case == "wide":
        d = torch.randint(-7, 8, shape, device="cuda", generator=g)
        q = (d + z).clamp(0, 255)
    else:
        q = torch.randint(0, 256, shape, device="cuda", generator=g)
        flat = q.view(-1)
        flat[:: 97] = 0
        flat[5:: 89] = 255
    return q.to(torch.uint8).contiguous()


def _acts(g, shape, case):
    """Exact activations: "wide": integers in [-3, 3] with one entry of 18 significant bits per row, 2^17 + 1024 a + 256 + odd: x_h keeps
    bits 17..10, the remainder 257..511 has 9 significant bits, so x_m and x_l are nonzero;
    "full": integers in [-3, 3].  "gauss": N(0, 1) rows of very different scale."""
    import torch
    if case == "gauss":
        t = torch.randn(shape, device="cuda", generator=g)
        return t * torch.exp(torch.randn(shape[:-1] + (1,), device="cuda", generator=g))
    x = torch.randint(-3, 4, shape, device="cuda", generator=g).float()
    if case == "wide":
        C = shape[-1]
        rows = x.numel() // C
        idx = torch.arange(rows, device="cuda") * 7 % C
        odd = torch.randint(0, 128, (rows,), device="cuda", generator=g).float() * 2 + 1
        sign = torch.randint(0, 2, (rows,), device="cuda", generator=g).float() * 2 - 1
        wide = sign * (131072 + 1024 * torch.randint(0, 32, (rows,), device="cuda", generator=g).float() + 256 + odd)
        x.view(rows, C)[torch.arange(rows, device="cuda"), idx] = wide
    return x


def _planes_nonzero(x):
    h = x.bfloat16().float(); m = (x - h).bfloat16().float(); lo = (x - h - m).bfloat16().float()
    return bool((h != 0).any()), bool((m != 0).any()), bool((lo != 0).any())


CONV_CASES = [
    # H, W, Cin, Cout, kh, kw, stride, pad top, bottom, left, right
    (128, 128, 320, 320, 3, 3, 1, 1, 1, 1, 1),    # SDXL's 128 x 128 x 320 level
    (64, 64, 640, 640, 3, 3, 1, 1, 1, 1, 1),      # its 64 x 64 x 640 level
    (32, 32, 1280, 1280, 3, 3, 1, 1, 1, 1, 1),    # its 32 x 32 x 1280 level
    (64, 64, 640, 1280, 1, 1, 1, 0, 0, 0, 0),     # a 1x1 shortcut
    (33, 47, 128, 128, 3, 3, 2, 0, 1, 1, 0),      # stride 2, asymmetric pads
    (20, 20, 48, 64, 3, 3, 1, 1, 1, 1, 1),        # Cin tails: the zero-filled plane tail
    (16, 16, 208, 64, 3, 3, 1, 1, 1, 1, 1),
    (64, 64, 128, 3, 3, 3, 1, 1, 1, 1, 1),        # ragged Cout
    (24, 24, 64, 200, 3, 3, 1, 1, 1, 1, 1),
]


@pytest.mark.parametrize("regime", ["exact", "gauss"])
@pytest.mark.parametrize("z", [0, 128, 255])
@pytest.mark.parametrize("H,W,Cin,Cout,kh,kw,st,pt,pb,pl,pr", CONV_CASES)
def test_f32x_u8w_conv(K, H, W, Cin, Cout, kh, kw, st, pt, pb, pl, pr, z, regime):
    import torch
    Ho, Wo = (H + pt + pb - kh) // st + 1, (W + pl + pr - kw) // st + 1
    assert K.osb_tc_conv_f32x_u8w_ok(H, W, Cin, Cout, kh, kw, st, Ho, Wo, z) == 1
    g = torch.Generator(device="cuda").manual_seed(H + 3 * Cin + 7 * Cout + kh + z)
    if regime == "exact":
        bias = torch.randint(-7, 8, (Cout,), device="cuda", generator=g).float()
        res = torch.randint(-7, 8, (Ho, Wo, Cout), device="cuda", generator=g).float()
        cases = [("wide", 2.0 ** -3), ("full", 2.0 ** -5)]
    else:
        bias = torch.randn(Cout, device="cuda", generator=g)
        res = torch.randn(Ho, Wo, Cout, device="cuda", generator=g)
        cases = [("gauss", 0.0123)]
    seen = [False, False, False]
    for i, (case, s) in enumerate(cases):
        x = _acts(g, (H, W, Cin), case)
        q = _weights(g, (Cout, kh, kw, Cin), z, case)
        epi = (None, None) if i == 0 else (bias, res)
        rc, n, y = _conv(K, x, q, s, z, *epi, st, pt, pl, Ho, Wo)
        assert rc == 0 and n in (2, 3), (rc, n)
        w = (q.double() - z) * s
        ref, absref = _epilogue(_conv64(x, w, st, pt, pl, Ho, Wo), _conv64(x.abs(), w.abs(), st, pt, pl, Ho, Wo), *epi)
        what = f"conv_f32x_u8w {(H, W, Cin, Cout, kh, kw, st, pt, pb, pl, pr)} z={z} {case}"
        if regime == "exact":
            seen = [a or b for a, b in zip(seen, _planes_nonzero(x))]
            _check_exact(y, ref, absref / s, what)
        else:
            _check(y, ref, absref, what, coef=BAR)
    if regime == "exact":
        assert all(seen), "every bf16 plane of x is nonzero somewhere"


GEMM_CASES = [
    # M (rows), K, N
    (4096, 640, 640), (4096, 1280, 1280), (1024, 640, 640), (1024, 1280, 1280), (77, 640, 640), (77, 1280, 1280),
    (333, 640, 640), (333, 1280, 1280),            # ragged rows
    (1024, 1280, 10240), (1024, 5120, 1280),       # SDXL's feed-forward
    (100, 200, 144),                               # a K tail (rows past K read the next plane of A) and a ragged last column tile
]


@pytest.mark.parametrize("regime", ["exact", "gauss"])
@pytest.mark.parametrize("z", [0, 128, 255])
@pytest.mark.parametrize("M,Kd,N", GEMM_CASES)
def test_f32x_u8w_gemm(K, M, Kd, N, z, regime):
    import torch
    assert K.osb_tc_gemm_f32x_u8w_ok(M, N, Kd, N, z) == 1
    g = torch.Generator(device="cuda").manual_seed(M + 3 * Kd + 7 * N + z)
    if regime == "exact":
        bias = torch.randint(-7, 8, (N,), device="cuda", generator=g).float()
        res = torch.randint(-7, 8, (M, N), device="cuda", generator=g).float()
        cases = [("wide", 2.0 ** -2), ("full", 2.0 ** -6)]
    else:
        bias = torch.randn(N, device="cuda", generator=g)
        res = torch.randn(M, N, device="cuda", generator=g)
        cases = [("gauss", 0.0071)]
    for i, (case, s) in enumerate(cases):
        a = _acts(g, (M, Kd), case)
        q = _weights(g, (Kd, N), z, case)
        epi = (None, None) if i == 0 else (bias, res)
        rc, n, c = _gemm(K, a, q, s, z, *epi)
        assert rc == 0 and n in (2, 3), (rc, n)
        w = (q.double() - z) * s
        ref, absref = _epilogue(a.double() @ w, a.double().abs() @ w.abs(), *epi)
        what = f"gemm_f32x_u8w {(M, Kd, N)} z={z} {case}"
        if regime == "exact":
            _check_exact(c, ref, absref / s, what)
        else:
            _check(c, ref, absref, what, coef=BAR)


def test_f32x_u8w_split_k(K):
    """Deep launches with few tiles -- a 3x3 conv 8 x 8 x 1280 -> 1280 (180 k-blocks) and a GEMM 77 x 5120 -> 1280 (80 k-blocks): forced
    splits agree with the unsplit launch bit for bit on exact operands (the partials are scaled before the workspace, the reduce adds bias
    and residual once), and the rule's own pick splits."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(5)
    z, s = 131, 2.0 ** -4
    x = _acts(g, (8, 8, 1280), "full")
    q = _weights(g, (1280, 3, 3, 1280), z, "full")
    a = _acts(g, (77, 5120), "full")
    qg = _weights(g, (5120, 1280), z, "full")
    bias = torch.randint(-7, 8, (1280,), device="cuda", generator=g).float()
    res = torch.randint(-7, 8, (8, 8, 1280), device="cuda", generator=g).float()
    resg = torch.randint(-7, 8, (77, 1280), device="cuda", generator=g).float()
    runs = {"conv": lambda: _conv(K, x, q, s, z, bias, res, 1, 1, 1, 8, 8), "gemm": lambda: _gemm(K, a, qg, s, z, bias, resg)}
    refs = {"conv": _epilogue(_conv64(x, (q.double() - z) * s, 1, 1, 1, 8, 8), _conv64(x.abs(), ((q.double() - z) * s).abs(), 1, 1, 1, 8, 8), bias, res),
            "gemm": _epilogue(a.double() @ ((qg.double() - z) * s), a.double().abs() @ ((qg.double() - z) * s).abs(), bias, resg)}
    try:
        for name, run in runs.items():
            K.osb_tc_set_tile(0, 0, 1)
            rc, n, y1 = run()
            assert (rc, n) == (0, 2), name
            ref, absref = refs[name]
            _check_exact(y1, ref, absref / s, f"{name} u8w split 1")
            for sp in (2, 3, 7, 13, 64):
                K.osb_tc_set_tile(0, 0, sp)
                rc, n, y = run()
                assert (rc, n) == (0, 3), (name, sp)
                assert torch.equal(y, y1), f"{name}: split {sp} differs from the unsplit launch"
            K.osb_tc_set_tile(0, 0, 0)
            rc, n, y = run()
            assert (rc, n) == (0, 3), f"{name}: the rule splits a launch of few tiles and many k-blocks"
            assert torch.equal(y, y1)
    finally:
        K.osb_tc_set_tile(0, 0, 0)


def test_f32x_u8w_one_hot_returns_the_weights(K):
    """One-hot activations return every weight (q - z) s bit for bit, at its own place: the GEMM reads row k of a [K][N] blob for the one-hot
    row k (a wrong swizzle, a transposed atom or a misplaced k-row moves values), the 1x1 conv filter row o of an OHWI blob for the one-hot
    pixel of channel c.  The q pattern is distinct per position."""
    import torch
    z, s = 77, 2.0 ** -7
    Kd, N = 200, 272
    q = ((torch.arange(Kd * N, device="cuda") * 37 + 11) % 256).to(torch.uint8).reshape(Kd, N)
    rc, _, c = _gemm(K, torch.eye(Kd, device="cuda"), q, s, z, None, None)
    assert rc == 0
    assert torch.equal(c, (q.float() - z) * s), "GEMM one-hot readback"
    Cin, Cout = 64, 200
    qc = ((torch.arange(Cout * Cin, device="cuda") * 101 + 3) % 256).to(torch.uint8).reshape(Cout, 1, 1, Cin)
    rc, _, y = _conv(K, torch.eye(Cin, device="cuda").reshape(8, 8, Cin), qc, s, z, None, None, 1, 0, 0, 8, 8)
    assert rc == 0
    assert torch.equal(y.reshape(Cin, Cout), (qc.reshape(Cout, Cin).t().float() - z) * s), "conv one-hot readback"


def test_f32x_u8w_refusals(K):
    """Shapes, zero points and pointers outside the kernels return cudaErrorNotSupported, launch nothing and leave the output untouched."""
    import torch
    buf = lambda n, dt=torch.float32: torch.zeros(n + 64, device="cuda", dtype=dt)
    x, w = buf(16 * 16 * 64), buf(128 * 9 * 64, torch.uint8)
    y = torch.full((16 * 16 * 128 + 64,), float("nan"), device="cuda")
    b, pl = buf(128), buf(3 * 16 * 16 * 64, torch.bfloat16)
    px, pw, py, pb, pp = x.data_ptr(), w.data_ptr(), y.data_ptr(), b.data_ptr(), pl.data_ptr()
    r = buf(16 * 16 * 128)
    pr = r.data_ptr()
    names = ("x", "w", "bias", "res", "y", "H", "W", "Cin", "Cout", "kh", "kw", "s", "pt", "pl", "Ho", "Wo", "scale", "z", "planes")
    ok = (px, pw, pb, pr, py, 16, 16, 64, 128, 3, 3, 1, 1, 1, 16, 16, 0.5, 128, pp)
    conv = lambda **kw: tuple(kw.get(k, v) for k, v in zip(names, ok))
    cases = [("Cin % 8", conv(Cin=60)), ("Cin < 16", conv(Cin=8)), ("kh kw Cin % 16", conv(Cin=24)), ("stride 3", conv(s=3, Ho=6, Wo=6)),
             ("kh > 7", conv(kh=8, Ho=11)), ("H W < 64", conv(H=7, W=8, Ho=7, Wo=8)), ("zero point -1", conv(z=-1)), ("zero point 256", conv(z=256)),
             ("unaligned x", conv(x=px + 4)), ("unaligned w", conv(w=pw + 8)), ("unaligned planes", conv(planes=pp + 8)), ("unaligned y", conv(y=py + 4)),
             ("unaligned residual", conv(res=pr + 4)), ("unaligned bias", conv(bias=pb + 2))]
    for what, args in cases:
        K.osb_launch_count_reset()
        rc = K.osb_tc_conv_f32x_u8w(*args, _stream())
        assert (rc, int(K.osb_launch_count())) == (NOT_SUPPORTED, 0), "conv " + what
    gnames = ("a", "b", "ldb", "c", "bias", "res", "M", "N", "K", "scale", "z", "planes")
    gok = (px, pw, 128, py, pb, pr, 32, 128, 64, 0.5, 128, pp)
    gemm = lambda **kw: tuple(kw.get(k, v) for k, v in zip(gnames, gok))
    gcases = [("K % 8", gemm(K=60)), ("ldb % 16", gemm(ldb=136, N=136)), ("ldb < N", gemm(N=144)), ("zero point -1", gemm(z=-1)),
              ("zero point 256", gemm(z=256)), ("unaligned A", gemm(a=px + 4)), ("unaligned B", gemm(b=pw + 8)), ("unaligned planes", gemm(planes=pp + 8)),
              ("unaligned C", gemm(c=py + 4)), ("unaligned residual", gemm(res=pr + 4)), ("unaligned bias", gemm(bias=pb + 2))]
    for what, args in gcases:
        K.osb_launch_count_reset()
        rc = K.osb_tc_gemm_f32x_u8w(*args, _stream())
        assert (rc, int(K.osb_launch_count())) == (NOT_SUPPORTED, 0), "gemm " + what
    torch.cuda.synchronize()
    assert torch.isnan(y).all(), "a refused launch wrote its output"
    assert K.osb_tc_conv_f32x_u8w_ok(16, 16, 64, 128, 3, 3, 1, 16, 16, 0) == 1
    assert K.osb_tc_conv_f32x_u8w_ok(448, 448, 128, 128, 3, 3, 1, 448, 448, 255) == 1, "no bound from the workspace"
    assert K.osb_tc_gemm_f32x_u8w_ok(1 << 20, 1280, 1280, 1280, 0) == 1, "no bound from the workspace"
    K.osb_launch_count_reset()
    assert K.osb_tc_conv_f32x_u8w(*ok, _stream()) == 0 and int(K.osb_launch_count()) == 2
    K.osb_launch_count_reset()
    assert K.osb_tc_gemm_f32x_u8w(*gok, _stream()) == 0 and int(K.osb_launch_count()) == 2
    torch.cuda.synchronize()


# ---- the engine: a W8A32 SDXL-shaped UNet ----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def workdir():
    with tempfile.TemporaryDirectory(prefix="osb200_u8w_") as d:
        yield d


# a tiny SDXL UNet at a 32 x 32 latent: levels 32, 16 and 8, every Conv input at least 64 pixels
UNET = emit.UNetConfig.tiny(32, sdxl=True)


def _unet(workdir, wdtype="uint8"):
    d = os.path.join(workdir, f"unet_{wdtype}") + "/"
    if not os.path.exists(d + "model.txt"):
        emit.emit_unet(d, UNET, wdtype, seed=5)
    return d


def _nodes(d):
    """Per op with a uint8 weight as input 1: (type, weight shape, input shape, zero point); and the number of uint8 weight references."""
    nodes, refs = [], 0
    for line in open(d + "model.txt").read().splitlines():
        m = re.match(r"[^:]*:(\w+)\*input:([^*]*)\*", line)
        if not m:
            continue
        ins = m.group(2).split(";")
        refs += sum("(uint8[" in i for i in ins)
        if len(ins) > 1 and "(uint8[" in ins[1]:
            zp = int(re.search(r"uint8\[[^,]*,(\d+)\]", ins[1]).group(1))
            ws = tuple(int(v) for v in re.search(r"\]:([0-9,]*)\)", ins[1]).group(1).split(",") if v)
            xs = tuple(int(v) for v in re.search(r"\(([0-9,]*)\)", ins[0]).group(1).split(","))
            nodes.append((m.group(1), ws, xs, zp))
    return nodes, refs


def _routed(node):
    """The engine's rule (engine_run.cpp: weight_route, mha_stored): a Conv the kernel takes, or a MatMul / Gemm with a 2-D
    weight and more than 2 rows."""
    op, ws, xs, zp = node
    if op == "Conv":
        cout, cin, kh, kw = ws
        return cin % 8 == 0 and cin >= 16 and xs[2] * xs[3] >= 64 and kh <= 7 and kw <= 7 and (kh * kw * cin) % 16 == 0
    if op in ("MatMul", "Gemm") and len(ws) == 2:
        return int(np.prod(xs[:-1])) > 2 and ws[0] % 8 == 0 and ws[1] % 16 == 0
    return False


def _count(names, key):
    return sum(key in n for n in names)


def test_w8a32_unet_route(engine_lib, workdir, monkeypatch):
    """A streamed W8A32 run launches the new kernels once per Conv, MatMul and attention projection the rule gives them, and converts none of
    their weights to fp32: against OSB_W8A32_TC=0 the run has exactly that many fewer uint8 -> fp32 conversions, two bf16x3 expansions fewer
    per routed conv, and fewer CUDA-core GEMMs (the attention projections left them)."""
    from kernel_trace import trace_run
    d = _unet(workdir)
    inputs = emit.unet_inputs(UNET, seed=5)
    nodes, _ = _nodes(d)
    convs = [n for n in nodes if n[0] == "Conv"]
    conv_new = sum(map(_routed, convs))
    mm_new = sum(_routed(n) for n in nodes if n[0] != "Conv")
    assert conv_new >= 10 and mm_new >= 10 and len(convs) - conv_new == 1
    _, new = trace_run(engine_lib, d, inputs, (), wp="ram+nocache")
    monkeypatch.setenv("OSB_W8A32_TC", "0")
    _, old = trace_run(engine_lib, d, inputs, (), wp="ram+nocache")
    diag = {k: (_count(new, k), _count(old, k)) for k in (CONV_KERNEL, GEMM_KERNEL, "dequant_kernel<float>", "bf16x3_expand", "igemm")}
    assert _count(new, CONV_KERNEL) == conv_new, diag
    assert _count(new, GEMM_KERNEL) == mm_new, diag
    assert _count(old, CONV_KERNEL) == 0 and _count(old, GEMM_KERNEL) == 0, diag
    assert _count(old, "dequant_kernel<float>") - _count(new, "dequant_kernel<float>") == conv_new + mm_new, diag
    assert _count(old, "bf16x3_expand") - _count(new, "bf16x3_expand") >= 2 * conv_new, diag
    assert _count(new, "igemm") < _count(old, "igemm"), diag


def test_w8a32_unet_resident_bytes(engine_lib, workdir):
    """Resident weights: every routed weight is held as its uint8 blob alone.  The count is exactly the routed blobs (1 byte per parameter),
    the other uint8 tensors as fp32 copies (4 bytes), the bf16x6 expansion of conv_in's filter (12 bytes per parameter) and the float32
    tensors (4 bytes)."""
    d = _unet(workdir)
    nodes, _ = _nodes(d)
    _, m = run_model(engine_lib, d, emit.unet_inputs(UNET, seed=5), (), wp="ram+nocache", b200_options=(("b200_resident_weights", 1),), runs=2)
    got = int(m.stats()["weight_resident_bytes"])
    m.close()
    routed = sum(int(np.prod(n[1])) for n in nodes if _routed(n))
    unrouted_conv = sum(int(np.prod(n[1])) for n in nodes if n[0] == "Conv" and not _routed(n))
    u8_total = f32_total = 0
    for f in os.listdir(d):
        if f.endswith(".bin"):
            size = os.path.getsize(os.path.join(d, f))
            txt = open(d + "model.txt").read()
            dt = re.search(re.escape(f.replace("_nhwc", "_nchw")) + r"\((\w+)", txt)
            if dt and dt.group(1) == "uint8":
                u8_total += size
            elif dt and dt.group(1) == "float32":
                f32_total += size
    want = routed + 4 * (u8_total - routed) + 12 * unrouted_conv + f32_total
    assert got == want, (got, want, routed, u8_total, f32_total, unrouted_conv)


def test_w8a32_unet_parity(engine_lib, oracle_lib, workdir, monkeypatch):
    """Against the reference's W8A32 run (which multiplies by fl((q - z) s)), streamed, resident and under graph replay; and against the
    fp32-copy route (OSB_W8A32_TC=0) within 2e-5 of max |out|."""
    from kernel_trace import trace_run
    d = _unet(workdir)
    inputs = emit.unet_inputs(UNET, seed=5)
    ref = reference_outputs(oracle_lib, d, inputs, ())["out_5F_sample"]
    outs = []
    for b200 in ((), (("b200_resident_weights", 1),), (("b200_resident_weights", 1), ("b200_cuda_graph", 1))):
        got, m = run_model(engine_lib, d, inputs, (), wp="ram+nocache", b200_options=b200, runs=3 if b200 else 1)
        r = report(got["out_5F_sample"], ref)
        assert r["rel_to_max"] <= 2e-4, (b200, r)
        outs.append(got["out_5F_sample"])
        m.close()
    monkeypatch.setenv("OSB_W8A32_TC", "0")
    old, names = trace_run(engine_lib, d, inputs, (), keep=("out_5F_sample",), wp="ram+nocache")
    assert _count(names, GEMM_KERNEL) == 0
    for o in outs:
        assert float(np.abs(o - old["out_5F_sample"]).max()) <= 2e-5 * float(np.abs(old["out_5F_sample"]).max())


def test_w8a16_and_decode_routes_unchanged(engine_lib, workdir, monkeypatch):
    """The same uint8 model under fp16 arithmetic (W8A16), and a 1-row MatMul on a uint8 weight (the decode GEMV, fp32 and fp16), launch the
    same kernels with the new route on and off, and none of the new kernels."""
    from kernel_trace import trace_run
    d = _unet(workdir)
    inputs = emit.unet_inputs(UNET, seed=5)
    g = emit.GraphBuilder(os.path.join(workdir, "gemv") + "/", "uint8", seed=2)
    x = g.input("x", (1, 1, 512))
    g.mark_output(g.linear(x, 768, bias=True))
    g.finish()
    dg = os.path.join(workdir, "gemv") + "/"
    gin = {"x": np.random.default_rng(1).standard_normal((1, 1, 512)).astype(np.float32)}
    runs = [(d, inputs, ("use_fp16_arithmetic",)), (dg, gin, ()), (dg, gin, ("use_fp16_arithmetic",))]
    traces = []
    for env in ("1", "0"):
        monkeypatch.setenv("OSB_W8A32_TC", env)
        traces.append([trace_run(engine_lib, dd, ii, oo, wp="ram+nocache")[1] for dd, ii, oo in runs])
    for new, old in zip(*traces):
        assert new == old
        assert _count(new, "u8w_kernel") == 0
    assert all(_count(t, "gemv_w8") >= 1 for t in traces[0][1:]), "the decode GEMV reads the uint8 weight"
