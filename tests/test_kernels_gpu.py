"""GPU parity tests for the hand-written kernels, called through the internal C ABI (include/onnxstream_b200_kernels.h)
with torch only providing device memory.  Reference = fp64 math on the same fp16-rounded inputs; the tolerance for the
fp16 tensor-core path is |err| <= 2^-9 * sum|a_i b_i| + 1 fp16 ulp of the result (fp32 accumulate, one final rounding)."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F16, F32 = 2, 3


@pytest.fixture(scope="module")
def K(engine_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = ctypes.CDLL(engine_lib)
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.osb_gemm.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_conv2d.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, ci, ci, vp]
    lib.osb_tc_launch_count.restype = ctypes.c_uint64
    lib.osb_launch_count_reset.restype = None
    lib.osb_tc_set_pair_mode.argtypes = [ci]
    lib.osb_tc_set_pair_mode.restype = None
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(out, ref, absref, what):
    import torch
    err = (out.double() - ref).abs()
    tol = absref * 2.0 ** -9 + ref.abs() * 2.0 ** -10 + 1e-6
    bad = (err > tol)
    assert not bad.any(), f"{what}: {int(bad.sum())} / {bad.numel()} outside tolerance, max err {float(err.max()):.4g} (ref max {float(ref.abs().max()):.4g})"


GEMM_CASES = [
    # batch, M, N, K, b_transposed, bias, residual
    (1, 256, 256, 128, 0, False, False),
    (1, 256, 256, 128, 1, False, False),
    (1, 128, 128, 64, 0, False, False),
    (1, 300, 136, 72, 0, True, True),
    (1, 300, 136, 72, 1, True, False),
    (3, 200, 64, 40, 0, False, False),     # attention-like: small K, ragged M
    (8, 4096, 40, 4096, 0, False, False) if False else (2, 512, 40, 512, 0, False, False),
    (1, 4096, 320, 320, 0, True, True),
    (1, 1024, 2560, 640, 0, True, False),
    (1, 77, 640, 768, 0, False, False),
    (1, 64, 1280, 11520, 1, True, False),    # few tiles, deep K: split-K path
    (1, 256, 1280, 2560, 0, True, True),     # split-K, MN-major B
    (1, 1, 1280, 1280, 0, True, False),      # time-embedding Gemm: weight-bandwidth GEMV
    (1, 4, 5632, 2048, 0, False, False),
    (1, 64, 32, 32, 0, True, False),         # VAE toy attention projections / score GEMMs
    (1, 64, 64, 32, 1, False, False),
    (1, 64, 32, 64, 0, False, True),
    (1, 1024, 16, 16, 0, True, False),
]


PAIR_GEMM_CASES = [
    # CTA pairs (2-CTA clusters sharing the B tile through TMA multicast) forced on: both B majors, ragged M / N / K, odd number
    # of 128-row tiles (the pair's second tile is empty), batch, bias / residual
    (1, 256, 256, 128, 1, False, False),
    (1, 256, 256, 128, 0, False, False),
    (1, 300, 136, 72, 1, True, True),
    (1, 300, 136, 72, 0, True, True),
    (1, 384, 64, 64, 1, True, False),
    (1, 640, 192, 200, 1, False, True),
    (1, 4096, 320, 320, 0, True, True),
    (1, 4096, 320, 1280, 1, True, True),
    (1, 1024, 2560, 640, 0, True, False),
    (1, 2048, 640, 5760, 1, True, False),
    (3, 520, 264, 136, 1, False, True),
    (2, 512, 512, 256, 0, True, False),
    (1, 8192, 1024, 512, 1, False, False),    # several tiles per pair: ring reuse across tiles
]


@pytest.mark.parametrize("case", PAIR_GEMM_CASES)
def test_gemm_f16_pair_kernel(K, case):
    K.osb_tc_set_pair_mode(2)
    try:
        test_gemm_f16(K, case, 2)
    finally:
        K.osb_tc_set_pair_mode(1)


PAIR_CONV_CASES = [
    (64, 64, 320, 320, 3, 1, 1, True, True),
    (32, 32, 96, 72, 3, 1, 1, False, False),      # ragged channels
    (24, 40, 32, 40, 3, 1, 1, True, False),       # non power-of-two width
    (256, 256, 32, 16, 3, 1, 1, True, False),     # wide image: bw = 128, one row segment per CTA
    (16, 16, 64, 64, 3, 2, 1, True, False),       # strided
    (64, 64, 320, 320, 3, 2, 1, True, False),
    (16, 16, 64, 128, 1, 1, 0, True, True),
    (32, 32, 640, 640, 3, 1, 1, True, True),
    (64, 64, 640, 640, 3, 1, 1, True, False),     # the 1.08-wave layer of the single-CTA kernel
    (128, 128, 128, 256, 3, 1, 1, True, True),    # VAE-decoder-like: many tiles per pair
]


@pytest.mark.parametrize("case", PAIR_CONV_CASES)
def test_conv_f16_pair_kernel(K, case):
    K.osb_tc_set_pair_mode(2)
    try:
        K.osb_launch_count_reset()
        test_conv_f16(K, case, 0)
        assert K.osb_tc_launch_count() >= 1
    finally:
        K.osb_tc_set_pair_mode(1)


@pytest.mark.parametrize("case", GEMM_CASES)
@pytest.mark.parametrize("impl", [1, 2])
def test_gemm_f16(K, case, impl):
    import torch
    batch, M, N, Kd, bt, has_bias, has_res = case
    if impl == 2 and M < 32:
        pytest.skip("skinny problems are served by the weight-bandwidth GEMV kernel, not the tensor-core tile kernel")
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + Kd)
    a = torch.randn(batch, M, Kd, device="cuda", generator=g).half()
    b = (torch.randn(batch, N, Kd, device="cuda", generator=g) if bt else torch.randn(batch, Kd, N, device="cuda", generator=g)).half()
    bias = torch.randn(N, device="cuda", generator=g).half() if has_bias else None
    res = torch.randn(batch, M, N, device="cuda", generator=g).half() if has_res else None
    c = torch.full((batch, M, N), float("nan"), device="cuda", dtype=torch.half)
    K.osb_launch_count_reset()
    rc = K.osb_gemm(a.data_ptr(), b.data_ptr(), c.data_ptr(), bias.data_ptr() if has_bias else None, res.data_ptr() if has_res else None,
                    batch, M, N, Kd, M * Kd, N * Kd, M * N, bt, F16, impl, _stream())
    assert rc == 0, f"osb_gemm rc={rc}"
    torch.cuda.synchronize()
    if impl == 2:
        assert K.osb_tc_launch_count() >= 1
    bd = b.double().transpose(1, 2) if bt else b.double()
    ref = a.double() @ bd
    absref = a.double().abs() @ bd.abs()
    if has_bias:
        ref = ref + bias.double(); absref = absref + bias.double().abs()
    if has_res:
        ref = ref + res.double(); absref = absref + res.double().abs()
    _check(c, ref, absref, f"gemm {case} impl {impl}")


CONV_CASES = [
    # H, W, Cin, Cout, k, stride, pad, bias, residual
    (16, 16, 64, 128, 3, 1, 1, True, False),
    (16, 16, 64, 128, 1, 1, 0, True, True),
    (8, 8, 128, 128, 3, 1, 1, True, False),
    (64, 64, 320, 320, 3, 1, 1, True, True),
    (32, 32, 96, 72, 3, 1, 1, False, False),      # ragged channels
    (24, 40, 32, 40, 3, 1, 1, True, False),       # non power-of-two width
    (256, 256, 32, 16, 3, 1, 1, True, False),     # wide image: one row segment per tile
    (16, 16, 64, 64, 3, 2, 1, True, False),       # strided: TMA traversal stride
    (64, 64, 320, 320, 3, 2, 1, True, False),
    (8, 8, 1280, 1280, 3, 2, 1, True, False),     # 4x4 output, split-K
    (8, 8, 1280, 1280, 3, 1, 1, True, True),      # weight-bound 8x8 level, split-K
    (64, 64, 320, 4, 3, 1, 1, True, False),       # conv_out: ragged Cout, scalar epilogue
    (64, 64, 4, 320, 3, 1, 1, True, False),       # conv_in: tiny Cin stays on the CUDA-core kernel
    (8, 8, 32, 32, 3, 1, 1, True, True),          # VAE-decoder toy shapes: narrow channels
    (16, 16, 32, 32, 3, 1, 1, True, False),
    (32, 32, 32, 16, 3, 1, 1, True, False),
    (32, 32, 16, 16, 3, 1, 1, True, True),
    (32, 32, 16, 3, 3, 1, 1, True, False),
    (32, 32, 32, 16, 1, 1, 0, True, True),
    (16, 16, 24, 40, 3, 1, 1, False, False),
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("impl", [1, 0])
def test_conv_f16(K, case, impl):
    import torch
    import torch.nn.functional as Fn
    H, W, Cin, Cout, k, s, pad, has_bias, has_res = case
    g = torch.Generator(device="cuda").manual_seed(H * 5 + Cin)
    x = torch.randn(H, W, Cin, device="cuda", generator=g).half()
    w = (torch.randn(Cout, k, k, Cin, device="cuda", generator=g) / (k * k * Cin) ** 0.5).half()
    bias = torch.randn(Cout, device="cuda", generator=g).half() if has_bias else None
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    res = torch.randn(Ho, Wo, Cout, device="cuda", generator=g).half() if has_res else None
    y = torch.full((Ho, Wo, Cout), float("nan"), device="cuda", dtype=torch.half)
    rc = K.osb_conv2d(x.data_ptr(), w.data_ptr(), bias.data_ptr() if has_bias else None, res.data_ptr() if has_res else None, y.data_ptr(),
                      H, W, Cin, Cout, k, k, s, pad, pad, Ho, Wo, F16, impl, _stream())
    assert rc == 0, f"osb_conv2d rc={rc}"
    torch.cuda.synchronize()
    xn = x.double().permute(2, 0, 1)[None]
    wn = w.double().permute(0, 3, 1, 2)
    ref = Fn.conv2d(xn, wn, None, stride=s, padding=pad)[0].permute(1, 2, 0)
    absref = Fn.conv2d(xn.abs(), wn.abs(), None, stride=s, padding=pad)[0].permute(1, 2, 0)
    if has_bias:
        ref = ref + bias.double(); absref = absref + bias.double().abs()
    if has_res:
        ref = ref + res.double(); absref = absref + res.double().abs()
    _check(y, ref, absref, f"conv {case} impl {impl}")


GN_CONV_CASES = [
    # H, W, Cin, Cout, k, stride, groups, residual, bias2, pair_mode
    (64, 64, 320, 320, 3, 1, 32, True, False, 1),     # cpg = 10: groups straddle 32-column chunks and 128-column tiles
    (64, 64, 320, 320, 3, 1, 32, False, True, 2),     # same through CTA pairs, with the time-embedding addend
    (32, 32, 320, 640, 3, 1, 32, False, True, 1),
    (32, 32, 640, 640, 1, 1, 32, True, False, 2),
    (16, 16, 1280, 1280, 3, 1, 32, True, False, 1),   # split-K: statistics in the reduce kernel (cpg = 40)
    (8, 8, 1280, 1280, 3, 1, 32, False, True, 1),
    (16, 16, 64, 64, 3, 1, 8, True, True, 1),         # tiny-model shapes (cpg = 8), ragged tile
    (24, 40, 32, 40, 3, 1, 5, False, False, 1),       # cpg = 8, non power-of-two width
    (128, 128, 128, 128, 3, 1, 32, True, False, 2),   # cpg = 4 (VAE decoder), several tiles per pair
]


@pytest.mark.parametrize("case", GN_CONV_CASES)
def test_conv_epilogue_gn_stats_and_bias2(K, case):
    """osb_conv2d_ex: conv + bias + bias2 (per-channel addend) + residual, with the GroupNorm statistics of the STORED fp16 output
    gathered in the epilogue (single-CTA or CTA-pair tile epilogue, or the split-K reduce kernel) -- then osb_group_norm_apply on them
    against a float64 GroupNorm of the same tensor."""
    import torch
    import torch.nn.functional as Fn
    vp, i64, ci, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    K.osb_conv2d_ex.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, ci, ci, vp, vp, ci, ctypes.POINTER(ci)]
    K.osb_group_norm_apply.argtypes = [vp, vp, ci, i64, i64, ci, vp, vp, cf, ci, vp, vp, vp]
    H, W, Cin, Cout, k, s, G, has_res, has_b2, pair_mode = case
    pad = k // 2
    g = torch.Generator(device="cuda").manual_seed(H * 3 + Cout)
    x = torch.randn(H, W, Cin, device="cuda", generator=g).half()
    w = (torch.randn(Cout, k, k, Cin, device="cuda", generator=g) / (k * k * Cin) ** 0.5).half()
    bias = torch.randn(Cout, device="cuda", generator=g).half()
    bias2 = torch.randn(Cout, device="cuda", generator=g).half() if has_b2 else None
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    res = torch.randn(Ho, Wo, Cout, device="cuda", generator=g).half() if has_res else None
    y = torch.full((Ho, Wo, Cout), float("nan"), device="cuda", dtype=torch.half)
    stats = torch.zeros(2 * G, device="cuda", dtype=torch.float64)
    done = ci(0)
    K.osb_tc_set_pair_mode(pair_mode)
    try:
        rc = K.osb_conv2d_ex(x.data_ptr(), w.data_ptr(), bias.data_ptr(), bias2.data_ptr() if has_b2 else None, res.data_ptr() if has_res else None, y.data_ptr(),
                             H, W, Cin, Cout, k, k, s, pad, pad, Ho, Wo, F16, 0, _stream(), stats.data_ptr(), G, ctypes.byref(done))
    finally:
        K.osb_tc_set_pair_mode(1)
    assert rc == 0
    torch.cuda.synchronize()
    xn = x.double().permute(2, 0, 1)[None]; wn = w.double().permute(0, 3, 1, 2)
    ref = Fn.conv2d(xn, wn, None, stride=s, padding=pad)[0].permute(1, 2, 0) + bias.double()
    absref = Fn.conv2d(xn.abs(), wn.abs(), None, stride=s, padding=pad)[0].permute(1, 2, 0) + bias.double().abs()
    if has_b2:
        ref = ref + bias2.double(); absref = absref + bias2.double().abs()
    if has_res:
        ref = ref + res.double(); absref = absref + res.double().abs()
    _check(y, ref, absref, f"conv_ex {case}")
    assert done.value == 1, "the kernel did not report the statistics"
    yd = y.double().reshape(Ho * Wo, G, Cout // G)
    want = torch.stack([yd.sum(dim=(0, 2)), (yd * yd).sum(dim=(0, 2))], dim=1).reshape(-1)
    err = (stats - want).abs() / (torch.stack([yd.abs().sum(dim=(0, 2)), (yd * yd).sum(dim=(0, 2))], dim=1).reshape(-1) + 1e-9)
    assert float(err.max()) <= 2e-5, f"statistics off by {float(err.max()):.3g} (relative to sum|y| / sum y^2)"
    # apply pass: GroupNorm + SiLU from those statistics; the `clear` buffer is zeroed on the way
    gamma = (1 + 0.1 * torch.randn(Cout, device="cuda", generator=g)).half(); beta = (0.1 * torch.randn(Cout, device="cuda", generator=g)).half()
    out = torch.empty_like(y); clear = torch.ones(2 * G, device="cuda", dtype=torch.float64)
    assert K.osb_group_norm_apply(y.data_ptr(), out.data_ptr(), F16, Cout, Ho * Wo, G, gamma.data_ptr(), beta.data_ptr(), 1e-5, 1, stats.data_ptr(), clear.data_ptr(), _stream()) == 0
    torch.cuda.synchronize()
    mean = yd.mean(dim=(0, 2), keepdim=True); var = yd.var(dim=(0, 2), unbiased=False, keepdim=True)
    gn = ((yd - mean) / torch.sqrt(var + 1e-5)).reshape(Ho, Wo, Cout) * gamma.double() + beta.double()
    gn = gn * torch.sigmoid(gn)
    assert float((out.double() - gn).abs().max()) <= 2e-3 * max(1.0, float(gn.abs().max()))
    assert float(clear.abs().max()) == 0.0


def test_channel_add_stats(K):
    import torch
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    K.osb_channel_add_stats.argtypes = [vp, vp, vp, ci, i64, i64, ci, vp, vp]
    for (HW, C, G) in [(4096, 320, 32), (256, 1280, 32), (64, 64, 8)]:
        g = torch.Generator(device="cuda").manual_seed(C)
        x = torch.randn(HW, C, device="cuda", generator=g).half(); t = torch.randn(C, device="cuda", generator=g).half()
        y = torch.empty_like(x); stats = torch.zeros(2 * G, device="cuda", dtype=torch.float64)
        assert K.osb_channel_add_stats(x.data_ptr(), t.data_ptr(), y.data_ptr(), F16, C, HW, G, stats.data_ptr(), _stream()) == 0
        torch.cuda.synchronize()
        want_y = (x.float() + t.float()).half()
        assert torch.equal(y, want_y)
        yd = y.double().reshape(HW, G, C // G)
        want = torch.stack([yd.sum(dim=(0, 2)), (yd * yd).sum(dim=(0, 2))], dim=1).reshape(-1)
        scale = torch.stack([yd.abs().sum(dim=(0, 2)), (yd * yd).sum(dim=(0, 2))], dim=1).reshape(-1)
        assert float(((stats - want).abs() / scale).max()) <= 2e-5


def test_qu8_gemm_and_conv_bit_exact(K):
    """W8A8 kernels against XNNPACK's fp32 requantisation, restated in numpy: acc = sum (x-zx)(w-zw) + bias;
    y = clamp(lrintf(acc * (sx*sw/sy)) + zy, 0, 255) (SURVEY section 8c: verified bit-exact against xnn qu8 FC).  Bit-exact."""
    import torch
    vp, i64, ci, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    K.osb_gemm_qu8.argtypes = [vp, vp, vp, vp, i64, i64, i64, ci, cf, ci, cf, ci, cf, vp]
    K.osb_conv2d_qu8.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, ci, cf, ci, cf, ci, cf, vp]
    rng = np.random.default_rng(3)
    zx, sx, zw, sw, zy, sy = 121, 0.031, 134, 0.0035, 117, 0.09
    scale = np.float32(np.float32(np.float32(sx) * np.float32(sw)) / np.float32(sy))

    def requant(acc):
        f = (acc.astype(np.float32) * scale).astype(np.float32)
        f = np.minimum(np.maximum(f, np.float32(0 - zy)), np.float32(255 - zy))
        return (np.rint(f).astype(np.int32) + zy).astype(np.uint8)

    M, N, Kd = 200, 136, 320
    a = rng.integers(0, 256, (M, Kd), dtype=np.uint8); b = rng.integers(0, 256, (Kd, N), dtype=np.uint8)
    bias = rng.integers(-2000, 2000, (N,), dtype=np.int32)
    ref = requant((a.astype(np.int32) - zx) @ (b.astype(np.int32) - zw) + bias)
    ta, tb, tbias = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), torch.from_numpy(bias).cuda()
    tc = torch.zeros((M, N), dtype=torch.uint8, device="cuda")
    assert K.osb_gemm_qu8(ta.data_ptr(), tb.data_ptr(), tc.data_ptr(), tbias.data_ptr(), M, N, Kd, zx, sx, zw, sw, zy, sy, _stream()) == 0
    torch.cuda.synchronize()
    assert np.array_equal(tc.cpu().numpy(), ref)

    H = W = 12; Cin, Cout, k = 24, 40, 3
    x = rng.integers(0, 256, (H, W, Cin), dtype=np.uint8); w = rng.integers(0, 256, (Cout, k, k, Cin), dtype=np.uint8)
    xp = np.full((H + 2, W + 2, Cin), zx, np.int32); xp[1:-1, 1:-1] = x          # XNNPACK pads with the input zero point
    acc = np.zeros((H, W, Cout), np.int64)
    for ky in range(k):
        for kx in range(k):
            acc += (xp[ky:ky + H, kx:kx + W].astype(np.int64) - zx) @ (w[:, ky, kx].astype(np.int64) - zw).T
    ref = requant(acc.astype(np.int32) + bias[:Cout])
    tx, tw = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda()
    ty = torch.zeros((H, W, Cout), dtype=torch.uint8, device="cuda")
    assert K.osb_conv2d_qu8(tx.data_ptr(), tw.data_ptr(), tbias.data_ptr(), ty.data_ptr(), H, W, Cin, Cout, k, k, 1, 1, 1, H, W, zx, sx, zw, sw, zy, sy, _stream()) == 0
    torch.cuda.synchronize()
    assert np.array_equal(ty.cpu().numpy(), ref)


def test_gemv_w8_in_register_dequant(K):
    """uint8-weight decode GEMV: identical operands to 'dequantise the blob to fp16, then GEMV' (the reference's load-time conversion)."""
    import torch
    vp, i64, ci, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    K.osb_gemv_w8.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, cf, ci, ci, vp]
    for (M, N, Kd) in [(1, 2048, 2048), (1, 5632, 2048), (2, 2048, 5632), (1, 32016, 2048)]:
        g = torch.Generator(device="cuda").manual_seed(N)
        a = torch.randn(M, Kd, device="cuda", generator=g).half()
        wq = torch.randint(0, 256, (Kd, N), device="cuda", generator=g, dtype=torch.uint8)
        scale, zp = 0.0037, 131
        res = torch.randn(M, N, device="cuda", generator=g).half()
        c = torch.empty(M, N, device="cuda", dtype=torch.half)
        assert K.osb_gemv_w8(a.data_ptr(), wq.data_ptr(), c.data_ptr(), None, res.data_ptr(), M, N, Kd, scale, zp, F16, _stream()) == 0
        torch.cuda.synchronize()
        wd = ((wq.int() - zp).float() * np.float32(scale)).half().double()
        ref = a.double() @ wd + res.double()
        absref = a.double().abs() @ wd.abs() + res.double().abs()
        _check(c, ref, absref, f"gemv_w8 {M}x{N}x{Kd}")


QU8_TC_GEMM = [(200, 144, 320, 0), (200, 144, 320, 1), (4096, 320, 320, 0), (1024, 1280, 640, 0), (77, 64, 768, 0), (512, 5120, 640, 1), (300, 48, 1040, 0)]


@pytest.mark.parametrize("M,N,Kd,bt", QU8_TC_GEMM)
def test_qu8_tensor_core_gemm_bit_exact(K, M, N, Kd, bt):
    """wgmma .u8 on raw uint8 bytes + zero-point terms from row / column sums + XNNPACK's fp32 requantisation: bit-exact
    against the integer restatement (the one tests/test_cpu.py and the model-level chain test pin to the reference's XNNPACK run).
    Both weight layouts: [K,N] (ONNX MatMul, MN-major B operand) and [N,K]."""
    import torch
    vp, i64, ci, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    K.osb_qu8_tc_gemm.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, ci, ci, cf, ci, cf, ci, cf, vp]
    K.osb_qu8_tc_gemm_ok.argtypes = [i64, i64, i64, vp, vp, vp]
    K.osb_rowsum_u8.argtypes = [vp, vp, i64, i64, vp]; K.osb_colsum_u8.argtypes = [vp, vp, i64, i64, vp]
    rng = np.random.default_rng(M + N)
    zx, sx, zw, sw, zy, sy = 121, 0.031, 134, 0.0035, 117, 0.09
    a = rng.integers(0, 256, (M, Kd), dtype=np.uint8)
    b = rng.integers(0, 256, (N, Kd) if bt else (Kd, N), dtype=np.uint8)
    bias = rng.integers(-2000, 2000, (N,), dtype=np.int32)
    bm = b.T if bt else b
    acc = (a.astype(np.int64) - zx) @ (bm.astype(np.int64) - zw) + bias
    scale = np.float32(np.float32(np.float32(sx) * np.float32(sw)) / np.float32(sy))
    f = (acc.astype(np.int32).astype(np.float32) * scale).astype(np.float32)
    f = np.minimum(np.maximum(f, np.float32(0 - zy)), np.float32(255 - zy))
    ref = (np.rint(f).astype(np.int32) + zy).astype(np.uint8)
    ta, tb, tbias = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), torch.from_numpy(bias).cuda()
    tc = torch.zeros((M, N), dtype=torch.uint8, device="cuda")
    assert K.osb_qu8_tc_gemm_ok(M, N, Kd, ta.data_ptr(), tb.data_ptr(), tc.data_ptr()) == 1
    rs = torch.zeros(M, dtype=torch.int32, device="cuda"); cs = torch.zeros(N, dtype=torch.int32, device="cuda")
    assert K.osb_rowsum_u8(ta.data_ptr(), rs.data_ptr(), M, Kd, _stream()) == 0
    if bt:
        assert K.osb_rowsum_u8(tb.data_ptr(), cs.data_ptr(), N, Kd, _stream()) == 0
    else:
        assert K.osb_colsum_u8(tb.data_ptr(), cs.data_ptr(), Kd, N, _stream()) == 0
    assert K.osb_qu8_tc_gemm(ta.data_ptr(), tb.data_ptr(), tc.data_ptr(), tbias.data_ptr(), rs.data_ptr(), cs.data_ptr(), M, N, Kd, bt, zx, sx, zw, sw, zy, sy, _stream()) == 0
    torch.cuda.synchronize()
    assert np.array_equal(rs.cpu().numpy(), a.astype(np.int64).sum(1))
    assert np.array_equal(cs.cpu().numpy(), bm.astype(np.int64).sum(0))
    got = tc.cpu().numpy()
    assert np.array_equal(got, ref), f"{int((got != ref).sum())} of {ref.size} bytes differ"


@pytest.mark.parametrize("H,W,Cin,Cout,k,s", [(12, 12, 32, 48, 3, 1), (64, 64, 320, 320, 3, 1), (32, 32, 640, 320, 1, 1), (33, 20, 64, 64, 3, 2), (16, 16, 1280, 1280, 3, 1)])
def test_qu8_tensor_core_conv_bit_exact(K, H, W, Cin, Cout, k, s):
    """kind::i8 implicit-GEMM conv on the zero-point-padded image (XNNPACK pads with the input zero point), bit-exact."""
    import torch
    vp, i64, ci, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    K.osb_qu8_tc_conv.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, i64, i64, ci, cf, ci, cf, ci, cf, vp]
    K.osb_pad_sum_u8.argtypes = [vp, vp, vp, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    K.osb_rowsum_u8.argtypes = [vp, vp, i64, i64, vp]
    rng = np.random.default_rng(H + Cin)
    zx, sx, zw, sw, zy, sy = 119, 0.027, 131, 0.0041, 120, 0.11 * (Cin / 64) ** 0.5
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    Hp, Wp = (Ho - 1) * s + k, (Wo - 1) * s + k
    x = rng.integers(0, 256, (H, W, Cin), dtype=np.uint8); w = rng.integers(0, 256, (Cout, k, k, Cin), dtype=np.uint8)
    bias = rng.integers(-3000, 3000, (Cout,), dtype=np.int32)
    xp = np.full((Hp, Wp, Cin), zx, np.int64); xp[pad:pad + H, pad:pad + W] = x
    acc = np.zeros((Ho, Wo, Cout), np.int64)
    for ky in range(k):
        for kx in range(k):
            acc += (xp[ky:ky + (Ho - 1) * s + 1:s, kx:kx + (Wo - 1) * s + 1:s] - zx) @ (w[:, ky, kx].astype(np.int64) - zw).T
    acc = acc + bias
    scale = np.float32(np.float32(np.float32(sx) * np.float32(sw)) / np.float32(sy))
    f = (acc.astype(np.int32).astype(np.float32) * scale).astype(np.float32)
    f = np.minimum(np.maximum(f, np.float32(0 - zy)), np.float32(255 - zy))
    ref = (np.rint(f).astype(np.int32) + zy).astype(np.uint8)
    tx, tw, tbias = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(bias).cuda()
    txp = torch.zeros((Hp, Wp, Cin), dtype=torch.uint8, device="cuda"); tps = torch.zeros(Hp * Wp, dtype=torch.int32, device="cuda")
    tcs = torch.zeros(Cout, dtype=torch.int32, device="cuda"); ty = torch.zeros((Ho, Wo, Cout), dtype=torch.uint8, device="cuda")
    assert K.osb_pad_sum_u8(tx.data_ptr(), txp.data_ptr(), tps.data_ptr(), H, W, Cin, Hp, Wp, pad, pad, zx, _stream()) == 0
    assert K.osb_rowsum_u8(tw.data_ptr(), tcs.data_ptr(), Cout, k * k * Cin, _stream()) == 0
    assert K.osb_qu8_tc_conv(txp.data_ptr(), tps.data_ptr(), tw.data_ptr(), tbias.data_ptr(), tcs.data_ptr(), ty.data_ptr(), Hp, Wp, Cin, Cout, k, k, s, Ho, Wo,
                             zx, sx, zw, sw, zy, sy, _stream()) == 0
    torch.cuda.synchronize()
    assert np.array_equal(txp.cpu().numpy(), xp.astype(np.uint8))
    got = ty.cpu().numpy()
    assert np.array_equal(got, ref), f"{int((got != ref).sum())} of {ref.size} bytes differ"


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("T,Tk,h,d", [(256, 256, 4, 40), (192, 77, 8, 40), (64, 64, 2, 160)])
def test_gemm_head_views(K, impl, T, Tk, h, d):
    """osb_gemm_ld on per-head slices of [T, h*d] projections (the fused multi-head-attention step): S = Q_h K_h^T with a padded
    leading dimension, then O[:, h*d:(h+1)*d] = P_h V_h written in place into the merged layout."""
    import torch
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    K.osb_gemm_ld.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    C = h * d
    Tkp = (Tk + 7) // 8 * 8
    g = torch.Generator(device="cuda").manual_seed(T + Tk)
    q = torch.randn(T, C, device="cuda", generator=g).half()
    k = torch.zeros(Tkp, C, device="cuda", dtype=torch.half); k[:Tk] = torch.randn(Tk, C, device="cuda", generator=g).half()
    v = torch.zeros(Tkp, C, device="cuda", dtype=torch.half); v[:Tk] = torch.randn(Tk, C, device="cuda", generator=g).half()
    S = torch.full((h, T, Tkp), float("nan"), device="cuda", dtype=torch.half)
    rc = K.osb_gemm_ld(q.data_ptr(), C, k.data_ptr(), C, S.data_ptr(), Tkp, None, None, h, T, Tkp, d, d, d, T * Tkp, 1, F16, impl, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    qh = q.double().view(T, h, d).permute(1, 0, 2)
    kh = k.double().view(Tkp, h, d).permute(1, 0, 2)
    ref = qh @ kh.transpose(1, 2)
    _check(S, ref, qh.abs() @ kh.abs().transpose(1, 2), "QK head views")
    P = torch.softmax(S.float(), dim=-1).half()
    P[:, :, Tk:] = 0
    O = torch.full((T, C), float("nan"), device="cuda", dtype=torch.half)
    rc = K.osb_gemm_ld(P.data_ptr(), Tkp, v.data_ptr(), C, O.data_ptr(), C, None, None, h, T, d, Tkp, T * Tkp, d, d, 0, F16, impl, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    vh = v.double().view(Tkp, h, d).permute(1, 0, 2)
    ref = (P.double() @ vh).permute(1, 0, 2).reshape(T, C)
    absref = (P.double().abs() @ vh.abs()).permute(1, 0, 2).reshape(T, C)
    _check(O, ref, absref, "PV head views")


@pytest.mark.parametrize("T,Tk,h,d", [(128, 128, 1, 64), (256, 384, 2, 40), (200, 77, 4, 40), (64, 30, 2, 32), (300, 200, 3, 64), (4096, 4096, 8, 40), (1024, 1024, 10, 64)])
def test_flash_attention(K, T, Tk, h, d):
    """Fused wgmma attention against softmax(QK^T s)V in fp64 on the fp16-rounded operands.  Tolerance: P is rounded to
    fp16 before the second MMA (as the reference's fp16 softmax output is), so |err| <= 2^-9 * sum|p_i v_i| + 2^-10 |ref|."""
    import torch
    vp, i64, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float
    K.osb_flash_attention.argtypes = [vp, i64, vp, i64, vp, i64, vp, i64, i64, i64, i64, i64, cf, vp]
    C = h * d
    g = torch.Generator(device="cuda").manual_seed(T * 3 + Tk)
    q = torch.randn(T, C, device="cuda", generator=g).half()
    k = torch.randn(Tk, C, device="cuda", generator=g).half()
    v = torch.randn(Tk, C, device="cuda", generator=g).half()
    o = torch.full((T, C), float("nan"), device="cuda", dtype=torch.half)
    scale = 1.0 / d ** 0.5
    rc = K.osb_flash_attention(q.data_ptr(), C, k.data_ptr(), C, v.data_ptr(), C, o.data_ptr(), C, h, T, Tk, d, scale, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    qh = q.double().view(T, h, d).permute(1, 0, 2); kh = k.double().view(Tk, h, d).permute(1, 0, 2); vh = v.double().view(Tk, h, d).permute(1, 0, 2)
    P = torch.softmax(qh @ kh.transpose(1, 2) * scale, dim=-1)
    ref = (P @ vh).permute(1, 0, 2).reshape(T, C)
    absref = (P @ vh.abs()).permute(1, 0, 2).reshape(T, C)
    err = (o.double() - ref).abs()
    tol = absref * 2.0 ** -8 + ref.abs() * 2.0 ** -9 + 1e-4
    assert not torch.isnan(o).any()
    assert not (err > tol).any(), f"max err {float(err.max()):.4g}, ref max {float(ref.abs().max()):.4g}, bad {(err > tol).sum().item()}"


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("rows,cols", [(4096, 320), (1024, 640), (256, 1280), (77, 768), (64, 1282), (33, 7), (5, 2048)])
def test_layer_norm(K, dtype, rows, cols):
    """Warp-per-row (register-resident) and block-per-row LayerNorm against fp64 math on the same inputs."""
    import torch
    torch.manual_seed(rows * 31 + cols)
    td = torch.float16 if dtype == F16 else torch.float32
    x = (torch.randn(rows, cols, device="cuda") * 3 + 0.5).to(td)
    g = torch.randn(cols, device="cuda").to(td)
    b = torch.randn(cols, device="cuda").to(td)
    y = torch.full((rows, cols), float("nan"), device="cuda", dtype=td)
    vp, i64, ci, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    K.osb_layer_norm.argtypes = [vp, vp, ci, i64, i64, vp, vp, cf, vp]
    rc = K.osb_layer_norm(x.data_ptr(), y.data_ptr(), dtype, rows, cols, g.data_ptr(), b.data_ptr(), 1e-5, _stream())
    torch.cuda.synchronize()
    assert rc == 0
    xd = x.double()
    ref = (xd - xd.mean(1, keepdim=True)) / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-5) * g.double() + b.double()
    tol = (2.0 ** -10 if dtype == F16 else 2.0 ** -20) * (ref.abs() + 4.0)
    err = (y.double() - ref).abs()
    assert not (err > tol).any(), f"max err {float(err.max()):.4g}"


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("C,HW,silu", [(320, 4096, 1), (640, 1024, 1), (1280, 64, 0), (2560, 256, 1), (960, 4096, 1), (32, 256, 0)])
def test_group_norm_nhwc(K, dtype, C, HW, silu):
    """GroupNorm(32) (+SiLU) on NHWC activations: single-launch rendezvous kernel / two-pass fallback vs fp64 math."""
    import torch
    torch.manual_seed(C + HW)
    td = torch.float16 if dtype == F16 else torch.float32
    x = (torch.randn(HW, C, device="cuda") * 2 + 0.25).to(td)
    g = torch.randn(C, device="cuda").to(td)
    b = torch.randn(C, device="cuda").to(td)
    y = torch.full((HW, C), float("nan"), device="cuda", dtype=td)
    scratch = torch.zeros(2048, device="cuda", dtype=torch.uint8)
    vp, i64, ci, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    K.osb_group_norm.argtypes = [vp, vp, ci, ci, i64, i64, ci, vp, vp, cf, ci, vp, vp]
    for _ in range(2):     # second launch checks that the kernel re-armed its scratch
        rc = K.osb_group_norm(x.data_ptr(), y.data_ptr(), dtype, 1, C, HW, 32, g.data_ptr(), b.data_ptr(), 1e-5, silu, scratch.data_ptr(), _stream())
        assert rc == 0
    torch.cuda.synchronize()
    xd = x.double().view(HW, 32, C // 32)
    mean = xd.mean(dim=(0, 2), keepdim=True)
    var = xd.var(dim=(0, 2), unbiased=False, keepdim=True)
    ref = ((xd - mean) / torch.sqrt(var + 1e-5)).view(HW, C) * g.double() + b.double()
    if silu:
        ref = ref * torch.sigmoid(ref)
    tol = (2.0 ** -9 if dtype == F16 else 2.0 ** -18) * (ref.abs() + 4.0)
    err = (y.double() - ref).abs()
    assert not (err > tol).any(), f"max err {float(err.max()):.4g}"


@pytest.mark.parametrize("groups,M,N,Kd", [(3, 4096, 320, 320), (3, 1024, 640, 640), (2, 77, 1280, 768), (3, 256, 1280, 1280), (2, 64, 1280, 1280), (3, 200, 136, 72)])
def test_gemm_grouped(K, groups, M, N, Kd):
    """q/k/v projections as one grouped tensor-core launch: every member must equal its stand-alone GEMM reference."""
    import torch
    torch.manual_seed(M + N + Kd)
    a = torch.randn(M, Kd, device="cuda").half()
    bs = [torch.randn(Kd, N, device="cuda").half() for _ in range(groups)]
    cs = [torch.full((M, N), float("nan"), device="cuda", dtype=torch.half) for _ in range(groups)]
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    K.osb_gemm_grouped.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(vp), ci, i64, i64, i64, ci, ci, ci, vp]
    B = (vp * groups)(*[b.data_ptr() for b in bs])
    C = (vp * groups)(*[c.data_ptr() for c in cs])
    K.osb_launch_count_reset()
    rc = K.osb_gemm_grouped(a.data_ptr(), B, C, groups, M, N, Kd, 0, F16, 0, _stream())
    torch.cuda.synchronize()
    assert rc == 0
    if N % 8 == 0 and Kd % 8 == 0 and M >= 32:
        assert K.osb_tc_launch_count() == 1, "expected ONE tensor-core launch for the whole group"
    for g in range(groups):
        ref = a.double() @ bs[g].double()
        absref = a.double().abs() @ bs[g].double().abs()
        _check(cs[g], ref, absref, f"grouped gemm member {g}")


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("rows,inner", [(4096, 1280), (256, 5120), (77, 12), (5, 7)])
def test_geglu(K, dtype, rows, inner):
    import torch
    torch.manual_seed(rows + inner)
    td = torch.float16 if dtype == F16 else torch.float32
    x = (torch.randn(rows, 2 * inner, device="cuda") * 2).to(td)
    y = torch.full((rows, inner), float("nan"), device="cuda", dtype=td)
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    K.osb_geglu.argtypes = [vp, vp, ci, i64, i64, vp]
    assert K.osb_geglu(x.data_ptr(), y.data_ptr(), dtype, rows, inner, _stream()) == 0
    torch.cuda.synchronize()
    xd = x.double()
    gate = xd[:, inner:]
    ref = xd[:, :inner] * (0.5 * gate * (1.0 + torch.erf(gate / 2.0 ** 0.5)))
    # fp32: 1 + erf(g / sqrt 2) cancels for negative gates, so the error scales with |a * g|, not with the (small) result
    scale = ref.abs() + (xd[:, :inner] * gate).abs() + 1.0
    tol = (2.0 ** -10 if dtype == F16 else 2.0 ** -20) * scale
    assert not ((y.double() - ref).abs() > tol).any()


ATTN_CASES = [
    # heads, Tq, Tk, d, dv, kv_group, mask, dtype
    (32, 1, 2048, 64, 64, 8, True, F16),      # TinyLlama decode: split-KV kernel
    (32, 1, 2048, 64, 64, 8, True, F32),
    (8, 1, 300, 64, 64, 2, False, F16),       # ragged last split
    (4, 3, 515, 80, 40, 1, True, F16),        # several query rows, d != dv, not a multiple of 8 halves per lane chunk
    (6, 2, 257, 20, 20, 3, True, F32),
    (4, 1, 100, 64, 64, 2, True, F16),        # short key axis: one warp per row
]


@pytest.mark.parametrize("heads,Tq,Tk,d,dv,group,with_mask,dtype", ATTN_CASES)
def test_attention_decode_matches_fp64(K, heads, Tq, Tk, d, dv, group, with_mask, dtype):
    import torch
    K.osb_attention.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_int64] * 5 + [ctypes.c_float, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]
    ty = torch.float16 if dtype == F16 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(heads * 1000 + Tk)
    q = torch.randn(heads, Tq, d, device="cuda", generator=g).to(ty)
    k = torch.randn(heads // group, Tk, d, device="cuda", generator=g).to(ty)
    v = torch.randn(heads // group, Tk, dv, device="cuda", generator=g).to(ty)
    mask = None
    if with_mask:
        mask = torch.zeros(Tq, Tk, device="cuda", dtype=ty)
        mask[:, Tk // 3: Tk // 3 + 40] = -65504.0 if dtype == F16 else -3.0e38     # a band of padded positions
        mask[:, :5] = -1.5
    scale = 1.0 / d ** 0.5
    out = torch.empty(heads, Tq, dv, device="cuda", dtype=ty)
    for rep in range(2):    # twice: the tickets must re-arm themselves
        out.zero_()
        rc = K.osb_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), mask.data_ptr() if with_mask else None, out.data_ptr(), heads, Tq, Tk, d, dv,
                             scale, 0, group, dtype, _stream())
        assert rc == 0
        torch.cuda.synchronize()
        kk = k.double().repeat_interleave(group, 0); vv = v.double().repeat_interleave(group, 0)
        s = q.double() @ kk.transpose(1, 2) * scale
        if with_mask:
            s = s + mask.double()
        ref = torch.softmax(s, -1) @ vv
        tol = 2e-3 if dtype == F16 else 1e-5
        assert float((out.double() - ref).abs().max()) <= tol * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("rows,cols,xd,wd,yd", [(1, 2048, F16, F16, F16), (3, 64, F32, F16, F32), (5, 1000, F16, F32, F32), (2, 5632, F32, F32, F32)])
def test_rms_norm_matches_fp64(K, rows, cols, xd, wd, yd):
    import torch
    K.osb_rms_norm.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p]
    T = {F16: torch.float16, F32: torch.float32}
    g = torch.Generator(device="cuda").manual_seed(rows * cols)
    x = (torch.randn(rows, cols, device="cuda", generator=g) * 3).to(T[xd])
    w = torch.randn(cols, device="cuda", generator=g).to(T[wd])
    y = torch.empty(rows, cols, device="cuda", dtype=T[yd])
    eps = 1e-5
    assert K.osb_rms_norm(x.data_ptr(), xd, w.data_ptr(), wd, y.data_ptr(), yd, rows, cols, eps, _stream()) == 0
    torch.cuda.synchronize()
    xx = x.double()
    ref = w.double() * (xx / torch.sqrt((xx * xx).mean(-1, keepdim=True) + eps))
    tol = 2e-3 if yd == F16 else 2e-6
    assert float((y.double() - ref).abs().max()) <= tol * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("rows,D,dtype", [(32, 64, F16), (4, 16, F32), (7, 128, F16)])
def test_rope_matches_the_op_chain(K, rows, D, dtype):
    """Slice / Neg / Concat / Mul / Mul / Add as separate roundings: the fused kernel must give the same bits in fp32 and the same
    values within one rounding in fp16 (src/onnxstream.cpp elementwise ops round after each op)."""
    import torch
    K.osb_rope.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p]
    ty = torch.float16 if dtype == F16 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(rows * D)
    x = torch.randn(rows, D, device="cuda", generator=g).to(ty)
    ang = torch.rand(D, device="cuda", generator=g) * 6.28
    cs, sn = torch.cos(ang).to(ty), torch.sin(ang).to(ty)
    y = torch.empty_like(x)
    assert K.osb_rope(x.data_ptr(), cs.data_ptr(), sn.data_ptr(), y.data_ptr(), dtype, rows, D, 1, _stream()) == 0
    torch.cuda.synchronize()
    rot = torch.cat([-x[:, D // 2:], x[:, :D // 2]], -1)
    ref = (x * cs).to(ty) + (rot * sn).to(ty)
    if dtype == F32:
        assert torch.equal(y, ref)
    else:
        assert float((y.float() - ref.float()).abs().max()) <= 2e-3 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("dtype,w8,M,Ns,Kd", [(F16, False, 1, (2048, 256, 256), 2048), (F16, False, 1, (5632, 5632), 2048), (F32, False, 3, (512, 264), 300),
                                              (F16, True, 1, (2048, 256, 256), 2048), (F16, True, 2, (5632, 5632), 2048), (F32, True, 1, (512, 272), 320)])
def test_gemv_grouped_matches_fp64(K, dtype, w8, M, Ns, Kd):
    """q/k/v (or gate/up) decode projections as one launch: every group equals its own fp64 product; run twice (scratch and counters re-arm)."""
    import torch
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    K.osb_gemv_grouped.argtypes = [vp, vp, vp, vp, vp, vp, ci, i64, i64, ci, ci, vp]
    ty = torch.float16 if dtype == F16 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(sum(Ns) + Kd)
    a = torch.randn(M, Kd, device="cuda", generator=g).to(ty)
    n = len(Ns)
    scales, zps = [0.0031 + 0.001 * i for i in range(n)], [128 + 3 * i for i in range(n)]
    if w8:
        ws = [torch.randint(0, 256, (Kd, N), device="cuda", generator=g, dtype=torch.uint8) for N in Ns]
        wd = [((w.int() - z).float() * np.float32(s)).to(ty).double() for w, s, z in zip(ws, scales, zps)]
    else:
        ws = [(torch.randn(Kd, N, device="cuda", generator=g) * 0.05).to(ty) for N in Ns]
        wd = [w.double() for w in ws]
    cs = [torch.empty(M, N, device="cuda", dtype=ty) for N in Ns]
    B = (vp * n)(*[w.data_ptr() for w in ws]); C = (vp * n)(*[c.data_ptr() for c in cs])
    Nv = (i64 * n)(*Ns); sc = (ctypes.c_float * n)(*scales); zp = (ci * n)(*zps)
    for rep in range(2):
        for c in cs:
            c.zero_()
        assert K.osb_gemv_grouped(a.data_ptr(), B, C, Nv, sc, zp, n, M, Kd, 1 if w8 else dtype, dtype, _stream()) == 0
        torch.cuda.synchronize()
        for c, w in zip(cs, wd):
            ref = a.double() @ w
            absref = a.double().abs() @ w.abs()
            if dtype == F16:
                _check(c, ref, absref, f"gemv_grouped {M}x{tuple(Ns)}x{Kd}")
            else:
                assert float((c.double() - ref).abs().max()) <= 1e-5 * float(absref.max())
    # shapes the grouped kernels do not cover are refused, not mangled
    Nbad = (i64 * n)(*([100] * n))
    assert K.osb_gemv_grouped(a.data_ptr(), B, C, Nbad, sc, zp, n, M, Kd, 1 if w8 else dtype, dtype, _stream()) == 801


def test_gemv_padded_rows_and_concat2_and_silu_mul(K):
    import torch
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    # GEMV against a row-padded weight (vocabulary 32003 -> ld 32008)
    K.osb_gemm_ld.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    g = torch.Generator(device="cuda").manual_seed(5)
    N, Np, Kd = 32003, 32008, 512
    a = torch.randn(1, Kd, device="cuda", generator=g).half()
    w = torch.zeros(Kd, Np, device="cuda", dtype=torch.half)
    w[:, :N] = (torch.randn(Kd, N, device="cuda", generator=g) * 0.05).half()
    w[:, N:] = 7.0                                       # padding must never reach an output
    c = torch.full((1, N + 8), -1.0, device="cuda", dtype=torch.half)
    K.osb_launch_count_reset()
    assert K.osb_gemm_ld(a.data_ptr(), Kd, w.data_ptr(), Np, c.data_ptr(), N, None, None, 1, 1, N, Kd, 0, 0, 0, 0, F16, 0, _stream()) == 0
    torch.cuda.synchronize()
    ref = a.double() @ w[:, :N].double()
    _check(c[:, :N], ref, a.double().abs() @ w[:, :N].double().abs(), "gemv padded ld")
    assert bool((c[:, N:] == -1.0).all())
    # two-source concat
    K.osb_concat2.argtypes = [vp, vp, vp, i64, i64, i64, vp]
    x = torch.randn(4, 2047, 64, device="cuda", generator=g).half(); y = torch.randn(4, 1, 64, device="cuda", generator=g).half()
    o = torch.empty(4, 2048, 64, device="cuda", dtype=torch.half)
    assert K.osb_concat2(x.data_ptr(), y.data_ptr(), o.data_ptr(), 4, 2047 * 64 * 2, 64 * 2, _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(o, torch.cat([x, y], 1))
    assert K.osb_concat2(x.data_ptr(), y.data_ptr(), o.data_ptr(), 4, 2047 * 64 * 2, 6, _stream()) == 801     # not 16-byte granular: refused
    # silu(a) * b
    K.osb_binary.argtypes = [ci, vp, vp, vp, vp, vp, vp, ci, ci, vp]
    n = 5632
    ga = torch.randn(n, device="cuda", generator=g).half() * 3; ub = torch.randn(n, device="cuda", generator=g).half()
    out = torch.empty(n, device="cuda", dtype=torch.half)
    one = (i64 * 1)(1); shp = (i64 * 1)(n)
    assert K.osb_binary(6, ga.data_ptr(), one, ub.data_ptr(), one, out.data_ptr(), shp, 1, F16, _stream()) == 0
    torch.cuda.synchronize()
    ref = torch.nn.functional.silu(ga.double()) * ub.double()
    assert float((out.double() - ref).abs().max()) <= 2e-3 * max(1.0, float(ref.abs().max()))


F32X_GEMM = [(77, 768, 768), (77, 3072, 768), (77, 768, 3072), (4096, 320, 320), (256, 64, 40), (1000, 136, 100)]


@pytest.mark.parametrize("M,N,Kd", F32X_GEMM)
def test_f32_gemm_on_tensor_cores_bf16_triple_split(K, M, N, Kd):
    """fp32 MatMul through the tensor cores (bf16 triple split, six cross products in one contraction): as accurate as an fp32 FMA loop.
    Bar: |err| <= 1e-5 * sum|a_i b_i| over every output (a sequential fp32 FMA loop is bounded by K * 2^-24 = 2e-5 at K = 320; the tensor core
    aligns each group of products to the largest one before adding) -- three orders of magnitude below what a single bf16 or tf32 pass gives."""
    import torch
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    K.osb_bf16x3_expand_cols.argtypes = [vp, vp, i64, i64, i64, ci, vp]
    K.osb_bf16x3_expand_rows.argtypes = [vp, vp, i64, i64, ci, vp]
    K.osb_tc_gemm_f32x.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, ci, vp]
    K.osb_tc_gemm_f32x_ok.argtypes = [i64, i64, i64]
    assert K.osb_tc_gemm_f32x_ok(M, N, Kd) == 1
    g = torch.Generator(device="cuda").manual_seed(M + N + Kd)
    a = torch.randn(M, Kd, device="cuda", generator=g) * torch.exp(torch.randn(M, 1, device="cuda", generator=g) * 2)     # rows of very different scale
    b = torch.randn(Kd, N, device="cuda", generator=g) * 0.05
    bias = torch.randn(N, device="cuda", generator=g); res = torch.randn(M, N, device="cuda", generator=g)
    a6 = torch.empty(M, 6 * Kd, device="cuda", dtype=torch.bfloat16); b6 = torch.empty(6 * Kd, N, device="cuda", dtype=torch.bfloat16)
    c = torch.empty(M, N, device="cuda")
    assert K.osb_bf16x3_expand_cols(a.data_ptr(), a6.data_ptr(), M, Kd, Kd, 0, _stream()) == 0
    assert K.osb_bf16x3_expand_rows(b.data_ptr(), b6.data_ptr(), Kd, N, 1, _stream()) == 0
    torch.cuda.synchronize()
    # the three parts re-assemble the fp32 value to 24 bits
    parts = a6.view(M, 6, Kd).double()
    assert float(((parts[:, 0] + parts[:, 2] + parts[:, 4]) - a.double()).abs().max()) <= 2.0 ** -23 * float(a.abs().max())
    K.osb_launch_count_reset()
    assert K.osb_tc_gemm_f32x(a6.data_ptr(), b6.data_ptr(), c.data_ptr(), bias.data_ptr(), res.data_ptr(), M, N, 6 * Kd, 0, _stream()) == 0
    torch.cuda.synchronize()
    assert K.osb_tc_launch_count() >= 1
    ref = a.double() @ b.double() + bias.double() + res.double()
    absref = a.double().abs() @ b.double().abs() + bias.double().abs() + res.double().abs()
    err = (c.double() - ref).abs()
    worst = float((err / absref).max())
    print(f"f32x gemm {M}x{N}x{Kd}: max err / sum|ab| = {worst:.3g}")
    assert worst <= 1e-5, f"f32x gemm {M}x{N}x{Kd}: max err / sum|ab| = {worst:.3g}"
    # K-major B ([N][K], the conv-weight layout) through expand_cols
    bt = b.t().contiguous()
    bt6 = torch.empty(N, 6 * Kd, device="cuda", dtype=torch.bfloat16)
    assert K.osb_bf16x3_expand_cols(bt.data_ptr(), bt6.data_ptr(), N, Kd, Kd, 1, _stream()) == 0
    c2 = torch.empty(M, N, device="cuda")
    assert K.osb_tc_gemm_f32x(a6.data_ptr(), bt6.data_ptr(), c2.data_ptr(), None, None, M, N, 6 * Kd, 1, _stream()) == 0
    torch.cuda.synchronize()
    ref2 = a.double() @ b.double()
    worst2 = float(((c2.double() - ref2).abs() / (a.double().abs() @ b.double().abs())).max())
    assert worst2 <= 1e-5, f"f32x gemm K-major B {M}x{N}x{Kd}: max err / sum|ab| = {worst2:.3g}"


@pytest.mark.parametrize("H,W,Cin,Cout,k,stride", [(64, 64, 320, 320, 3, 1), (32, 32, 64, 128, 3, 2), (16, 16, 1280, 640, 1, 1), (40, 24, 12, 40, 3, 1)])
def test_f32_conv_on_tensor_cores_bf16_triple_split(K, H, W, Cin, Cout, k, stride):
    import torch
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    K.osb_bf16x3_expand_cols.argtypes = [vp, vp, i64, i64, i64, ci, vp]
    K.osb_tc_conv_f32x.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, vp]
    K.osb_tc_conv_f32x_ok.argtypes = [i64, i64, i64, i64, ci, ci, ci, i64, i64]
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    assert K.osb_tc_conv_f32x_ok(H, W, Cin, Cout, k, k, stride, Ho, Wo) == 1
    g = torch.Generator(device="cuda").manual_seed(H * Cin + Cout)
    x = torch.randn(1, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * 0.05
    bias = torch.randn(Cout, device="cuda", generator=g)
    xh = x[0].permute(1, 2, 0).contiguous()                     # [H][W][Cin]
    wo = w.permute(0, 2, 3, 1).contiguous()                     # OHWI
    x6 = torch.empty(H * W, 6 * Cin, device="cuda", dtype=torch.bfloat16); w6 = torch.empty(Cout * k * k, 6 * Cin, device="cuda", dtype=torch.bfloat16)
    y = torch.empty(Ho, Wo, Cout, device="cuda")
    assert K.osb_bf16x3_expand_cols(xh.data_ptr(), x6.data_ptr(), H * W, Cin, Cin, 0, _stream()) == 0
    assert K.osb_bf16x3_expand_cols(wo.data_ptr(), w6.data_ptr(), Cout * k * k, Cin, Cin, 1, _stream()) == 0
    assert K.osb_tc_conv_f32x(x6.data_ptr(), w6.data_ptr(), bias.data_ptr(), None, y.data_ptr(), H, W, 6 * Cin, Cout, k, k, stride, pad, pad, Ho, Wo, _stream()) == 0
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(x.double(), w.double(), bias.double(), stride=stride, padding=pad)[0].permute(1, 2, 0)
    absref = torch.nn.functional.conv2d(x.double().abs(), w.double().abs(), bias.double().abs(), stride=stride, padding=pad)[0].permute(1, 2, 0)
    worst = float(((y.double() - ref).abs() / absref).max())
    assert worst <= 1e-5, f"f32x conv: max err / sum|xw| = {worst:.3g}"
