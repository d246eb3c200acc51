"""The contraction kernels (osb_gemm_ld, osb_conv2d_ex, the GEMV family, the fp32 bf16-triple-split and uint8 entry points) on every
dispatch path, each case in two data regimes (tests/test_kernels_gpu.py: bit-exact on integer operands, and the fp32-accumulation bar
on Gaussian operands with rows of very different scale).

Tensor-core cases are pinned by the launch profile (osb_tc_profile_dump: one line "M N K taps batch split conv ..." per launch) or by
the launch counters.  CUDA-core cases cannot be observed from outside; each names the predicate in osb_gemm_ld / osb_conv2d_ex that
selects its kernel, and asserts the tensor-core eligibility predicates where they apply."""
import ctypes

import numpy as np
import pytest

from test_kernels_gpu import F16, F32, _check, _check_exact, _operands, _verify

pytestmark = pytest.mark.gpu

REGIMES = ("exact", "gauss")
INVALID_VALUE, NOT_READY, NOT_SUPPORTED = 1, 600, 801


@pytest.fixture(scope="module")
def K(engine_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = ctypes.CDLL(engine_lib)
    vp, i64, ci, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    lib.osb_gemm_ld.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_gemm.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_conv2d_ex.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, ci, ci, vp, vp, ci, ctypes.POINTER(ci)]
    lib.osb_conv2d_fusable.argtypes = [vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci]
    lib.osb_gemm_tc_eligible.argtypes = [i64, i64, i64, ci]
    lib.osb_gemv_w8.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, cf, ci, ci, vp]
    lib.osb_gemv_grouped.argtypes = [vp, vp, vp, vp, vp, vp, ci, i64, i64, ci, ci, vp]
    lib.osb_bf16x3_expand_cols.argtypes = [vp, vp, i64, i64, i64, ci, vp]
    lib.osb_bf16x3_expand_rows.argtypes = [vp, vp, i64, i64, ci, vp]
    lib.osb_tc_gemm_f32x.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, ci, vp]
    lib.osb_tc_gemm_f32x_ok.argtypes = [i64, i64, i64]
    lib.osb_tc_conv_f32x.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, vp]
    lib.osb_tc_conv_f32x_ok.argtypes = [i64, i64, i64, i64, ci, ci, ci, i64, i64]
    lib.osb_gemm_qu8.argtypes = [vp, vp, vp, vp, i64, i64, i64, ci, cf, ci, cf, ci, cf, vp]
    lib.osb_conv2d_qu8.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, ci, cf, ci, cf, ci, cf, vp]
    lib.osb_qu8_tc_conv.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, i64, i64, ci, cf, ci, cf, ci, cf, vp]
    lib.osb_qu8_tc_conv_ok.argtypes = [i64, i64, i64, i64, ci, ci, ci, vp, vp, vp]
    lib.osb_qu8_tc_gemm_ok.argtypes = [i64, i64, i64, vp, vp, vp]
    lib.osb_pad_sum_u8.argtypes = [vp, vp, vp, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_rowsum_u8.argtypes = [vp, vp, i64, i64, vp]
    lib.osb_workspace_release.argtypes = [vp]
    lib.osb_workspace_release.restype = None
    lib.osb_tc_profile.argtypes = [ci]
    lib.osb_tc_profile.restype = None
    lib.osb_tc_profile_dump.argtypes = [ctypes.c_char_p, ci]
    lib.osb_launch_count.restype = ctypes.c_uint64
    lib.osb_tc_launch_count.restype = ctypes.c_uint64
    lib.osb_launch_count_reset.restype = None
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _tc_profile(K, fn):
    """Runs fn() with the tensor-core launch profile on; returns one dict per launch (M, N, K, taps, batch, split, conv)."""
    import torch
    torch.cuda.synchronize()
    K.osb_tc_profile(1)
    try:
        fn()
        torch.cuda.synchronize()
        buf = ctypes.create_string_buffer(1 << 16)
        n = K.osb_tc_profile_dump(buf, len(buf))
        assert n >= 0
    finally:
        K.osb_tc_profile(0)
    keys = ("M", "N", "K", "taps", "batch", "split", "conv")
    return [dict(zip(keys, map(int, line.split()[:7]))) for line in buf.value.decode().splitlines()]


def _counted(K, fn):
    """Runs fn(); returns (launches, tensor-core launches)."""
    K.osb_launch_count_reset()
    fn()
    return int(K.osb_launch_count()), int(K.osb_tc_launch_count())


# ---- osb_gemm_ld: reference and one call ----------------------------------------------------------------------------------------------

def _gemm_problem(K, regime, seed, dtype, batch, M, N, Kd, bt, has_bias, has_res, lda=None, ldb=None, ldc=None, a_off=0, b_off=0, r_off=0,
                  shared=""):
    """Operands for C[b] = A[b] B[b] (+ bias) (+ residual) with the given leading dimensions / element offsets; `shared` = "a" / "b" makes
    that operand one matrix for every batch (stride 0).  Pad elements hold 7, so a read past a row shows."""
    import torch
    td = torch.half if dtype == F16 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(seed)
    lda, ldb, ldc = lda or Kd, ldb or (Kd if bt else N), ldc or N
    ba, bb = (1 if shared == "a" else batch), (1 if shared == "b" else batch)
    a, b, bias, res = _operands(regime, g, [(ba, M, Kd), (bb, N, Kd) if bt else (bb, Kd, N), (N,) if has_bias else None,
                                            (batch, M, N) if has_res else None], td, lim=3, row_scaled=1)
    if regime == "gauss" and dtype == F16:
        b = (b.float() * 0.25).half()

    def place(t, rows, ld, off):        # [nb, rows, cols] -> a padded, offset buffer; returns (buffer, view pointer)
        nb, _, cols = t.shape
        buf = torch.full((off + nb * rows * ld + 8,), 7.0, device="cuda", dtype=td)
        buf[off:off + nb * rows * ld].view(nb, rows, ld)[:, :, :cols] = t
        return buf, buf.data_ptr() + off * buf.element_size()

    abuf, pa = place(a, M, lda, a_off)
    bbuf, pb = place(b, N if bt else Kd, ldb, b_off)
    rbuf, pr = place(res, M, ldc, r_off) if has_res else (None, None)
    cbuf = torch.full((batch * M * ldc,), float("nan"), device="cuda", dtype=td)
    bd = b.double().transpose(1, 2) if bt else b.double()
    ref = a.double() @ bd
    absref = a.double().abs() @ bd.abs()
    if has_bias:
        ref = ref + bias.double(); absref = absref + bias.double().abs()
    if has_res:
        ref = ref + res.double(); absref = absref + res.double().abs()
    sa = 0 if shared == "a" else M * lda
    sb = 0 if shared == "b" else (N if bt else Kd) * ldb
    keep = (abuf, bbuf, rbuf, bias)

    def run(impl=0):
        return K.osb_gemm_ld(pa, lda, pb, ldb, cbuf.data_ptr(), ldc, _ptr(bias), pr, batch, M, N, Kd, sa, sb, M * ldc, bt, dtype, impl, _stream())

    def result():
        c = cbuf.view(batch, M, ldc)
        if ldc > N:
            assert bool(torch.isnan(c[:, :, N:]).all()), "a store landed in the pad columns of C"
        return c[:, :, :N]

    return run, result, ref, absref, keep


def _gemm_check(K, regime, path, case_id, seed, dtype, batch, M, N, Kd, bt, has_bias, has_res, impl=0, **kw):
    import torch
    run, result, ref, absref, keep = _gemm_problem(K, regime, seed, dtype, batch, M, N, Kd, bt, has_bias, has_res, **kw)
    launches = _counted(K, lambda: _rc0(run(impl)))
    torch.cuda.synchronize()
    _verify(regime, result(), ref, absref, f"{path} {case_id} {regime}")
    return launches


def _rc0(rc):
    assert rc == 0, f"rc = {rc}"


# ---- GEMV panel kernel (gemv_panel_kernel) ---------------------------------------------------------------------------------------------
# predicate in osb_gemm_ld: lda == K, ldc == N, M <= 8, batch == 1, !bt, ldb >= N, ldb % vec == 0, B 16-byte aligned, N >= 256, K >= 64,
# M * N <= OSB_WS_GEMV_FLOATS (and a scratch outside capture).  MAXM instantiations: M = 1, 2, <= 4, <= 8.

@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("epi", ["none", "bias", "bias+res"])
@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 8])
def test_gemv_panel_rows(K, M, dtype, epi, regime):
    N, Kd = 1000, 700      # ragged last column panel; K split over many k-slice CTAs, the last one short
    assert K.osb_gemm_tc_eligible(M, N, Kd, dtype) == 0
    n, tc = _gemm_check(K, regime, "gemv_panel", f"M={M} dt={dtype} {epi}", M * 31 + dtype, dtype, 1, M, N, Kd, 0, epi != "none", epi == "bias+res")
    assert (n, tc) == (1, 0), "one GEMV launch: panel kernel with in-kernel finish"


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("dtype,M", [(F16, 5), (F32, 3)])
def test_gemv_panel_row_padded_ldb(K, dtype, M, regime):
    """ldb > N (a row-padded weight, e.g. a 32003-entry vocabulary stored 32008 wide): the pad columns (7.0) never reach C."""
    N, ldb = 1003, 1008
    n, tc = _gemm_check(K, regime, "gemv_panel", f"ldb={ldb}", 7 + M, dtype, 1, M, N, 512, 0, True, True, ldb=ldb)
    assert (n, tc) == (1, 0)


# ---- skinny_gemm_kernel: dense, M <= 8, batch 1, when the GEMV predicate fails ----------------------------------------------------------

SKINNY = [
    # id, dtype, M, N, K, bt, b_off: the failing GEMV condition
    ("bt-M1", F16, 1, 300, 1000, 1, 0),         # b_transposed: warp-per-column branch
    ("bt-M3", F32, 3, 300, 1000, 1, 0),
    ("bt-M8", F16, 8, 520, 333, 1, 0),
    ("N<256", F16, 4, 200, 300, 0, 0),          # [K, N] branch: N < 256
    ("K<64", F32, 2, 512, 40, 0, 0),            # K < 64
    ("B+1", F16, 3, 512, 256, 0, 1),            # B offset by one element: not 16-byte aligned, scalar loads
    ("ldb%8", F16, 2, 1001, 128, 0, 0),         # ldb = N = 1001: ldb % vec != 0
]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("cid,dtype,M,N,Kd,bt,b_off", SKINNY)
def test_skinny_gemm(K, cid, dtype, M, N, Kd, bt, b_off, regime):
    n, tc = _gemm_check(K, regime, "skinny", cid, N + Kd, dtype, 1, M, N, Kd, bt, True, True, b_off=b_off)
    assert (n, tc) == (1, 0)


@pytest.mark.parametrize("regime", REGIMES)
def test_skinny_gemm_beyond_gemv_scratch(K, regime):
    """M * N = 8 * 262152 > OSB_WS_GEMV_FLOATS (2^21): the panel GEMV has no room for its sums, the skinny kernel takes it."""
    n, tc = _gemm_check(K, regime, "skinny", "M*N>scratch", 5, F16, 1, 8, 262152, 64, 0, True, False)
    assert (n, tc) == (1, 0)


# ---- igemm_kernel (CUDA cores): every fp32 GEMM with M > 8 or batch > 1, and fp16 shapes the tensor cores refuse -------------------------

IGEMM = [
    # id, dtype, batch, M, N, K, bt, bias, res, a_off
    ("f32", F32, 1, 100, 72, 200, 0, True, True, 0),
    ("f32-bt", F32, 1, 77, 130, 96, 1, True, False, 0),
    ("f32-batch3", F32, 3, 40, 64, 48, 0, False, True, 0),
    ("f32-M1-batch2", F32, 2, 1, 300, 100, 1, True, False, 0),   # M <= 8 but batch > 1: not skinny
    ("f16-M<32-batch2", F16, 2, 20, 64, 64, 0, True, True, 0),   # osb_tc_gemm_ok: M < 32
    ("f16-N%8", F16, 1, 64, 100, 64, 0, True, True, 0),          # N % 8 != 0
    ("f16-K%8", F16, 1, 64, 64, 100, 1, True, False, 0),         # K % 8 != 0
    ("f16-A+1", F16, 1, 64, 64, 64, 0, False, True, 1),          # A not 16-byte aligned
]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("cid,dtype,batch,M,N,Kd,bt,has_bias,has_res,a_off", IGEMM)
def test_igemm_gemm(K, cid, dtype, batch, M, N, Kd, bt, has_bias, has_res, a_off, regime):
    if dtype == F16 and not a_off:
        assert K.osb_gemm_tc_eligible(M, N, Kd, dtype) == 0
    n, tc = _gemm_check(K, regime, "gemm_igemm", cid, M + N + Kd, dtype, batch, M, N, Kd, bt, has_bias, has_res, a_off=a_off)
    assert (n, tc) == (1, 0)


# ---- tensor-core GEMM launcher ----------------------------------------------------------------------------------------------------------
# split-K shapes: 2 output tiles and 64 k-blocks -> choose_split gives min(SMs / 2, 32) splits on any H100 (>= 114 SMs)

TC_GEMM = [
    # id, batch, M, N, K, bt, bias, res, kwargs, expected (batch, split) per launch: split ">1" or 1
    ("K8-N8", 1, 64, 8, 8, 0, True, True, {}, [(1, 1)]),
    ("K16-N8-bt", 1, 200, 8, 16, 1, True, False, {}, [(1, 1)]),
    ("K24", 1, 130, 136, 24, 0, True, True, {}, [(1, 1)]),
    ("K24-bt", 1, 130, 136, 24, 1, False, True, {}, [(1, 1)]),
    ("splitK", 1, 128, 256, 4096, 0, True, True, {}, [(1, ">1")]),
    ("splitK-bt", 1, 128, 256, 4096, 1, True, True, {}, [(1, ">1")]),      # bias and residual with K-major B through the reduce
    ("splitK-batch2", 2, 128, 128, 4096, 0, True, True, {}, [(2, ">1")]),
    ("ldc!=N", 1, 128, 128, 4096, 0, True, True, {"ldc": 136}, [(1, 1)]),   # split-K forced off: the reduce writes dense rows
    ("fold-shared-B", 3, 128, 64, 128, 0, True, True, {"shared": "b"}, [(1, 1)] * 3),
    ("fold-shared-A", 3, 64, 64, 136, 1, True, False, {"shared": "a"}, [(1, 1)] * 3),
    ("residual+1", 1, 128, 256, 4096, 0, True, True, {"r_off": 1}, [(1, 1)]),   # residual not 8-byte aligned: unsplit, scalar reads
]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("cid,batch,M,N,Kd,bt,has_bias,has_res,kw,want", TC_GEMM)
def test_tc_gemm(K, cid, batch, M, N, Kd, bt, has_bias, has_res, kw, want, regime):
    import torch
    run, result, ref, absref, keep = _gemm_problem(K, regime, M + Kd, F16, batch, M, N, Kd, bt, has_bias, has_res, **kw)
    prof = _tc_profile(K, lambda: _rc0(run(2)))
    got = [(p["batch"], p["split"] if p["split"] == 1 else ">1") for p in prof]
    assert got == want, f"launches {prof}"
    assert all((p["M"], p["N"], p["K"], p["conv"]) == (M, N, Kd, 0) for p in prof)
    torch.cuda.synchronize()
    _verify(regime, result(), ref, absref, f"gemm_tc {cid} {regime}")


def test_tc_gemm_pair_residual_misaligned(K):
    """The CTA-pair path reads the residual as scalars too: a residual offset by one element is fine there."""
    import torch
    K.osb_tc_set_pair_mode.argtypes = [ctypes.c_int]
    K.osb_tc_set_pair_mode.restype = None
    K.osb_tc_set_pair_mode(2)
    try:
        for regime in REGIMES:
            run, result, ref, absref, keep = _gemm_problem(K, regime, 3, F16, 1, 256, 128, 256, 0, True, True, r_off=1)
            n, tc = _counted(K, lambda: _rc0(run(2)))
            assert tc == 1
            torch.cuda.synchronize()
            _verify(regime, result(), ref, absref, f"gemm_tc pair residual+1 {regime}")
    finally:
        K.osb_tc_set_pair_mode(1)


# ---- convolution: tensor-core split-K and residual alignment; fp32 on the CUDA cores -------------------------------------------------------

def _conv_problem(K, regime, seed, dtype, H, W, Cin, Cout, kh, kw, s, pt, pl, has_bias, has_res, r_off=0, lim=3):
    import torch
    import torch.nn.functional as Fn
    td = torch.half if dtype == F16 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(seed)
    Ho, Wo = (H + 2 * pt - kh) // s + 1, (W + 2 * pl - kw) // s + 1
    x, w, bias, res = _operands(regime, g, [(H, W, Cin), (Cout, kh, kw, Cin), (Cout,) if has_bias else None, (Ho, Wo, Cout) if has_res else None],
                                torch.float32, lim=lim)
    if regime == "gauss":
        w = w / (kh * kw * Cin) ** 0.5
    x, w = x.to(td), w.to(td)
    bias = bias.to(td) if has_bias else None
    rbuf = None
    if has_res:
        res = res.to(td)
        rbuf = torch.empty(r_off + res.numel() + 8, device="cuda", dtype=td)
        rbuf[r_off:r_off + res.numel()] = res.reshape(-1)
    y = torch.full((Ho, Wo, Cout), float("nan"), device="cuda", dtype=td)
    xn, wn = x.double().permute(2, 0, 1)[None], w.double().permute(0, 3, 1, 2)
    ref = Fn.conv2d(xn, wn, None, stride=s, padding=(pt, pl))[0].permute(1, 2, 0)
    absref = Fn.conv2d(xn.abs(), wn.abs(), None, stride=s, padding=(pt, pl))[0].permute(1, 2, 0)
    if has_bias:
        ref = ref + bias.double(); absref = absref + bias.double().abs()
    if has_res:
        ref = ref + res.double(); absref = absref + res.double().abs()
    pr = rbuf.data_ptr() + r_off * rbuf.element_size() if has_res else None

    def run(impl, bias2=None):
        return K.osb_conv2d_ex(x.data_ptr(), w.data_ptr(), _ptr(bias), bias2, pr, y.data_ptr(), H, W, Cin, Cout, kh, kw, s, pt, pl, Ho, Wo, dtype, impl,
                      _stream(), None, 0, None)

    return run, y, ref, absref, (x, w, bias, rbuf)


TC_CONV = [
    # id, H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left, residual offset, expected split
    ("splitK-Cout132", 8, 8, 1280, 132, 3, 3, 1, 1, 1, 0, ">1"),     # Cout % 4 == 0, % 8 != 0, through the reduce kernel
    ("splitK-Conv1D", 64, 1, 1280, 128, 3, 1, 1, 1, 0, 0, ">1"),     # Conv1D (bw = 1, bh = 128) through the reduce kernel
    ("splitK-residual+1", 8, 8, 1280, 128, 3, 3, 1, 1, 1, 1, 1),     # residual not 8-byte aligned: unsplit
    ("Cout3", 32, 32, 16, 3, 3, 3, 1, 1, 1, 0, 1),                   # ragged Cout: scalar epilogue
]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("cid,H,W,Cin,Cout,kh,kw,s,pt,pl,r_off,want", TC_CONV)
def test_tc_conv(K, cid, H, W, Cin, Cout, kh, kw, s, pt, pl, r_off, want, regime):
    import torch
    run, y, ref, absref, keep = _conv_problem(K, regime, H * Cin + Cout, F16, H, W, Cin, Cout, kh, kw, s, pt, pl, True, True, r_off=r_off)
    prof = _tc_profile(K, lambda: _rc0(run(2)))
    assert len(prof) == 1 and prof[0]["conv"] == 1 and prof[0]["taps"] == kh * kw, prof
    assert (prof[0]["split"] if prof[0]["split"] == 1 else ">1") == want, prof
    torch.cuda.synchronize()
    _verify(regime, y, ref, absref, f"conv_tc {cid} {regime}")


IGEMM_CONV_F32 = [
    # H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left: osb_conv2d_ex with dtype f32 always takes igemm_kernel<float, CONV>
    (16, 16, 8, 24, 3, 3, 1, 1, 1),
    (33, 20, 4, 12, 3, 3, 2, 1, 1),
    (64, 1, 16, 16, 5, 1, 1, 2, 0),      # Conv1D
    (20, 24, 8, 8, 1, 7, 1, 0, 3),
    (32, 32, 3, 16, 7, 7, 2, 3, 3),
]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("H,W,Cin,Cout,kh,kw,s,pt,pl", IGEMM_CONV_F32)
def test_igemm_conv_f32(K, H, W, Cin, Cout, kh, kw, s, pt, pl, regime):
    import torch
    run, y, ref, absref, keep = _conv_problem(K, regime, H + Cin * 3 + kh, F32, H, W, Cin, Cout, kh, kw, s, pt, pl, True, True)
    assert K.osb_conv2d_fusable(None, None, None, H, W, Cin, Cout, kh, kw, s, F32, 0) == 0
    n, tc = _counted(K, lambda: _rc0(run(0)))
    assert (n, tc) == (1, 0)
    torch.cuda.synchronize()
    _verify(regime, y, ref, absref, f"conv_igemm f32 {(H, W, Cin, Cout, kh, kw, s, pt, pl)} {regime}")


# ---- fp32 on the tensor cores (bf16 triple split) ---------------------------------------------------------------------------------------

F32X_CONV = [
    # H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left, residual
    (32, 32, 4, 320, 3, 3, 1, 1, 1, False),     # the fp32 UNet's conv_in: 6 Cin = 24 < one k-block
    (32, 32, 64, 3, 3, 3, 1, 1, 1, True),       # the VAE's conv_out: Cout = 3, scalar partial writes
    (16, 16, 32, 40, 3, 3, 2, 1, 1, True),      # residual on the conv
    (64, 1, 16, 32, 3, 1, 1, 1, 0, True),       # Conv1D
]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("H,W,Cin,Cout,kh,kw,s,pt,pl,has_res", F32X_CONV)
def test_f32x_conv(K, H, W, Cin, Cout, kh, kw, s, pt, pl, has_res, regime):
    import torch
    import torch.nn.functional as Fn
    Ho, Wo = (H + 2 * pt - kh) // s + 1, (W + 2 * pl - kw) // s + 1
    assert K.osb_tc_conv_f32x_ok(H, W, Cin, Cout, kh, kw, s, Ho, Wo) == 1
    g = torch.Generator(device="cuda").manual_seed(H * Cin + Cout)
    x, w, bias, res = _operands(regime, g, [(H, W, Cin), (Cout, kh, kw, Cin), (Cout,), (Ho, Wo, Cout) if has_res else None], torch.float32,
                                lim=7, row_scaled=1)
    if regime == "gauss":
        w = w * 0.05
    x6 = torch.empty(H * W, 6 * Cin, device="cuda", dtype=torch.bfloat16); w6 = torch.empty(Cout * kh * kw, 6 * Cin, device="cuda", dtype=torch.bfloat16)
    y = torch.full((Ho, Wo, Cout), float("nan"), device="cuda")
    assert K.osb_bf16x3_expand_cols(x.data_ptr(), x6.data_ptr(), H * W, Cin, Cin, 0, _stream()) == 0
    assert K.osb_bf16x3_expand_cols(w.data_ptr(), w6.data_ptr(), Cout * kh * kw, Cin, Cin, 1, _stream()) == 0
    prof = _tc_profile(K, lambda: _rc0(K.osb_tc_conv_f32x(x6.data_ptr(), w6.data_ptr(), bias.data_ptr(), _ptr(res), y.data_ptr(), H, W, 6 * Cin, Cout,
                                                           kh, kw, s, pt, pl, Ho, Wo, _stream())))
    assert len(prof) == 1 and prof[0]["conv"] == 1 and prof[0]["K"] == 6 * Cin, prof
    xn, wn = x.double().permute(2, 0, 1)[None], w.double().permute(0, 3, 1, 2)
    ref = Fn.conv2d(xn, wn, bias.double(), stride=s, padding=(pt, pl))[0].permute(1, 2, 0)
    absref = Fn.conv2d(xn.abs(), wn.abs(), bias.double().abs(), stride=s, padding=(pt, pl))[0].permute(1, 2, 0)
    if has_res:
        ref = ref + res.double(); absref = absref + res.double().abs()
    _verify(regime, y, ref, absref, f"conv_f32x {(H, W, Cin, Cout, kh, kw)} {regime}")


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("M,N,Kd,bt", [(64, 8, 8, 1), (200, 136, 1500, 1), (96, 64, 40, 0)])
def test_f32x_gemm_bias_residual(K, M, N, Kd, bt, regime):
    """Bias and residual through the fp32 reduce, K-major B included (the existing f32x test runs K-major B without them)."""
    import torch
    assert K.osb_tc_gemm_f32x_ok(M, N, Kd) == 1
    g = torch.Generator(device="cuda").manual_seed(M + N + Kd)
    a, b, bias, res = _operands(regime, g, [(M, Kd), (N, Kd) if bt else (Kd, N), (N,), (M, N)], torch.float32, lim=7, row_scaled=1)
    a6 = torch.empty(M, 6 * Kd, device="cuda", dtype=torch.bfloat16)
    b6 = torch.empty((N, 6 * Kd) if bt else (6 * Kd, N), device="cuda", dtype=torch.bfloat16)
    c = torch.full((M, N), float("nan"), device="cuda")
    assert K.osb_bf16x3_expand_cols(a.data_ptr(), a6.data_ptr(), M, Kd, Kd, 0, _stream()) == 0
    if bt:
        assert K.osb_bf16x3_expand_cols(b.data_ptr(), b6.data_ptr(), N, Kd, Kd, 1, _stream()) == 0
    else:
        assert K.osb_bf16x3_expand_rows(b.data_ptr(), b6.data_ptr(), Kd, N, 1, _stream()) == 0
    prof = _tc_profile(K, lambda: _rc0(K.osb_tc_gemm_f32x(a6.data_ptr(), b6.data_ptr(), c.data_ptr(), bias.data_ptr(), res.data_ptr(), M, N, 6 * Kd, bt, _stream())))
    assert len(prof) == 1 and prof[0]["K"] == 6 * Kd and prof[0]["conv"] == 0, prof
    bd = b.double().t() if bt else b.double()
    ref = a.double() @ bd + bias.double() + res.double()
    absref = a.double().abs() @ bd.abs() + bias.double().abs() + res.double().abs()
    _verify(regime, c, ref, absref, f"gemm_f32x {(M, N, Kd, bt)} {regime}")


# ---- uint8: igemm fallbacks, tensor-core geometry, zero points and clamping ---------------------------------------------------------------

def _requant(acc, sx, sw, sy, zy):
    scale = np.float32(np.float32(np.float32(sx) * np.float32(sw)) / np.float32(sy))
    f = (acc.astype(np.int32).astype(np.float32) * scale).astype(np.float32)
    f = np.minimum(np.maximum(f, np.float32(0 - zy)), np.float32(255 - zy))
    return (np.rint(f).astype(np.int32) + zy).astype(np.uint8)


def _qu8_conv_ref(x, w, bias, zx, zw, s, pt, pl):
    H, W, Cin = x.shape
    Cout, kh, kw, _ = w.shape
    Ho, Wo = (H + 2 * pt - kh) // s + 1, (W + 2 * pl - kw) // s + 1
    xp = np.full((H + 2 * pt + s, W + 2 * pl + s, Cin), zx, np.int64)      # XNNPACK pads with the input zero point
    xp[pt:pt + H, pl:pl + W] = x
    acc = np.zeros((Ho, Wo, Cout), np.int64)
    for ky in range(kh):
        for kx in range(kw):
            acc += (xp[ky:ky + (Ho - 1) * s + 1:s, kx:kx + (Wo - 1) * s + 1:s] - zx) @ (w[:, ky, kx].astype(np.int64) - zw).T
    return acc + bias, Ho, Wo


QU8_ZP = [
    # zx, sx, zw, sw, zy, sy: every zero point at 0 and at 255 (the other operand's zero point mid-range, so that the products take both
    # signs); the output scale is small enough that both requantisation clamps fire
    (0, 0.02, 128, 0.004, 0, 0.01),
    (255, 0.02, 128, 0.004, 255, 0.01),
    (121, 0.031, 0, 0.0035, 117, 0.02),
    (121, 0.031, 255, 0.0035, 117, 0.02),
]

QU8_IGEMM_CONV = [
    # H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left: what osb_qu8_tc_conv_ok refuses
    (32, 32, 3, 16, 7, 7, 2, 3, 3),      # Cin = 3 stem
    (12, 12, 16, 24, 3, 3, 1, 1, 1),     # Cout % 16 != 0
    (20, 20, 16, 16, 1, 3, 1, 0, 1),     # non-square kernel (Cin, Cout fit the tensor cores, exercised on igemm here)
    (40, 1, 16, 16, 5, 1, 2, 2, 0),      # Conv1D, Ho * Wo = 20 < 64
]


@pytest.mark.parametrize("zp", range(len(QU8_ZP)))
@pytest.mark.parametrize("H,W,Cin,Cout,kh,kw,s,pt,pl", QU8_IGEMM_CONV)
def test_qu8_igemm_conv(K, H, W, Cin, Cout, kh, kw, s, pt, pl, zp):
    import torch
    zx, sx, zw, sw, zy, sy = QU8_ZP[zp]
    rng = np.random.default_rng(H * W + Cin + zp)
    x = rng.integers(0, 256, (H, W, Cin), dtype=np.uint8); w = rng.integers(0, 256, (Cout, kh, kw, Cin), dtype=np.uint8)
    bias = rng.integers(-3000, 3000, (Cout,), dtype=np.int32)
    acc, Ho, Wo = _qu8_conv_ref(x, w, bias, zx, zw, s, pt, pl)
    ref = _requant(acc, sx, sw, sy, zy)
    tx, tw, tb = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(bias).cuda()
    ty = torch.zeros((Ho, Wo, Cout), dtype=torch.uint8, device="cuda")
    if Ho * Wo >= 64 and kh == kw:
        assert K.osb_qu8_tc_conv_ok(Cin, Cout, Ho, Wo, kh, kw, s, tx.data_ptr(), tw.data_ptr(), ty.data_ptr()) == 0
    n, tc = _counted(K, lambda: _rc0(K.osb_conv2d_qu8(tx.data_ptr(), tw.data_ptr(), tb.data_ptr(), ty.data_ptr(), H, W, Cin, Cout, kh, kw, s, pt, pl, Ho, Wo,
                                                      zx, sx, zw, sw, zy, sy, _stream())))
    assert (n, tc) == (1, 0)
    torch.cuda.synchronize()
    got = ty.cpu().numpy()
    assert np.array_equal(got, ref), f"{int((got != ref).sum())} of {ref.size} bytes differ"
    assert (ref == 0).any() and (ref == 255).any(), "both requantisation clamps must be exercised"


@pytest.mark.parametrize("zp", range(len(QU8_ZP)))
@pytest.mark.parametrize("M,N,Kd", [(5, 64, 96), (40, 24, 100), (64, 48, 40)])
def test_qu8_igemm_gemm(K, M, N, Kd, zp):
    """osb_gemm_qu8 (igemm_kernel<uint8_t>) at shapes osb_qu8_tc_gemm_ok refuses: M < 32, N or K not a multiple of 16."""
    import torch
    zx, sx, zw, sw, zy, sy = QU8_ZP[zp]
    rng = np.random.default_rng(M * N + Kd + zp)
    a = rng.integers(0, 256, (M, Kd), dtype=np.uint8); b = rng.integers(0, 256, (Kd, N), dtype=np.uint8)
    bias = rng.integers(-3000, 3000, (N,), dtype=np.int32)
    ref = _requant((a.astype(np.int64) - zx) @ (b.astype(np.int64) - zw) + bias, sx, sw, sy, zy)
    ta, tb, tbias = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), torch.from_numpy(bias).cuda()
    tc_ = torch.zeros((M, N), dtype=torch.uint8, device="cuda")
    assert K.osb_qu8_tc_gemm_ok(M, N, Kd, ta.data_ptr(), tb.data_ptr(), tc_.data_ptr()) == 0
    n, tc = _counted(K, lambda: _rc0(K.osb_gemm_qu8(ta.data_ptr(), tb.data_ptr(), tc_.data_ptr(), tbias.data_ptr(), M, N, Kd, zx, sx, zw, sw, zy, sy, _stream())))
    assert (n, tc) == (1, 0)
    torch.cuda.synchronize()
    assert np.array_equal(tc_.cpu().numpy(), ref)
    assert (ref == 0).any() and (ref == 255).any()


QU8_TC_CONV = [
    # H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left
    (16, 20, 32, 48, 1, 3, 1, 0, 1),     # non-square
    (20, 16, 32, 48, 3, 1, 1, 1, 0),
    (128, 1, 32, 32, 3, 1, 1, 1, 0),     # Conv1D
    (129, 1, 32, 32, 5, 1, 2, 2, 0),
    (64, 64, 16, 32, 7, 7, 2, 3, 3),     # 7x7 stride-2 stem at Cin = 16
]


@pytest.mark.parametrize("zp", range(len(QU8_ZP)))
@pytest.mark.parametrize("H,W,Cin,Cout,kh,kw,s,pt,pl", QU8_TC_CONV)
def test_qu8_tc_conv_geometry(K, H, W, Cin, Cout, kh, kw, s, pt, pl, zp):
    import torch
    zx, sx, zw, sw, zy, sy = QU8_ZP[zp]
    rng = np.random.default_rng(H * W + Cin + kh * 7 + zp)
    x = rng.integers(0, 256, (H, W, Cin), dtype=np.uint8); w = rng.integers(0, 256, (Cout, kh, kw, Cin), dtype=np.uint8)
    bias = rng.integers(-3000, 3000, (Cout,), dtype=np.int32)
    acc, Ho, Wo = _qu8_conv_ref(x, w, bias, zx, zw, s, pt, pl)
    ref = _requant(acc, sx, sw, sy, zy)
    Hp, Wp = (Ho - 1) * s + kh, (Wo - 1) * s + kw
    tx, tw, tb = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(bias).cuda()
    txp = torch.zeros((Hp, Wp, Cin), dtype=torch.uint8, device="cuda"); tps = torch.zeros(Hp * Wp, dtype=torch.int32, device="cuda")
    tcs = torch.zeros(Cout, dtype=torch.int32, device="cuda"); ty = torch.zeros((Ho, Wo, Cout), dtype=torch.uint8, device="cuda")
    assert K.osb_qu8_tc_conv_ok(Cin, Cout, Ho, Wo, kh, kw, s, txp.data_ptr(), tw.data_ptr(), ty.data_ptr()) == 1
    assert K.osb_pad_sum_u8(tx.data_ptr(), txp.data_ptr(), tps.data_ptr(), H, W, Cin, Hp, Wp, pt, pl, zx, _stream()) == 0
    assert K.osb_rowsum_u8(tw.data_ptr(), tcs.data_ptr(), Cout, kh * kw * Cin, _stream()) == 0
    n, tc = _counted(K, lambda: _rc0(K.osb_qu8_tc_conv(txp.data_ptr(), tps.data_ptr(), tw.data_ptr(), tb.data_ptr(), tcs.data_ptr(), ty.data_ptr(), Hp, Wp, Cin, Cout,
                                                       kh, kw, s, Ho, Wo, zx, sx, zw, sw, zy, sy, _stream())))
    assert (n, tc) == (1, 1)
    torch.cuda.synchronize()
    xp = np.full((Hp, Wp, Cin), zx, np.int64)
    xp[pt:pt + H, pl:pl + W] = x[:Hp - pt, :Wp - pl]
    assert np.array_equal(txp.cpu().numpy(), xp.astype(np.uint8))
    assert np.array_equal(tps.cpu().numpy(), xp.sum(axis=2).reshape(-1)), "per-pixel channel sums of the padded image"
    got = ty.cpu().numpy()
    assert np.array_equal(got, ref), f"{int((got != ref).sum())} of {ref.size} bytes differ"
    assert (ref == 0).any() and (ref == 255).any()


# ---- GEMV users interleaved on one stream; scratch fallbacks under CUDA-graph capture ----------------------------------------------------

def _gemv_decode_step(K, g, dtype=F16):
    """A decode step's GEMV users in order: a plain GEMV (osb_gemm_ld), a grouped q/k/v GEMV, a uint8-weight GEMV, each with its own N.
    Returns (launch closures, checkers)."""
    import torch
    Kd = 1024
    a = (torch.randint(-3, 4, (1, Kd), device="cuda", generator=g)).half()
    w0 = torch.randint(-3, 4, (Kd, 2048), device="cuda", generator=g).half(); c0 = torch.full((1, 2048), float("nan"), device="cuda", dtype=torch.half)
    Ns = (512, 256, 256)
    wg = [torch.randint(-3, 4, (Kd, n), device="cuda", generator=g).half() for n in Ns]
    cg = [torch.full((1, n), float("nan"), device="cuda", dtype=torch.half) for n in Ns]
    wq = torch.randint(0, 256, (Kd, 5632), device="cuda", generator=g, dtype=torch.uint8)
    bq = torch.randint(-3, 4, (5632,), device="cuda", generator=g).half()
    cq = torch.full((1, 5632), float("nan"), device="cuda", dtype=torch.half)
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    B = (vp * 3)(*[w.data_ptr() for w in wg]); C = (vp * 3)(*[c.data_ptr() for c in cg]); Nv = (i64 * 3)(*Ns)
    sc = (ctypes.c_float * 3)(1.0, 1.0, 1.0); zp = (ci * 3)(0, 0, 0)

    def gemv():
        return K.osb_gemm_ld(a.data_ptr(), Kd, w0.data_ptr(), 2048, c0.data_ptr(), 2048, None, None, 1, 1, 2048, Kd, 0, 0, 0, 0, F16, 0, _stream())

    def grouped():
        return K.osb_gemv_grouped(a.data_ptr(), B, C, Nv, sc, zp, 3, 1, Kd, F16, F16, _stream())

    def w8():       # scale 1, zero point 128: integer weights in [-128, 127], S < 2^24
        return K.osb_gemv_w8(a.data_ptr(), wq.data_ptr(), cq.data_ptr(), bq.data_ptr(), None, 1, 5632, Kd, 1.0, 128, F16, _stream())

    ad = a.double()
    checks = [(c0, ad @ w0.double(), ad.abs() @ w0.double().abs())]
    checks += [(c, ad @ w.double(), ad.abs() @ w.double().abs()) for c, w in zip(cg, wg)]
    wqd = wq.double() - 128
    checks.append((cq, ad @ wqd + bq.double(), ad.abs() @ wqd.abs() + bq.double().abs()))
    keep = (a, w0, wg, wq, bq, B, C, Nv, sc, zp)
    return (gemv, grouped, w8), checks, keep


def test_gemv_users_interleaved(K):
    """GEMV, grouped GEMV and osb_gemv_w8 share one stream's scratch sums and arrival counters: each must leave them re-armed."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(11)
    fns, checks, keep = _gemv_decode_step(K, g)
    for step in range(3):
        for c, _, _ in checks:
            c.fill_(float("nan"))
        for fn in fns:
            assert fn() == 0
        torch.cuda.synchronize()
        for i, (c, ref, S) in enumerate(checks):
            _check_exact(c, ref, S, f"decode step {step} GEMV user {i}")


def test_capture_falls_back_without_scratch(K):
    """osb_workspace returns null while a stream captures and has no scratch yet: a split-K candidate runs unsplit, the GEMV takes the
    skinny kernel, osb_gemv_w8 reports cudaErrorNotReady.  Three replays of the graph give identical bits that pass the bars."""
    import torch
    s = torch.cuda.Stream()
    K.osb_workspace_release(ctypes.c_void_p(s.cuda_stream))      # torch pools its streams: this one may own scratch from an earlier test
    g = torch.Generator(device="cuda").manual_seed(12)
    split_run, split_result, split_ref, split_S, keep1 = _gemm_problem(K, "gauss", 4, F16, 1, 128, 256, 4096, 0, True, True)
    fns, checks, keep2 = _gemv_decode_step(K, g)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    K.osb_launch_count_reset()
    with torch.cuda.graph(graph, stream=s):
        assert split_run(0) == 0
        assert fns[0]() == 0
        assert fns[2]() == NOT_READY
    assert (int(K.osb_launch_count()), int(K.osb_tc_launch_count())) == (2, 1), "split-K candidate unsplit (no reduce launch) + skinny GEMV"
    outs = []
    for _ in range(3):
        split_result().fill_(float("nan")); checks[0][0].fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        outs.append((split_result().clone(), checks[0][0].clone()))
    for o in outs[1:]:
        assert torch.equal(o[0], outs[0][0]) and torch.equal(o[1], outs[0][1]), "graph replays differ"
    _check(outs[0][0], split_ref, split_S, "gemm_tc captured split-K candidate")
    c0, ref0, S0 = checks[0]
    _check_exact(outs[0][1], ref0, S0, "captured GEMV (skinny fallback)")
    del graph
    K.osb_workspace_release(ctypes.c_void_p(s.cuda_stream))


# ---- host-side refusals: no launch ----------------------------------------------------------------------------------------------------

def test_host_refusals(K):
    import torch
    h = torch.zeros(1 << 16, device="cuda", dtype=torch.half)
    u8 = torch.zeros(1 << 16, device="cuda", dtype=torch.uint8)
    p = h.data_ptr()
    cases = [
        ("impl 2, M < 32", lambda: K.osb_gemm(p, p, p, None, None, 1, 16, 64, 64, 0, 0, 0, 0, F16, 2, _stream()), INVALID_VALUE),
        ("impl 2, A misaligned", lambda: K.osb_gemm(p + 2, p, p, None, None, 1, 64, 64, 64, 0, 0, 0, 0, F16, 2, _stream()), INVALID_VALUE),
        ("impl 2, fp32", lambda: K.osb_gemm(p, p, p, None, None, 1, 64, 64, 64, 0, 0, 0, 0, F32, 2, _stream()), INVALID_VALUE),
        ("bias2 on a CUDA-core conv", lambda: K.osb_conv2d_ex(p, p, None, p, None, p, 16, 16, 3, 16, 3, 3, 1, 1, 1, 16, 16, F16, 0, _stream(), None, 0, None),
         INVALID_VALUE),
        ("gemv_w8 N % 16", lambda: K.osb_gemv_w8(p, u8.data_ptr(), p, None, None, 1, 264, 64, 1.0, 0, F16, _stream()), INVALID_VALUE),
        ("f32x gemm N % 8", lambda: K.osb_tc_gemm_f32x(p, p, p, None, None, 64, 36, 48, 0, _stream()), NOT_SUPPORTED),
        ("pad_sum_u8 C % 16", lambda: K.osb_pad_sum_u8(u8.data_ptr(), u8.data_ptr(), p, 4, 4, 8, 6, 6, 1, 1, 0, _stream()), INVALID_VALUE),
    ]
    for what, fn, want in cases:
        K.osb_launch_count_reset()
        assert fn() == want, what
        assert K.osb_launch_count() == 0, f"{what}: launched"
    torch.cuda.synchronize()
