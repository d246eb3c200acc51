"""The tensor-core kernel's tile epilogue (gemm_wgmma.cu: the bias, bias2 and residual values of a group of 8-column blocks are loaded
before the group's stores, as one 4-byte word per column pair where the operand is aligned to it) at every tile, with the operand
placements that change how it loads: bias / bias2 and residual offset by one element (two 2-byte loads per pair) and the residual being
C itself (a residual Add done in place).  Integer operands: the output must be the fp64 result rounded once to fp16, bit for bit."""
import ctypes

import pytest

from test_gemm_conv_paths_gpu import K  # noqa: F401  (the module fixture)
from test_kernels_gpu import F16, _check_exact, _stream
from test_tc_tiles_gpu import TILES_K, TILES_MN, _profile, _rc0, _tid, tile  # noqa: F401  (tile: fixture)

pytestmark = pytest.mark.gpu

GEMM_TILES = [(0, t) for t in TILES_MN] + [(1, t) for t in TILES_K]
# id, bias offset, residual offset (elements), residual is C
PLACEMENTS = [("aligned", 0, 0, False), ("bias+1", 1, 0, False), ("residual+1", 0, 1, False), ("in-place", 0, 0, True)]


def _ints(g, *shape):
    import torch
    return torch.randint(-3, 4, shape, device="cuda", generator=g).half()


def _offset(t, off):
    """t's values in a fresh buffer, starting `off` elements in (off = 1: only 2-byte aligned)."""
    import torch
    buf = torch.zeros(t.numel() + 8, device="cuda", dtype=t.dtype)
    buf[off:off + t.numel()] = t.reshape(-1)
    return buf[off:off + t.numel()].view(t.shape), buf


@pytest.mark.parametrize("pid,bias_off,r_off,inplace", PLACEMENTS, ids=[p[0] for p in PLACEMENTS])
@pytest.mark.parametrize("bt,t", GEMM_TILES, ids=[f"{'K' if bt else 'MN'}-{_tid(t)}" for bt, t in GEMM_TILES])
def test_epilogue_gemm(K, tile, bt, t, pid, bias_off, r_off, inplace):
    """M = 1100 and N = 328 are ragged against every tile; at 64-row tiles there are more tiles than SMs, so CTAs run several."""
    import torch
    M, N, Kd = 1100, 328, 192
    g = torch.Generator(device="cuda").manual_seed(M + bt + bias_off + 2 * r_off)
    a, b = _ints(g, M, Kd), (_ints(g, N, Kd) if bt else _ints(g, Kd, N))
    bias, bbuf = _offset(_ints(g, N), bias_off)
    res, rbuf = _offset(_ints(g, M, N), r_off)
    ref = a.double() @ (b.double().t() if bt else b.double()) + bias.double() + res.double()
    absref = a.double().abs() @ (b.double().abs().t() if bt else b.double().abs()) + 6
    c = res if inplace else torch.full((M, N), float("nan"), device="cuda", dtype=torch.half)
    tile(t[0], t[1], 1)
    prof = _profile(K, lambda: _rc0(K.osb_gemm_ld(a.data_ptr(), Kd, b.data_ptr(), Kd if bt else N, c.data_ptr(), N, bias.data_ptr(), res.data_ptr(),
                                                  1, M, N, Kd, 0, 0, M * N, bt, F16, 2, _stream())))
    assert [(p["bm"], p["bn"], p["split"]) for p in prof] == [(t[0], t[1], 1)], prof
    torch.cuda.synchronize()
    _check_exact(c, ref, absref, f"gemm epilogue {t} bt {bt} {pid}")


CONV_PLACEMENTS = [("aligned", 0, False), ("bias+1", 1, False), ("in-place", 0, True)]


@pytest.mark.parametrize("pid,bias_off,inplace", CONV_PLACEMENTS, ids=[p[0] for p in CONV_PLACEMENTS])
@pytest.mark.parametrize("t", TILES_K, ids=_tid)
def test_epilogue_conv_extras(K, tile, t, pid, bias_off, inplace):
    """bias, bias2 (both offset by one element in 'bias+1'), residual and the GroupNorm statistics: the EXTRAS instantiation of every
    tile on a 20 x 20 image (boxes cross the image edge), Cout = 136 (ragged against every BN)."""
    import torch
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    K.osb_conv2d_ex.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, ci, ci, vp, vp, ci, ctypes.POINTER(ci)]
    H, Cin, Cout, G = 20, 64, 136, 17
    g = torch.Generator(device="cuda").manual_seed(Cout + bias_off + int(inplace))
    x, w = _ints(g, H, H, Cin), _ints(g, Cout, 3, 3, Cin)
    bias, b1buf = _offset(_ints(g, Cout), bias_off)
    bias2, b2buf = _offset(_ints(g, Cout), bias_off)
    res = _ints(g, H, H, Cout)
    import torch.nn.functional as Fn
    xn, wn = x.double().permute(2, 0, 1)[None], w.double().permute(0, 3, 1, 2)
    ref = Fn.conv2d(xn, wn, None, padding=1)[0].permute(1, 2, 0) + bias.double() + res.double() + bias2.double()
    absref = Fn.conv2d(xn.abs(), wn.abs(), None, padding=1)[0].permute(1, 2, 0) + 9
    y = res if inplace else torch.full((H, H, Cout), float("nan"), device="cuda", dtype=torch.half)
    stats = torch.zeros(2 * G, device="cuda", dtype=torch.float64)
    done = ci(0)
    tile(t[0], t[1], 1)
    prof = _profile(K, lambda: _rc0(K.osb_conv2d_ex(x.data_ptr(), w.data_ptr(), bias.data_ptr(), bias2.data_ptr(), res.data_ptr(), y.data_ptr(),
                                                    H, H, Cin, Cout, 3, 3, 1, 1, 1, H, H, F16, 2, _stream(), stats.data_ptr(), G, ctypes.byref(done))))
    assert [(p["bm"], p["bn"], p["split"]) for p in prof] == [(t[0], t[1], 1)], prof
    torch.cuda.synchronize()
    _check_exact(y, ref, absref, f"conv epilogue {t} {pid}")
    assert done.value == 1, "the kernel did not report the statistics"
    yd = y.double().reshape(H * H, G, Cout // G)
    want = torch.stack([yd.sum(dim=(0, 2)), (yd * yd).sum(dim=(0, 2))], dim=1).reshape(-1)
    scale = torch.stack([yd.abs().sum(dim=(0, 2)), (yd * yd).sum(dim=(0, 2))], dim=1).reshape(-1) + 1e-9
    err = float(((stats - want).abs() / scale).max())
    assert err <= 2e-5, f"statistics off by {err:.3g} (relative to sum|y| / sum y^2)"
