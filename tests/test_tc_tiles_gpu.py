"""Every tile shape of the tensor-core GEMM / conv kernel (tc_gemm_kernel<BM, BN, ...>), forced through osb_tc_set_tile and pinned by the
launch profile (osb_tc_profile_dump: "... bm bn kmajor" after the nine original fields), in the two data regimes of
tests/test_gemm_conv_paths_gpu.py: bit-exact on integer operands, and the fp32-accumulation bar on Gaussian operands."""
import ctypes

import pytest

from test_gemm_conv_paths_gpu import K, REGIMES, _conv_problem, _gemm_problem  # noqa: F401  (K: the module fixture)
from test_kernels_gpu import F16, _check, _stream, _verify

pytestmark = pytest.mark.gpu

# the instantiated tiles (gemm_wgmma.cu: TC_TILES_KMAJOR, TC_TILES_MNMAJOR)
TILES_K = [(128, 128), (128, 64), (128, 80), (128, 160), (64, 64), (64, 128), (64, 160)]
TILES_MN = [(128, 128), (128, 64), (64, 128)]
KEYS = ("M", "N", "K", "taps", "batch", "split", "conv", "ms", "gflop", "bm", "bn", "kmajor")


def _tid(t):
    return "%dx%d" % t


@pytest.fixture()
def tile(K):
    """tile(bm, bn, split) forces the next launches; the rule is restored afterwards."""
    K.osb_tc_set_tile.argtypes = [ctypes.c_int] * 3
    K.osb_tc_set_tile.restype = None
    yield K.osb_tc_set_tile
    K.osb_tc_set_tile(0, 0, 0)


def _profile(K, fn):
    import torch
    torch.cuda.synchronize()
    K.osb_tc_profile(1)
    try:
        fn()
        torch.cuda.synchronize()
        buf = ctypes.create_string_buffer(1 << 16)
        assert K.osb_tc_profile_dump(buf, len(buf)) >= 0
    finally:
        K.osb_tc_profile(0)
    return [dict(zip(KEYS, (float(v) if k in ("ms", "gflop") else int(v) for k, v in zip(KEYS, line.split()))))
            for line in buf.value.decode().splitlines()]


def _rc0(rc):
    assert rc == 0, f"rc = {rc}"


def _clamped_split(split, k_blocks, allowed):
    """The split a forced `split` becomes (gemm_wgmma.cu: choose_tile): at most one per k-block, no empty split."""
    if not allowed or k_blocks < 2:
        return 1
    sp = min(split, k_blocks)
    kb_per = -(-k_blocks // sp)
    return -(-k_blocks // kb_per)


# ---- GEMM: every tile of both B layouts, ragged M and N, split forced off and on ---------------------------------------------------------

GEMM_TILES = [(0, t) for t in TILES_MN] + [(1, t) for t in TILES_K]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("split", [1, 3])
@pytest.mark.parametrize("bt,t", GEMM_TILES, ids=[f"{'K' if bt else 'MN'}-{_tid(t)}" for bt, t in GEMM_TILES])
def test_tile_gemm(K, tile, bt, t, split, regime):
    """M = 200 and N = 328 are ragged against every tile (N: 5.1 tiles of 64, 4.1 of 80, 2.6 of 128, 2.05 of 160); bias and residual
    through the tile epilogue (split 1) and the reduce kernel (split 3)."""
    import torch
    M, N, Kd = 200, 328, 640
    run, result, ref, absref, keep = _gemm_problem(K, regime, M + split + bt, F16, 1, M, N, Kd, bt, True, True)
    tile(t[0], t[1], split)
    prof = _profile(K, lambda: _rc0(run(2)))
    assert [(p["bm"], p["bn"], p["split"], p["kmajor"]) for p in prof] == [(t[0], t[1], split, bt)], prof
    torch.cuda.synchronize()
    _verify(regime, result(), ref, absref, f"gemm {t} split {split} bt {bt} {regime}")


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("bt,t", GEMM_TILES, ids=[f"{'K' if bt else 'MN'}-{_tid(t)}" for bt, t in GEMM_TILES])
def test_tile_gemm_batched(K, tile, bt, t, regime):
    """A batch of 2 with a forced split: the workspace planes and the reduce index batch and split correctly for every tile."""
    import torch
    run, result, ref, absref, keep = _gemm_problem(K, regime, 17 + bt, F16, 2, 136, 200, 512, bt, True, True)
    tile(t[0], t[1], 2)
    prof = _profile(K, lambda: _rc0(run(2)))
    assert [(p["bm"], p["bn"], p["split"], p["batch"]) for p in prof] == [(t[0], t[1], 2, 2)], prof
    torch.cuda.synchronize()
    _verify(regime, result(), ref, absref, f"gemm batch 2 {t} bt {bt} {regime}")


@pytest.mark.parametrize("bt,t", GEMM_TILES, ids=[f"{'K' if bt else 'MN'}-{_tid(t)}" for bt, t in GEMM_TILES])
def test_tile_grouped(K, tile, bt, t):
    """The grouped q/k/v launch stays ONE launch at every tile (a forced split does not apply to it); integer operands, bit-exact."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(5 + bt)
    M, N, Kd = 300, 320, 320
    a = torch.randint(-3, 4, (M, Kd), device="cuda", generator=g).half()
    ws = [torch.randint(-3, 4, (N, Kd) if bt else (Kd, N), device="cuda", generator=g).half() for _ in range(3)]
    cs = [torch.full((M, N), float("nan"), device="cuda", dtype=torch.half) for _ in range(3)]
    vp = ctypes.c_void_p
    B = (vp * 3)(*[w.data_ptr() for w in ws]); C = (vp * 3)(*[c.data_ptr() for c in cs])
    K.osb_gemm_grouped.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.c_int, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                   ctypes.c_int, ctypes.c_int, ctypes.c_int, vp]
    tile(t[0], t[1], 3)
    prof = _profile(K, lambda: _rc0(K.osb_gemm_grouped(a.data_ptr(), B, C, 3, M, N, Kd, bt, F16, 2, _stream())))
    assert [(p["bm"], p["bn"], p["split"], p["batch"]) for p in prof] == [(t[0], t[1], 1, 3)], prof
    torch.cuda.synchronize()
    for w, c in zip(ws, cs):
        ref = a.double() @ (w.double().t() if bt else w.double())
        assert torch.equal(c.double(), ref.half().double()), f"grouped {t} bt {bt}"


# ---- convolution: every K-major tile at the geometries that change the pixel box ----------------------------------------------------------

CONV_GEOMS = [
    # id, H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left
    ("8x8-Cout132", 8, 8, 128, 132, 3, 3, 1, 1, 1),     # BM = 64: the box is exactly the image; Cout % 8 != 0
    ("16x16", 16, 16, 64, 136, 3, 3, 1, 1, 1),
    ("stride2", 32, 32, 64, 64, 3, 3, 2, 1, 1),
    ("1x1", 16, 16, 96, 320, 1, 1, 1, 0, 0),
    ("Conv1D", 64, 1, 64, 128, 3, 1, 1, 1, 0),          # bw = 1, bh = BM
    ("Wo<bw", 20, 5, 32, 64, 3, 3, 1, 1, 1),            # Wo = 5: bw = 8, boxes stick out of the image
    ("Cout4", 16, 16, 32, 4, 3, 3, 1, 1, 1),
    ("Cout3", 16, 16, 16, 3, 3, 3, 1, 1, 1),            # ragged Cout: no split whatever is forced
]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("split", [1, 3])
@pytest.mark.parametrize("cid,H,W,Cin,Cout,kh,kw,s,pt,pl", CONV_GEOMS, ids=[c[0] for c in CONV_GEOMS])
@pytest.mark.parametrize("t", TILES_K, ids=_tid)
def test_tile_conv(K, tile, t, cid, H, W, Cin, Cout, kh, kw, s, pt, pl, split, regime):
    import torch
    run, y, ref, absref, keep = _conv_problem(K, regime, H * Cin + Cout + split, F16, H, W, Cin, Cout, kh, kw, s, pt, pl, True, True)
    tile(t[0], t[1], split)
    prof = _profile(K, lambda: _rc0(run(2)))
    want_split = _clamped_split(split, kh * kw * -(-Cin // 64), Cout % 4 == 0)
    assert [(p["bm"], p["bn"], p["split"], p["conv"], p["taps"]) for p in prof] == [(t[0], t[1], want_split, 1, kh * kw)], prof
    torch.cuda.synchronize()
    _verify(regime, y, ref, absref, f"conv {cid} {t} split {split} {regime}")


@pytest.mark.parametrize("split", [1, 3])
@pytest.mark.parametrize("H,Cout,G", [(16, 256, 32), (8, 160, 8)], ids=["16x16-cpg8", "8x8-cpg20"])
@pytest.mark.parametrize("t", TILES_K, ids=_tid)
def test_tile_conv_extras(K, tile, t, H, Cout, G, split):
    """bias2 and the GroupNorm statistics (the EXTRAS instantiation of every tile): in the tile epilogue (split 1) or the reduce kernel
    (split 3); the statistics must be those of the stored fp16 output."""
    import torch
    import torch.nn.functional as Fn
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    K.osb_conv2d_ex.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, ci, ci, vp, vp, ci, ctypes.POINTER(ci)]
    Cin = 64
    g = torch.Generator(device="cuda").manual_seed(H + Cout + split)
    x = torch.randn(H, H, Cin, device="cuda", generator=g).half()
    w = (torch.randn(Cout, 3, 3, Cin, device="cuda", generator=g) / (9 * Cin) ** 0.5).half()
    bias, bias2 = torch.randn(Cout, device="cuda", generator=g).half(), torch.randn(Cout, device="cuda", generator=g).half()
    res = torch.randn(H, H, Cout, device="cuda", generator=g).half()
    y = torch.full((H, H, Cout), float("nan"), device="cuda", dtype=torch.half)
    stats = torch.zeros(2 * G, device="cuda", dtype=torch.float64)
    done = ci(0)
    tile(t[0], t[1], split)
    prof = _profile(K, lambda: _rc0(K.osb_conv2d_ex(x.data_ptr(), w.data_ptr(), bias.data_ptr(), bias2.data_ptr(), res.data_ptr(), y.data_ptr(),
                                                    H, H, Cin, Cout, 3, 3, 1, 1, 1, H, H, F16, 2, _stream(), stats.data_ptr(), G, ctypes.byref(done))))
    assert [(p["bm"], p["bn"], p["split"]) for p in prof] == [(t[0], t[1], split)], prof
    torch.cuda.synchronize()
    xn, wn = x.double().permute(2, 0, 1)[None], w.double().permute(0, 3, 1, 2)
    ref = Fn.conv2d(xn, wn, None, padding=1)[0].permute(1, 2, 0) + bias.double() + bias2.double() + res.double()
    absref = Fn.conv2d(xn.abs(), wn.abs(), None, padding=1)[0].permute(1, 2, 0) + bias.double().abs() + bias2.double().abs() + res.double().abs()
    _check(y, ref, absref, f"conv extras {t} split {split}")
    assert done.value == 1, "the kernel did not report the statistics"
    yd = y.double().reshape(H * H, G, Cout // G)
    want = torch.stack([yd.sum(dim=(0, 2)), (yd * yd).sum(dim=(0, 2))], dim=1).reshape(-1)
    scale = torch.stack([yd.abs().sum(dim=(0, 2)), (yd * yd).sum(dim=(0, 2))], dim=1).reshape(-1) + 1e-9
    err = float(((stats - want).abs() / scale).max())
    assert err <= 2e-5, f"statistics off by {err:.3g} (relative to sum|y| / sum y^2)"


# ---- the k order is the tile's own business: unsplit, every tile gives the 128 x 128 tile's bits ----------------------------------------

@pytest.mark.parametrize("bt,t", GEMM_TILES, ids=[f"{'K' if bt else 'MN'}-{_tid(t)}" for bt, t in GEMM_TILES])
def test_tile_invariance_gemm(K, tile, bt, t):
    import torch
    run, result, ref, absref, keep = _gemm_problem(K, "gauss", 23 + bt, F16, 1, 200, 328, 1280, bt, True, True)
    tile(128, 128, 1)
    _rc0(run(2))
    torch.cuda.synchronize()
    base = result().clone()
    tile(t[0], t[1], 1)
    _rc0(run(2))
    torch.cuda.synchronize()
    assert torch.equal(result(), base), f"tile {t} differs from 128 x 128 in {int((result() != base).sum())} elements"


@pytest.mark.parametrize("t", TILES_K, ids=_tid)
def test_tile_invariance_conv(K, tile, t):
    import torch
    run, y, ref, absref, keep = _conv_problem(K, "gauss", 29, F16, 16, 16, 128, 136, 3, 3, 1, 1, 1, True, True)
    tile(128, 128, 1)
    _rc0(run(2))
    torch.cuda.synchronize()
    base = y.clone()
    tile(t[0], t[1], 1)
    _rc0(run(2))
    torch.cuda.synchronize()
    assert torch.equal(y, base), f"tile {t} differs from 128 x 128 in {int((y != base).sum())} elements"


# ---- the rule: its own picks run, and a forced shape that a launch cannot take leaves it to the rule -----------------------------------

def test_rule_and_unavailable_tile(K, tile):
    import torch
    run, result, ref, absref, keep = _gemm_problem(K, "exact", 3, F16, 1, 256, 320, 640, 0, True, True)
    tile(128, 80, 1)          # K-major only: the MN-major launch takes the rule's shape for its layout
    prof = _profile(K, lambda: _rc0(run(2)))
    assert len(prof) == 1 and (prof[0]["bm"], prof[0]["bn"]) in TILES_MN, prof
    torch.cuda.synchronize()
    _verify("exact", result(), ref, absref, "MN-major with a K-major-only tile forced")
    tile(-1, 0, 0)            # the previous rule: 128 x 128
    prof = _profile(K, lambda: _rc0(run(2)))
    assert [(p["bm"], p["bn"]) for p in prof] == [(128, 128)], prof
    tile(0, 0, 0)
    prof = _profile(K, lambda: _rc0(run(2)))
    assert len(prof) == 1 and (prof[0]["bm"], prof[0]["bn"]) in TILES_MN, prof
    torch.cuda.synchronize()
    _verify("exact", result(), ref, absref, "the rule's pick")


# ---- CUDA-graph capture with a non-default tile ---------------------------------------------------------------------------------------

def test_tile_graph_replay(K, tile):
    """A split GEMM at 64 x 128 and a conv at 64 x 160 captured into one graph: three replays give identical bits that pass the bars."""
    import torch
    s = torch.cuda.Stream()
    gemm_run, gemm_result, gemm_ref, gemm_S, keep1 = _gemm_problem(K, "gauss", 41, F16, 1, 256, 640, 1280, 0, True, True)
    conv_run, y, conv_ref, conv_S, keep2 = _conv_problem(K, "gauss", 43, F16, 16, 16, 64, 320, 3, 3, 1, 1, 1, True, True)
    with torch.cuda.stream(s):      # a workspace for the split before capture
        tile(64, 128, 4)
        _rc0(gemm_run(2))
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        tile(64, 128, 4)
        _rc0(gemm_run(2))
        tile(64, 160, 1)
        _rc0(conv_run(2))
    tile(0, 0, 0)
    outs = []
    for _ in range(3):
        gemm_result().fill_(float("nan")); y.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        outs.append((gemm_result().clone(), y.clone()))
    for o in outs[1:]:
        assert torch.equal(o[0], outs[0][0]) and torch.equal(o[1], outs[0][1]), "graph replays differ"
    _check(outs[0][0], gemm_ref, gemm_S, "captured split GEMM at 64 x 128")
    _check(outs[0][1], conv_ref, conv_S, "captured conv at 64 x 160")
    del graph
