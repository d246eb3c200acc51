"""fp32-arithmetic convolution on fp16 weights read in place: the tensor-core conv that splits the fp16 filter tile into its bf16 hi / lo
parts in shared memory and stores fp32 from its registers (osb_tc_conv_f32x_f16w), and the engine routing that hands it the fp16 blob of a
Conv instead of an fp32 copy and its bf16x6 expansion.

Kernel cases run in the two regimes of tests/test_gemm_f32x_f16w_gpu.py.  The exact regime uses fixed-point operands built so that each of
the five products the kernel computes (x_h w_hi, x_h w_lo, x_m w_hi, x_l w_hi, x_m w_lo) is nonzero somewhere and the one it drops (x_l
w_lo) is zero everywhere; the result is then the fp64 result rounded once to fp32, bit for bit.  The Gaussian regime holds _check's bar."""
import ctypes
import os
import re
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from test_kernels_gpu import _check, _check_exact, _operands
from util import reference_outputs, report, run_model

pytestmark = pytest.mark.gpu

NOT_SUPPORTED = 801
TOL32 = 2e-4        # tests/test_models_gpu.py TOL["float32"]
KERNEL = "tc_gemm_f16w_kernel<true>"
WS_BYTES = 96 << 20     # the split-K workspace (workspace.h OSB_WS_SPLITK_BYTES)


@pytest.fixture(scope="module")
def K(engine_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = ctypes.CDLL(engine_lib)
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.osb_tc_conv_f32x_f16w_ok.argtypes = [i64, i64, i64, i64, ci, ci, ci, i64, i64]
    lib.osb_tc_conv_f32x_f16w.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, vp, vp]
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


def _out_size(H, W, kh, kw, s, pt, pb, pl, pr):
    return (H + pt + pb - kh) // s + 1, (W + pl + pr - kw) // s + 1


def _run(K, x, w, bias, res, s, pt, pl, Ho, Wo):
    """osb_tc_conv_f32x_f16w on x [H, W, Cin] fp32 and w [Cout, kh, kw, Cin] fp16: (rc, launches, y [Ho, Wo, Cout])."""
    import torch
    H, W, Cin = x.shape
    Cout, kh, kw, _ = w.shape
    assert x.is_contiguous() and w.is_contiguous()
    y = torch.full((Ho, Wo, Cout), float("nan"), device="cuda")
    planes = torch.empty(3 * H * W * Cin, device="cuda", dtype=torch.bfloat16)
    K.osb_launch_count_reset()
    rc = K.osb_tc_conv_f32x_f16w(x.data_ptr(), w.data_ptr(), _ptr(bias), _ptr(res), y.data_ptr(), H, W, Cin, Cout, kh, kw, s, pt, pl, Ho, Wo,
                                 planes.data_ptr(), _stream())
    n = int(K.osb_launch_count())
    torch.cuda.synchronize()
    return rc, n, y


def _conv64(x, w, s, pt, pl, Ho, Wo):
    """fp64 conv on the device of x [H, W, Cin] and w [Cout, kh, kw, Cin] (any float types) with pads (pt, pl) and the output size (Ho, Wo):
    the bottom / right pads follow from it (negative: rows the conv never reaches)."""
    import torch.nn.functional as Fn
    H, W, _ = x.shape
    _, kh, kw, _ = w.shape
    pb, pr = (Ho - 1) * s + kh - H - pt, (Wo - 1) * s + kw - W - pl
    xn = Fn.pad(x.double().permute(2, 0, 1)[None], (pl, pr, pt, pb))
    return Fn.conv2d(xn, w.double().permute(0, 3, 1, 2), None, stride=s)[0].permute(1, 2, 0)


def _ref(x, w, bias, res, s, pt, pl, Ho, Wo):
    ref = _conv64(x, w, s, pt, pl, Ho, Wo)
    absref = _conv64(x.abs(), w.abs(), s, pt, pl, Ho, Wo)
    if bias is not None:
        ref = ref + bias.double(); absref = absref + bias.double().abs()
    if res is not None:
        ref = ref + res.double(); absref = absref + res.double().abs()
    return ref, absref


def _exact_operands(case, H, W, Cin, Cout, kh, kw, seed):
    """Integers in [-7, 7] with sparse wide entries.  Case "m": x entries of 9 significant bits (x_m != 0, x_l = 0) and w entries of 9 (w_lo !=
    0); case "l": x entries of 18 significant bits whose remainder past x_h needs 9 (x_l != 0), w entries of at most 3 (w_lo = 0).  A pixel
    holds at most one wide x entry (its channel c has (c + 7 pixel) % P == 0, P >= Cin) and a filter row at most kh kw Cin / Pw + 1 wide w
    entries, so with kh kw <= 9 every partial sum S = sum |x w| stays below 2^24: each is exact in fp32."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randint(-7, 8, (H, W, Cin), device="cuda", generator=g).float()
    w = torch.randint(-7, 8, (Cout, kh, kw, Cin), device="cuda", generator=g).float()
    P = max(Cin, 8)
    pix = torch.arange(H * W, device="cuda").reshape(H, W, 1)
    sx = (torch.arange(Cin, device="cuda") + 7 * pix) % P == 0
    sign = lambda shp: torch.randint(0, 2, shp, device="cuda", generator=g).float() * 2 - 1
    odd = lambda shp, hi: torch.randint(0, hi // 2, shp, device="cuda", generator=g).float() * 2 + 1
    if case == "m":
        x = torch.where(sx, sign(x.shape) * (256 + odd(x.shape, 256)), x)
        Kt = kh * kw * Cin
        Pw = max(8, Kt // 8)
        k2, n2 = torch.meshgrid(torch.arange(Kt, device="cuda"), torch.arange(Cout, device="cuda"), indexing="ij")
        sw = ((k2 * 3 + n2) % Pw == 0).t().contiguous().reshape(Cout, kh, kw, Cin)
        w = torch.where(sw, sign(w.shape) * (256 + odd(w.shape, 256)), w)
    else:
        # 2^17 + 1024 a + 256 + odd: x_h keeps bits 17..10, the remainder (257..511 or -511..-257) has 9 bits, its lowest is x_l
        wide = 131072 + 1024 * torch.randint(0, 32, x.shape, device="cuda", generator=g).float() + 256 + odd(x.shape, 512)
        x = torch.where(sx, sign(x.shape) * wide, x)
        w = torch.randint(-3, 4, w.shape, device="cuda", generator=g).float()
    return x, w.half()


def _products(x, w, s, pt, pl, Ho, Wo):
    """{name: is the product nonzero for some output} of the six triple-split products with an fp16 filter."""
    h = x.bfloat16().float(); m = (x - h).bfloat16().float(); lo_x = (x - h - m).bfloat16().float()
    wf = w.float()
    hi = wf.bfloat16().float(); lo = (wf - hi).bfloat16().float()
    nz = lambda a, b: bool((_conv64((a != 0).float(), (b != 0).float(), s, pt, pl, Ho, Wo) > 0).any())
    return {"h.hi": nz(h, hi), "h.lo": nz(h, lo), "m.hi": nz(m, hi), "l.hi": nz(lo_x, hi), "m.lo": nz(m, lo), "l.lo": nz(lo_x, lo)}


CASES = [
    # H, W, Cin, Cout, kh, kw, stride, pad top, bottom, left, right
    (32, 32, 512, 512, 3, 3, 1, 1, 1, 1, 1),      # the SD VAE decoder's 3x3 convs
    (48, 48, 512, 256, 3, 3, 1, 1, 1, 1, 1),
    (64, 64, 256, 256, 3, 3, 1, 1, 1, 1, 1),
    (64, 64, 256, 128, 3, 3, 1, 1, 1, 1, 1),
    (96, 96, 128, 128, 3, 3, 1, 1, 1, 1, 1),
    (48, 48, 512, 256, 1, 1, 1, 0, 0, 0, 0),      # its 1x1 shortcuts
    (64, 64, 256, 128, 1, 1, 1, 0, 0, 0, 0),
    (64, 64, 128, 3, 3, 3, 1, 1, 1, 1, 1),        # conv_out: Cout = 3
    (24, 24, 16, 64, 3, 3, 1, 1, 1, 1, 1),        # Cin not a multiple of 64: the zero-filled plane tail
    (20, 20, 40, 64, 3, 3, 1, 1, 1, 1, 1),
    (18, 18, 72, 136, 3, 3, 1, 1, 1, 1, 1),
    (16, 16, 200, 64, 3, 3, 1, 1, 1, 1, 1),
    (37, 53, 64, 128, 3, 3, 1, 1, 1, 1, 1),       # odd H and W, not multiples of the box
    (33, 47, 128, 128, 3, 3, 2, 0, 1, 1, 0),      # stride 2, asymmetric pads
    (40, 40, 64, 64, 3, 3, 2, 1, 1, 1, 1),
    (40, 36, 64, 96, 3, 1, 1, 1, 1, 0, 0),        # non-square kernels
    (30, 40, 48, 64, 1, 3, 1, 0, 0, 2, 0),
    (448, 448, 128, 128, 3, 3, 1, 1, 1, 1, 1),    # an fp32 output above the split-K workspace: unsplit, stored from the registers
]


@pytest.mark.parametrize("regime", ["exact", "gauss"])
@pytest.mark.parametrize("epi", ["none", "bias", "bias+res"])
@pytest.mark.parametrize("H,W,Cin,Cout,kh,kw,s,pt,pb,pl,pr", CASES)
def test_f32x_f16w_conv(K, H, W, Cin, Cout, kh, kw, s, pt, pb, pl, pr, epi, regime):
    import torch
    Ho, Wo = _out_size(H, W, kh, kw, s, pt, pb, pl, pr)
    big = Ho * Wo * Cout * 4 > WS_BYTES
    if big and epi == "bias":
        pytest.skip("the largest shape runs without and with the full epilogue")
    assert K.osb_tc_conv_f32x_f16w_ok(H, W, Cin, Cout, kh, kw, s, Ho, Wo) == 1
    g = torch.Generator(device="cuda").manual_seed(H + 3 * Cin + 7 * Cout + kh)
    bias = res = None
    if epi != "none":
        bias, res = _operands("exact" if regime == "exact" else "gauss", g, [(Cout,), (Ho, Wo, Cout) if epi == "bias+res" else None], torch.float32, lim=7)
    if regime == "exact":
        cases = [_exact_operands(c, H, W, Cin, Cout, kh, kw, H + Cin + Cout + i) for i, c in enumerate(("m", "l"))]
    else:
        x, w = _operands("gauss", g, [(H, W, Cin), (Cout, kh, kw, Cin)], torch.float32, row_scaled=1)
        cases = [(x, (w * 0.05).half())]
    seen = {}
    for x, w in cases:
        rc, n, y = _run(K, x, w, bias, res, s, pt, pl, Ho, Wo)
        assert rc == 0 and n in (2, 3), (rc, n)          # the split of x, the conv, the fp32 reduce when split
        if big:
            assert n == 2, "an output above the workspace runs unsplit"
        ref, absref = _ref(x, w, bias, res, s, pt, pl, Ho, Wo)
        what = f"conv_f32x_f16w {(H, W, Cin, Cout, kh, kw, s, pt, pb, pl, pr)} {epi} {regime}"
        if regime == "exact":
            prods = _products(x, w, s, pt, pl, Ho, Wo)
            assert not prods["l.lo"], "the dropped product x_l w_lo must be zero for the exact regime"
            for k_, v in prods.items():
                seen[k_] = seen.get(k_, False) or v
            _check_exact(y, ref, absref, what)
        else:
            _check(y, ref, absref, what)
    if regime == "exact":
        assert all(seen[p] for p in ("h.hi", "h.lo", "m.hi", "l.hi", "m.lo")), seen


def test_f32x_f16w_conv_split_k(K):
    """A deep small conv (8 x 8 x 1280 -> 1280, 180 k-blocks): forced splits agree with the unsplit launch bit for bit in the exact regime,
    and launch the split of x, the conv and the reduce (unsplit: no reduce); the rule's own pick is a split launch."""
    import torch
    H = W = 8
    Cin = Cout = 1280
    g = torch.Generator(device="cuda").manual_seed(11)
    bias, res = _operands("exact", g, [(Cout,), (H, W, Cout)], torch.float32, lim=7)
    try:
        for case in ("m", "l"):
            x, w = _exact_operands(case, H, W, Cin, Cout, 3, 3, 3 if case == "m" else 4)
            ref, absref = _ref(x, w, bias, res, 1, 1, 1, H, W)
            K.osb_tc_set_tile(0, 0, 1)
            rc, n, y1 = _run(K, x, w, bias, res, 1, 1, 1, H, W)
            assert (rc, n) == (0, 2)
            _check_exact(y1, ref, absref, f"conv_f32x_f16w split 1 {case}")
            for sp in (2, 3, 7, 13, 64):
                K.osb_tc_set_tile(0, 0, sp)
                rc, n, y = _run(K, x, w, bias, res, 1, 1, 1, H, W)
                assert (rc, n) == (0, 3), sp
                assert torch.equal(y, y1), f"split {sp} differs from the unsplit launch"
            K.osb_tc_set_tile(0, 0, 0)
            rc, n, y = _run(K, x, w, bias, res, 1, 1, 1, H, W)
            assert (rc, n) == (0, 3), "the rule splits a 10-tile launch of 180 k-blocks"
            assert torch.equal(y, y1)
    finally:
        K.osb_tc_set_tile(0, 0, 0)


def test_f32x_f16w_conv_one_hot_returns_the_filter(K):
    """A 1x1 conv on a one-hot image (pixel p = channel p) returns every fp16 filter value bit for bit as fp32: full 11-bit significands,
    subnormals, +-65504 and signed zeros."""
    import torch
    Cin, Cout = 64, 256
    bits = torch.arange(Cin * Cout, dtype=torch.int64) * 2654435761 % 65536 - 32768
    w = bits.to(torch.int16).view(torch.float16).reshape(Cout, 1, 1, Cin).cuda()
    w = torch.where(torch.isfinite(w), w, torch.zeros_like(w))
    w[:8, 0, 0, 0] = torch.tensor([65504, -65504, 6e-8, -6e-8, 0.0, -0.0, 2047 / 1024, 1.0009765625], dtype=torch.half)
    w[:4, 0, 0, 1] = torch.tensor([6.1e-5, 3.05e-5, -1.5e-7, 0.000999], dtype=torch.half)
    x = torch.eye(Cin, device="cuda").reshape(8, 8, Cin)
    rc, n, y = _run(K, x, w, None, None, 1, 0, 0, 8, 8)
    assert rc == 0
    got = y.reshape(Cin, Cout)
    want = w.reshape(Cout, Cin).t().float()
    assert torch.equal(got.view(torch.int32)[want != 0], want.view(torch.int32)[want != 0]), "nonzero values bit for bit"
    assert torch.equal(got[want == 0], want[want == 0])


def test_f32x_f16w_conv_refusals(K):
    """Shapes and pointers outside the kernel return cudaErrorNotSupported and launch nothing."""
    import torch
    x = torch.zeros(16 * 16 * 64 + 16, device="cuda")
    w = torch.zeros(128 * 9 * 64 + 16, device="cuda", dtype=torch.half)
    y = torch.zeros(16 * 16 * 128 + 16, device="cuda")
    b = torch.zeros(128 + 4, device="cuda")
    pl = torch.empty(3 * 16 * 16 * 64 + 16, device="cuda", dtype=torch.bfloat16)
    px, pw, py, pb, pp = x.data_ptr(), w.data_ptr(), y.data_ptr(), b.data_ptr(), pl.data_ptr()
    ok = (px, pw, pb, py, py, 16, 16, 64, 128, 3, 3, 1, 1, 1, 16, 16, pp)
    def with_(**kw):
        names = ("x", "w", "bias", "res", "y", "H", "W", "Cin", "Cout", "kh", "kw", "s", "pt", "pl", "Ho", "Wo", "planes")
        return tuple(kw.get(k, v) for k, v in zip(names, ok))
    for what, args in [("Cin % 8", with_(Cin=60)), ("Cin < 16", with_(Cin=8)), ("stride 3", with_(s=3, Ho=6, Wo=6)), ("kh > 7", with_(kh=8, Ho=11)),
                       ("kw > 7", with_(kw=8, Wo=11)), ("H W < 64", with_(H=7, W=8, Ho=7, Wo=8)), ("unaligned x", with_(x=px + 4)),
                       ("unaligned w", with_(w=pw + 2)), ("unaligned planes", with_(planes=pp + 8)), ("unaligned y", with_(y=py + 4)),
                       ("unaligned residual", with_(res=py + 4)), ("unaligned bias", with_(bias=pb + 2))]:
        K.osb_launch_count_reset()
        rc = K.osb_tc_conv_f32x_f16w(*args, _stream())
        assert (rc, int(K.osb_launch_count())) == (NOT_SUPPORTED, 0), what
    assert K.osb_tc_conv_f32x_f16w_ok(16, 16, 64, 128, 3, 3, 1, 16, 16) == 1
    assert K.osb_tc_conv_f32x_f16w_ok(448, 448, 128, 128, 3, 3, 1, 448, 448) == 1, "no bound from the workspace"
    assert K.osb_tc_conv_f32x_f16w_ok(16, 16, 60, 128, 3, 3, 1, 16, 16) == 0
    K.osb_launch_count_reset()
    assert K.osb_tc_conv_f32x_f16w(*ok, _stream()) == 0 and int(K.osb_launch_count()) == 2
    torch.cuda.synchronize()


# ---- the engine: fp32-arithmetic VAE decoder / UNet on fp16 blobs ---------------------------------------------------------------------------

@pytest.fixture(scope="module")
def workdir():
    with tempfile.TemporaryDirectory(prefix="osb200_f16wconv_") as d:
        yield d


def _convs(d):
    """(Cin, Cout, kh, kw, Ho Wo) of every Conv with an fp16 weight in model.txt, and the number of fp16 weight references outside those
    weights."""
    convs, other = [], 0
    for line in open(d + "model.txt").read().splitlines():
        refs = re.findall(r"\(float16:([0-9,]*)\)", line)
        if ":Conv*" in line:
            o, i, kh, kw = (int(v) for v in refs[0].split(","))
            _, _, ho, wo = (int(v) for v in re.search(r"\*output:[^(]*\(([0-9,]*)\)", line).group(1).split(","))
            convs.append((i, o, kh, kw, ho * wo))
            other += len(refs) - 1
        else:
            other += len(refs)
    return convs, other


def _new_route(c):
    """The engine's shape rule (engine_run.cpp op_conv): Cin % 8 == 0, Cin >= 16 and an output of at least 128 x 128 pixels (every output
    of these graphs fits the expanded route's workspace)."""
    return c[0] % 8 == 0 and c[0] >= 16 and c[4] >= 128 * 128


# levels 32 x 32, 64 x 64 and 128 x 128: the last one's convs take the new route, the others the expanded one
ROUTE_VAE = emit.VAEConfig(latent=32, block_ch=(32, 32, 16), layers_per_block=1, groups=8, mid_attention=False)
VAE_IN = {"input_2E_1": np.random.default_rng(7).standard_normal((1, 4, 32, 32)).astype(np.float32)}


def _vae(workdir, tag, cfg, wdtype):
    d = os.path.join(workdir, f"{tag}_{wdtype}") + "/"
    if not os.path.exists(d + "model.txt"):
        emit.emit_vae_decoder(d, cfg, wdtype)
    return d


def test_f32_conv_route_reads_f16_weights(engine_lib, workdir):
    """A streamed fp32 VAE-decoder-shaped run on fp16 blobs launches the new kernel once per Conv the shape rule gives it, and for those convs
    no bf16x3 expansion, no CUDA-core conv and no fp16 -> fp32 weight conversion: every other conv keeps the expanded route (two expansions
    each, its fp16 weight converted), and the run converts exactly the fp16 weights outside the new route's convs."""
    from kernel_trace import trace_run
    d = _vae(workdir, "route", ROUTE_VAE, "float16")
    _, names = trace_run(engine_lib, d, VAE_IN, (), wp="ram+nocache")
    convs, other = _convs(d)
    new = [c for c in convs if _new_route(c)]
    assert len(new) >= 4 and len(convs) - len(new) >= 4
    assert sum(KERNEL in n for n in names) == len(new), names
    assert sum("bf16x3_expand" in n for n in names) == 2 * (len(convs) - len(new)), names
    assert not [n for n in names if "igemm" in n], names
    converts = sum("convert_kernel<__half, float>" in n for n in names)
    assert converts == other + (len(convs) - len(new)), (converts, other)


def test_f32_conv_resident_bytes(engine_lib, workdir):
    """Resident weights: each new-route conv weight is cached once as its fp16 blob (2 bytes per parameter).  The fp32-blob model caches it
    in fp32 and its bf16x6 expansion (4 + 12 bytes per parameter); every other weight costs the same in both.  At the parent the fp16 model
    cached the same fp32 copies and expansions as the fp32 one."""
    res = {}
    for wdtype in ("float16", "float32"):
        d = _vae(workdir, "bytes", ROUTE_VAE, wdtype)
        _, m = run_model(engine_lib, d, VAE_IN, (), wp="ram+nocache", b200_options=(("b200_resident_weights", 1),), runs=2)
        res[wdtype] = int(m.stats()["weight_resident_bytes"])
        m.close()
    convs, _ = _convs(os.path.join(workdir, "bytes_float16") + "/")
    params = sum(i * o * kh * kw for i, o, kh, kw, _ in filter(_new_route, convs))
    assert params > 0
    assert res["float16"] == res["float32"] - 16 * params + 2 * params, (res, params)


# a decoder whose 448 x 448 x 128 convs have an fp32 output above the split-K workspace, and a small UNet at a 256 x 256 latent (its
# 256 x 256 -> 128 x 128 downsampler and the resnet convs with a fused residual take the new route)
PARITY_VAE = emit.VAEConfig(latent=56, block_ch=(128,) * 4, layers_per_block=1)
PARITY_UNET = emit.UNetConfig(latent=256, block_ch=(32, 64, 64), attn_levels=(False, False, False), heads=4, depth=(0, 0, 0), mid_depth=1, ctx_len=7,
                              ctx_dim=48, groups=8)


def _parity_case(workdir, arch):
    if arch == "vae":
        d = _vae(workdir, "parity_vae", PARITY_VAE, "float16")
        rng = np.random.default_rng(9)
        return d, {"input_2E_1": rng.standard_normal((1, 4, 56, 56)).astype(np.float32)}, "outsample"
    d = os.path.join(workdir, "parity_unet_float16") + "/"
    if not os.path.exists(d + "model.txt"):
        emit.emit_unet(d, PARITY_UNET, "float16", seed=3)
    return d, emit.unet_inputs(PARITY_UNET, seed=3), "out_5F_sample"


@pytest.mark.parametrize("arch", ["vae", "unet"])
def test_f32_conv_on_f16_weights_parity(engine_lib, oracle_lib, workdir, arch):
    """fp32 arithmetic on fp16 blobs, streamed, resident and graph replay, against the reference's fp32 run."""
    d, inputs, out = _parity_case(workdir, arch)
    convs, _ = _convs(d)
    assert any(_new_route(c) for c in convs)
    ref = reference_outputs(oracle_lib, d, inputs, ())
    for b200 in ((), (("b200_resident_weights", 1),), (("b200_resident_weights", 1), ("b200_cuda_graph", 1))):
        got, m = run_model(engine_lib, d, inputs, (), wp="ram+nocache", b200_options=b200, runs=3 if b200 else 1)
        assert got[out].shape == ref[out].shape, b200
        r = report(got[out], ref[out])
        assert r["rel_to_max"] <= TOL32, (b200, r)
        m.close()
