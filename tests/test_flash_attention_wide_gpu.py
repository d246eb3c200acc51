"""The wide-head flash attention (osb_flash_attention_wide, 160 < d <= 512): the kernel against fp64 math with both K layouts, at the
VAE's single-head d = 512 and at ragged shapes; the scope osb_flash_attention_wide_ok and the launch entry accept; bit-identical repeat
launches; the engine route for MatMul-Mul-Softmax-MatMul with a wide head -- one launch, no [T, Tk] score buffer in the activation
pool -- and a VAE decoder with a 512-wide mid block, whole and tiled, against the reference (stored reference outputs under
tests/golden/oracle, tests/util.py)."""
import ctypes
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from util import reference_outputs, report, run_model, stored_reference, model_text

pytestmark = pytest.mark.gpu

F16, F32 = 2, 3
FP16 = ("use_fp16_arithmetic", "fuse_ops_in_attention")
MB = 1 << 20


@pytest.fixture(autouse=True)
def _device():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.fixture(scope="module")
def K(engine_lib):
    lib = ctypes.CDLL(engine_lib)
    vp, i64, cf, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int
    lib.osb_flash_attention_wide.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, cf, ci, ci, vp]
    lib.osb_flash_attention_wide_ok.argtypes = [i64, i64, i64, ci]
    lib.osb_launch_count.restype = ctypes.c_uint64
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _inputs(T, Tk, h, d, row_scales=False):
    """q [h,T,d], k [h,Tk,d], v [h,Tk,d] in fp16.  row_scales: query rows spread over four decades and key rows whose norm grows along
    the sequence, so a row's maximum score keeps moving to later key tiles and the running maximum and the rescaling of O matter."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(T * 7 + Tk * 3 + d + h)
    q = torch.randn(h, T, d, device="cuda", generator=g)
    k = torch.randn(h, Tk, d, device="cuda", generator=g)
    v = torch.randn(h, Tk, d, device="cuda", generator=g)
    if row_scales:
        q *= torch.logspace(-2, 2, T, device="cuda")[torch.randperm(T, device="cuda", generator=g)].view(1, T, 1)
        k *= torch.linspace(0.25, 2.0, Tk, device="cuda").view(1, Tk, 1)
    return q.half(), k.half(), v.half()


def _wide(K, q, k, v, kt, scale=None):
    """out [h,T,d] from the kernel; kt: K passed pre-transposed as [h,d,Tk]."""
    import torch
    h, T, d = q.shape
    Tk = k.shape[1]
    kk = k.transpose(1, 2).contiguous() if kt else k
    o = torch.full((h, T, d), float("nan"), device="cuda", dtype=torch.half)
    s = 1.0 / d ** 0.5 if scale is None else scale
    rc = K.osb_flash_attention_wide(q.data_ptr(), kk.data_ptr(), v.data_ptr(), o.data_ptr(), h, T, Tk, d, s, int(kt), F16, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    return o


def _check(o, q, k, v, scale=None):
    """Against softmax(QK^T s)V in fp64 on the fp16-rounded operands, with the bar of test_flash_attention_gpu.py: P is rounded to fp16
    before the second MMA, so |err| <= 2^-8 * sum|p_i v_i| + 2^-9 |ref| + 1e-4."""
    import torch
    d = q.shape[-1]
    s = 1.0 / d ** 0.5 if scale is None else scale
    P = torch.softmax(q.double() @ k.double().transpose(-1, -2) * s, dim=-1)
    ref = P @ v.double()
    absref = P @ v.double().abs()
    err = (o.double() - ref).abs()
    tol = absref * 2.0 ** -8 + ref.abs() * 2.0 ** -9 + 1e-4
    assert not torch.isnan(o).any()
    assert not (err > tol).any(), f"max err {float(err.max()):.4g}, max err/bar {float((err / tol).max()):.3g}, bad {(err > tol).sum().item()}"


# (T, Tk, heads, d, K pre-transposed): the VAE's single head at d = 512 (64^2 latent: T = 4096), T / Tk that end inside a query tile and
# a key tile, every head-dim class above 160 (168: one partial 64-column chunk; 320 / 448: a partial second slice of V), several heads
SHAPES = [(64, 64, 1, 512, True), (64, 64, 1, 512, False), (77, 77, 1, 512, False), (1000, 1000, 1, 512, True), (1000, 1000, 1, 512, False),
          (4096, 4096, 1, 512, True), (4096, 4096, 1, 512, False), (200, 333, 1, 512, False), (130, 72, 1, 512, True), (65, 1000, 1, 512, True),
          (300, 240, 1, 168, True), (300, 241, 1, 168, False), (256, 256, 1, 256, True), (300, 240, 1, 320, True), (190, 77, 1, 320, False),
          (300, 240, 1, 448, False), (129, 136, 1, 448, True), (256, 256, 2, 256, True), (256, 256, 2, 256, False), (128, 200, 8, 256, True),
          (100, 333, 8, 256, False)]


@pytest.mark.parametrize("T,Tk,h,d,kt", SHAPES)
def test_flash_attention_wide_matches_fp64(K, T, Tk, h, d, kt):
    q, k, v = _inputs(T, Tk, h, d)
    _check(_wide(K, q, k, v, kt), q, k, v)


@pytest.mark.parametrize("T,Tk,d,kt", [(1000, 1000, 512, True), (333, 777, 512, False), (256, 1024, 320, True)])
def test_flash_attention_wide_running_max(K, T, Tk, d, kt):
    """Query rows four decades apart in scale and key norms growing along the sequence: most rows find a new maximum in later key tiles
    (scores up to several hundred in log2 units), so a kernel that kept the first tile's maximum or skipped the rescaling of O fails."""
    q, k, v = _inputs(T, Tk, 1, d, row_scales=True)
    _check(_wide(K, q, k, v, kt), q, k, v)


def test_flash_attention_wide_scope(K):
    """fp16, 160 < d <= 512, d % 8 == 0; the launch entry refuses what *_ok refuses, a transposed K with Tk % 8 != 0 and misaligned
    pointers, and launches nothing (the output stays as it was)."""
    import torch
    for d in (168, 256, 512):
        assert K.osb_flash_attention_wide_ok(1024, 77, d, F16)
    for d, dt in ((160, F16), (516, F16), (520, F16), (512, F32), (164, F16), (80, F16)):
        assert not K.osb_flash_attention_wide_ok(1024, 1024, d, dt), (d, dt)
    buf = torch.zeros(4 * 64 * 520 + 8, device="cuda", dtype=torch.half)
    out = torch.full((64 * 520,), 7.0, device="cuda", dtype=torch.half)
    p = buf.data_ptr()

    def refused(d, dt=F16, kt=0, Tk=64, off=0, scale=1.0):
        n0 = K.osb_launch_count()
        rc = K.osb_flash_attention_wide(p + off, p, p, out.data_ptr(), 1, 64, Tk, d, scale, kt, dt, _stream())
        torch.cuda.synchronize()
        return rc != 0 and K.osb_launch_count() == n0
    for d in (160, 516, 520):
        assert refused(d)
    assert refused(512, dt=F32)
    assert refused(512, kt=1, Tk=60)          # K^T rows of 120 bytes: not a TMA row stride
    assert refused(512, off=2)                # q one element off 16-byte alignment
    assert refused(512, scale=0.0) and refused(512, scale=-0.05)     # the running maximum is taken over the raw scores
    assert bool((out == 7.0).all())
    assert not refused(512, kt=1, Tk=64) and not refused(512, kt=0, Tk=60)


@pytest.mark.parametrize("T,Tk,h,d,kt", [(1000, 1000, 1, 512, True), (300, 241, 2, 320, False)])
def test_flash_attention_wide_repeatable(K, T, Tk, h, d, kt):
    """Two launches on the same inputs give the same bits."""
    import torch
    q, k, v = _inputs(T, Tk, h, d)
    a = _wide(K, q, k, v, kt)
    b = _wide(K, q, k, v, kt)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---- through the engine ------------------------------------------------------------------------------------------------------------


def _attention_block(d, T, D, scale=None):
    """One attention as the VAE decoder writes it: graph inputs q [1,T,D], kt [1,D,T] (K already transposed), v [1,T,D];
    MatMul(q, kt) -> Mul(scale, default 1/sqrt(D)) -> Softmax -> MatMul(., v) -> out."""
    g = emit.GraphBuilder(d, "float16", 0)
    q, kt, v = g.input("q", (1, T, D)), g.input("kt", (1, D, T)), g.input("v", (1, T, D))
    s = g.node("MatMul", [q, kt], [(1, T, T)])
    s = g.node("Mul", [s, g.scalar(1.0 / D ** 0.5 if scale is None else scale)], [s.shape])
    p = g.node("Softmax", [s], [s.shape], [("axis", "-1")])
    g.node("MatMul", [p, v], [(1, T, D)], out_names=["out"])
    g.mark_output(emit.T("out", (1, T, D)))
    g.finish()


@pytest.mark.parametrize("T", [16384, 16383])
def test_engine_wide_attention_memory(engine_lib, T):
    """T = 16384 and T = 16383 (a transposed K whose rows are no TMA row stride: the route transposes it to [T, d] first, 16 MB), d = 512,
    one head: the activation pool's high-water minus the device copies of the inputs and the output stays below
    32 MB on the flash route.  The copies live while the attention runs: the fp32 upload of each input (h2d_input_bytes), its fp16 copy
    and the fp16 result (the fp32 copy of the result for the download is made after the fp16 inputs are released).  With
    b200_flash_attention = 0 the remainder holds the fp16 [T, T] score buffer (512 MB).  Output rows against fp64 on a seeded sample."""
    import torch
    D = 512
    rng = np.random.default_rng(11)
    q = rng.standard_normal((1, T, D), dtype=np.float32)
    k = rng.standard_normal((1, T, D), dtype=np.float32)
    v = rng.standard_normal((1, T, D), dtype=np.float32)
    inputs = {"q": q, "kt": np.ascontiguousarray(k.transpose(0, 2, 1)), "v": v}
    with tempfile.TemporaryDirectory(prefix="osb200_faw_") as d:
        _attention_block(d, T, D)
        rest = {}
        for flash in (1, 0):
            got, m = run_model(engine_lib, d + "/", inputs, FP16, b200_options=(("b200_flash_attention", flash),))
            st = m.stats()
            m.close()
            assert st["h2d_input_bytes"] == 3 * T * D * 4
            rest[flash] = st["act_high_water_bytes"] - (st["h2d_input_bytes"] * 1.5 + T * D * 2)
            if flash:
                out = got["out"]
    assert rest[1] < 32 * MB, rest
    assert rest[0] >= T * T * 2, rest
    rows = np.sort(np.random.default_rng(3).choice(T, 48, replace=False))
    qh, kh, vh = (torch.from_numpy(x[0]).cuda().half() for x in (q, k, v))
    scale = float(np.float16(1.0 / D ** 0.5))
    _check(torch.from_numpy(out[0][rows]).cuda().half(), qh[rows], kh, vh, scale)


def test_engine_negative_scale_keeps_the_chain(engine_lib):
    """The kernel's running maximum assumes scale > 0: an attention whose Mul scalar is negative keeps the three-kernel chain, so the
    output and the tensor-core launches are the same with b200_flash_attention on and off."""
    T, D = 256, 512
    rng = np.random.default_rng(12)
    inputs = {"q": rng.standard_normal((1, T, D), dtype=np.float32), "kt": rng.standard_normal((1, D, T), dtype=np.float32),
              "v": rng.standard_normal((1, T, D), dtype=np.float32)}
    with tempfile.TemporaryDirectory(prefix="osb200_faw_neg_") as d:
        _attention_block(d, T, D, scale=-1.0 / D ** 0.5)
        res = {}
        for flash in (1, 0):
            got, m = run_model(engine_lib, d + "/", inputs, FP16, b200_options=(("b200_flash_attention", flash),))
            res[flash] = (got["out"], int(m.stats()["tc_launches"]))
            m.close()
    assert res[1][1] == res[0][1], (res[1][1], res[0][1])
    assert np.array_equal(res[1][0], res[0][0])


def _vae_wide(latent):
    # a 512-wide mid block (one head, d = 512) ahead of a narrow up path: T = latent^2 tokens
    return emit.VAEConfig(latent=latent, block_ch=(512, 32), layers_per_block=1, groups=32)


@pytest.fixture(scope="module")
def vae_wide():
    # latent 48: T = 2304; the chain's QK^T (18 x 18 tiles) and PV (18 x 4) GEMMs fill the SMs unsplit, one launch each
    with tempfile.TemporaryDirectory(prefix="osb200_faw_vae_") as d:
        cfg = _vae_wide(48)
        emit.emit_vae_decoder(d + "/", cfg, "float16", seed=7)
        yield d + "/", {"input_2E_1": np.random.default_rng(9).standard_normal((1, 4, 48, 48)).astype(np.float32)}


def test_vae_wide_takes_the_flash_route(engine_lib, vae_wide):
    """The mid-block attention becomes one flash launch instead of QK^T GEMM, scaled softmax and PV GEMM: two launches fewer in all and
    one fewer on the tensor cores than with b200_flash_attention off."""
    d, inputs = vae_wide
    with open(d + "model.txt") as f:
        n_attn = sum(1 for line in f if line.split("*")[0].split(":")[-1] == "Softmax")
    assert n_attn == 1

    def launches(flash):
        _, m = run_model(engine_lib, d, inputs, FP16, wp="ram+nocache", b200_options=(("b200_flash_attention", flash),), runs=2)
        st = m.stats()
        m.close()
        return int(st["kernel_launches"]), int(st["tc_launches"])

    (on_k, on_tc), (off_k, off_tc) = launches(1), launches(0)
    assert (off_k - on_k, off_tc - on_tc) == (2 * n_attn, n_attn), (on_k, on_tc, off_k, off_tc)


def test_vae_wide_parity(engine_lib, oracle_lib, vae_wide):
    """The decoder's output against the reference's fp16 mode (DESIGN section 4's fp16 model bar), and flash on against flash off."""
    d, inputs = vae_wide
    out = "outsample"
    ref = reference_outputs(oracle_lib, d, inputs, FP16)
    got, _ = run_model(engine_lib, d, inputs, FP16)
    off, _ = run_model(engine_lib, d, inputs, FP16, b200_options=(("b200_flash_attention", 0),))
    assert report(got[out], ref[out])["rel_to_max"] <= 3e-2, report(got[out], ref[out])
    assert report(got[out], off[out])["rel_to_max"] <= 1e-2, report(got[out], off[out])


def test_vae_wide_tiled_decode(engine_lib, oracle_lib):
    """tiled_vae.py's batched decode (every tile a batch sibling of one run) through a decoder built for 12 x 12 latent tiles: T = 144,
    which ends inside a query tile and a key tile.  Each sibling's attention takes the flash route (one tensor-core launch fewer per
    tile), the batched image equals the tile-by-tile one, and it matches the reference decoding tile by tile."""
    from onnxstream_b200 import tiled_vae as tv
    from onnxstream_b200.model import Model
    latent = np.random.default_rng(4).standard_normal((1, 4, 20, 20)).astype(np.float32)     # 2 x 2 tiles (stride 8)
    kw = dict(tile=12, stride=8)
    with tempfile.TemporaryDirectory(prefix="osb200_faw_tiles_") as d:
        d += "/"
        emit.emit_vae_decoder(d, _vae_wide(12), "float16", seed=8)

        def mk(lib, flash=1):
            m = Model(lib, 4, "nocache")
            for o in FP16:
                m.set_option(o, True)
            if lib == engine_lib:
                m.lib.model_set_option(m.h, b"b200_flash_attention", flash)
            m.read_file(d + "model.txt")
            return m

        m_on, m_off = mk(engine_lib, 1), mk(engine_lib, 0)
        img_b, n = tv.tiled_decode(m_on, latent, "input_2E_1", "outsample", batched=True, **kw)
        tc_on = int(m_on.stats()["tc_launches"])
        img_off, _ = tv.tiled_decode(m_off, latent, "input_2E_1", "outsample", batched=True, **kw)
        tc_off = int(m_off.stats()["tc_launches"])
        img_s, _ = tv.tiled_decode(mk(engine_lib), latent, "input_2E_1", "outsample", batched=False, **kw)
        img_r = stored_reference(("tiled_decode", model_text(d), {"latent": latent}, sorted(kw.items())),
                                 lambda: {"img": tv.tiled_decode(mk(oracle_lib), latent, "input_2E_1", "outsample", batched=False, **kw)[0]})["img"]
    assert n == 4 and tc_off - tc_on == n, (n, tc_on, tc_off)
    assert report(img_b, img_s)["rel_to_max"] <= 2e-3
    assert report(img_b, img_off)["rel_to_max"] <= 1e-2, report(img_b, img_off)
    assert report(img_b, img_r)["rel_to_max"] <= 3e-2, report(img_b, img_r)
