"""The fp32 wide-head flash attention on the tensor cores (osb_flash_attention_wide_f32x, 160 < d <= 512: bf16 triple split): the
kernel against fp64 math with both K layouts at the VAE's single-head d = 512 and at ragged shapes, held to the bar of
test_flash_attention_f32_gpu.py (relative to torch's own fp32 attention); the scope osb_flash_attention_wide_f32x_ok and the launch
refusals; bit-identical repeat launches; the engine route for an fp32 MatMul-Mul-Softmax-MatMul with a wide head -- no [T, Tk] score
buffer in the activation pool -- and a VAE decoder with a 512-wide mid block in fp32 and in fp32 arithmetic on fp16 weights, whole
and tiled, against the reference (stored reference outputs under tests/golden/oracle, tests/util.py)."""
import ctypes
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from test_flash_attention_f32_gpu import _check as _check_merged
from util import model_text, reference_outputs, report, run_model, stored_reference

pytestmark = pytest.mark.gpu

F16, F32 = 2, 3
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
    lib.osb_flash_attention_wide_f32x.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, cf, ci, vp, vp]
    lib.osb_flash_attention_wide_f32x_ok.argtypes = [i64, i64, i64, ci]
    lib.osb_flash_attention_wide_ok.argtypes = [i64, i64, i64, ci]
    lib.osb_launch_count.restype = ctypes.c_uint64
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _inputs(T, Tk, h, d, row_scales=False):
    """q [h,T,d], k / v [h,Tk,d] fp32.  row_scales: query rows spread over three decades and key rows whose norm grows along the
    sequence, so the rows' maxima keep moving to later key tiles and logits reach several hundred."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(T * 5 + Tk * 3 + d + h)
    q = torch.randn(h, T, d, device="cuda", generator=g)
    k = torch.randn(h, Tk, d, device="cuda", generator=g)
    v = torch.randn(h, Tk, d, device="cuda", generator=g)
    if row_scales:
        q *= torch.logspace(-1, 2, T, device="cuda")[torch.randperm(T, device="cuda", generator=g)].view(1, T, 1)
        k *= torch.linspace(0.25, 2.0, Tk, device="cuda").view(1, Tk, 1)
    return q, k, v


def _planes(T, Tk, h, d):
    import torch
    return torch.empty(3 * (T + 2 * Tk) * h * d, device="cuda", dtype=torch.bfloat16)


def _wide32(K, q, k, v, kt):
    """out [h,T,d] from the kernel at scale 1/sqrt(d); kt: K passed pre-transposed as [h,d,Tk]."""
    import torch
    h, T, d = q.shape
    Tk = k.shape[1]
    kk = k.transpose(1, 2).contiguous() if kt else k
    o = torch.full((h, T, d), float("nan"), device="cuda")
    pl = _planes(T, Tk, h, d)
    rc = K.osb_flash_attention_wide_f32x(q.data_ptr(), kk.data_ptr(), v.data_ptr(), o.data_ptr(), h, T, Tk, d, 1.0 / d ** 0.5, int(kt),
                                         pl.data_ptr(), _stream())
    assert rc == 0
    torch.cuda.synchronize()
    return o


def _merge(x):
    return x.permute(1, 0, 2).reshape(x.shape[1], -1)


def _check(o, q, k, v):
    """test_flash_attention_f32_gpu.py's bar on [h, T, d] tensors: max and RMS error against fp64 at most 4x those of torch's fp32
    attention (TF32 off), and at most 1e-4 max|ref|."""
    h, d = q.shape[0], q.shape[2]
    _check_merged(_merge(o), _merge(q), _merge(k), _merge(v), h, d)


# (T, Tk, heads, d, K pre-transposed): the VAE's single head at d = 512 (32^2 and 64^2 latents), T / Tk that end inside a query tile
# and a key tile (a transposed K with Tk % 8 != 0 included), every head-dim class above 160 (168: one partial 64-column chunk;
# 320 / 448: a partial second slice of V), several heads
SHAPES = [(1024, 1024, 1, 512, True), (1024, 1024, 1, 512, False), (4096, 4096, 1, 512, True), (4096, 4096, 1, 512, False),
          (77, 77, 1, 512, False), (77, 77, 1, 512, True), (1000, 1000, 1, 512, True), (1000, 1000, 1, 512, False), (130, 72, 1, 512, True),
          (65, 1000, 1, 512, True), (200, 333, 1, 512, True), (300, 240, 1, 168, True), (300, 241, 1, 168, False), (256, 256, 1, 256, True),
          (300, 240, 1, 320, True), (190, 77, 1, 320, False), (300, 240, 1, 448, False), (129, 137, 1, 448, True), (256, 256, 2, 256, True),
          (128, 200, 8, 256, True), (100, 333, 8, 256, False), (300, 241, 2, 512, True)]


@pytest.mark.parametrize("T,Tk,h,d,kt", SHAPES)
def test_flash_attention_wide_f32x_matches_fp64(K, T, Tk, h, d, kt):
    q, k, v = _inputs(T, Tk, h, d)
    _check(_wide32(K, q, k, v, kt), q, k, v)


@pytest.mark.parametrize("T,Tk,d,kt", [(1000, 1000, 512, True), (333, 777, 512, False), (256, 1024, 320, True)])
def test_flash_attention_wide_f32x_running_max(K, T, Tk, d, kt):
    """Rows of very different scale: a kernel that kept the first tile's maximum or skipped the rescaling of O fails."""
    q, k, v = _inputs(T, Tk, 1, d, row_scales=True)
    _check(_wide32(K, q, k, v, kt), q, k, v)


def test_flash_attention_wide_f32x_scope(K):
    """fp32, 160 < d <= 512, d % 8 == 0, T, Tk >= 1; the fp16 wide entry keeps refusing fp32.  The launch refuses what *_ok refuses,
    misaligned pointers, scale <= 0 or non-finite and heads outside 1..65535, and enqueues nothing: the output stays as it was.  A
    transposed K with Tk % 8 != 0 is accepted."""
    import torch
    for d in (168, 256, 320, 512):
        assert K.osb_flash_attention_wide_f32x_ok(1024, 77, d, F32), d
    for T, Tk, d, dt in ((1024, 77, 160, F32), (1024, 77, 516, F32), (1024, 77, 520, F32), (1024, 77, 164, F32), (1024, 77, 80, F32),
                         (1024, 77, 512, F16), (0, 77, 512, F32), (1024, 0, 512, F32)):
        assert not K.osb_flash_attention_wide_f32x_ok(T, Tk, d, dt), (T, Tk, d, dt)
    assert not K.osb_flash_attention_wide_ok(1024, 1024, 512, F32)
    T, Tk = 64, 64
    buf = torch.zeros(64 * 520 + 16, device="cuda")
    out = torch.full((64 * 520 + 16,), 7.0, device="cuda")
    pl = _planes(T, Tk, 1, 520)
    p = buf.data_ptr()

    def refused(d=512, h=1, kt=1, Tk=Tk, off=0, ooff=0, ploff=0, scale=0.05):
        n0 = K.osb_launch_count()
        rc = K.osb_flash_attention_wide_f32x(p + off, p, p, out.data_ptr() + ooff, h, T, Tk, d, scale, kt, pl.data_ptr() + ploff, _stream())
        torch.cuda.synchronize()
        return rc != 0 and K.osb_launch_count() == n0
    for d in (160, 164, 516, 520):
        assert refused(d=d), d
    assert refused(off=4) and refused(ooff=8) and refused(ploff=8)       # q, out, planes off 16-byte alignment
    assert refused(scale=0.0) and refused(scale=-0.05) and refused(scale=float("inf")) and refused(scale=float("nan"))
    assert refused(h=0) and refused(h=65536)
    assert bool((out == 7.0).all())
    assert not refused(kt=1, Tk=60) and not refused(kt=0, Tk=60)


@pytest.mark.parametrize("T,Tk,h,d,kt", [(1000, 1000, 1, 512, True), (300, 241, 2, 320, False)])
def test_flash_attention_wide_f32x_repeatable(K, T, Tk, h, d, kt):
    """Two launches on the same inputs give the same bits."""
    import torch
    q, k, v = _inputs(T, Tk, h, d)
    a = _wide32(K, q, k, v, kt)
    b = _wide32(K, q, k, v, kt)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- through the engine ------------------------------------------------------------------------------------------------------------


def _attention_block(d, T, D, scale=None):
    """One fp32 attention as the VAE decoder writes it: graph inputs q [1,T,D], kt [1,D,T] (K already transposed), v [1,T,D];
    MatMul(q, kt) -> Mul(scale, default 1/sqrt(D)) -> Softmax -> MatMul(., v) -> out."""
    g = emit.GraphBuilder(d, "float32", 0)
    q, kt, v = g.input("q", (1, T, D)), g.input("kt", (1, D, T)), g.input("v", (1, T, D))
    s = g.node("MatMul", [q, kt], [(1, T, T)])
    s = g.node("Mul", [s, g.scalar(1.0 / D ** 0.5 if scale is None else scale)], [s.shape])
    p = g.node("Softmax", [s], [s.shape], [("axis", "-1")])
    g.node("MatMul", [p, v], [(1, T, D)], out_names=["out"])
    g.mark_output(emit.T("out", (1, T, D)))
    g.finish()


@pytest.mark.parametrize("T", [16384, 16383])
def test_engine_wide_f32_attention_memory(engine_lib, T):
    """T = 16384 and T = 16383 (a transposed K whose rows are no TMA row stride: the K split transposes it), d = 512, one head, fp32:
    the activation pool's high-water minus the fp32 inputs and output stays within the bf16 planes (18 T d bytes) + 32 MB on the
    flash route; with b200_flash_attention = 0 the remainder holds the fp32 [T, T] score buffer (1 GB).  Output rows against fp64 on a
    seeded sample."""
    import torch
    D = 512
    rng = np.random.default_rng(11)
    q = rng.standard_normal((1, T, D), dtype=np.float32)
    k = rng.standard_normal((1, T, D), dtype=np.float32)
    v = rng.standard_normal((1, T, D), dtype=np.float32)
    inputs = {"q": q, "kt": np.ascontiguousarray(k.transpose(0, 2, 1)), "v": v}
    with tempfile.TemporaryDirectory(prefix="osb200_faw32_") as d:
        _attention_block(d, T, D)
        rest = {}
        for flash in (1, 0):
            got, m = run_model(engine_lib, d + "/", inputs, (), b200_options=(("b200_flash_attention", flash),))
            st = m.stats()
            m.close()
            assert st["h2d_input_bytes"] == 3 * T * D * 4
            rest[flash] = st["act_high_water_bytes"] - (st["h2d_input_bytes"] + T * D * 4)
            if flash:
                out = got["out"]
    assert rest[1] <= 18 * T * D + 32 * MB, rest
    assert rest[0] >= 4 * T * T, rest
    rows = np.sort(np.random.default_rng(3).choice(T, 48, replace=False))
    qt, kt_, vt = (torch.from_numpy(x).cuda() for x in (q, k, v))
    _check(torch.from_numpy(out[:, rows]).cuda(), qt[:, rows], kt_, vt)


@pytest.mark.parametrize("T,sign", [(2304, -1.0), (1024, 1.0), (1600, 1.0)])
def test_engine_wide_f32_keeps_the_chain(engine_lib, T, sign):
    """The kernel's running maximum assumes scale > 0: an fp32 attention whose Mul scalar is negative keeps the three-kernel chain.  So
    does one whose grid (one CTA per 64 queries and 256 columns of d) covers fewer than half of the SMs, where the chain is faster:
    T = 1024 and 1600 at d = 512 (32 and 50 CTAs).  The output and the launch counts are the same with b200_flash_attention on and
    off."""
    D = 512
    rng = np.random.default_rng(12)
    inputs = {"q": rng.standard_normal((1, T, D), dtype=np.float32), "kt": rng.standard_normal((1, D, T), dtype=np.float32),
              "v": rng.standard_normal((1, T, D), dtype=np.float32)}
    with tempfile.TemporaryDirectory(prefix="osb200_faw32_chain_") as d:
        _attention_block(d, T, D, scale=sign / D ** 0.5)
        res = {}
        for flash in (1, 0):
            got, m = run_model(engine_lib, d + "/", inputs, (), b200_options=(("b200_flash_attention", flash),))
            st = m.stats()
            res[flash] = (got["out"], int(st["kernel_launches"]), int(st["tc_launches"]))
            m.close()
    assert res[1][1:] == res[0][1:], (res[1][1:], res[0][1:])
    assert np.array_equal(res[1][0], res[0][0])


def _vae_wide(latent):
    # a 512-wide mid block (one head, d = 512) ahead of a narrow up path: T = latent^2 tokens
    return emit.VAEConfig(latent=latent, block_ch=(512, 32), layers_per_block=1, groups=32)


# the decoder's weights: fp32, or fp16 run in fp32 arithmetic (no options: SDXL's default decode)
WEIGHTS = ["float32", "float16"]


@pytest.fixture(scope="module", params=WEIGHTS)
def vae_wide32(request):
    with tempfile.TemporaryDirectory(prefix="osb200_faw32_vae_") as d:
        emit.emit_vae_decoder(d + "/", _vae_wide(48), request.param, seed=7)
        yield d + "/", {"input_2E_1": np.random.default_rng(9).standard_normal((1, 4, 48, 48)).astype(np.float32)}


def test_vae_wide_f32_takes_the_flash_route(engine_lib, vae_wide32):
    """The mid-block attention becomes the three plane splits and one tensor-core flash launch instead of the QK^T GEMM, scaled softmax
    and PV GEMM (fp32: on the CUDA cores): per attention one launch and one tensor-core launch more than with b200_flash_attention
    off."""
    d, inputs = vae_wide32
    with open(d + "model.txt") as f:
        n_attn = sum(1 for line in f if line.split("*")[0].split(":")[-1] == "Softmax")
    assert n_attn == 1

    def launches(flash):
        _, m = run_model(engine_lib, d, inputs, (), wp="ram+nocache", b200_options=(("b200_flash_attention", flash),), runs=2)
        st = m.stats()
        m.close()
        return int(st["kernel_launches"]), int(st["tc_launches"])

    (on_k, on_tc), (off_k, off_tc) = launches(1), launches(0)
    assert (on_k - off_k, on_tc - off_tc) == (n_attn, n_attn), (on_k, on_tc, off_k, off_tc)


def test_vae_wide_f32_parity(engine_lib, oracle_lib, vae_wide32):
    """The decoder's output against the reference's fp32 arithmetic (DESIGN section 4's fp32 model bar), flash on against flash off,
    and the resident + CUDA-graph replay against the eager run."""
    d, inputs = vae_wide32
    out = "outsample"
    ref = reference_outputs(oracle_lib, d, inputs, ())
    got, _ = run_model(engine_lib, d, inputs, ())
    off, _ = run_model(engine_lib, d, inputs, (), b200_options=(("b200_flash_attention", 0),))
    gr, m = run_model(engine_lib, d, inputs, (), wp="ram+nocache", b200_options=(("b200_resident_weights", 1), ("b200_cuda_graph", 1)), runs=5)
    assert m.stats()["graph_replays"] >= 1
    m.close()
    assert report(got[out], ref[out])["rel_to_max"] <= 2e-4, report(got[out], ref[out])
    assert report(got[out], off[out])["rel_to_max"] <= 2e-5, report(got[out], off[out])
    assert report(gr[out], got[out])["rel_to_max"] <= 2e-5, report(gr[out], got[out])


def test_vae_wide_f32_tiled_decode(engine_lib, oracle_lib):
    """tiled_vae.py's batched decode in fp32 arithmetic on fp16 weights through a decoder built for 48 x 48 latent tiles: T = 2304,
    which ends inside a key tile.  Each sibling's attention takes the flash route (one tensor-core launch more per tile), the batched
    image equals the tile-by-tile one, and it matches the reference decoding tile by tile."""
    from onnxstream_b200 import tiled_vae as tv
    from onnxstream_b200.model import Model
    latent = np.random.default_rng(4).standard_normal((1, 4, 56, 56)).astype(np.float32)     # 2 x 2 tiles (stride 8)
    kw = dict(tile=48, stride=8)
    with tempfile.TemporaryDirectory(prefix="osb200_faw32_tiles_") as d:
        d += "/"
        emit.emit_vae_decoder(d, _vae_wide(48), "float16", seed=8)

        def mk(lib, flash=1):
            m = Model(lib, 4, "nocache")
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
        img_r = stored_reference(("tiled_decode_fp32_arithmetic", model_text(d), {"latent": latent}, sorted(kw.items())),
                                 lambda: {"img": tv.tiled_decode(mk(oracle_lib), latent, "input_2E_1", "outsample", batched=False, **kw)[0]})["img"]
    assert n == 4 and tc_on - tc_off == n, (n, tc_on, tc_off)
    assert report(img_b, img_s)["rel_to_max"] <= 2e-5, report(img_b, img_s)
    assert report(img_b, img_off)["rel_to_max"] <= 2e-5, report(img_b, img_off)
    assert report(img_b, img_r)["rel_to_max"] <= 2e-4, report(img_b, img_r)
