"""The fp32 multi-head flash attention on the tensor cores (osb_flash_attention_f32x: bf16 triple split): the kernel against fp64 math at
the SD 1.5 and SDXL head dims (40, 64, 80, 160) and at ragged shapes, held to a bar relative to torch's own fp32 attention; the scope
osb_flash_attention_f32x_ok accepts and the launch refusals; bit-identical repeat launches; the engine route for one fp32 multi-head
attention block -- no [heads, T, Tk] score buffer in the activation pool -- and a small fp32 UNet with d = 48 / 80 / 160 attention levels
against the reference (stored reference outputs under tests/golden/oracle, tests/util.py), eager and in resident + CUDA-graph mode."""
import ctypes
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from util import reference_outputs, report, run_model

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
    lib.osb_flash_attention_f32x.argtypes = [vp, i64, vp, i64, vp, i64, vp, i64, i64, i64, i64, i64, cf, vp, vp]
    lib.osb_flash_attention_f32x_ok.argtypes = [i64, i64, i64, ci]
    lib.osb_flash_attention_ok.argtypes = [i64, i64, i64, ci]
    lib.osb_launch_count.restype = ctypes.c_uint64
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _inputs(T, Tk, h, d, row_scales=False):
    """q [T, h*d], k / v [Tk, h*d] fp32.  row_scales: query rows spread over three decades and key rows whose norm grows along the
    sequence, so the rows' maxima keep moving to later key tiles and logits reach several hundred."""
    import torch
    C = h * d
    g = torch.Generator(device="cuda").manual_seed(T * 5 + Tk * 3 + d + h)
    q = torch.randn(T, C, device="cuda", generator=g)
    k = torch.randn(Tk, C, device="cuda", generator=g)
    v = torch.randn(Tk, C, device="cuda", generator=g)
    if row_scales:
        q *= torch.logspace(-1, 2, T, device="cuda")[torch.randperm(T, device="cuda", generator=g)].view(T, 1)
        k *= torch.linspace(0.25, 2.0, Tk, device="cuda").view(Tk, 1)
    return q, k, v


def _planes(T, Tk, C):
    import torch
    return torch.empty(3 * (T + 2 * Tk) * C, device="cuda", dtype=torch.bfloat16)


def _flash(K, q, k, v, h, d, scale=None):
    import torch
    T, C = q.shape
    Tk = k.shape[0]
    o = torch.full((T, C), float("nan"), device="cuda")
    pl = _planes(T, Tk, C)
    s = 1.0 / d ** 0.5 if scale is None else scale
    rc = K.osb_flash_attention_f32x(q.data_ptr(), C, k.data_ptr(), C, v.data_ptr(), C, o.data_ptr(), C, h, T, Tk, d, s, pl.data_ptr(), _stream())
    assert rc == 0
    torch.cuda.synchronize()
    return o


def _heads(x, h):
    return x.view(x.shape[0], h, -1).permute(1, 0, 2)


def _merge(x):
    return x.permute(1, 0, 2).reshape(x.shape[1], -1)


def _torch_fp32(q, k, v, h, d):
    """torch's fp32 attention on the math path, TF32 off."""
    import torch
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        P = torch.softmax(_heads(q, h) @ _heads(k, h).transpose(1, 2) * (1.0 / d ** 0.5), dim=-1)
        return _merge(P @ _heads(v, h))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _check(o, q, k, v, h, d):
    """Max and RMS error against fp64 at most 4x those of torch's fp32 attention on the same inputs, and a loose absolute bound.  A
    relative bar is what catches a dropped product: hl / lh are ~2^-18 of a score, the fp32 rounding ~2^-24."""
    import torch
    P = torch.softmax(_heads(q.double(), h) @ _heads(k.double(), h).transpose(1, 2) * (1.0 / d ** 0.5), dim=-1)
    ref = _merge(P @ _heads(v.double(), h))
    t = _torch_fp32(q, k, v, h, d).double()
    assert not torch.isnan(o).any()
    e, et = (o.double() - ref).abs(), (t - ref).abs()
    mx, mxt = float(e.max()), float(et.max())
    rms, rmst = float(e.square().mean().sqrt()), float(et.square().mean().sqrt())
    msg = f"max {mx:.3g} (torch {mxt:.3g}), rms {rms:.3g} (torch {rmst:.3g}), ref max {float(ref.abs().max()):.3g}"
    assert mx <= 4 * mxt and rms <= 4 * rmst, msg
    assert mx <= 1e-4 * max(float(ref.abs().max()), 1.0), msg


# SD 1.5 levels (8 heads: 64^2 d 40, 32^2 d 80, 16^2 and 8^2 d 160; self-attention and the 77-token context), SDXL's d = 64 (10 heads at
# 64^2, 20 at 32^2), and ragged T / Tk that end inside a query tile and a key tile at every tile configuration
SHAPES = [(4096, 4096, 8, 40), (4096, 77, 8, 40), (1024, 1024, 8, 80), (1024, 77, 8, 80), (256, 256, 8, 160), (256, 77, 8, 160),
          (64, 64, 8, 160), (64, 77, 8, 160), (4096, 77, 10, 64), (1024, 1024, 20, 64), (200, 77, 4, 80), (300, 200, 3, 128),
          (130, 333, 2, 160), (96, 100, 2, 72), (65, 30, 2, 136), (320, 1000, 2, 48), (1, 5, 1, 8), (77, 77, 2, 16), (129, 65, 3, 56)] + \
    [(100, 77, 2, d) for d in range(8, 161, 8)]     # every accepted head dim on one ragged shape


@pytest.mark.parametrize("T,Tk,h,d", SHAPES)
def test_flash_attention_f32x_matches_fp64(K, T, Tk, h, d):
    q, k, v = _inputs(T, Tk, h, d)
    _check(_flash(K, q, k, v, h, d), q, k, v, h, d)


@pytest.mark.parametrize("T,Tk,h,d", [(1000, 1000, 2, 40), (333, 777, 2, 80), (256, 1024, 1, 160), (500, 500, 2, 64)])
def test_flash_attention_f32x_running_max(K, T, Tk, h, d):
    """Rows of very different scale: a kernel that kept the first tile's maximum or skipped the rescaling of O fails."""
    q, k, v = _inputs(T, Tk, h, d, row_scales=True)
    _check(_flash(K, q, k, v, h, d), q, k, v, h, d)


def test_flash_attention_f32x_scope(K):
    """fp32, 8 <= d <= 160, d % 8 == 0, T, Tk >= 1; the fp16 kernel keeps refusing fp32.  The launch refuses what *_ok refuses,
    misaligned pointers and strides and scale <= 0, and enqueues nothing: the output stays as it was."""
    import torch
    for d in (8, 40, 64, 80, 128, 160):
        assert K.osb_flash_attention_f32x_ok(1024, 77, d, F32), d
    assert K.osb_flash_attention_f32x_ok(1, 1, 40, F32)
    for T, Tk, d, dt in ((1024, 77, 168, F32), (1024, 77, 84, F32), (1024, 77, 0, F32), (1024, 77, 80, F16), (0, 77, 80, F32), (1024, 0, 80, F32)):
        assert not K.osb_flash_attention_f32x_ok(T, Tk, d, dt), (T, Tk, d, dt)
    assert not K.osb_flash_attention_ok(1024, 77, 80, F32)
    T, Tk, h, d = 64, 64, 2, 80
    C = h * d
    buf = torch.zeros(3 * 64 * 168 * 2 + 16, device="cuda")
    out = torch.full((T * 336 + 16,), 7.0, device="cuda")
    pl = _planes(T, Tk, 2 * 168)
    p = buf.data_ptr()

    def refused(d=d, h=h, ld=C, off=0, ooff=0, ploff=0, scale=0.1):
        n0 = K.osb_launch_count()
        rc = K.osb_flash_attention_f32x(p + off, ld, p, ld, p, ld, out.data_ptr() + ooff, ld, h, T, Tk, d, scale, pl.data_ptr() + ploff, _stream())
        torch.cuda.synchronize()
        return rc != 0 and K.osb_launch_count() == n0
    assert refused(d=168, ld=336) and refused(d=84, ld=168)
    assert refused(off=4) and refused(ooff=8) and refused(ploff=8)       # q, out, planes off 16-byte alignment
    assert refused(ld=C + 2) and refused(ld=C - 8)                        # a row stride that is no multiple of 4 floats / shorter than a row
    assert refused(scale=0.0) and refused(scale=-0.1) and refused(scale=float("inf"))
    assert bool((out == 7.0).all())
    assert not refused()


@pytest.mark.parametrize("T,Tk,h,d", [(1024, 1024, 8, 40), (1024, 77, 8, 80), (256, 256, 8, 160)])
def test_flash_attention_f32x_repeatable(K, T, Tk, h, d):
    """Two launches on the same inputs give the same bits."""
    import torch
    q, k, v = _inputs(T, Tk, h, d)
    a = _flash(K, q, k, v, h, d)
    b = _flash(K, q, k, v, h, d)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- through the engine ------------------------------------------------------------------------------------------------------------


def _mha_block(dirname, T, C, heads):
    """One self-attention block as the UNet exporter writes it (emit.GraphBuilder.attention): x [1, T, C] -> q / k / v projections ->
    head split -> MatMul-Mul-Softmax-MatMul -> head merge -> output projection; returns the output's name."""
    g = emit.GraphBuilder(dirname, "float32", 0)
    x = g.input("x", (1, T, C))
    o = g.attention(x, x, heads)
    g.mark_output(o)
    g.finish()
    return o.name


def test_engine_f32_mha_route_and_memory(engine_lib):
    """T = 4096, 8 heads, d = 40 (C = 320), fp32: the activation pool's high-water minus the fp32 input upload and the fp32 output stays
    below 64 MB on the flash route (q / k / v projections 16 MB + their bf16 planes 24 MB); with b200_flash_attention = 0 the remainder
    holds the fp32 [8, T, T] score buffer (512 MB).  The flash route is one tensor-core launch more (the chain's fp32 GEMMs run on the
    CUDA cores) and fewer launches in all; its output matches the chain's."""
    T, C, heads = 4096, 320, 8
    x = np.random.default_rng(21).standard_normal((1, T, C), dtype=np.float32)
    with tempfile.TemporaryDirectory(prefix="osb200_fa32_") as d:
        name = _mha_block(d, T, C, heads)
        res = {}
        for flash in (1, 0):
            got, m = run_model(engine_lib, d + "/", {"x": x}, (), b200_options=(("b200_flash_attention", flash),))
            st = m.stats()
            m.close()
            assert st["h2d_input_bytes"] == T * C * 4
            res[flash] = (got[name], st["act_high_water_bytes"] - 2 * T * C * 4, int(st["tc_launches"]), int(st["kernel_launches"]))
    (o1, rest1, tc1, k1), (o0, rest0, tc0, k0) = res[1], res[0]
    assert rest1 < 64 * MB, rest1
    assert rest0 >= heads * T * T * 4, rest0
    assert tc1 - tc0 == 1 and k1 < k0, (tc1, tc0, k1, k0)
    assert report(o1, o0)["rel_to_max"] <= 2e-5, report(o1, o0)


def _unet_cfg():
    # 2 heads per level: 32 x 32 = 1024 tokens at 96 channels = d 48 (the reference refuses this graph at d = 40: a Reshape shape check);
    # 16 x 16 = 256 tokens at 160 = d 80; 8 x 8 = 64 tokens at 320 = d 160 (and the mid block); cross-attention over a 7-token context
    return emit.UNetConfig(latent=32, block_ch=(96, 160, 320), attn_levels=(True, True, True), layers_per_block=1, heads=2, depth=(1, 1, 1),
                           mid_depth=1, ctx_len=7, ctx_dim=48, groups=8)


@pytest.fixture(scope="module")
def unet32():
    with tempfile.TemporaryDirectory(prefix="osb200_fa32_unet_") as d:
        cfg = _unet_cfg()
        emit.emit_unet(d + "/", cfg, "float32", seed=6)
        yield d + "/", emit.unet_inputs(cfg)


def test_unet_f32_takes_the_flash_route(engine_lib, unet32):
    """Every attention of the model (one Softmax node each) becomes one tensor-core flash launch (after its plane split) instead of the
    QK^T GEMM, softmax and PV GEMM on the CUDA cores: per attention one tensor-core launch more and one launch fewer in all."""
    d, inputs = unet32
    with open(d + "model.txt") as f:
        n_attn = sum(1 for line in f if line.split("*")[0].split(":")[-1] == "Softmax")
    assert n_attn == 20

    def launches(flash):
        _, m = run_model(engine_lib, d, inputs, (), wp="ram+nocache", b200_options=(("b200_flash_attention", flash),), runs=2)
        st = m.stats()
        m.close()
        return int(st["kernel_launches"]), int(st["tc_launches"])

    (on_k, on_tc), (off_k, off_tc) = launches(1), launches(0)
    assert (off_k - on_k, on_tc - off_tc) == (n_attn, n_attn), (on_k, on_tc, off_k, off_tc)


def test_unet_f32_parity(engine_lib, oracle_lib, unet32):
    """The model's output against the reference's fp32 mode (DESIGN section 4's fp32 model bar), flash on against flash off, and the
    resident + CUDA-graph replay against the eager run."""
    d, inputs = unet32
    out = "out_5F_sample"
    ref = reference_outputs(oracle_lib, d, inputs, ())
    got, _ = run_model(engine_lib, d, inputs, ())
    off, _ = run_model(engine_lib, d, inputs, (), b200_options=(("b200_flash_attention", 0),))
    gr, m = run_model(engine_lib, d, inputs, (), wp="ram+nocache", b200_options=(("b200_resident_weights", 1), ("b200_cuda_graph", 1)), runs=5)
    assert m.stats()["graph_replays"] >= 1
    m.close()
    assert report(got[out], ref[out])["rel_to_max"] <= 2e-4, report(got[out], ref[out])
    assert report(got[out], off[out])["rel_to_max"] <= 2e-5, report(got[out], off[out])
    assert report(gr[out], got[out])["rel_to_max"] <= 2e-5, report(gr[out], got[out])
