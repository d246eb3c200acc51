"""The fused multi-head flash attention (osb_flash_attention) at every head dim the SD 1.5 UNet uses (40, 80, 160) and at d = 128:
the kernel against fp64 math at the UNet's shapes, at ragged ones, at every accepted head dim and on rows of very different scale, the scope osb_flash_attention_ok accepts, bit-identical repeat
launches, and a small UNet whose attention levels have d = 80 and d = 160 -- that it takes the flash route and matches the reference
(stored reference output under tests/golden/oracle, tests/util.py)."""
import ctypes
import os
import tempfile

import pytest

from onnxstream_b200 import emit
from util import reference_outputs, report, run_model

pytestmark = pytest.mark.gpu

F16, F32 = 2, 3
FP16 = ("use_fp16_arithmetic", "fuse_ops_in_attention")


@pytest.fixture(scope="module")
def K(engine_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = ctypes.CDLL(engine_lib)
    vp, i64, cf, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int
    lib.osb_flash_attention.argtypes = [vp, i64, vp, i64, vp, i64, vp, i64, i64, i64, i64, i64, cf, vp]
    lib.osb_flash_attention_ok.argtypes = [i64, i64, i64, ci]
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _inputs(T, Tk, h, d, row_scales=False):
    """q [T, h*d], k / v [Tk, h*d] fp16.  row_scales: query rows spread over three decades (|q| stays below 1e3, well inside fp16) and
    key rows whose norm grows along the sequence, so the rows' maxima keep moving to later key tiles."""
    import torch
    C = h * d
    g = torch.Generator(device="cuda").manual_seed(T * 5 + Tk * 3 + d)
    q = torch.randn(T, C, device="cuda", generator=g)
    k = torch.randn(Tk, C, device="cuda", generator=g)
    v = torch.randn(Tk, C, device="cuda", generator=g)
    if row_scales:
        q *= torch.logspace(-1, 2, T, device="cuda")[torch.randperm(T, device="cuda", generator=g)].view(T, 1)
        k *= torch.linspace(0.25, 2.0, Tk, device="cuda").view(Tk, 1)
    return q.half(), k.half(), v.half()


def _flash(K, q, k, v, T, Tk, h, d):
    import torch
    C = h * d
    o = torch.full((T, C), float("nan"), device="cuda", dtype=torch.half)
    rc = K.osb_flash_attention(q.data_ptr(), C, k.data_ptr(), C, v.data_ptr(), C, o.data_ptr(), C, h, T, Tk, d, 1.0 / d ** 0.5, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    return o


# SD 1.5 UNet levels (8 heads: 64^2 d 40, 32^2 d 80, 16^2 and 8^2 d 160; self-attention and the 77-token context), d = 128, ragged
# T / Tk that end inside a query tile and a key tile, and every head dim the kernel accepts (8 to 160: instantiations change at 48 / 64 /
# 80 / 128)
SHAPES = [(4096, 77, 8, 40), (1024, 1024, 8, 80), (1024, 77, 8, 80), (256, 256, 8, 160), (256, 77, 8, 160), (64, 64, 8, 160),
          (64, 77, 8, 160), (512, 512, 4, 128), (200, 77, 4, 80), (300, 200, 3, 128), (130, 333, 2, 160), (96, 100, 2, 72),
          (64, 30, 2, 136), (320, 1000, 2, 48)] + [(100, 77, 2, d) for d in range(8, 161, 8)]     # every accepted head dim, one ragged shape


def _check(o, q, k, v, h, d):
    """Against softmax(QK^T s)V in fp64 on the fp16-rounded operands, with the bar of test_kernels_gpu.py::test_flash_attention: P is
    rounded to fp16 before the second MMA, so |err| <= 2^-8 * sum|p_i v_i| + 2^-9 |ref| + 1e-4."""
    import torch
    T, Tk = q.shape[0], k.shape[0]
    qh = q.double().view(T, h, d).permute(1, 0, 2); kh = k.double().view(Tk, h, d).permute(1, 0, 2); vh = v.double().view(Tk, h, d).permute(1, 0, 2)
    P = torch.softmax(qh @ kh.transpose(1, 2) / d ** 0.5, dim=-1)
    ref = (P @ vh).permute(1, 0, 2).reshape(T, h * d)
    absref = (P @ vh.abs()).permute(1, 0, 2).reshape(T, h * d)
    err = (o.double() - ref).abs()
    tol = absref * 2.0 ** -8 + ref.abs() * 2.0 ** -9 + 1e-4
    assert not torch.isnan(o).any()
    assert not (err > tol).any(), f"max err {float(err.max()):.4g}, ref max {float(ref.abs().max()):.4g}, bad {(err > tol).sum().item()}"


@pytest.mark.parametrize("T,Tk,h,d", SHAPES)
def test_flash_attention_head_dims(K, T, Tk, h, d):
    q, k, v = _inputs(T, Tk, h, d)
    _check(_flash(K, q, k, v, T, Tk, h, d), q, k, v, h, d)


@pytest.mark.parametrize("T,Tk,h,d", [(1000, 1000, 2, 40), (333, 777, 2, 80), (500, 500, 2, 128), (256, 1024, 1, 160)])
def test_flash_attention_running_max(K, T, Tk, h, d):
    """Rows of very different scale: a kernel that kept the first tile's maximum or skipped the rescaling of O fails."""
    q, k, v = _inputs(T, Tk, h, d, row_scales=True)
    _check(_flash(K, q, k, v, T, Tk, h, d), q, k, v, h, d)


def test_flash_attention_scope(K):
    """fp16, 8 <= d <= 160, d % 8 == 0, T >= 64; a head dim outside the scope is refused by the kernel entry too."""
    import torch
    assert K.osb_flash_attention_ok(1024, 77, 160, F16)
    assert K.osb_flash_attention_ok(1024, 77, 72, F16)
    assert not K.osb_flash_attention_ok(1024, 77, 168, F16)
    assert not K.osb_flash_attention_ok(1024, 77, 84, F16)
    assert not K.osb_flash_attention_ok(1024, 77, 80, F32)
    assert not K.osb_flash_attention_ok(1024, 77, 512, F16)
    q = torch.zeros(64, 168, device="cuda", dtype=torch.half)
    assert K.osb_flash_attention(q.data_ptr(), 168, q.data_ptr(), 168, q.data_ptr(), 168, q.data_ptr(), 168, 1, 64, 64, 168, 1.0, _stream()) != 0


def test_flash_attention_refuses_scales_it_cannot_compute(K):
    """The kernel takes the running maximum over the raw scores times the scale, which is the maximum of the scaled logits only for
    scale > 0: scale 0, a negative scale, inf and NaN are refused before anything is enqueued, and the output stays as it was."""
    import torch
    T, Tk, h, d = 128, 77, 2, 80
    q, k, v = _inputs(T, Tk, h, d)
    C = h * d
    o = torch.full((T, C), 7.0, device="cuda", dtype=torch.half)
    for scale in (0.0, -1.0, -1.0 / d ** 0.5, float("inf"), float("nan")):
        n0 = K.osb_launch_count()
        rc = K.osb_flash_attention(q.data_ptr(), C, k.data_ptr(), C, v.data_ptr(), C, o.data_ptr(), C, h, T, Tk, d, scale, _stream())
        torch.cuda.synchronize()
        assert rc != 0 and K.osb_launch_count() == n0, scale
    assert bool((o == 7.0).all())


@pytest.mark.parametrize("T,Tk,h,d", [(1024, 1024, 8, 40), (1024, 77, 8, 80), (256, 256, 8, 160)])
def test_flash_attention_repeatable(K, T, Tk, h, d):
    """Two launches on the same inputs give the same bits."""
    import torch
    q, k, v = _inputs(T, Tk, h, d)
    a = _flash(K, q, k, v, T, Tk, h, d)
    b = _flash(K, q, k, v, T, Tk, h, d)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def _unet_d80_d160():
    # level 0: 16 x 16 = 256 tokens at 160 channels / 2 heads = d 80; level 1 and the mid block: 8 x 8 = 64 tokens, d 160
    return emit.UNetConfig(latent=16, block_ch=(160, 320), attn_levels=(True, True), layers_per_block=1, heads=2, depth=(1, 1),
                           mid_depth=1, ctx_len=7, ctx_dim=48, groups=8)


@pytest.fixture(scope="module")
def unet_d80_d160():
    with tempfile.TemporaryDirectory(prefix="osb200_fa_") as d:
        cfg = _unet_d80_d160()
        emit.emit_unet(d + "/", cfg, "float16", seed=5)
        yield d + "/", emit.unet_inputs(cfg)


def test_unet_attention_takes_the_flash_route(engine_lib, unet_d80_d160):
    """Every attention of the model (one Softmax node each, all with T >= 64) becomes one flash launch instead of the QK^T and PV
    tensor-core GEMMs: the tensor-core launches of one run with b200_flash_attention off, minus those with it on, are the attention
    count."""
    d, inputs = unet_d80_d160
    with open(d + "model.txt") as f:
        n_attn = sum(1 for line in f if line.split("*")[0].split(":")[-1] == "Softmax")     # <name>:<op type>*<inputs>...
    assert n_attn == 14

    def tc_launches(flash):
        _, m = run_model(engine_lib, d, inputs, FP16, wp="ram+nocache", b200_options=(("b200_flash_attention", flash),), runs=2)
        n = int(m.stats()["tc_launches"])
        m.close()
        return n

    on, off = tc_launches(1), tc_launches(0)
    assert off - on == n_attn, (on, off)


def test_unet_d80_d160_parity(engine_lib, oracle_lib, unet_d80_d160):
    """The model's output against the reference's fp16 mode, and flash on against flash off."""
    d, inputs = unet_d80_d160
    out = "out_5F_sample"
    ref = reference_outputs(oracle_lib, d, inputs, FP16)
    got, _ = run_model(engine_lib, d, inputs, FP16)
    off, _ = run_model(engine_lib, d, inputs, FP16, b200_options=(("b200_flash_attention", 0),))
    assert report(got[out], ref[out])["rel_to_max"] <= 3e-2, report(got[out], ref[out])
    assert report(got[out], off[out])["rel_to_max"] <= 1e-2, report(got[out], off[out])


def test_engine_fp16_mha_negative_scale_keeps_the_chain(engine_lib):
    """An fp16 multi-head attention block whose Mul scalar is -1 (d = 80).  On the flash kernel the running maximum would be the smallest
    logit, and P = 2^(x - m) overflows fp16 once a row's logits spread over more than ~16 log2 units, as they do here.  The engine runs
    the chain instead: as many tensor-core launches as with b200_flash_attention = 0, the same bits, finite, and softmax(-QK^T)V in fp64."""
    import numpy as np
    T, C, heads = 256, 160, 2
    d = C // heads
    x = np.random.default_rng(3).standard_normal((1, T, C), dtype=np.float32)
    with tempfile.TemporaryDirectory(prefix="osb200_fa_neg_") as dirname:
        g = emit.GraphBuilder(dirname + "/", "float16", 0, keep_in_memory=True)
        xi = g.input("x", (1, T, C))
        o = g.attention(xi, xi, heads, scale=-1.0)
        g.mark_output(o)
        g.finish()
        res = {}
        for flash in (1, 0):
            got, m = run_model(engine_lib, dirname + "/", {"x": x}, FP16, b200_options=(("b200_flash_attention", flash),))
            res[flash] = (np.asarray(got[o.name], dtype=np.float64), int(m.stats()["tc_launches"]))
            m.close()
    (on, tc_on), (off, tc_off) = res[1], res[0]
    assert tc_on == tc_off, (tc_on, tc_off)
    assert np.isfinite(on).all()
    assert np.array_equal(on, off)
    # fp64 on the fp16 input and weights: q / k / v projections (bias-free), per-head softmax(-q k^T) v, output projection with bias
    blobs = [a for _, a in g.blobs.values() if a.dtype == np.float16]
    wq, wk, wv, wo = [a.astype(np.float64) for a in blobs if a.ndim == 2]
    bo = [a for a in blobs if a.ndim == 1 and a.size == C][-1].astype(np.float64)
    xh = x[0].astype(np.float16).astype(np.float64)
    qh, kh, vh = [(xh @ w).reshape(T, heads, d).transpose(1, 0, 2) for w in (wq, wk, wv)]
    s = -(qh @ kh.transpose(0, 2, 1))
    spread = (s.max(axis=-1) - s.min(axis=-1)).min() / np.log(2.0)
    assert spread > 16, spread
    p = np.exp(s - s.max(axis=-1, keepdims=True))
    p /= p.sum(axis=-1, keepdims=True)
    ref = (p @ vh).transpose(1, 0, 2).reshape(T, C) @ wo + bo
    assert report(on.reshape(T, C), ref)["rel_to_max"] <= 3e-2, report(on.reshape(T, C), ref)
