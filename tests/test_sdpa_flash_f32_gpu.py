"""fp32 prompt prefill on the tensor cores: the grouped-KV masked flash attention for fp32 (osb_sdpa_flash_f32x: bf16 triple split).

The kernel against fp64 math at the prefill shapes of test_prefill_gpu.py (TinyLlama 32 / 4 heads, Mistral 32 / 8 at d = 128, equal
heads, Tq just above the decode threshold, ragged tiles, fully masked rows) and with rows of very different scale, held to the bar of
test_flash_attention_f32_gpu.py (4x torch's own fp32 attention, and 1e-4 of the output's magnitude); llm.cpp's fp32 mask values
(-3.4028235e38 on part of a row and on whole rows) and -inf over a row's leading key tiles; any finite scale; bit-identical repeat
launches; the scope and the launch refusals.  Through the engine: a Llama prefill in fp32 arithmetic takes one tensor-core launch per
layer, matches the reference (stored reference outputs under tests/golden/oracle, tests/util.py) streamed, resident and with the flash
route off, and an equal-heads prefill at T = 2048 no longer holds the [heads, T, T] fp32 score buffer."""
import ctypes
import os
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from test_prefill_gpu import DYN, MID64, MID128, OPTS32, SDPA_CASES, _prefill_case
from util import reference_outputs, report, run_model

pytestmark = pytest.mark.gpu

F16, F32 = 2, 3
FLT_MAX = float(np.finfo(np.float32).max)


@pytest.fixture(autouse=True)
def _device():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.fixture(scope="module")
def K(engine_lib):
    lib = ctypes.CDLL(engine_lib)
    vp, i64, cf, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int
    lib.osb_sdpa_flash_f32x.argtypes = [vp] * 5 + [i64] * 5 + [cf, vp, vp]
    lib.osb_sdpa_flash_f32x_ok.argtypes = [i64] * 6 + [ci]
    lib.osb_sdpa_flash_ok.argtypes = [i64] * 6 + [ci]
    lib.osb_launch_count.restype = ctypes.c_uint64
    return lib


@pytest.fixture(scope="module")
def workdir():
    with tempfile.TemporaryDirectory(prefix="osb200_pf32_") as d:
        yield d


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _inputs(Hq, Hkv, Tq, Tk, d, row_scales=False):
    """q [Hq, Tq, d], k / v [Hkv, Tk, d] fp32.  row_scales: query rows spread over three decades and key rows whose norm grows along
    the sequence, so the rows' maxima keep moving to later key tiles."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(Hq * 7919 + Tq * 31 + Tk + d)
    q = torch.randn(Hq, Tq, d, device="cuda", generator=g)
    k = torch.randn(Hkv, Tk, d, device="cuda", generator=g)
    v = torch.randn(Hkv, Tk, d, device="cuda", generator=g)
    if row_scales:
        q *= torch.logspace(-1, 2, Tq, device="cuda")[torch.randperm(Tq, device="cuda", generator=g)].view(1, Tq, 1)
        k *= torch.linspace(0.25, 2.0, Tk, device="cuda").view(1, Tk, 1)
    return q, k, v


def _mask(kind, Tq, Tk, past, fill=-65504.0):
    """fp32 additive mask [Tq, Tk]: causal after `past` cached positions (keep[t, j] = j <= past + t) with `fill` on the masked keys;
    band: a padded band inside the cache; full_rows: finite non-trivial values and rows whose every key is masked."""
    import torch
    keep = torch.arange(Tk)[None, :] <= past + torch.arange(Tq)[:, None]
    if kind == "band":
        keep[:, 100:160] = False
    m = torch.where(keep, 0.0, fill).float()
    if kind == "full_rows":
        m[:, :7] = -1.5
        m[[0, 9, 33, 63], :] = fill
    return m.cuda()


def _planes(Hq, Hkv, Tq, Tk, d):
    import torch
    return torch.empty(3 * (Hq * Tq + 2 * Hkv * Tk) * d, device="cuda", dtype=torch.bfloat16)


def _flash(K, q, k, v, mask, scale):
    import torch
    Hq, Tq, d = q.shape
    Hkv, Tk, _ = k.shape
    o = torch.full((Hq, Tq, d), float("nan"), device="cuda")
    pl = _planes(Hq, Hkv, Tq, Tk, d)
    rc = K.osb_sdpa_flash_f32x(q.data_ptr(), k.data_ptr(), v.data_ptr(), mask.data_ptr() if mask is not None else None, o.data_ptr(),
                               Hq, Hkv, Tq, Tk, d, scale, pl.data_ptr(), _stream())
    assert rc == 0
    torch.cuda.synchronize()
    return o


def _logits(q, k, mask, scale, fp32_logits):
    """Q K^T * scale + mask per query head (KV head h // G).  fp32_logits: the logits as fp32 attention forms them -- the exact product
    rounded to fp32, times the scale and plus the mask in fp32 -- for masks whose values swamp the scores (a row masked at -3.4e38
    everywhere is uniform in fp32 and a softmax of the scores in fp64)."""
    G = q.shape[0] // k.shape[0]
    s = q.double() @ k.double().repeat_interleave(G, 0).transpose(1, 2)
    if fp32_logits:
        return (s.float() * scale + mask).double()
    return s * scale + mask.double()


def _torch_fp32(q, k, v, mask, scale):
    """torch's fp32 attention on the math path, TF32 off."""
    import torch
    G = q.shape[0] // k.shape[0]
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        P = torch.softmax(q @ k.repeat_interleave(G, 0).transpose(1, 2) * scale + mask, dim=-1)
        return P @ v.repeat_interleave(G, 0)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _check(o, q, k, v, mask, scale, fp32_logits=False):
    """Max and RMS error against fp64 at most 4x those of torch's fp32 attention (same mask), and at most 1e-4 of max |ref|; no NaN or
    Inf anywhere."""
    import torch
    G = q.shape[0] // k.shape[0]
    ref = torch.softmax(_logits(q, k, mask, scale, fp32_logits), dim=-1) @ v.double().repeat_interleave(G, 0)
    t = _torch_fp32(q, k, v, mask, scale).double()
    assert bool(torch.isfinite(o).all()), "NaN or Inf in the output"
    e, et = (o.double() - ref).abs(), (t - ref).abs()
    mx, mxt = float(e.max()), float(et.max())
    rms, rmst = float(e.square().mean().sqrt()), float(et.square().mean().sqrt())
    msg = f"max {mx:.3g} (torch {mxt:.3g}), rms {rms:.3g} (torch {rmst:.3g}), ref max {float(ref.abs().max()):.3g}"
    assert mx <= 4 * mxt and rms <= 4 * rmst, msg
    assert mx <= 1e-4 * max(float(ref.abs().max()), 1.0), msg
    return ref


@pytest.mark.parametrize("Hq,Hkv,Tq,Tk,d,kind,past", SDPA_CASES)
def test_sdpa_flash_f32x_matches_fp64(K, Hq, Hkv, Tq, Tk, d, kind, past):
    """The prefill shapes of the fp16 kernel's test with fp32 masks; a second launch gives the same bits."""
    import torch
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d)
    mask = _mask(kind, Tq, Tk, past)
    scale = float(np.float32(1.0 / d ** 0.5))
    assert K.osb_sdpa_flash_f32x_ok(Hq, Hkv, Tq, Tk, d, d, F32) == 1
    a = _flash(K, q, k, v, mask, scale)
    b = _flash(K, q, k, v, mask, scale)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "second launch differs"
    _check(a, q, k, v, mask, scale, fp32_logits=kind == "full_rows")


@pytest.mark.parametrize("Hq,Hkv,Tq,Tk,d,past", [(32, 4, 512, 512, 64, 0), (8, 2, 333, 777, 128, 444), (4, 4, 300, 300, 40, 0)])
def test_sdpa_flash_f32x_running_max(K, Hq, Hkv, Tq, Tk, d, past):
    """Rows of very different scale under a causal mask: a kernel that kept the first tile's maximum or skipped the rescaling of O fails."""
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d, row_scales=True)
    mask = _mask("causal", Tq, Tk, past)
    scale = float(np.float32(1.0 / d ** 0.5))
    _check(_flash(K, q, k, v, mask, scale), q, k, v, mask, scale)


@pytest.mark.parametrize("d", [64, 128])
def test_sdpa_flash_f32x_flt_max_mask(K, d):
    """llm.cpp's fp32 mask value: -3.4028235e38 on the masked part of each causal row gives those keys exactly 0 (compared with fp64
    on the same mask); rows masked at -3.4028235e38 everywhere get the softmax of the logits as fp32 forms them, which are all -FLT_MAX:
    uniform weights.  A kernel that folded log2e into the mask would turn the mask into -inf (NaN on the full rows)."""
    import torch
    Hq, Hkv, Tq, Tk, past = 8, 2, 150, 250, 100
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d)
    scale = float(np.float32(1.0 / d ** 0.5))
    mask = _mask("causal", Tq, Tk, past, fill=-FLT_MAX)
    _check(_flash(K, q, k, v, mask, scale), q, k, v, mask, scale)
    full = [0, 17, 77, 149]
    mask[full, :] = -FLT_MAX
    o = _flash(K, q, k, v, mask, scale)
    ref = _check(o, q, k, v, mask, scale, fp32_logits=True)
    G = Hq // Hkv
    uniform = v.double().mean(dim=1).repeat_interleave(G, 0)                # [Hq, d]
    for t in full:
        assert float((ref[:, t] - uniform).abs().max()) <= 1e-12
        assert float((o[:, t].double() - uniform).abs().max()) <= 1e-5


@pytest.mark.parametrize("d", [64, 128])
def test_sdpa_flash_f32x_leading_neg_inf_tiles(K, d):
    """-inf over the first 192 keys of every row (three 64-key tiles at d = 64, six 32-key tiles at d = 128) of rows that have finite
    keys later: those tiles must leave the running maximum, the sums and O untouched instead of making them NaN."""
    Hq, Hkv, Tq, Tk, past = 8, 2, 200, 456, 256
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d)
    scale = float(np.float32(1.0 / d ** 0.5))
    mask = _mask("causal", Tq, Tk, past, fill=float("-inf"))
    mask[:, :192] = float("-inf")
    _check(_flash(K, q, k, v, mask, scale), q, k, v, mask, scale)


@pytest.mark.parametrize("scale", [-0.125, 0.9, 1e-3])
def test_sdpa_flash_f32x_any_scale(K, scale):
    """Any finite scale, negative included: the running maximum is taken over the masked, scaled logits."""
    Hq, Hkv, Tq, Tk, d = 8, 2, 130, 200, 64
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d)
    mask = _mask("causal", Tq, Tk, Tk - Tq)
    _check(_flash(K, q, k, v, mask, scale), q, k, v, mask, scale)


def test_sdpa_flash_f32x_no_mask(K):
    """A null mask is softmax(Q K^T * scale) V."""
    import torch
    Hq, Hkv, Tq, Tk, d = 4, 2, 100, 170, 64
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d)
    scale = float(np.float32(1.0 / d ** 0.5))
    _check(_flash(K, q, k, v, None, scale), q, k, v, torch.zeros(Tq, Tk, device="cuda"), scale)


def test_sdpa_flash_f32x_scope(K):
    """fp32, d % 8 == 0 with 8 <= d <= 128, dv == d, Hq a multiple of Hkv; the fp16 kernel keeps refusing fp32.  The launch refuses what
    *_ok refuses, q / k / v / out / planes off 16-byte alignment, a mask off 4-byte alignment and a scale that is not finite, and
    enqueues nothing: the output stays as it was."""
    import torch
    for d in (8, 40, 64, 80, 128):
        assert K.osb_sdpa_flash_f32x_ok(32, 4, 2048, 2048, d, d, F32), d
    assert K.osb_sdpa_flash_f32x_ok(32, 8, 1, 1, 128, 128, F32)
    for Hq, Hkv, d, dv, dt in ((32, 4, 136, 136, F32), (32, 4, 60, 60, F32), (32, 4, 64, 32, F32), (32, 5, 64, 64, F32), (32, 4, 64, 64, F16),
                               (2, 4, 64, 64, F32), (32, 0, 64, 64, F32)):
        assert not K.osb_sdpa_flash_f32x_ok(Hq, Hkv, 64, 64, d, dv, dt), (Hq, Hkv, d, dv, dt)
    assert not K.osb_sdpa_flash_f32x_ok(32, 4, 0, 64, 64, 64, F32) and not K.osb_sdpa_flash_f32x_ok(32, 4, 64, 0, 64, 64, F32)
    assert not K.osb_sdpa_flash_ok(32, 4, 64, 64, 64, 64, F32)
    Hq, Hkv, Tq, Tk, d = 4, 2, 64, 64, 64
    buf = torch.zeros(Hq * Tq * d + 64, device="cuda")
    mask = torch.zeros(Tq * Tk + 4, device="cuda")
    out = torch.full((Hq * Tq * d + 16,), 7.0, device="cuda")
    pl = torch.empty(3 * (Hq * Tq + 2 * Hkv * Tk) * 136 + 64, device="cuda", dtype=torch.bfloat16)
    p = buf.data_ptr()

    def refused(d=d, Hkv=Hkv, qoff=0, koff=0, voff=0, ooff=0, ploff=0, moff=0, scale=0.125):
        n0 = K.osb_launch_count()
        rc = K.osb_sdpa_flash_f32x(p + qoff, p + koff, p + voff, mask.data_ptr() + moff, out.data_ptr() + ooff, Hq, Hkv, Tq, Tk, d, scale,
                                   pl.data_ptr() + ploff, _stream())
        torch.cuda.synchronize()
        return rc != 0 and K.osb_launch_count() == n0
    assert refused(d=136) and refused(d=60) and refused(Hkv=3)
    assert refused(qoff=4) and refused(koff=8) and refused(voff=4) and refused(ooff=8) and refused(ploff=8)
    assert refused(moff=2)                                                   # mask off 4-byte alignment
    assert refused(scale=float("inf")) and refused(scale=float("-inf")) and refused(scale=float("nan"))
    assert bool((out == 7.0).all())
    assert not refused(moff=4) and not refused(scale=-0.5)                  # a 4-byte-aligned mask and a negative scale are taken


# ---- through the engine ------------------------------------------------------------------------------------------------------------


def _tc_launches(engine_lib, d, inputs, opts, flash):
    from onnxstream_b200.model import Model
    m = Model(engine_lib, 0, "ram+nocache")
    for o in opts:
        m.set_option(o, True)
    m.lib.model_set_option(m.h, b"b200_flash_attention", int(flash))
    m.read_file(d + "model.txt")
    for _ in range(2):                                  # the second run is the counted one
        m.clear_tensors()
        for k, v in inputs.items():
            m.add_tensor(k, v)
        m.run()
    n = int(m.stats()["tc_launches"])
    m.close()
    return n


@pytest.mark.parametrize("turn", ["first", "later"])
@pytest.mark.parametrize("cfgkw", [MID64, MID128], ids=["d64", "d128"])
def test_f32_prefill_attention_takes_the_flash_route(engine_lib, workdir, cfgkw, turn):
    """fp32 arithmetic (use_scaled_dp_attn_op, no use_fp16_arithmetic): one tensor-core attention launch per layer -- the tensor-core
    launches with b200_flash_attention on, minus those with it off, are the layer count."""
    cfg, d, inputs, dyn = _prefill_case(workdir, cfgkw, turn)
    on, off = _tc_launches(engine_lib, d, inputs, OPTS32 + dyn, 1), _tc_launches(engine_lib, d, inputs, OPTS32 + dyn, 0)
    assert on - off == cfg.layers, (on, off)


@pytest.mark.parametrize("turn", ["first", "later"])
@pytest.mark.parametrize("cfgkw", [MID64, MID128], ids=["d64", "d128"])
def test_f32_prefill_parity(engine_lib, oracle_lib, workdir, cfgkw, turn):
    """fp32 arithmetic: logits of every new token and the grown caches, streamed, resident and with the flash route off, against ONE
    reference run at the fp32 model bar (2e-4 of max |ref|); flash on and off agree within 2e-5."""
    cfg, d, inputs, dyn = _prefill_case(workdir, cfgkw, turn)
    names = ("logits", "opkv0", "opkv3")
    ref = reference_outputs(oracle_lib, d, inputs, OPTS32 + dyn, extra_outputs=("opkv0", "opkv3"))
    got = {}
    for b200 in ((), (("b200_resident_weights", 1),), (("b200_flash_attention", 0),)):
        got[b200], _ = run_model(engine_lib, d, inputs, OPTS32 + dyn, extra_outputs=("opkv0", "opkv3"), wp="ram+nocache", b200_options=b200,
                                 runs=2 if b200 else 1)
        for n in names:
            assert got[b200][n].shape == ref[n].shape, (n, b200)
            assert report(got[b200][n], ref[n])["rel_to_max"] <= 2e-4, (n, b200, report(got[b200][n], ref[n]))
    off = got[(("b200_flash_attention", 0),)]
    for n in names:
        assert report(got[()][n], off[n])["rel_to_max"] <= 2e-5, (n, report(got[()][n], off[n]))


def test_f32_prefill_equal_heads_memory(engine_lib, workdir):
    """An equal-heads fp32 prefill of T = 2048 tokens (4 heads, d = 64): the flash route's activation high-water is below the chain's by
    at least the chain's [heads, T, T] fp32 score buffer less the flash route's bf16 planes, and the logits agree."""
    T = 2048
    cfg = emit.LlamaConfig(vocab=259, hidden=256, heads=4, kv_heads=4, head_dim=64, mlp=512, layers=1, past=0, max_pos=T)
    d = os.path.join(workdir, "prefill_f32_eq_2048") + "/"
    emit.emit_llama_decode(d, cfg, "float16", new_tokens=T)
    inputs = emit.llama_inputs(cfg, new_tokens=T)
    res = {}
    for flash in (1, 0):
        got, m = run_model(engine_lib, d, inputs, OPTS32 + DYN, b200_options=(("b200_flash_attention", flash),))
        res[flash] = (got["logits"], m.stats()["act_high_water_bytes"])
        m.close()
    scores = cfg.heads * T * T * 4                                          # 64 MiB
    planes = 6 * (cfg.heads * T + 2 * cfg.kv_heads * T) * cfg.head_dim     # 9 MiB
    slack = 64 << 10                                                        # the pool's 256-byte rounding of the other buffers live then
    assert res[0][1] - res[1][1] >= scores - planes - slack, (res[0][1], res[1][1], scores, planes)
    assert report(res[1][0], res[0][0])["rel_to_max"] <= 2e-5, report(res[1][0], res[0][0])
