"""Kernel-level tests of the bandwidth-bound node kernels (kernels_basic.cu, and the softmax / attention-rows kernels of kernels_gemm.cu)
on every dispatch path, called through the C ABI (include/onnxstream_b200_kernels.h) with torch only providing device memory.

References: fp64 math on the stored inputs for the floating-point kernels, bit-exact fp32 / integer restatements for the elementwise
and data-movement kernels, and oracle/np_oracle.py for the uint8 path.  Output buffers start as NaN (0xAB bytes for integer data) so that
an element a kernel never writes fails.  Each case names the kernel path it targets; each test states its error bar."""
import ctypes
import math
import os
import sys
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
from np_oracle import qu8_add, qu8_mul, qu8_percentiles, qu8_quantize  # noqa: E402

U8, F16, F32, I64 = 1, 2, 3, 4
CUDA_ERROR_INVALID_VALUE = 1
NP = {F16: np.float16, F32: np.float32}


@pytest.fixture(scope="module")
def K(engine_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = ctypes.CDLL(engine_lib)
    vp, i64, ci, cf, sz = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
    pi = ctypes.POINTER(ctypes.c_int64)
    lib.osb_softmax.argtypes = [vp, vp, ci, i64, i64, vp]
    lib.osb_softmax_scaled_ld.argtypes = [vp, vp, ci, i64, i64, i64, cf, vp, i64, vp]
    lib.osb_attention.argtypes = [vp] * 5 + [i64] * 5 + [cf, ci, i64, ci, vp]
    lib.osb_group_norm.argtypes = [vp, vp, ci, ci, i64, i64, ci, vp, vp, cf, ci, vp, vp]
    lib.osb_group_norm_apply.argtypes = [vp, vp, ci, i64, i64, ci, vp, vp, cf, ci, vp, vp, vp]
    lib.osb_channel_add_stats.argtypes = [vp, vp, vp, ci, i64, i64, ci, vp, vp]
    lib.osb_conv2d_ex.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, ci, ci, vp, vp, ci, ctypes.POINTER(ci)]
    lib.osb_instance_norm.argtypes = [vp, vp, ci, i64, i64, vp, vp, cf, vp]
    lib.osb_reduce_mean.argtypes = [vp, vp, ci, i64, i64, vp]
    lib.osb_unary.argtypes = [ci, vp, vp, ci, sz, cf, vp]
    lib.osb_binary.argtypes = [ci, vp, pi, vp, pi, vp, pi, ci, ci, vp]
    lib.osb_convert.argtypes = [vp, ci, vp, ci, sz, cf, ci, vp]
    lib.osb_strided_copy.argtypes = [vp, vp, ci, ci, pi, pi, pi, i64, pi, i64, vp]
    lib.osb_transpose2d.argtypes = [vp, vp, ci, i64, i64, i64, vp]
    lib.osb_gather_rows.argtypes = [vp, vp, vp, i64, i64, i64, vp]
    lib.osb_scatter_elems.argtypes = [vp, vp, vp, i64, ci, vp]
    lib.osb_maxpool_nhwc.argtypes = [vp, vp, ci, i64, i64, i64, ci, ci, ci, ci, ci, i64, i64, vp]
    lib.osb_fill.argtypes = [vp, ci, sz, cf, vp]
    lib.osb_percentiles.argtypes = [vp, ci, sz, ci, cf, cf, vp, vp]
    lib.osb_percentile_key_to_float.argtypes = [ctypes.c_uint, ci]
    lib.osb_percentile_key_to_float.restype = ctypes.c_float
    lib.osb_binary_qu8.argtypes = [ci, vp, pi, cf, ci, vp, pi, cf, ci, vp, cf, ci, pi, ci, vp]
    lib.osb_softmax_qu8.argtypes = [vp, vp, i64, i64, cf, cf, ci, vp]
    lib.osb_launch_count.restype = ctypes.c_uint64
    lib.osb_launch_count_reset.restype = None
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _i64(vals):
    return (ctypes.c_int64 * len(vals))(*[int(v) for v in vals])


def _tdt(dtype):
    import torch
    return {F16: torch.float16, F32: torch.float32}[dtype]


def _offset_view(n, dtype, off, fill=float("nan")):
    """A length-n device vector whose data pointer is `off` elements past a 256-byte aligned allocation (off = 1: misaligned)."""
    import torch
    buf = torch.full((n + 16,), fill, device="cuda", dtype=_tdt(dtype))
    return buf[off:off + n]


def _ulp(ref, dtype):
    """Spacing of the storage type at |ref| (fp16 subnormals included)."""
    return np.spacing(np.abs(ref).astype(NP[dtype])).astype(np.float64)


def _assert_within(got, ref, tol, what):
    got = np.asarray(got, np.float64)
    bad = ~(np.abs(got - ref) <= tol)          # NaN fails
    assert not bad.any(), (f"{what}: {int(bad.sum())} / {bad.size} outside the bar, first at {np.argwhere(bad)[0].tolist()}: "
                           f"got {got[bad][0]!r} want {ref[bad][0]!r} (bar {np.broadcast_to(tol, ref.shape)[bad][0]:.3g})")


# ============================================================================================================================
# 1. softmax family
# ============================================================================================================================

def _softmax_fp32_bar(p, lgap, n, threads, fast_exp):
    """Relative error of an fp32 softmax from fp32 logits: the rounding of x = l - max (2^-24 |x|), exp (expf <= 2 ulp; __expf <= 2 +
    1.17 |x| ulp), the same weighted over the row for the sum, fp32 accumulation of n terms in chains of ceil(n / threads) plus a log2(threads) tree, and
    the final 1/sum and product (2 roundings).  One ulp = 2^-23 relative."""
    e = (2.0 + (1.17 * lgap if fast_exp else 0.0)) * 2.0 ** -23 + lgap * 2.0 ** -24
    acc = (math.ceil(n / threads) + math.log2(max(threads, 1)) + 2) * 2.0 ** -24
    return e + (p * e).sum(-1, keepdims=True) + acc + 2 * 2.0 ** -24


def _softmax_check(got, logits32, dtype, n, threads, fast_exp, what):
    """got vs the fp64 softmax of the fp32 logits the kernel forms: fp32 error (above) plus, for fp16, one rounding of the result
    (half an ulp: 2^-11 relative, 2^-25 absolute below the fp16 normal range).  A -inf logit must give 0 (its gap counts as 0 in the
    bar, which leaves the bar of that element at 1e-38 / 2^-25)."""
    lg = logits32.astype(np.float64)
    mx = lg.max(-1, keepdims=True)
    e = np.exp(lg - mx)
    ref = e / e.sum(-1, keepdims=True)
    rel = _softmax_fp32_bar(ref, np.where(np.isfinite(lg), mx - lg, 0.0), n, threads, fast_exp)
    tol = ref * rel + 1e-38
    if dtype == F16:
        tol = tol + ref * 2.0 ** -11 + 2.0 ** -25
    _assert_within(got, ref, tol, what)


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("rows,cols", [(2500, 1), (2500, 7), (300, 255), (300, 256), (64, 1023), (64, 1024), (33, 5000)])
def test_softmax(K, dtype, rows, cols):
    """osb_softmax (softmax_kernel): 32 threads below 256 columns, 128 below 1024, 256 above; rows > 16 * SMs walk the grid-stride
    row loop.  Bar: see _softmax_check (expf)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(rows * 7 + cols)
    x = (torch.randn(rows, cols, device="cuda", generator=g) * 4).to(_tdt(dtype))
    y = torch.full_like(x, float("nan"))
    assert K.osb_softmax(x.data_ptr(), y.data_ptr(), dtype, rows, cols, _stream()) == 0
    torch.cuda.synchronize()
    threads = 256 if cols >= 1024 else (128 if cols >= 256 else 32)
    _softmax_check(y.cpu().numpy(), x.float().cpu().numpy(), dtype, cols, threads, False, f"softmax {rows}x{cols}")


SCALE = 0.125     # a power of two: x * scale is exact in fp32, so the logit x * scale + mask is ONE rounding with or without an FMA


def _mask_rows(mask_rows, cols, dtype, rng, neg_inf=False):
    """mask row 0: a band of -65504 (fp16) / -3e38 (fp32); row 1: small finite values; row 2: every column masked with the same value.
    neg_inf: -inf instead, over keys [0, 40) on row 0 and over every key but the last on row 2, so that every row keeps a finite key."""
    neg = -65504.0 if dtype == F16 else -3.0e38
    m = np.zeros((mask_rows, cols), np.float32)
    if neg_inf:
        m[0, :min(40, cols - 1)] = -np.inf
    else:
        m[0, cols // 3: cols // 3 + max(cols // 4, 1)] = neg
    if mask_rows > 1:
        m[1, :5] = -1.5
        m[1] += rng.standard_normal(cols).astype(np.float32) * 0.25
    if mask_rows > 2:
        m[2, :] = -np.inf if neg_inf else neg
        if neg_inf:
            m[2, -1] = 0.0
    return m.astype(NP[dtype])


SOFTMAX_LD_CASES = [
    # path, cols, ld, pointer offset (elements)
    ("warp", 1, 1, 0),
    ("warp", 77, 80, 0),          # pad columns [77, 80) must come out exactly 0
    ("warp", 256, 256, 0),
    ("smem", 512, 512, 0),
    ("smem", 4096, 4096, 0),
    ("smem", 12288, 12288, 0),
    ("generic", 300, 300, 0),
    ("generic", 12296, 12296, 0),  # above the shared-memory row limit
    ("generic", 4102, 4102, 0),    # not a multiple of either vector width (8 halves / 4 floats)
    ("generic", 4096, 4096, 1),    # misaligned base pointer
]


@pytest.mark.parametrize("inplace", [False, True])
@pytest.mark.parametrize("masked", [False, True, "ninf"])
@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("path,cols,ld,off", SOFTMAX_LD_CASES)
def test_softmax_scaled_ld(K, path, cols, ld, off, dtype, masked, inplace):
    """osb_softmax_scaled_ld on each of its kernels (warp: ld <= 256, __expf, zero-filled pad columns; smem: 512 <= cols <= 12288,
    aligned, cols % vec == 0, __expf; generic: expf), out of place and in place (x == y, as the engine calls it), with a [3, cols] mask
    broadcast over 7 rows (row r reads mask row r % 3): a masked band, small finite values, and a fully masked row ("ninf": -inf over
    the leading 40 keys and a row whose only finite key is the last).  Row 4 holds logits near 125, which overflow expf unless the row
    maximum is subtracted.  Bar: _softmax_check on the fp32 logits (exact: SCALE is a power of two); a row masked everywhere with -3e38
    (fp32) must be exactly uniform; the pad columns must be exactly 0."""
    import torch
    rows, mask_rows = 7, 3
    rng = np.random.default_rng(cols * 3 + ld + off)
    xv = (rng.standard_normal((rows, ld)) * 6).astype(np.float32)
    xv[4, :] += 1000.0
    xv[:, cols:] = np.nan                      # input pad columns are never read
    xs = xv.astype(NP[dtype])
    tdt = _tdt(dtype)
    xbuf = _offset_view(rows * ld, dtype, off)
    xbuf.copy_(torch.from_numpy(xs.reshape(-1)).cuda())
    if inplace:
        ybuf = xbuf
    else:
        ybuf = _offset_view(rows * ld, dtype, off)
    mask = _mask_rows(mask_rows, cols, dtype, rng, neg_inf=masked == "ninf") if masked else None
    tmask = torch.from_numpy(mask).cuda() if masked else None
    rc = K.osb_softmax_scaled_ld(xbuf.data_ptr(), ybuf.data_ptr(), dtype, rows, cols, ld, SCALE,
                                 tmask.data_ptr() if masked else None, mask_rows if masked else 0, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    got = ybuf.view(rows, ld).cpu().numpy().astype(np.float64)
    logits = xs[:, :cols].astype(np.float32) * np.float32(SCALE)
    if masked:
        logits = (logits + mask[np.arange(rows) % mask_rows].astype(np.float32)).astype(np.float32)
    threads = 256 if cols >= 1024 else (128 if cols >= 256 else 32)
    fast = path != "generic"
    if path == "smem":
        threads = 256
    elif path == "warp":
        threads = 32
    _softmax_check(got[:, :cols], logits, dtype, cols, threads, fast, f"{path} softmax cols {cols} ld {ld}")
    if ld > cols:
        assert (got[:, cols:] == 0).all(), f"pad columns not zero-filled: {got[:, cols:]}"
    if masked is True and dtype == F32:
        full = got[2::mask_rows, :cols]            # rows whose mask row masks every column with -3e38: the logits are all equal
        assert (full == np.float32(1.0) / np.float32(cols)).all(), "a fully masked row is not uniform"


def test_softmax_scaled_ld_refuses_long_padded_rows(K):
    """Padded rows (ld != cols) exist only for the warp kernel (ld <= 256): anything else is refused before any launch."""
    assert K.osb_softmax_scaled_ld(None, None, F16, 4, 300, 304, 1.0, None, 0, _stream()) == CUDA_ERROR_INVALID_VALUE


# ============================================================================================================================
# 2. osb_attention beyond decode: the rows kernel (attention_rows_kernel)
# ============================================================================================================================

NEG_INF_MASKS = ("ninf_lead40", "ninf_splits", "ninf_one_key")


def neg_inf_mask(kind, Tq, Tk, ty):
    """[Tq, Tk] additive mask holding -inf, as an fp32 -FLT_MAX mask or two added -65504 masks become in fp16 and as a left-padded
    prompt masks the leading keys.  ninf_lead40: keys [0, 40); ninf_splits: keys [0, 128) and [256, 384), the first and the third
    128-key split of the split-KV decode kernel; ninf_one_key: every key but the last.  The last 5 keys get -1.5 on top.  Every row
    keeps at least one finite key, so the fp64 answer is finite."""
    import torch
    m = torch.zeros(Tq, Tk, dtype=torch.float64)
    m[:, Tk - 5:] = -1.5
    if kind == "ninf_lead40":
        m[:, :40] = float("-inf")
    elif kind == "ninf_splits":
        m[:, :128] = float("-inf")
        m[:, 256:384] = float("-inf")
    else:
        assert kind == "ninf_one_key", kind
        m[:, :Tk - 1] = float("-inf")
    assert bool(torch.isfinite(m).any(-1).all()), (kind, Tk)
    return m.to(ty).cuda()


ATTN_ROWS_CASES = [
    # heads, Tq, Tk, d, dv, kv_group, k_transposed, mask (True: finite block masks; or a NEG_INF_MASKS kind), dtype
    (4, 3, 20, 40, 40, 1, 1, False, F16),      # K stored [h, d, Tk], Tk < 32
    (4, 5, 77, 64, 64, 2, 1, True, F16),       # Tk not a multiple of 32, grouped KV
    (2, 9, 300, 80, 80, 1, 1, True, F32),
    (2, 17, 300, 40, 72, 2, 1, True, F16),     # k_transposed with dv != d, dv % 32 != 0
    (32, 160, 300, 64, 64, 4, 0, True, F16),   # Tq > 16, grouped KV, heads * Tq > 4096: too many rows for the split-KV decode kernel
    (32, 130, 256, 64, 64, 8, 0, False, F32),
    (4, 20, 100, 40, 72, 2, 0, True, F16),     # dv != d, dv % 32 != 0
    (3, 24, 200, 48, 24, 3, 0, True, F32),
    # -inf over a row's first 32-key block: the running maximum stays -inf through it
    (4, 5, 77, 64, 64, 2, 1, "ninf_lead40", F16),
    (4, 5, 77, 64, 64, 2, 1, "ninf_lead40", F32),
    (4, 5, 77, 64, 64, 2, 0, "ninf_lead40", F16),
    (4, 5, 77, 64, 64, 2, 0, "ninf_lead40", F32),
    (2, 9, 400, 80, 80, 1, 1, "ninf_splits", F32),     # K^T at Tk >= 256
    (2, 17, 400, 40, 72, 2, 1, "ninf_splits", F16),
    (32, 160, 400, 64, 64, 4, 0, "ninf_splits", F16),  # heads * Tq > 4096
    (4, 3, 20, 40, 40, 1, 1, "ninf_one_key", F16),     # the finite key inside the first block
    (3, 24, 200, 48, 24, 3, 0, "ninf_one_key", F32),
    (4, 20, 100, 40, 72, 2, 0, "ninf_one_key", F16),
]


@pytest.mark.parametrize("heads,Tq,Tk,d,dv,group,kt,with_mask,dtype", ATTN_ROWS_CASES)
def test_attention_rows_matches_fp64(K, heads, Tq, Tk, d, dv, group, kt, with_mask, dtype):
    """osb_attention on the per-row online-softmax kernel against fp64 softmax(Q K^T s + mask) V.  The finite mask masks whole 32-key
    blocks with -65504 / -3e38: keys [0, 32) on even query rows -- the first block a row sees -- and keys [64, 96) everywhere; the last
    5 keys get -1.5.  The -inf masks are those of neg_inf_mask.  Bars of test_attention_decode_matches_fp64: 2e-3 (fp16) / 1e-5 (fp32)
    of max(1, max|ref|); every output finite."""
    import torch
    ty = _tdt(dtype)
    g = torch.Generator(device="cuda").manual_seed(heads * 1000 + Tq * 10 + Tk)
    q = torch.randn(heads, Tq, d, device="cuda", generator=g).to(ty)
    k = torch.randn(heads // group, Tk, d, device="cuda", generator=g).to(ty)
    v = torch.randn(heads // group, Tk, dv, device="cuda", generator=g).to(ty)
    kin = k.transpose(1, 2).contiguous() if kt else k
    mask = None
    if with_mask in NEG_INF_MASKS:
        mask = neg_inf_mask(with_mask, Tq, Tk, ty)
    elif with_mask:
        neg = -65504.0 if dtype == F16 else -3.0e38
        mask = torch.zeros(Tq, Tk, device="cuda", dtype=ty)
        mask[0::2, :32] = neg
        mask[:, 64:96] = neg
        mask[:, Tk - 5:] = -1.5
    scale = 1.0 / d ** 0.5
    out = torch.full((heads, Tq, dv), float("nan"), device="cuda", dtype=ty)
    rc = K.osb_attention(q.data_ptr(), kin.data_ptr(), v.data_ptr(), mask.data_ptr() if mask is not None else None, out.data_ptr(),
                         heads, Tq, Tk, d, dv, scale, kt, group, dtype, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    kk = k.double().repeat_interleave(group, 0)
    vv = v.double().repeat_interleave(group, 0)
    s = q.double() @ kk.transpose(1, 2) * scale
    if mask is not None:
        s = s + mask.double()
    ref = torch.softmax(s, -1) @ vv
    tol = (2e-3 if dtype == F16 else 1e-5) * max(1.0, float(ref.abs().max()))
    assert bool(torch.isfinite(out).all()), f"{int((~torch.isfinite(out)).sum())} / {out.numel()} outputs not finite"
    err = float((out.double() - ref).abs().max())
    assert err <= tol, f"max err {err:.3g} > {tol:.3g}"


# ============================================================================================================================
# 3. normalisation and reductions
# ============================================================================================================================

GN_CASES = [
    # path, dtype, nhwc, C, HW, groups, x offset, y offset (elements), launches
    ("fused one-launch NHWC", F16, 1, 320, 1024, 32, 0, 0, 1),
    ("fused one-launch NHWC", F32, 1, 640, 256, 32, 0, 0, 1),
    ("two-pass: vector stats (groups = 64 > 48)", F16, 1, 640, 512, 64, 0, 0, 2),
    ("two-pass: vector stats (groups = 64 > 48)", F32, 1, 256, 300, 64, 0, 0, 2),
    ("two-pass: scalar stats (C = 36, C % vec != 0)", F16, 1, 36, 500, 4, 0, 0, 2),
    ("two-pass: scalar stats (C = 18, C % vec != 0)", F32, 1, 18, 300, 3, 0, 0, 2),
    ("two-pass: scalar stats (C / 8 = 520 > 512)", F16, 1, 4160, 64, 32, 0, 0, 2),
    ("two-pass: vector stats + scalar apply (y misaligned)", F16, 1, 320, 256, 32, 0, 1, 2),
    ("two-pass: scalar stats + scalar apply (x misaligned)", F32, 1, 64, 200, 8, 1, 0, 2),
    ("NCHW, vector apply (HW % 8 == 0)", F16, 0, 64, 256, 8, 0, 0, 2),
    ("NCHW, scalar apply (HW % 8 != 0)", F16, 0, 48, 99, 6, 0, 0, 2),
    ("NCHW, vector apply", F32, 0, 320, 64, 32, 0, 0, 2),
]


def _gn_ref(xd, nhwc, C, HW, G, gamma, beta, silu):
    """fp64 GroupNorm(+SiLU) of x ([HW, C] or [C, HW]); also the per-element mean and rstd it used."""
    xc = xd.reshape(HW, C).T if nhwc else xd.reshape(C, HW)            # [C, HW]
    grp = xc.reshape(G, -1)
    mean = grp.mean(1)
    var = ((grp - mean[:, None]) ** 2).mean(1)
    rstd = 1.0 / np.sqrt(var + 1e-5)
    cpg = C // G
    m_c, r_c = np.repeat(mean, cpg)[:, None], np.repeat(rstd, cpg)[:, None]
    out = (xc - m_c) * r_c * gamma[:, None] + beta[:, None]
    if silu:
        out = out / (1.0 + np.exp(-out))
    to_layout = (lambda a: a.T.reshape(-1)) if nhwc else (lambda a: a.reshape(-1))
    return to_layout(out), to_layout(np.broadcast_to(m_c, xc.shape)), to_layout(np.broadcast_to(r_c * np.abs(gamma[:, None]), xc.shape))


def _run_group_norm(K, dtype, nhwc, C, HW, G, xoff, yoff, silu, offset_mean, seed):
    import torch
    rng = np.random.default_rng(seed)
    n = C * HW
    xs = (offset_mean + rng.standard_normal(n) * (1.0 if offset_mean else 2.0) + (0.0 if offset_mean else 0.25)).astype(NP[dtype])
    gamma = rng.standard_normal(C).astype(NP[dtype])
    beta = rng.standard_normal(C).astype(NP[dtype])
    x = _offset_view(n, dtype, xoff)
    x.copy_(torch.from_numpy(xs).cuda())
    tg, tb = torch.from_numpy(gamma).cuda(), torch.from_numpy(beta).cuda()
    scratch = torch.zeros(2048, device="cuda", dtype=torch.uint8)
    outs, counts = [], []
    for _ in range(2):          # two launches on the same scratch: the path must re-arm (fused) or clear (two-pass) it
        y = _offset_view(n, dtype, yoff)
        K.osb_launch_count_reset()
        rc = K.osb_group_norm(x.data_ptr(), y.data_ptr(), dtype, nhwc, C, HW, G, tg.data_ptr(), tb.data_ptr(), 1e-5, silu, scratch.data_ptr(), _stream())
        assert rc == 0
        torch.cuda.synchronize()
        counts.append(int(K.osb_launch_count()))
        outs.append(y.cpu().numpy().astype(np.float64))
    ref, mean, rg = _gn_ref(xs.astype(np.float64), nhwc, C, HW, G, gamma.astype(np.float64), beta.astype(np.float64), silu)
    return outs, counts, ref, mean, rg


def _gn_tol(ref, mean, rg, dtype):
    """The bar of test_group_norm_nhwc, 2^-9 (fp16) / 2^-18 (fp32) x (|ref| + 4), plus one fp32 ulp of the mean times rstd |gamma|:
    the apply pass subtracts the mean rounded to fp32, which is not negligible against an fp32 input at an offset of 1024."""
    base = (2.0 ** -9 if dtype == F16 else 2.0 ** -18) * (np.abs(ref) + 4.0)
    return base + np.spacing(np.abs(mean).astype(np.float32)).astype(np.float64) * rg * 1.5


@pytest.mark.parametrize("silu", [0, 1])
@pytest.mark.parametrize("path,dtype,nhwc,C,HW,G,xoff,yoff,launches", GN_CASES)
def test_group_norm_paths(K, path, dtype, nhwc, C, HW, G, xoff, yoff, launches, silu):
    """osb_group_norm on every path: the fused rendezvous kernel (1 launch) or statistics + apply (2 launches, counted by
    osb_launch_count), against fp64 GroupNorm(+SiLU) of the stored input.  Both launches on the same scratch must meet the bar (stale
    statistics would double the sums); their bits may differ, as the fp32 shared-memory atomics fold channels in any order.  Bar: _gn_tol."""
    outs, counts, ref, mean, rg = _run_group_norm(K, dtype, nhwc, C, HW, G, xoff, yoff, silu, 0.0, C * 31 + HW + silu)
    assert counts == [launches, launches], f"{path}: expected {launches} launch(es), got {counts}"
    for i, out in enumerate(outs):
        _assert_within(out, ref, _gn_tol(ref, mean, rg, dtype), f"{path}, launch {i + 1}")


GN_OFFSET_CASES = [
    ("fused one-launch NHWC", 1, 320, 4096, 32, 0, 1),
    ("two-pass: vector stats (groups = 64)", 1, 640, 1024, 64, 0, 2),
    ("two-pass: scalar stats (C = 18)", 1, 18, 4096, 3, 0, 2),
    ("NCHW", 0, 320, 4096, 32, 0, 2),
]


@pytest.mark.parametrize("m", [256.0, 1024.0])
@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("path,nhwc,C,HW,G,yoff,launches", GN_OFFSET_CASES)
def test_group_norm_offset_mean(K, path, nhwc, C, HW, G, yoff, launches, dtype, m):
    """x = m + N(0, 1): the group mean is large against the spread, which cancels catastrophically in var = E[x^2] - mean^2 when the
    sums are plain fp32 sums of x and x^2 (at m = 1024 in fp16 rstd came out up to 9 % off).  Bar: _gn_tol."""
    outs, counts, ref, mean, rg = _run_group_norm(K, dtype, nhwc, C, HW, G, 0, yoff, 1, m, int(m) + C)
    assert counts == [launches, launches]
    for i, out in enumerate(outs):
        _assert_within(out, ref, _gn_tol(ref, mean, rg, dtype), f"{path} m = {m}, launch {i + 1}")


# ---- producer statistics (plain fp64 sums of y and y^2 in a two-slot ring) -> osb_group_norm_apply, at large means ----------------

STATS_M = [0.0, 16.0, 64.0, 256.0, 1024.0]         # mean / spread of the GroupNorm input


def _check_gn_slot(stats, yd, HW, C, G, what):
    """The mean and variance osb_group_norm_apply derives from a statistics slot (plain sums S, Q: mean = S/n, var = Q/n - mean^2, in fp64)
    against the fp64 two-pass statistics of the stored y ([HW, C]).  Bar, relative to the variance (not to sum y^2, which is larger by
    1 + mean^2/var): the producers sum y - p in fp32 (p: one stored y of the group, so sum (y - p)^2 is a small multiple of n var) over
    chains of at most a few hundred values, then shift back in fp64 -- |d var| <= 2^-14 var; and the fp64 sums themselves carry a few
    ulps at the mean's scale -- + 2^-48 mean^2.  The mean: |d mean| <= 2^-14 sqrt(var) + 2^-48 |mean|.  Returns the worst error / bar."""
    st = stats.cpu().numpy().astype(np.float64).reshape(-1)[:2 * G].reshape(G, 2)
    grp = yd.reshape(HW, G, C // G).transpose(1, 0, 2).reshape(G, -1)
    n = grp.shape[1]
    mean = grp.mean(1)
    var = ((grp - mean[:, None]) ** 2).mean(1)
    gm = st[:, 0] / n
    gv = st[:, 1] / n - gm * gm
    bar_m = 2.0 ** -14 * np.sqrt(var) + 2.0 ** -48 * np.abs(mean)
    bar_v = 2.0 ** -14 * var + 2.0 ** -48 * mean * mean
    rm, rv = np.abs(gm - mean) / bar_m, np.abs(gv - var) / bar_v
    worst = float(max(rm.max(), rv.max()))
    print(f"[bar] gn-slot {what}: mean {float(rm.max()):.3g}, var {float(rv.max()):.3g} of the bar")
    assert rm.max() <= 1.0 and rv.max() <= 1.0, (f"{what}: slot statistics off: mean err/bar {float(rm.max()):.3g} (group {int(rm.argmax())}), "
                                                 f"var err/bar {float(rv.max()):.3g} (group {int(rv.argmax())}, var {var[rv.argmax()]:.4g}, "
                                                 f"got {gv[rv.argmax()]:.6g}, mean {mean[rv.argmax()]:.4g})")
    return worst


def _check_gn_apply_from_slot(K, y, stats, dtype, HW, C, G, seed, what):
    """osb_group_norm_apply (GroupNorm + SiLU) on the slot against fp64 GroupNorm of the stored y; the other slot must come back zeroed.
    Bar: _gn_tol."""
    import torch
    rng = np.random.default_rng(seed)
    gamma = rng.standard_normal(C).astype(NP[dtype]); beta = rng.standard_normal(C).astype(NP[dtype])
    tg, tb = torch.from_numpy(gamma).cuda(), torch.from_numpy(beta).cuda()
    out = torch.full_like(y, float("nan"))
    clear = torch.ones(2 * G, device="cuda", dtype=torch.float64)
    assert K.osb_group_norm_apply(y.data_ptr(), out.data_ptr(), dtype, C, HW, G, tg.data_ptr(), tb.data_ptr(), 1e-5, 1, stats.data_ptr(), clear.data_ptr(), _stream()) == 0
    torch.cuda.synchronize()
    ref, mean, rg = _gn_ref(y.double().cpu().numpy().reshape(-1), 1, C, HW, G, gamma.astype(np.float64), beta.astype(np.float64), 1)
    _assert_within(out.cpu().numpy().reshape(-1), ref, _gn_tol(ref, mean, rg, dtype), what)
    assert float(clear.abs().max()) == 0.0, f"{what}: the other slot was not cleared"


# HW, C, G: cpg 10, 4 (G = 64), 8 (G = 64) and 40; HW ragged against the CTA pixel strips
CHANNEL_ADD_SHAPES = [(4096, 320, 32), (1000, 256, 64), (999, 512, 64), (333, 960, 24)]


@pytest.mark.parametrize("m", STATS_M)
@pytest.mark.parametrize("addv", [True, False], ids=["add", "stats-only"])
@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("HW,C,G", CHANNEL_ADD_SHAPES)
def test_channel_add_stats_offset_mean(K, HW, C, G, dtype, addv, m):
    """osb_channel_add_stats (gn_stats_nhwc_vec_kernel): with addv, y = x + t[c] is written and its statistics gathered (a resnet's
    time-embedding Add feeding a GroupNorm); without, the statistics of x (a GroupNorm whose producer gathered none).  x = m + 0.5 N(0,1)
    per channel + N(0,1): the group mean is large against the spread at m >= 64.  The slot: _check_gn_slot; GroupNorm(+SiLU) of the
    stored y from it: _gn_tol."""
    import torch
    rng = np.random.default_rng(HW + C + int(m) + 7 * dtype + int(addv))
    xs = (m + 0.5 * rng.standard_normal((1, C)) + rng.standard_normal((HW, C))).astype(NP[dtype])
    x = torch.from_numpy(xs).cuda()
    stats = torch.zeros(2 * G, device="cuda", dtype=torch.float64)
    if addv:
        t = torch.from_numpy(rng.standard_normal(C).astype(NP[dtype])).cuda()
        y = torch.full_like(x, float("nan"))
        assert K.osb_channel_add_stats(x.data_ptr(), t.data_ptr(), y.data_ptr(), dtype, C, HW, G, stats.data_ptr(), _stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(y, (x.float() + t.float()).to(x.dtype))
    else:
        y = x
        assert K.osb_channel_add_stats(x.data_ptr(), None, None, dtype, C, HW, G, stats.data_ptr(), _stream()) == 0
        torch.cuda.synchronize()
    what = f"channel_add_stats {'add' if addv else 'stats-only'} {'f16' if dtype == F16 else 'f32'} HW {HW} C {C} G {G} m {m}"
    _check_gn_slot(stats, y.double().cpu().numpy(), HW, C, G, what)
    _check_gn_apply_from_slot(K, y, stats, dtype, HW, C, G, HW + C, what)


# route, forced (bm, bn, split) or None, CTA-pair mode, Cout, G: every EXTRAS tile, the CTA pairs and the split-K reduce, with cpg
# 10, 4, 8 and 40 spread over them
CONV_STATS_ROUTES = [
    ("tile-128x128", (128, 128, 1), 1, 320, 32),
    ("tile-128x64", (128, 64, 1), 1, 256, 64),
    ("tile-128x80", (128, 80, 1), 1, 320, 8),
    ("tile-128x160", (128, 160, 1), 1, 320, 32),
    ("tile-64x64", (64, 64, 1), 1, 136, 17),
    ("tile-64x128", (64, 128, 1), 1, 256, 64),
    ("tile-64x160", (64, 160, 1), 1, 320, 8),
    ("cta-pair", None, 2, 320, 32),
    ("split-k", (128, 128, 3), 1, 320, 8),
    ("split-k", (64, 128, 2), 1, 256, 64),
]


@pytest.mark.parametrize("m", STATS_M)
@pytest.mark.parametrize("route,force,pair,Cout,G", CONV_STATS_ROUTES, ids=[f"{r[0]}-cpg{r[3] // r[4]}" for r in CONV_STATS_ROUTES])
def test_conv_epilogue_gn_stats_offset_mean(K, route, force, pair, Cout, G, m):
    """osb_conv2d_ex with statistics: the tile epilogue (gn_stats_pair) at every EXTRAS tile, forced with osb_tc_set_tile and pinned by
    the launch profile, through CTA pairs, and the split-K reduce kernel -- the conv output sits at m + O(1) through a large bias (and a
    residual: half of m each in the split-K cases, so the reduce kernel adds both).  On a 25 x 19 image every tile is ragged and some
    warps hold no valid row.  The slot: _check_gn_slot; GroupNorm(+SiLU) of the stored output from it: _gn_tol (fp16)."""
    import torch
    from test_tc_tiles_gpu import _profile
    ci = ctypes.c_int
    K.osb_tc_set_tile.argtypes = [ci] * 3
    K.osb_tc_set_pair_mode.argtypes = [ci]
    H, W, Cin = 25, 19, 64
    g = torch.Generator(device="cuda").manual_seed(Cout * 7 + G + int(m))
    x = torch.randn(H, W, Cin, device="cuda", generator=g).half()
    w = (torch.randn(Cout, 3, 3, Cin, device="cuda", generator=g) / (9 * Cin) ** 0.5).half()
    split = force is not None and force[2] > 1
    bias = ((m / 2 if split else m) + 0.5 * torch.randn(Cout, device="cuda", generator=g)).half()
    bias2 = torch.randn(Cout, device="cuda", generator=g).half()
    res = (m / 2 + torch.randn(H, W, Cout, device="cuda", generator=g)).half() if split else None
    y = torch.full((H, W, Cout), float("nan"), device="cuda", dtype=torch.half)
    stats = torch.zeros(2 * G, device="cuda", dtype=torch.float64)
    done = ci(0)
    if force:
        K.osb_tc_set_tile(*force)
    K.osb_tc_set_pair_mode(pair)
    try:
        prof = _profile(K, lambda: K.osb_conv2d_ex(x.data_ptr(), w.data_ptr(), bias.data_ptr(), bias2.data_ptr(), res.data_ptr() if split else None,
                                                   y.data_ptr(), H, W, Cin, Cout, 3, 3, 1, 1, 1, H, W, F16, 2 if force else 0, _stream(),
                                                   stats.data_ptr(), G, ctypes.byref(done)))
    finally:
        K.osb_tc_set_tile(0, 0, 0)
        K.osb_tc_set_pair_mode(1)
    torch.cuda.synchronize()
    assert len(prof) == 1, prof
    if force:
        assert (prof[0]["bm"], prof[0]["bn"], prof[0]["split"]) == force, prof
    else:
        assert (prof[0]["bm"], prof[0]["bn"], prof[0]["split"]) == (128, 128, 1), prof
    assert done.value == 1, "the kernel did not report the statistics"
    what = f"conv epilogue {route} Cout {Cout} G {G} m {m}"
    _check_gn_slot(stats, y.double().cpu().numpy(), H * W, Cout, G, what)
    _check_gn_apply_from_slot(K, y, stats, F16, H * W, Cout, G, Cout + G, what)


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("C,n,affine,m", [(8, 700, True, 0.0), (3, 200000, True, 0.0), (5, 65536, False, 0.0), (4, 50000, True, 256.0), (4, 50000, True, 1024.0), (16, 900, True, 1024.0)])
def test_instance_norm(K, dtype, C, n, affine, m):
    """osb_instance_norm: n_per_c < 1024 (one split) and large n_per_c (up to 64 splits), null scale / bias, offset means; fp64
    statistics as the reference.  Bar of test_layer_norm, 2^-10 (fp16) / 2^-20 (fp32) x (|ref| + 4), plus one fp32 ulp of the mean
    times rstd |scale| (the apply pass subtracts the mean rounded to fp32)."""
    import torch
    rng = np.random.default_rng(C * n + int(m))
    xs = (m + rng.standard_normal((C, n)) * (1.0 if m else 3.0) + (0.0 if m else 0.5)).astype(NP[dtype])
    sc = rng.standard_normal(C).astype(NP[dtype]); bi = rng.standard_normal(C).astype(NP[dtype])
    x = torch.from_numpy(xs).cuda(); y = torch.full_like(x, float("nan"))
    ts, tb = torch.from_numpy(sc).cuda(), torch.from_numpy(bi).cuda()
    assert K.osb_instance_norm(x.data_ptr(), y.data_ptr(), dtype, C, n, ts.data_ptr() if affine else None, tb.data_ptr() if affine else None, 1e-5, _stream()) == 0
    torch.cuda.synchronize()
    xd = xs.astype(np.float64)
    mean = xd.mean(1, keepdims=True)
    rstd = 1.0 / np.sqrt(((xd - mean) ** 2).mean(1, keepdims=True) + 1e-5)
    g = sc.astype(np.float64)[:, None] if affine else np.ones((C, 1))
    b = bi.astype(np.float64)[:, None] if affine else np.zeros((C, 1))
    ref = (xd - mean) * rstd * g + b
    tol = (2.0 ** -10 if dtype == F16 else 2.0 ** -20) * (np.abs(ref) + 4.0) + np.spacing(np.abs(mean).astype(np.float32)) * rstd * np.abs(g) * 1.5
    _assert_within(y.cpu().numpy(), ref, tol, f"instance_norm C {C} n {n} m {m}")


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("rows,cols", [(2500, 1), (2500, 31), (300, 255), (300, 256), (64, 1023), (64, 1024), (16, 70000)])
def test_reduce_mean(K, dtype, rows, cols):
    """osb_reduce_mean at the 32 / 128 / 256-thread boundaries.  Bar: fp32 accumulation of n terms in chains of ceil(n / threads) plus a
    log2(threads) tree, (chain + log2 T + 2) 2^-24 sum|x| / n, plus one rounding of the result for fp16."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(rows + cols)
    x = (torch.randn(rows, cols, device="cuda", generator=g) * 2 + 1).to(_tdt(dtype))
    y = torch.full((rows,), float("nan"), device="cuda", dtype=x.dtype)
    assert K.osb_reduce_mean(x.data_ptr(), y.data_ptr(), dtype, rows, cols, _stream()) == 0
    torch.cuda.synchronize()
    xd = x.double().cpu().numpy()
    ref = xd.mean(1)
    T = 256 if cols >= 1024 else (128 if cols >= 256 else 32)
    tol = (math.ceil(cols / T) + math.log2(T) + 2) * 2.0 ** -24 * np.abs(xd).mean(1)
    if dtype == F16:
        tol = tol + _ulp(ref, F16) / 2
    _assert_within(y.cpu().numpy(), ref, tol, f"reduce_mean {rows}x{cols}")


# ============================================================================================================================
# 4. elementwise
# ============================================================================================================================

BIN_ADD, BIN_SUB, BIN_MUL, BIN_DIV, BIN_MUL_GELU, BIN_MUL_SIGMOID, BIN_SILU_MUL = range(7)
BIN_OPS = [BIN_ADD, BIN_SUB, BIN_MUL, BIN_DIV, BIN_MUL_GELU, BIN_MUL_SIGMOID, BIN_SILU_MUL]
_SQRT1_2 = 0.70710678118654752


def _bin_ref(op, a, b):
    """fp64 value of the op on the stored inputs, and the absolute error a fp32 evaluation may add beyond its final rounding: erff /
    expf are within 2 ulp; 1 + erf(b / sqrt 2) cancels for negative b, so MUL_GELU may err by ~2^-22 |a b| whatever the result."""
    from scipy.special import erf
    if op == BIN_MUL_GELU:
        return a * (0.5 * b * (1.0 + erf(b * _SQRT1_2))), 2.0 ** -21 * np.abs(a * b) * (1.0 + np.abs(b))
    if op == BIN_MUL_SIGMOID:
        return a / (1.0 + np.exp(-b)), 0.0
    if op == BIN_SILU_MUL:
        return (a / (1.0 + np.exp(-a))) * b, 0.0
    raise ValueError(op)


def _bin_exact(op, a32, b32):
    """ADD / SUB / MUL / DIV in fp32 (IEEE, round to nearest) on the stored inputs: what the kernel computes before rounding to storage."""
    with np.errstate(all="ignore"):
        return {BIN_ADD: a32 + b32, BIN_SUB: a32 - b32, BIN_MUL: a32 * b32, BIN_DIV: a32 / b32}[op]


BIN_PATHS = [
    # path, out shape, a shape, b shape, a pointer offset (elements)
    ("flat", (37, 64), (37, 64), (37, 64), 0),
    ("flat, n % VEC != 0 (block-0 tail)", (5, 13), (5, 13), (5, 13), 0),
    ("flat, scalar a", (33, 40), (1, 1), (33, 40), 0),
    ("flat, scalar b", (33, 40), (33, 40), (1, 1), 0),
    ("flat, unaligned a (VEC = 1)", (33, 40), (33, 40), (33, 40), 1),
    ("per-column, swap = 0", (3, 12, 64), (3, 12, 64), (1, 1, 64), 0),
    ("per-column, swap = 1", (3, 12, 64), (1, 1, 64), (3, 12, 64), 0),
    ("per-row, swap = 0", (3, 12, 64), (3, 12, 64), (3, 12, 1), 0),
    ("per-row, swap = 1", (3, 12, 64), (3, 12, 1), (3, 12, 64), 0),
    ("generic: per-column with cols % VEC != 0", (9, 13), (9, 13), (1, 13), 0),
    ("generic 4-D broadcast", (2, 3, 5, 7), (2, 1, 5, 7), (1, 3, 1, 7), 0),
    ("generic 6-D broadcast", (2, 2, 3, 4, 2, 5), (2, 1, 3, 1, 2, 5), (1, 2, 1, 4, 2, 1), 0),
]


def _bcast_strides(shape, out_shape):
    st, s = [], 1
    for d in range(len(shape) - 1, -1, -1):
        st.append(0 if shape[d] == 1 and out_shape[d] != 1 else s)
        s *= shape[d]
    return st[::-1]


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("op", BIN_OPS)
@pytest.mark.parametrize("path,oshape,ashape,bshape,aoff", BIN_PATHS)
def test_binary(K, path, oshape, ashape, bshape, aoff, op, dtype):
    """osb_binary on each dispatch path.  ADD / SUB / MUL / DIV: bit-exact against the fp32 op on the stored inputs, rounded to the
    storage type.  MUL_GELU / MUL_SIGMOID / SILU_MUL against fp64: 2^-20 relative in fp32 (2-3 operations of <= 2 ulp
    each, an ulp being at most 2^-23 relative) or 1 fp16 ulp (that fp32 value rounded once), plus the cancellation term of _bin_ref."""
    import torch
    rng = np.random.default_rng(zlib.crc32(path.encode()) + op * 10 + dtype)
    av = (rng.standard_normal(ashape) * 2).astype(NP[dtype])
    bv = rng.standard_normal(bshape).astype(np.float32)
    if op == BIN_DIV:
        bv = np.sign(bv) * (0.5 + np.abs(bv))      # keep divisors away from 0
    bv = (bv * 2).astype(NP[dtype])
    n_a = int(np.prod(ashape))
    ta = _offset_view(n_a, dtype, aoff)
    ta.copy_(torch.from_numpy(av.reshape(-1)).cuda())
    tb = torch.from_numpy(bv.copy()).cuda()
    out = torch.full(oshape, float("nan"), device="cuda", dtype=_tdt(dtype))
    nd = len(oshape)
    rc = K.osb_binary(op, ta.data_ptr(), _i64(_bcast_strides(ashape, oshape)), tb.data_ptr(), _i64(_bcast_strides(bshape, oshape)),
                      out.data_ptr(), _i64(oshape), nd, dtype, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    a = np.broadcast_to(av, oshape).astype(np.float32)
    b = np.broadcast_to(bv, oshape).astype(np.float32)
    if op in (BIN_ADD, BIN_SUB, BIN_MUL, BIN_DIV):
        want = _bin_exact(op, a, b).astype(NP[dtype])
        assert np.array_equal(got, want), f"{path}: {int((got != want).sum())} of {want.size} differ"
    else:
        ref, extra = _bin_ref(op, a.astype(np.float64), b.astype(np.float64))
        tol = (_ulp(ref, F16) if dtype == F16 else 2.0 ** -20 * np.abs(ref)) + extra
        _assert_within(got, ref, tol, path)


UN_SIGMOID, UN_SILU, UN_ERF, UN_SQRT, UN_SIN, UN_COS, UN_POW, UN_NEG, UN_GELU_ERF, UN_COPY, UN_MULC, UN_ADDC, UN_RECIP_SQRT = range(13)
UNARY_OPS = [
    # op, alpha, input kind
    (UN_SIGMOID, 0.0, "normal"), (UN_SILU, 0.0, "normal"), (UN_ERF, 0.0, "normal"), (UN_SQRT, 0.0, "positive"),
    (UN_SIN, 0.0, "normal"), (UN_COS, 0.0, "normal"), (UN_POW, 3.0, "normal"), (UN_POW, 2.0, "normal"), (UN_POW, 0.5, "positive"),
    (UN_NEG, 0.0, "normal"), (UN_GELU_ERF, 0.0, "normal"), (UN_COPY, 0.0, "normal"), (UN_MULC, 0.37, "normal"),
    (UN_ADDC, 1.25, "normal"), (UN_RECIP_SQRT, 0.0, "positive"),
]


def _unary_exact(op, x32, alpha):
    a = np.float32(alpha)
    return {UN_NEG: -x32, UN_COPY: x32, UN_MULC: x32 * a, UN_ADDC: x32 + a}.get(op)


def _unary_ref(op, x, alpha):
    from scipy.special import erf
    if op == UN_SIGMOID: return 1.0 / (1.0 + np.exp(-x)), 0.0
    if op == UN_SILU: return x / (1.0 + np.exp(-x)), 0.0
    if op == UN_ERF: return erf(x), 0.0
    if op == UN_SQRT: return np.sqrt(x), 0.0
    if op == UN_SIN: return np.sin(x), 0.0
    if op == UN_COS: return np.cos(x), 0.0
    if op == UN_POW: return np.power(x, alpha), 0.0
    if op == UN_GELU_ERF: return 0.5 * x * (1.0 + erf(x * _SQRT1_2)), 2.0 ** -21 * np.abs(x) * (1.0 + np.abs(x))
    if op == UN_RECIP_SQRT: return 1.0 / np.sqrt(x), 0.0
    raise ValueError(op)


@pytest.mark.parametrize("off", [0, 1])
@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("op,alpha,kind", UNARY_OPS)
def test_unary(K, op, alpha, kind, dtype, off):
    """osb_unary, vectorised (aligned) and VEC = 1 (misaligned base pointer), n = 8 * 1000 + 5 so the block-0 tail runs.  NEG / COPY /
    MULC / ADDC: bit-exact against the fp32 op rounded to storage.  The rest against fp64: 2^-20 relative in fp32 (CUDA's expf / erff /
    sinf / cosf / powf / rsqrtf are within 2 ulp, plus the division / addition they feed) or 1 fp16 ulp, plus GELU's cancellation term."""
    import torch
    n = 8 * 1000 + 5
    rng = np.random.default_rng(op * 100 + int(alpha * 10) + dtype + off)
    xv = rng.standard_normal(n) * 3
    if kind == "positive":
        xv = np.abs(xv) + 1e-2
    xs = xv.astype(NP[dtype])
    x = _offset_view(n, dtype, off)
    x.copy_(torch.from_numpy(xs).cuda())
    y = _offset_view(n, dtype, off)
    assert K.osb_unary(op, x.data_ptr(), y.data_ptr(), dtype, n, alpha, _stream()) == 0
    torch.cuda.synchronize()
    got = y.cpu().numpy()
    exact = _unary_exact(op, xs.astype(np.float32), alpha)
    if exact is not None:
        want = exact.astype(NP[dtype])
        assert np.array_equal(got, want), f"{int((got != want).sum())} of {n} differ"
    else:
        ref, extra = _unary_ref(op, xs.astype(np.float64), alpha)
        tol = (_ulp(ref, F16) if dtype == F16 else 2.0 ** -20 * np.abs(ref)) + extra
        _assert_within(got, ref, tol, f"unary op {op}")


def test_convert_float_int64(K):
    """osb_convert fp16 <-> fp32 and int64 -> fp32: bit-exact against round-to-nearest-even conversions (int64 values beyond 2^24
    exercise the rounding)."""
    import torch
    n = 10007
    rng = np.random.default_rng(1)
    f32 = (rng.standard_normal(n) * 1000).astype(np.float32)
    f32[:4] = [70000.0, -70000.0, 1e-6, 65519.0]          # fp16 overflow to inf, subnormal, round to 65504
    with np.errstate(over="ignore"):
        want_h = f32.astype(np.float16)
    t32 = torch.from_numpy(f32).cuda()
    h = torch.full((n,), float("nan"), device="cuda", dtype=torch.half)
    assert K.osb_convert(t32.data_ptr(), F32, h.data_ptr(), F16, n, 1.0, 0, _stream()) == 0
    back = torch.full((n,), float("nan"), device="cuda", dtype=torch.float32)
    assert K.osb_convert(h.data_ptr(), F16, back.data_ptr(), F32, n, 1.0, 0, _stream()) == 0
    i64 = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    i64[:3] = [(1 << 24) + 1, -(1 << 53) - 3, 0]
    ti = torch.from_numpy(i64).cuda()
    fi = torch.full((n,), float("nan"), device="cuda", dtype=torch.float32)
    assert K.osb_convert(ti.data_ptr(), I64, fi.data_ptr(), F32, n, 1.0, 0, _stream()) == 0
    torch.cuda.synchronize()
    assert np.array_equal(h.cpu().numpy().view(np.uint16), want_h.view(np.uint16))
    assert np.array_equal(back.cpu().numpy(), want_h.astype(np.float32))
    assert np.array_equal(fi.cpu().numpy(), i64.astype(np.float32))


@pytest.mark.parametrize("dtype", [F16, F32])
def test_convert_dequantize_u8(K, dtype):
    """osb_convert uint8 -> float: (q - zp) * scale in fp32, rounded to storage.  Bit-exact."""
    import torch
    q = np.arange(256 * 41, dtype=np.int64).astype(np.uint8)
    scale, zp = np.float32(0.0371), 131
    tq = torch.from_numpy(q).cuda()
    y = torch.full((q.size,), float("nan"), device="cuda", dtype=_tdt(dtype))
    assert K.osb_convert(tq.data_ptr(), U8, y.data_ptr(), dtype, q.size, float(scale), zp, _stream()) == 0
    torch.cuda.synchronize()
    want = ((q.astype(np.int32) - zp).astype(np.float32) * scale).astype(NP[dtype])
    assert np.array_equal(y.cpu().numpy(), want)


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("scale,zp", [(0.25, 100), (0.0371, 3), (0.5, 250)])
def test_convert_quantize_u8(K, dtype, scale, zp):
    """osb_convert float -> uint8 (XNNPACK f32-qu8 convert): bit-exact against np_oracle.qu8_quantize, with exact .5 ties (x * (1 /
    scale) = k + 0.5 when scale is a power of two), values past both clamps, and large finite extremes."""
    import torch
    rng = np.random.default_rng(int(scale * 1000) + zp)
    n = 4099
    xv = rng.uniform(-(zp + 20) * scale, (275 - zp) * scale, n)
    if scale == 0.25 or scale == 0.5:
        k = rng.integers(-zp - 3, 258 - zp, 1000)
        xv[:1000] = (k + 0.5) * scale                     # ties: round half to even
    xv[1000:1004] = [-60000.0, 60000.0, -1e-3 * scale, 65504.0]
    xs = xv.astype(NP[dtype])
    x = torch.from_numpy(xs).cuda()
    y = torch.full((n,), 0xAB, device="cuda", dtype=torch.uint8)
    assert K.osb_convert(x.data_ptr(), dtype, y.data_ptr(), U8, n, scale, zp, _stream()) == 0
    torch.cuda.synchronize()
    want = qu8_quantize(xs.astype(np.float32), np.float32(scale), zp)
    got = y.cpu().numpy()
    assert np.array_equal(got, want), f"{int((got != want).sum())} of {n} differ, first at {np.argwhere(got != want)[0]}"


# ============================================================================================================================
# 5. data movement (bit-exact)
# ============================================================================================================================

def _copy_ref(src, dst, shape, ist, idiv, ioff, ost, ooff):
    """out[out_off + sum i_k os_k] = in[in_off + sum (i_k / in_div_k) is_k] over every index of `shape` (flat element arrays)."""
    idx = np.indices(shape).reshape(len(shape), -1)
    io = ioff + sum((idx[d] // idiv[d]) * ist[d] for d in range(len(shape)))
    oo = ooff + sum(idx[d] * ost[d] for d in range(len(shape)))
    out = dst.copy()
    out[oo] = src[io]
    return out


COPY_CASES = [
    # name, elem size, in elements, out elements, shape, in stride, in div, in offset, out stride, out offset, in pointer offset (bytes)
    ("transpose (no widening)", 2, 64 * 48, 64 * 48, (48, 64), (1, 48), (1, 1), 0, (64, 1), 0, 0),
    ("slice widened to 16 bytes", 2, 9 * 40, 9 * 16, (9, 16), (40, 1), (1, 1), 8, (16, 1), 0, 0),
    ("slice widened to 8 bytes", 2, 9 * 36, 9 * 12, (9, 12), (36, 1), (1, 1), 4, (12, 1), 0, 0),
    ("slice widened to 4 bytes", 2, 9 * 34, 9 * 6, (9, 6), (34, 1), (1, 1), 2, (6, 1), 0, 0),
    ("slice, odd offset (no widening)", 1, 9 * 40, 9 * 7, (9, 7), (40, 1), (1, 1), 1, (7, 1), 0, 0),
    ("byte slice widened to 8 bytes", 1, 9 * 40, 9 * 24, (9, 24), (40, 1), (1, 1), 8, (24, 1), 0, 0),
    ("expand (stride 0), widened to 16 bytes", 4, 64, 50 * 64, (50, 64), (0, 1), (1, 1), 0, (64, 1), 0, 0),
    ("expand a row to columns (stride 0 innermost)", 4, 50, 50 * 9, (50, 9), (1, 0), (1, 1), 0, (9, 1), 0, 0),
    ("nearest resize x2 (in_div), NHWC", 2, 5 * 7 * 24, 10 * 14 * 24, (10, 14, 24), (7 * 24, 24, 1), (2, 2, 1), 0, (14 * 24, 24, 1), 0, 0),
    ("nearest resize x2 (in_div), NCHW innermost", 4, 3 * 5 * 7, 3 * 10 * 14, (3, 10, 14), (35, 7, 1), (1, 2, 2), 0, (140, 14, 1), 0, 0),
    ("concat half: write at an output offset", 2, 6 * 16, 6 * 40, (6, 16), (16, 1), (1, 1), 0, (40, 1), 24, 0),
    ("unaligned base pointer (no widening)", 2, 9 * 40, 9 * 16, (9, 16), (40, 1), (1, 1), 8, (16, 1), 0, 2),
]


@pytest.mark.parametrize("name,es,n_in,n_out,shape,ist,idiv,ioff,ost,ooff,pbytes", COPY_CASES)
def test_strided_copy(K, name, es, n_in, n_out, shape, ist, idiv, ioff, ost, ooff, pbytes):
    """osb_strided_copy: transpose, slice, expand, nearest resize and an output offset, on cases that do and do not qualify for the
    2 / 4 / 8 / 16-byte widening.  Bit-exact; elements outside the written set keep their 0xAB fill."""
    import torch
    udt = {1: np.uint8, 2: np.uint16, 4: np.uint32}[es]
    rng = np.random.default_rng(n_in + n_out)
    src = rng.integers(0, np.iinfo(udt).max, n_in, dtype=np.uint64).astype(udt)
    raw = torch.zeros(n_in * es + 64, dtype=torch.uint8, device="cuda")
    tin = raw[pbytes:pbytes + n_in * es]
    tin.copy_(torch.from_numpy(src.view(np.uint8).copy()).cuda())
    tout = torch.full((n_out * es,), 0xAB, dtype=torch.uint8, device="cuda")
    nd = len(shape)
    rc = K.osb_strided_copy(tin.data_ptr(), tout.data_ptr(), es, nd, _i64(shape), _i64(ist), _i64(idiv), ioff, _i64(ost), ooff, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    init = np.full(n_out * es, 0xAB, np.uint8).view(udt)
    want = _copy_ref(src, init, shape, ist, idiv, ioff, ost, ooff)
    got = tout.cpu().numpy().view(udt)
    assert np.array_equal(got, want), f"{name}: {int((got != want).sum())} of {n_out} differ"


@pytest.mark.parametrize("es", [1, 2, 4])
@pytest.mark.parametrize("batch,rows,cols", [(3, 37, 70), (1, 1, 65), (2, 64, 32), (4, 33, 1)])
def test_transpose2d(K, es, batch, rows, cols):
    """osb_transpose2d [B, R, C] -> [B, C, R] with ragged tiles, batch > 1.  Bit-exact."""
    import torch
    udt = {1: np.uint8, 2: np.uint16, 4: np.uint32}[es]
    rng = np.random.default_rng(batch * rows * cols + es)
    src = rng.integers(0, np.iinfo(udt).max, (batch, rows, cols), dtype=np.uint64).astype(udt)
    tin = torch.from_numpy(src.view(np.uint8).reshape(-1).copy()).cuda()
    tout = torch.full((batch * rows * cols * es,), 0xAB, dtype=torch.uint8, device="cuda")
    assert K.osb_transpose2d(tin.data_ptr(), tout.data_ptr(), es, batch, rows, cols, _stream()) == 0
    torch.cuda.synchronize()
    got = tout.cpu().numpy().view(udt).reshape(batch, cols, rows)
    assert np.array_equal(got, src.transpose(0, 2, 1))


def test_transpose2d_refuses_tall_grid(K):
    """More than 65535 32-row tiles does not fit grid.y: refused before any launch."""
    assert K.osb_transpose2d(None, None, 2, 1, 65536 * 32 + 1, 1, _stream()) == CUDA_ERROR_INVALID_VALUE


@pytest.mark.parametrize("row_bytes,off", [(320, 0), (10, 0), (320, 2)])
def test_gather_rows(K, row_bytes, off):
    """osb_gather_rows: the 16-byte path (row_bytes % 16 == 0, aligned) and the byte path (ragged row, or misaligned table); negative
    indices count from the end, out-of-range ones clamp to the first / last row.  Bit-exact."""
    import torch
    rows, n_idx = 50, 300
    rng = np.random.default_rng(row_bytes + off)
    table = rng.integers(0, 256, (rows, row_bytes), dtype=np.uint8)
    idx = rng.integers(-rows, rows, n_idx, dtype=np.int64)
    idx[:6] = [0, rows - 1, -1, -rows, rows + 7, -rows - 9]
    raw = torch.zeros(rows * row_bytes + 32, dtype=torch.uint8, device="cuda")
    tt = raw[off:off + rows * row_bytes]
    tt.copy_(torch.from_numpy(table.reshape(-1)).cuda())
    ti = torch.from_numpy(idx).cuda()
    out = torch.full((n_idx * row_bytes,), 0xAB, dtype=torch.uint8, device="cuda")
    assert K.osb_gather_rows(tt.data_ptr(), ti.data_ptr(), out.data_ptr(), n_idx, rows, row_bytes, _stream()) == 0
    torch.cuda.synchronize()
    src = np.where(idx < 0, idx + rows, idx).clip(0, rows - 1)
    assert np.array_equal(out.cpu().numpy().reshape(n_idx, row_bytes), table[src])


@pytest.mark.parametrize("es", [2, 4])
def test_scatter_elems(K, es):
    """osb_scatter_elems with unique in-range positions: out[pos[i]] = updates[i], everything else untouched.  Bit-exact."""
    import torch
    udt = {2: np.uint16, 4: np.uint32}[es]
    n_out, n = 5000, 1234
    rng = np.random.default_rng(es)
    base = rng.integers(0, np.iinfo(udt).max, n_out, dtype=np.uint64).astype(udt)
    pos = rng.permutation(n_out)[:n].astype(np.int64)
    upd = rng.integers(0, np.iinfo(udt).max, n, dtype=np.uint64).astype(udt)
    tout = torch.from_numpy(base.view(np.uint8).copy()).cuda()
    tp = torch.from_numpy(pos).cuda(); tu = torch.from_numpy(upd.view(np.uint8).copy()).cuda()
    assert K.osb_scatter_elems(tout.data_ptr(), tp.data_ptr(), tu.data_ptr(), n, es, _stream()) == 0
    torch.cuda.synchronize()
    want = base.copy(); want[pos] = upd
    assert np.array_equal(tout.cpu().numpy().view(udt), want)


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("H,W,C,k,s,pad", [(9, 11, 13, 3, 2, 1), (16, 16, 8, 2, 2, 0), (7, 5, 3, 3, 1, 1), (10, 10, 5, 3, 2, 0)])
def test_maxpool_nhwc(K, dtype, H, W, C, k, s, pad):
    """osb_maxpool_nhwc with padding (padded taps ignored), stride 2 and ragged C against torch's max_pool2d.  Bit-exact (a max)."""
    import torch
    import torch.nn.functional as Fn
    g = torch.Generator(device="cuda").manual_seed(H * W * C)
    x = torch.randn(H, W, C, device="cuda", generator=g).to(_tdt(dtype))
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    y = torch.full((Ho, Wo, C), float("nan"), device="cuda", dtype=x.dtype)
    assert K.osb_maxpool_nhwc(x.data_ptr(), y.data_ptr(), dtype, H, W, C, k, k, s, pad, pad, Ho, Wo, _stream()) == 0
    torch.cuda.synchronize()
    ref = Fn.max_pool2d(x.double().permute(2, 0, 1)[None], k, s, pad)[0].permute(1, 2, 0).to(x.dtype)
    assert torch.equal(y, ref)


@pytest.mark.parametrize("dtype", [F16, F32])
def test_fill(K, dtype):
    """osb_fill: every element equals the fp32 value rounded to storage.  Bit-exact."""
    import torch
    for n, v in [(1, 1.5), (1000003, -3.1), (77, 0.0)]:
        y = torch.full((n + 3,), float("nan"), device="cuda", dtype=_tdt(dtype))
        assert K.osb_fill(y.data_ptr(), dtype, n, v, _stream()) == 0
        torch.cuda.synchronize()
        got = y.cpu().numpy()
        assert (got[:n] == np.float32(v).astype(NP[dtype])).all()
        assert np.isnan(got[n:]).all(), "wrote past n"


# ============================================================================================================================
# 6. uint8 path (bit-exact against oracle/np_oracle.py)
# ============================================================================================================================

def _pct_chunk_count(x, threads, from_left, from_right):
    """Chunks that yield a percentile pair in np_oracle.qu8_percentiles' walk (finite count > k on both sides)."""
    flat = np.asarray(x).ravel()
    size = flat.size
    chunk = 16384 if flat.dtype == np.float32 else 32768
    per = size // threads or 1
    count = 0
    for i in range(threads):
        st, en = i * per, (size if i >= threads - 1 else (i + 1) * per)
        if st >= en or st >= size:
            continue
        for j in range(st, en, chunk):
            nn = min(en, j + chunk) - j
            fin = int(np.isfinite(flat[j:j + nn].astype(np.float32)).sum())
            kl, kr = int(np.float32(nn) * np.float32(from_left)), int(np.float32(nn) * np.float32(from_right))
            count += kl < fin and kr < fin
    return count


PCT_CASES = [
    # name, n in chunks (float: 1.0 = one chunk), threads, content
    ("below one chunk", 0.03, 1, "normal"),
    ("exactly one chunk", 1.0, 1, "normal"),
    ("many chunks, 4 spans of two chunks", 5.37, 4, "normal"),
    ("many chunks, 7 spans, the last one ragged", 5.37, 7, "normal"),
    ("±inf and NaN mixed in", 3.0, 4, "nonfinite"),
    ("a chunk with fewer finite values than k", 3.0, 1, "sparse"),
    ("all inf: no chunk", 2.0, 4, "allinf"),
]


@pytest.mark.parametrize("dtype", [F16, F32])
@pytest.mark.parametrize("name,chunks,threads,content", PCT_CASES)
def test_percentiles(K, name, chunks, threads, content, dtype):
    """osb_percentiles (per-chunk radix select) against np_oracle.qu8_percentiles: low / high bit-exact, and the number of chunks
    that produced a result equal to the oracle's walk."""
    import torch
    chunk = 32768 if dtype == F16 else 16384
    n = int(chunks * chunk)
    rng = np.random.default_rng(n + threads)
    xv = rng.standard_normal(n) * 3
    if content == "nonfinite":
        pick = rng.choice(n, 3000, replace=False)
        xv[pick[:1000]] = np.inf; xv[pick[1000:2000]] = -np.inf; xv[pick[2000:]] = np.nan
    elif content == "sparse":
        xv[chunk:2 * chunk] = np.inf                       # the middle chunk keeps 10 finite values, fewer than k = 32 (fp16) / 16 (fp32)
        keep = chunk + rng.choice(chunk, 10, replace=False)
        xv[keep] = np.linspace(-5000, 5000, 10)            # extremes that would widen the range if the chunk contributed
    elif content == "allinf":
        xv[:] = np.inf
        xv[::2] = -np.inf
    xs = xv.astype(NP[dtype])
    fl = fr = 0.001
    x = torch.from_numpy(xs).cuda()
    out3 = torch.from_numpy(np.array([0xFFFFFFFF, 0, 0], np.uint32).view(np.int32)).cuda()
    assert K.osb_percentiles(x.data_ptr(), dtype, n, threads, fl, fr, out3.data_ptr(), _stream()) == 0
    torch.cuda.synchronize()
    lo_key, hi_key, count = (int(v) for v in out3.cpu().numpy().view(np.uint32))
    assert count == _pct_chunk_count(xs, threads, fl, fr), f"{name}: {count} chunks reported"
    want = qu8_percentiles(xs, threads, fl, fr)
    if count == 0:
        assert want is None
        return
    assert want is not None
    lo, hi = K.osb_percentile_key_to_float(lo_key, dtype), K.osb_percentile_key_to_float(hi_key, dtype)
    assert (np.float32(lo), np.float32(hi)) == (want[0], want[1]), f"{name}: got ({lo}, {hi}), oracle {want}"


QU8_BIN_CASES = [
    # name, out shape, a shape, b shape, sa, sb, so
    ("flat", (1000,), (1000,), (1000,), 0.031, 0.027, 0.05),
    ("broadcast b over rows", (4, 5, 33), (4, 5, 33), (1, 5, 1), 0.5, 0.7, 0.9),
    ("broadcast both", (3, 7, 9), (3, 1, 9), (1, 7, 1), 3.0, 0.01, 0.25),
    ("ratio near the shift limit (shift = 31)", (257,), (257,), (257,), 0.03 * 2.0 ** -11 * 1.5, 0.03 * 2.0 ** -12, 0.03),
]


@pytest.mark.parametrize("op", [BIN_ADD, BIN_MUL])
@pytest.mark.parametrize("name,oshape,ashape,bshape,sa,sb,so", QU8_BIN_CASES)
def test_binary_qu8(K, name, oshape, ashape, bshape, sa, sb, so, op):
    """osb_binary_qu8 ADD (fixed point) and MUL (fp32 requantisation) against np_oracle.qu8_add / qu8_mul.  Bit-exact."""
    import torch
    sa, sb, so = float(np.float32(sa)), float(np.float32(sb)), float(np.float32(so))
    za, zb, zo = 121, 90, 130
    rng = np.random.default_rng(len(name) + op)
    qa = rng.integers(0, 256, ashape, dtype=np.uint8); qb = rng.integers(0, 256, bshape, dtype=np.uint8)
    ta, tb = torch.from_numpy(qa).cuda(), torch.from_numpy(qb).cuda()
    out = torch.full(oshape, 0xAB, dtype=torch.uint8, device="cuda")
    rc = K.osb_binary_qu8(op, ta.data_ptr(), _i64(_bcast_strides(ashape, oshape)), sa, za, tb.data_ptr(), _i64(_bcast_strides(bshape, oshape)), sb, zb,
                          out.data_ptr(), so, zo, _i64(oshape), len(oshape), _stream())
    assert rc == 0
    torch.cuda.synchronize()
    fn = qu8_add if op == BIN_ADD else qu8_mul
    want = np.broadcast_to(fn(qa, sa, za, qb, sb, zb, so, zo), oshape)
    got = out.cpu().numpy()
    assert np.array_equal(got, want), f"{name}: {int((got != want).sum())} of {want.size} differ"


def test_binary_qu8_refuses_tiny_scale_ratio(K):
    """ADD with max(|sa / so|, |sb / so|) < 2^-11 needs a shift > 31: refused before any launch."""
    s = float(np.float32(0.03 * 2.0 ** -12))
    rc = K.osb_binary_qu8(BIN_ADD, None, _i64([1]), s, 0, None, _i64([1]), s, 0, None, 0.03, 0, _i64([16]), 1, _stream())
    assert rc == CUDA_ERROR_INVALID_VALUE


@pytest.mark.parametrize("rows,cols,in_scale", [(64, 77, 0.05), (9, 1024, 0.11), (3, 4097, 0.02)])
def test_softmax_qu8(K, rows, cols, in_scale):
    """osb_softmax_qu8 against a numpy restatement of its documented arithmetic: dequantise (x * in_scale, zero point 0), fp32 softmax,
    lrintf(p / out_scale) + out_zp, clamp to [0, 255].  Within 1 code: the device expf and numpy's exp may round differently, and the
    sums add in different orders, which can move a value across a rounding boundary."""
    import torch
    rng = np.random.default_rng(rows * cols)
    q = rng.integers(0, 256, (rows, cols), dtype=np.uint8)
    out_scale, out_zp = np.float32(2.0 ** -8), 0
    tq = torch.from_numpy(q).cuda()
    y = torch.full((rows, cols), 0xAB, dtype=torch.uint8, device="cuda")
    assert K.osb_softmax_qu8(tq.data_ptr(), y.data_ptr(), rows, cols, in_scale, float(out_scale), out_zp, _stream()) == 0
    torch.cuda.synchronize()
    f = q.astype(np.float32) * np.float32(in_scale)
    e = np.exp(f - f.max(1, keepdims=True)).astype(np.float32)
    p = e * (np.float32(1.0) / e.sum(1, keepdims=True, dtype=np.float32))
    want = np.clip(np.rint(p / out_scale).astype(np.int64) + out_zp, 0, 255)
    got = y.cpu().numpy().astype(np.int64)
    assert np.abs(got - want).max() <= 1
