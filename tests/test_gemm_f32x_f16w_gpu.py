"""fp32-arithmetic prefill on fp16 weights read in place: the tensor-core GEMM that splits the fp16 B tile into its bf16 hi / lo parts in
shared memory (osb_tc_gemm_f32x_f16w), and the engine routing that hands it the fp16 blob of a prefill-shaped MatMul / Gemm instead of an
fp32 copy and its bf16x6 expansion.

Kernel cases run in the two regimes of tests/test_gemm_conv_paths_gpu.py::test_f32x_gemm_bias_residual.  The exact regime uses fixed-point
operands built so that each of the five products the kernel computes (a_h b_hi, a_h b_lo, a_m b_hi, a_l b_hi, a_m b_lo) is nonzero
somewhere and the one it drops (a_l b_lo) is zero everywhere; the result is then the fp64 result rounded once to fp32, bit for bit.  The
Gaussian regime holds the test's error bar."""
import ctypes
import os
import re
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from test_kernels_gpu import _check, _check_exact, _operands
from test_prefill_gpu import DYN, OPTS32
from util import reference_outputs, report, run_model

pytestmark = pytest.mark.gpu

NOT_SUPPORTED = 801
TOL32 = 2e-4        # tests/test_models_gpu.py TOL["float32"]
KERNEL = "tc_gemm_f16w_kernel"


@pytest.fixture(scope="module")
def K(engine_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = ctypes.CDLL(engine_lib)
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.osb_tc_gemm_f32x_f16w_ok.argtypes = [i64] * 4
    lib.osb_tc_gemm_f32x_f16w.argtypes = [vp, vp, i64, vp, vp, vp, i64, i64, i64, vp, vp]
    lib.osb_bf16x3_expand_cols.argtypes = [vp, vp, i64, i64, i64, ci, vp]
    lib.osb_bf16x3_expand_rows.argtypes = [vp, vp, i64, i64, ci, vp]
    lib.osb_tc_gemm_f32x.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, ci, vp]
    lib.osb_launch_count.restype = ctypes.c_uint64
    lib.osb_launch_count_reset.restype = None
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _planes(M, Kd):
    import torch
    return torch.empty(3 * M * Kd, device="cuda", dtype=torch.bfloat16)


def _run(K, a, w, bias, res, N=None):
    """osb_tc_gemm_f32x_f16w on a [M, K] fp32 and w [K, ldb] fp16, of which the first N columns are used; (rc, launches, C [M, N])."""
    import torch
    M, Kd = a.shape
    N = w.shape[1] if N is None else N
    c = torch.full((M, N), float("nan"), device="cuda")
    K.osb_launch_count_reset()
    rc = K.osb_tc_gemm_f32x_f16w(a.data_ptr(), w.data_ptr(), w.shape[1], c.data_ptr(), _ptr(bias), _ptr(res), M, N, Kd, _planes(M, Kd).data_ptr(), _stream())
    n = int(K.osb_launch_count())
    torch.cuda.synchronize()
    return rc, n, c


def _parts(a, w):
    """The triple split of a (h, m, l) and the hi / lo parts of the fp16 w, as float64."""
    import torch
    h = a.bfloat16().float(); m = (a - h).bfloat16().float(); lo_a = (a - h - m).bfloat16().float()
    wf = w.float()
    hi = wf.bfloat16().float(); lo = (wf - hi).bfloat16().float()
    assert torch.equal(hi + lo, wf), "an fp16 value is exactly hi + lo"
    return h.double(), m.double(), lo_a.double(), hi.double(), lo.double()


def _exact_operands(case, M, N, Kd, seed):
    """Integers in [-7, 7] with sparse wide entries: case "m", A entries of 9 significant bits (a_m != 0, a_l = 0) and B entries of 9
    (b_lo != 0); case "l", A entries of 18 significant bits whose remainder past a_h needs 9 (a_l != 0) and B entries of at most 8 (b_lo =
    0).  At most 17 (case m) or 9 (case l) wide entries per dot product keep S = sum |a_k b_k| < 2^24: every partial sum is exact in fp32."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randint(-7, 8, (M, Kd), device="cuda", generator=g).float()
    w = torch.randint(-7, 8, (Kd, N), device="cuda", generator=g).float()
    P = max(8, Kd // (16 if case == "m" else 8))
    r, k = torch.meshgrid(torch.arange(M, device="cuda"), torch.arange(Kd, device="cuda"), indexing="ij")
    sa = (r * 7 + k) % P == 0
    sign = lambda shp: torch.randint(0, 2, shp, device="cuda", generator=g).float() * 2 - 1
    odd = lambda shp, hi: torch.randint(0, hi // 2, shp, device="cuda", generator=g).float() * 2 + 1
    if case == "m":
        a = torch.where(sa, sign((M, Kd)) * (256 + odd((M, Kd), 256)), a)
        k2, n2 = torch.meshgrid(torch.arange(Kd, device="cuda"), torch.arange(N, device="cuda"), indexing="ij")
        sb = (k2 * 3 + n2) % P == 0
        w = torch.where(sb, sign((Kd, N)) * (256 + odd((Kd, N), 256)), w)
    else:
        # 2^17 + 1024 x + 256 + odd: a_h keeps bits 17..10, the remainder (257..511 or -511..-257) has 9 bits, its lowest is a_l
        wide = 131072 + 1024 * torch.randint(0, 32, (M, Kd), device="cuda", generator=g).float() + 256 + odd((M, Kd), 512)
        a = torch.where(sa, sign((M, Kd)) * wide, a)
    return a, w.half()


def _products(a, w):
    """{name: is the product nonzero for some output} of the six triple-split products with fp16 B."""
    h, m, l, hi, lo = _parts(a, w)
    nz = lambda x, y: bool(((x != 0).double() @ (y != 0).double()).any())
    return {"h.hi": nz(h, hi), "h.lo": nz(h, lo), "m.hi": nz(m, hi), "l.hi": nz(l, hi), "m.lo": nz(m, lo), "l.lo": nz(l, lo)}


# the prefill projections of TinyLlama (hidden 2048, kv 256, mlp 5632) and Mistral 7B (4096, 1024, 14336): (K, N)
PROJ = [(2048, 2048), (2048, 256), (2048, 5632), (5632, 2048), (4096, 4096), (4096, 1024), (4096, 14336), (14336, 4096)]
CASES = [(M, Kd, N) for (Kd, N) in PROJ for M in (9, 17, 128, 300, 2048)]
CASES += [(17, 5632, 256), (64, 72, 264), (300, 200, 264), (9, 200, 264)]      # a split-K launch; ragged K


def _ref(a, w, bias, res):
    ref = a.double() @ w.double()
    absref = a.double().abs() @ w.double().abs()
    if bias is not None:
        ref = ref + bias.double(); absref = absref + bias.double().abs()
    if res is not None:
        ref = ref + res.double(); absref = absref + res.double().abs()
    return ref, absref


@pytest.mark.parametrize("regime", ["exact", "gauss"])
@pytest.mark.parametrize("epi", ["none", "bias+res"])
@pytest.mark.parametrize("M,Kd,N", CASES)
def test_f32x_f16w_gemm(K, M, Kd, N, epi, regime):
    import torch
    if M * Kd * N > 2048 * 4096 * 4096 and (epi != "none" or regime == "exact"):
        pytest.skip("the largest shapes run once, Gaussian, without epilogue")
    g = torch.Generator(device="cuda").manual_seed(M + 3 * Kd + 7 * N)
    bias = res = None
    if epi != "none":
        bias, res = _operands("exact" if regime == "exact" else "gauss", g, [(N,), (M, N)], torch.float32, lim=7)
    cases = [_exact_operands(c, M, N, Kd, M + Kd + N + i) for i, c in enumerate(("m", "l"))] if regime == "exact" else \
        [(lambda a, w: (a, w.half()))(*_operands("gauss", g, [(M, Kd), (Kd, N)], torch.float32, row_scaled=1))]
    seen = {}
    for a, w in cases:
        rc, n, c = _run(K, a, w, bias, res)
        assert rc == 0 and n >= 3, (rc, n)          # the split of A, the GEMM, the fp32 reduce
        ref, absref = _ref(a, w, bias, res)
        what = f"gemm_f32x_f16w {(M, Kd, N)} {epi} {regime}"
        if regime == "exact":
            prods = _products(a, w)
            assert not prods["l.lo"], "the dropped product a_l b_lo must be zero for the exact regime"
            for k_, v in prods.items():
                seen[k_] = seen.get(k_, False) or v
            _check_exact(c, ref, absref, what)
        else:
            _check(c, ref, absref, what)
    if regime == "exact":
        assert all(seen[p] for p in ("h.hi", "h.lo", "m.hi", "l.hi", "m.lo")), seen


@pytest.mark.parametrize("regime", ["exact", "gauss"])
def test_f32x_f16w_padded_weight(K, regime):
    """A 259-column weight stored 264 wide (the row-padded vocabulary): the pad columns (7.0) never reach the output."""
    import torch
    M, Kd, N, ldb = 300, 256, 259, 264
    g = torch.Generator(device="cuda").manual_seed(5)
    a, w = _exact_operands("m", M, N, Kd, 9) if regime == "exact" else \
        (lambda a, w: (a, w.half()))(*_operands("gauss", g, [(M, Kd), (Kd, N)], torch.float32, row_scaled=1))
    bias, res = _operands("exact", g, [(N,), (M, N)], torch.float32, lim=7)
    wp = torch.full((Kd, ldb), 7.0, device="cuda", dtype=torch.half)
    wp[:, :N] = w
    rc, n, c = _run(K, a, wp, bias, res, N)
    assert rc == 0
    ref, absref = _ref(a, w, bias, res)
    (_check_exact if regime == "exact" else _check)(c, ref, absref, f"gemm_f32x_f16w ldb={ldb} {regime}")


def test_f32x_f16w_one_hot_returns_the_weight(K):
    """A one-hot A returns the fp16 B bit for bit as fp32: full 11-bit significands, subnormals, +-65504 and signed zeros."""
    import torch
    Kd, N = 64, 256
    bits = torch.arange(Kd * N, dtype=torch.int64) * 2654435761 % 65536 - 32768
    w = bits.to(torch.int16).view(torch.float16).reshape(Kd, N).cuda()
    w = torch.where(torch.isfinite(w), w, torch.zeros_like(w))
    w[0, :8] = torch.tensor([65504, -65504, 6e-8, -6e-8, 0.0, -0.0, 2047 / 1024, 1.0009765625], dtype=torch.half)
    w[1, :4] = torch.tensor([6.1e-5, 3.05e-5, -1.5e-7, 0.000999], dtype=torch.half)
    a = torch.eye(Kd, device="cuda")
    rc, n, c = _run(K, a, w, None, None)
    assert rc == 0
    want = w.float()
    assert torch.equal(c.view(torch.int32)[want != 0], want.view(torch.int32)[want != 0]), "nonzero values bit for bit"
    assert torch.equal(c[want == 0], want[want == 0])


def test_f32x_f16w_refusals(K):
    """Shapes and pointers outside the kernel return cudaErrorNotSupported and launch nothing."""
    import torch
    a = torch.zeros(64, 264, device="cuda")
    w = torch.zeros(264 * 272 + 8, device="cuda", dtype=torch.half)
    c = torch.zeros(64 * 272 + 4, device="cuda")
    pl = _planes(64, 264 + 8)
    pa, pw, pc, pp = a.data_ptr(), w.data_ptr(), c.data_ptr(), pl.data_ptr()
    for what, args in [("K % 8", (pa, pw, 264, pc, None, None, 64, 264, 260, pp)), ("ldb % 8", (pa, pw, 268, pc, None, None, 64, 264, 256, pp)),
                       ("ldb < N", (pa, pw, 256, pc, None, None, 64, 264, 256, pp)), ("unaligned A", (pa + 4, pw, 264, pc, None, None, 32, 264, 256, pp)),
                       ("unaligned B", (pa, pw + 2, 264, pc, None, None, 64, 264, 256, pp)), ("unaligned planes", (pa, pw, 264, pc, None, None, 64, 264, 256, pp + 8)),
                       ("unaligned C", (pa, pw, 264, pc + 2, None, None, 64, 264, 256, pp)), ("M = 0", (pa, pw, 264, pc, None, None, 0, 264, 256, pp))]:
        K.osb_launch_count_reset()
        rc = K.osb_tc_gemm_f32x_f16w(*args, _stream())
        assert (rc, int(K.osb_launch_count())) == (NOT_SUPPORTED, 0), what
    assert K.osb_tc_gemm_f32x_f16w_ok(64, 264, 256, 264) == 1
    assert K.osb_tc_gemm_f32x_f16w_ok(64, 264, 260, 264) == 0 and K.osb_tc_gemm_f32x_f16w_ok(64, 264, 256, 260) == 0


# ---- the engine: fp32-arithmetic Llama prefill on fp16 blobs ----------------------------------------------------------------------------

# every MatMul width a multiple of 8, so the streamed prefill takes the new route for all of them
ROUTE_CFG = dict(vocab=264, hidden=256, heads=4, kv_heads=2, head_dim=64, mlp=512, layers=2, max_pos=512)


@pytest.fixture(scope="module")
def workdir():
    with tempfile.TemporaryDirectory(prefix="osb200_f16wgemm_") as d:
        yield d


def _matmul_weights(d):
    """(K, N) of every MatMul with a static 2-D fp16 weight in model.txt, and the number of fp16 weight references outside them."""
    mm, other = [], 0
    for line in open(d + "model.txt").read().splitlines():
        refs = re.findall(r"\(float16:([0-9,]*)\)", line)
        if ":MatMul*" in line:
            for s in refs:
                dims = [int(x) for x in s.split(",") if x]
                if len(dims) == 2:
                    mm.append(tuple(dims))
        else:
            other += len(refs)
    return mm, other


def _case(workdir, tag, cfgkw, T, past):
    cfg = emit.LlamaConfig(past=past, **cfgkw)
    d = os.path.join(workdir, f"{tag}_{T}_{past}") + "/"
    if not os.path.exists(d + "model.txt"):
        emit.emit_llama_decode(d, cfg, "float16", new_tokens=T)
    return cfg, d, emit.llama_inputs(cfg, new_tokens=T), (DYN if past == 0 else ())


def test_f32_prefill_route_reads_f16_weights(engine_lib, workdir):
    """A streamed fp32 prefill of 64 tokens launches the new kernel once per MatMul and no bf16x3 expansion; the decode step of the same
    model still launches only the fp16-weight GEMVs.  The prefill converts exactly as many fp16 weights to fp32 as the model text has fp16
    weight references outside its MatMuls: every one of those once, no MatMul weight (test_f32_prefill_resident_bytes shows, byte for
    byte, that no MatMul weight gets an fp32 copy)."""
    from kernel_trace import trace_run
    cfg, d, inputs, dyn = _case(workdir, "route", ROUTE_CFG, 64, 0)
    _, names = trace_run(engine_lib, d, inputs, OPTS32 + dyn, wp="ram+nocache")
    mm, other = _matmul_weights(d)
    assert len(mm) == 7 * cfg.layers + 1
    assert sum(KERNEL in n for n in names) == len(mm), names
    assert not [n for n in names if "bf16x3_expand" in n], names
    converts = sum("convert_kernel<__half, float>" in n for n in names)
    cfg1, d1, inputs1, dyn1 = _case(workdir, "route", ROUTE_CFG, 1, 300)
    _, names1 = trace_run(engine_lib, d1, inputs1, OPTS32 + dyn1, wp="ram+nocache")
    assert not [n for n in names1 if "tc_gemm_kernel" in n or "bf16x3_expand" in n], names1
    assert sum("gemv_panel" in n and "<__half, float," in n for n in names1) == 4 * cfg.layers + 1, names1
    assert converts == other, (converts, other)


def test_f32_prefill_resident_bytes(engine_lib, workdir):
    """Resident weights: every prefill MatMul weight is cached once as its fp16 blob (2 bytes per parameter), plus the row-padded fp16
    copy of a 259-entry vocabulary; the other weights cost what they cost in the fp32-blob model.  That model caches each MatMul weight in
    fp32 and, where N % 8 == 0, its bf16x6 expansion (4 + 12 bytes per parameter); its 259-wide vocabulary runs the CUDA-core GEMM on the
    fp32 copy alone.  At the parent the fp16 model cached the same fp32 copies and expansions."""
    cfgkw = dict(ROUTE_CFG, vocab=259)
    res = {}
    for wdtype in ("float16", "float32"):
        cfg = emit.LlamaConfig(past=0, **cfgkw)
        d = os.path.join(workdir, f"bytes_{wdtype}") + "/"
        emit.emit_llama_decode(d, cfg, wdtype, new_tokens=64)
        _, m = run_model(engine_lib, d, emit.llama_inputs(cfg, new_tokens=64), OPTS32 + DYN, wp="ram+nocache",
                         b200_options=(("b200_resident_weights", 1),), runs=2)
        res[wdtype] = int(m.stats()["weight_resident_bytes"])
        m.close()
    mm, _ = _matmul_weights(os.path.join(workdir, "bytes_float16") + "/")
    params = sum(k * n for k, n in mm)
    vocab = cfg.hidden * cfg.vocab
    pad16 = cfg.hidden * ((cfg.vocab + 7) // 8 * 8)
    assert res["float16"] == res["float32"] - 16 * (params - vocab) - 4 * vocab + 2 * params + 2 * pad16, (res, params)


MISTRAL_HEADS = dict(vocab=259, hidden=4096, heads=32, kv_heads=8, head_dim=128, mlp=512, layers=1, max_pos=512)
TINY_HEADS = dict(vocab=259, hidden=2048, heads=32, kv_heads=4, head_dim=64, mlp=512, layers=1, max_pos=512)


@pytest.mark.parametrize("Tq,past", [(17, 0), (128, 300)], ids=["first", "later"])
@pytest.mark.parametrize("cfgkw", [TINY_HEADS, MISTRAL_HEADS], ids=["tinyllama_heads", "mistral_heads"])
def test_f32_prefill_on_f16_weights_parity(engine_lib, oracle_lib, workdir, cfgkw, Tq, past):
    """TinyLlama (32 / 4 heads, d 64) and Mistral (32 / 8, d 128) heads at a reduced MLP and depth: fp32 prefill on fp16 blobs, a first turn
    and a later turn over a cache, streamed, resident and graph replay, against the reference's fp32 run."""
    cfg, d, inputs, dyn = _case(workdir, f"parity_h{cfgkw['heads']}_{cfgkw['kv_heads']}", cfgkw, Tq, past)
    names = ("logits", "opkv0")
    ref = reference_outputs(oracle_lib, d, inputs, OPTS32 + dyn, extra_outputs=("opkv0",))
    for b200 in ((), (("b200_resident_weights", 1),), (("b200_resident_weights", 1), ("b200_cuda_graph", 1))):
        got, m = run_model(engine_lib, d, inputs, OPTS32 + dyn, extra_outputs=("opkv0",), wp="ram+nocache", b200_options=b200,
                           runs=3 if b200 else 1)
        for n in names:
            assert got[n].shape == ref[n].shape, (n, b200)
            assert report(got[n], ref[n])["rel_to_max"] <= TOL32, (n, b200, report(got[n], ref[n]))
        m.close()
