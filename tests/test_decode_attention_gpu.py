"""Decode attention (osb_attention): which kernel each side of every routing condition runs, and the decode attention chain through the
engine with a -inf mask.

osb_attention sends a launch to the split-KV decode kernel (attention_decode_kernel) when K is [h, Tk, d], Tk >= 256, heads * Tq <= 4096
and the key splits fit (nsplit = ceil(Tk / 128) <= 4 dv), and to the per-row online-softmax kernel (attention_rows_kernel) otherwise
(kernels_gemm.cu, osb_attention).  Each boundary case runs on both sides, fp16 and fp32, with real decode shapes besides (d = 128 with
32 heads, dv = 64 at the largest key count the split kernel takes, and the fp16 scalar paths of its K dot product and P V loop).  The
kernel each case ran is read from a torch.profiler trace taken in a child process (tests/kernel_trace.py says why); every output is
held to the fp64 bar of test_kernels_gpu.py::test_attention_decode_matches_fp64.  Every case masks keys [0, 40) with -inf.

Through the engine: the decode attention chain as emit_llama_decode spells it (Concat of the cache, Transpose, MatMul, Div, Add of
the mask, Softmax, MatMul; Tq = 1 and 4 new tokens after 100 cached positions, 32 query heads over 8 KV heads, d = 64), the additive
mask a graph input holding -inf on the first 40 positions, in fp16 and fp32 arithmetic, against fp64 and against the reference's
output (stored under tests/golden/oracle, tests/util.py)."""
import json
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from util import reference_outputs, report, run_model

pytestmark = pytest.mark.gpu

F16, F32 = 2, 3
DECODE, ROWS = "attention_decode_kernel", "attention_rows_kernel"

# name: heads, Tq, Tk, d, dv, kv_group, k_transposed, K / V offset (elements), dtypes, the kernel osb_attention must choose
ROUTE_CASES = {
    "Tk255": (8, 1, 255, 64, 64, 2, 0, 0, (F16, F32), ROWS),
    "Tk256": (8, 1, 256, 64, 64, 2, 0, 0, (F16, F32), DECODE),
    "nsplit_eq_4dv": (8, 1, 4096, 8, 8, 2, 0, 0, (F16, F32), DECODE),          # dv = 8: 32 splits
    "nsplit_gt_4dv": (8, 1, 4097, 8, 8, 2, 0, 0, (F16, F32), ROWS),            # 33 splits
    "rows4096": (32, 128, 256, 64, 64, 4, 0, 0, (F16, F32), DECODE),
    "rows4097": (17, 241, 256, 64, 64, 1, 0, 0, (F16, F32), ROWS),
    "k_transposed": (8, 1, 2048, 64, 64, 2, 1, 0, (F16, F32), ROWS),
    "d128_G4": (32, 1, 4096, 128, 128, 4, 0, 0, (F16, F32), DECODE),
    "d128_G1": (32, 1, 4096, 128, 128, 1, 0, 0, (F16, F32), DECODE),
    "dv64_Tk32768": (32, 1, 32768, 64, 64, 8, 0, 0, (F16, F32), DECODE),       # nsplit = 256 = 4 dv
    "d20_scalar": (6, 2, 300, 20, 20, 3, 0, 0, (F16,), DECODE),                # d, dv % 8 != 0: scalar K dot product and P V loop
    "kv_off2_scalar": (8, 1, 2048, 64, 64, 2, 0, 1, (F16,), DECODE),           # K / V 2 bytes off 16-byte alignment
}
ROUTE_IDS = [(name, dt) for name, c in ROUTE_CASES.items() for dt in c[8]]

_CHILD = """
import ctypes, json, sys
import torch
from torch.profiler import ProfilerActivity, profile
lib_path, cases, out_path = sys.argv[1], json.loads(sys.argv[2]), sys.argv[3]
lib = ctypes.CDLL(lib_path)
vp, i64 = ctypes.c_void_p, ctypes.c_int64
lib.osb_attention.argtypes = [vp] * 5 + [i64] * 5 + [ctypes.c_float, ctypes.c_int, i64, ctypes.c_int, vp]
F16 = 2
runs = []
for name, dt, (heads, Tq, Tk, d, dv, group, kt, off) in cases:
    ty = torch.float16 if dt == F16 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(heads * 1000 + Tq * 10 + Tk + d)
    q = torch.randn(heads, Tq, d, device="cuda", generator=g).to(ty)
    k = torch.randn(heads // group, Tk, d, device="cuda", generator=g).to(ty)
    v = torch.randn(heads // group, Tk, dv, device="cuda", generator=g).to(ty)
    mask = (torch.randn(Tq, Tk, device="cuda", generator=g) * 0.5).to(ty)
    mask[:, :40] = float("-inf")
    kin = k.transpose(1, 2).contiguous() if kt else k
    kbuf = torch.empty(kin.numel() + off, device="cuda", dtype=ty)[off:]
    vbuf = torch.empty(v.numel() + off, device="cuda", dtype=ty)[off:]
    kbuf.copy_(kin.reshape(-1)); vbuf.copy_(v.reshape(-1))
    out = torch.full((heads, Tq, dv), float("nan"), device="cuda", dtype=ty)
    runs.append((name, dt, q, k, v, mask, kbuf, vbuf, out, (heads, Tq, Tk, d, dv, group, kt)))
torch.cuda.synchronize()
rcs = []
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for name, dt, q, k, v, mask, kbuf, vbuf, out, (heads, Tq, Tk, d, dv, group, kt) in runs:
        rcs.append(lib.osb_attention(q.data_ptr(), kbuf.data_ptr(), vbuf.data_ptr(), mask.data_ptr(), out.data_ptr(), heads, Tq, Tk, d, dv,
                                     1.0 / d ** 0.5, kt, group, dt, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
evs = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "attention" in e.name), key=lambda e: e.time_range.start)
names = [e.name for e in evs]
res = {}
for i, (name, dt, q, k, v, mask, kbuf, vbuf, out, (heads, Tq, Tk, d, dv, group, kt)) in enumerate(runs):
    kk = k.double().repeat_interleave(group, 0)
    vv = v.double().repeat_interleave(group, 0)
    ref = torch.softmax(q.double() @ kk.transpose(1, 2) / d ** 0.5 + mask.double(), -1) @ vv
    res[f"{name}-{dt}"] = dict(rc=rcs[i], kernel=names[i] if len(names) == len(runs) else None, kernels=len(names),
                               finite=bool(torch.isfinite(out).all()), err=float((out.double() - ref).abs().max()),
                               ref_max=float(ref.abs().max()))
json.dump(res, open(out_path, "w"))
"""


@pytest.fixture(scope="module")
def routes(engine_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    cases = [(name, dt, ROUTE_CASES[name][:8]) for name, dt in ROUTE_IDS]
    with tempfile.TemporaryDirectory(prefix="osb200_routes_") as d:
        out = os.path.join(d, "routes.json")
        env = dict(os.environ)
        env.pop("OSB_DECODE_ATTN", None)            # read once per process: the split kernel on (its default)
        r = subprocess.run([sys.executable, "-c", _CHILD, engine_lib, json.dumps(cases), out], stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, env=env)
        assert r.returncode == 0, r.stdout[-4000:]
        with open(out) as f:
            return json.load(f)


@pytest.mark.parametrize("name,dtype", ROUTE_IDS, ids=[f"{n}-{'f16' if dt == F16 else 'f32'}" for n, dt in ROUTE_IDS])
def test_attention_route(routes, name, dtype):
    """The kernel osb_attention chose (one attention launch per case, in order), and its output against fp64: 2e-3 (fp16) / 1e-5 (fp32)
    of max(1, max|ref|), every output finite."""
    r = routes[f"{name}-{dtype}"]
    want = ROUTE_CASES[name][9]
    assert r["rc"] == 0
    assert r["kernel"] is not None, f"{r['kernels']} attention launches traced for {len(ROUTE_IDS)} calls"
    print(f"[route] {name} {'f16' if dtype == F16 else 'f32'}: {r['kernel']}")
    assert want in r["kernel"], (want, r["kernel"])
    assert r["finite"], "NaN or Inf in the output"
    tol = (2e-3 if dtype == F16 else 1e-5) * max(1.0, r["ref_max"])
    assert r["err"] <= tol, f"max err {r['err']:.3g} > {tol:.3g}"


# ---- through the engine ------------------------------------------------------------------------------------------------------------

HEADS, KV_HEADS, D, PAST = 32, 8, 64, 100
OPTS = {F32: ("use_scaled_dp_attn_op",), F16: ("use_scaled_dp_attn_op", "use_fp16_arithmetic")}


def _decode_attention(dirname, T):
    """The attention of one emit_llama_decode layer on its own: q [1, H, T, D], the new k / v [1, KV, T, D] appended to the cache
    pkv0 / pkv1 [1, KV, PAST, D], scores divided by sqrt(D), plus the additive mask input [1, 1, T, PAST + T], softmax, times V."""
    TT = PAST + T
    g = emit.GraphBuilder(dirname, "float16", 0)
    q = g.input("q", (1, HEADS, T, D))
    k = g.input("k", (1, KV_HEADS, T, D))
    v = g.input("v", (1, KV_HEADS, T, D))
    pk = g.input("pkv0", (1, KV_HEADS, PAST, D))
    pv = g.input("pkv1", (1, KV_HEADS, PAST, D))
    mask = g.input("mask", (1, 1, T, TT))
    kc = g.node("Concat", [pk, k], [(1, KV_HEADS, TT, D)], [("axis", "2")])
    vc = g.node("Concat", [pv, v], [(1, KV_HEADS, TT, D)], [("axis", "2")])
    kt = g.node("Transpose", [kc], [(1, KV_HEADS, D, TT)], [("perm", "0,1,3,2")])
    s = g.node("MatMul", [q, kt], [(1, HEADS, T, TT)])
    s = g.node("Div", [s, g.scalar(math.sqrt(D))], [(1, HEADS, T, TT)])
    s = g.node("Add", [s, mask], [(1, HEADS, T, TT)])
    p = g.node("Softmax", [s], [(1, HEADS, T, TT)], [("axis", "-1")])
    o = g.node("MatMul", [p, vc], [(1, HEADS, T, D)], out_names=["attn_5F_out"])
    g.mark_output(o)
    g.finish()
    rng = np.random.default_rng(T)
    inputs = {n: rng.standard_normal(shape, dtype=np.float32) for n, shape in
              (("q", (1, HEADS, T, D)), ("k", (1, KV_HEADS, T, D)), ("v", (1, KV_HEADS, T, D)), ("pkv0", (1, KV_HEADS, PAST, D)),
               ("pkv1", (1, KV_HEADS, PAST, D)))}
    m = np.zeros((1, 1, T, TT), np.float32)
    m[..., :40] = -np.inf
    inputs["mask"] = m
    return inputs


@pytest.mark.parametrize("dtype", [F16, F32], ids=["f16", "f32"])
@pytest.mark.parametrize("T", [1, 4])
def test_engine_decode_attention_neg_inf_mask(engine_lib, oracle_lib, T, dtype):
    """Finite, within 2e-3 (fp16) / 1e-5 (fp32) of max(1, max|ref|) of fp64 on the operands as the arithmetic type rounds them, and
    within the same of the reference's output."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    with tempfile.TemporaryDirectory(prefix="osb200_dec_attn_") as d:
        d += "/"
        inputs = _decode_attention(d, T)
        ref = reference_outputs(oracle_lib, d, inputs, OPTS[dtype])["attn_5F_out"]
        got, m = run_model(engine_lib, d, inputs, OPTS[dtype])
        m.close()
    got = np.asarray(got["attn_5F_out"], np.float64)
    assert got.shape == (1, HEADS, T, D)
    assert np.isfinite(got).all(), f"{int((~np.isfinite(got)).sum())} / {got.size} outputs not finite"
    rnd = (lambda a: a.astype(np.float16).astype(np.float64)) if dtype == F16 else (lambda a: a.astype(np.float64))
    G = HEADS // KV_HEADS
    kc = np.repeat(np.concatenate([rnd(inputs["pkv0"]), rnd(inputs["k"])], 2), G, 1)
    vc = np.repeat(np.concatenate([rnd(inputs["pkv1"]), rnd(inputs["v"])], 2), G, 1)
    s = rnd(inputs["q"]) @ kc.transpose(0, 1, 3, 2) / math.sqrt(D) + inputs["mask"].astype(np.float64)
    p = np.exp(s - s.max(-1, keepdims=True))
    want = (p / p.sum(-1, keepdims=True)) @ vc
    tol = (2e-3 if dtype == F16 else 1e-5) * max(1.0, float(np.abs(want).max()))
    assert float(np.abs(got - want).max()) <= tol, (float(np.abs(got - want).max()), tol)
    assert report(got, ref)["max_abs"] <= tol, report(got, ref)
