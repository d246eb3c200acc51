"""Prompt prefill: one Model::run over T new tokens with a KV cache (src/llm.cpp:472-480).

GPU tests (gpu marker): the grouped-KV masked flash attention kernel (osb_sdpa_flash) against fp64 math -- at every accepted head dim,
with -inf masks, rows of very different scale, any scale and no mask -- and its launch refusals, the emitted Llama prefill
graphs against the reference's own Model::run() (stored reference outputs under tests/golden/oracle, tests/util.py), the routing of
the prefill attention onto the kernel, and a decode step fed with each side's prefill cache.  CPU tests (no marker): the fusion plan
of a prefill graph, the unchanged decode model text, and the numpy restatement of the prefill graph (mask construction included)
against the stored reference output."""
import ctypes
import hashlib
import os
import re
import sys
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from util import reference_outputs, report, run_model

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
from np_oracle import NumpyOracle  # noqa: E402

F16 = 2
UPCAST = ("_2F_input_5F_layernorm_2F_", "_2F_post_5F_attention_5F_layernorm_2F_", "_2F_norm_2F_")
OPTS32 = ("use_scaled_dp_attn_op",)
OPTS16 = ("use_scaled_dp_attn_op", "use_fp16_arithmetic")
# llm.cpp reads every model with support_dynamic_shapes (src/llm.cpp:376): that is what lets the first turn's (1, kv_heads, 0, d)
# caches through the model text
DYN = ("support_dynamic_shapes",)

MID64 = dict(vocab=259, hidden=256, heads=4, kv_heads=2, head_dim=64, mlp=512, layers=2, max_pos=512)
MID128 = dict(vocab=259, hidden=256, heads=2, kv_heads=1, head_dim=128, mlp=512, layers=2, max_pos=512)
# turn -> (new tokens, cached positions, attention_mask positions set to 0)
TURNS = {"first": (40, 0, None), "later": (33, 300, (5, 40))}


@pytest.fixture(scope="module")
def workdir():
    with tempfile.TemporaryDirectory(prefix="osb200_pf_") as d:
        yield d


def _prefill_case(workdir, cfgkw, turn, wdtype="float16"):
    T, past, masked = TURNS[turn]
    cfg = emit.LlamaConfig(past=past, **cfgkw)
    d = os.path.join(workdir, f"prefill_d{cfg.head_dim}_{turn}_{wdtype}") + "/"
    if not os.path.exists(d + "model.txt"):
        emit.emit_llama_decode(d, cfg, wdtype, new_tokens=T)
    inputs = emit.llama_inputs(cfg, new_tokens=T)
    if masked:
        inputs["attention_5F_mask"][0, masked[0]:masked[1]] = 0
    dyn = DYN if past == 0 else ()
    return cfg, d, inputs, dyn


# ---- kernel ------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def K(engine_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = ctypes.CDLL(engine_lib)
    vp, i64, cf = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float
    lib.osb_sdpa_flash.argtypes = [vp] * 5 + [i64] * 5 + [cf, vp]
    lib.osb_sdpa_flash_ok.argtypes = [i64] * 6 + [ctypes.c_int]
    lib.osb_rope.argtypes = [vp] * 4 + [ctypes.c_int, i64, i64, i64, vp]
    lib.osb_launch_count.restype = ctypes.c_uint64
    return lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _mask(kind, Tq, Tk, past):
    """0 / -65504 additive mask [Tq, Tk] as the prefill graph builds it: keep[t, j] = (j <= past + t) * attention_mask[j].  The ninf_*
    kinds put -inf on every masked key (an fp32 -FLT_MAX mask in fp16): ninf_lead40 also masks keys [0, 40) (a left-padded prompt),
    ninf_splits keys [0, 128) and [256, 384), ninf_one_key leaves every third row its last causal key only."""
    import torch
    keep = (torch.arange(Tk)[None, :] <= past + torch.arange(Tq)[:, None]).double()
    if kind == "band":
        keep[:, 100:160] = 0                                  # padded positions inside the cache
    elif kind == "ninf_lead40":
        keep[:, :40] = 0
    elif kind == "ninf_splits":
        keep[:, :128] = 0
        keep[:, 256:384] = 0
    elif kind == "ninf_one_key":
        for t in range(0, Tq, 3):
            keep[t, :past + t] = 0
    if kind.startswith("ninf"):
        assert bool((keep.sum(-1) > 0).all()), kind         # every row keeps a finite key
        return torch.where(keep > 0, 0.0, float("-inf")).half().cuda()
    m = (1 - keep) * -65504.0
    if kind == "full_rows":
        m[:, :7] = -1.5                                       # finite non-trivial values too
        m[[0, 9, 33, 63], :] = -65504.0                       # rows whose every key is masked
    return m.half().cuda()


SDPA_CASES = [
    # Hq, Hkv, Tq, Tk, d, mask kind, past
    (32, 4, 512, 512, 64, "causal", 0),          # TinyLlama heads, first turn
    (32, 8, 300, 1000, 128, "band", 700),        # Mistral heads, d = 128, a later turn with a padded band
    (4, 4, 77, 77, 64, "causal", 0),             # equal head counts
    (8, 2, 17, 17, 64, "causal", 0),             # Tq just above the decode threshold
    (4, 1, 130, 131, 40, "causal", 1),           # ragged: partial query and key tiles, odd Tk, d < 64
    (2, 2, 64, 129, 128, "full_rows", 65),       # rows fully masked at -65504
] + [(4, 2, 33, 70, d, "causal", 37) for d in range(8, 129, 8)]     # every accepted head dim on one ragged shape

# -inf masks (fp16 kernel only: the fp32 kernel's own tests hold it to -inf and -FLT_MAX masks)
SDPA_NEG_INF_CASES = [
    (8, 2, 64, 300, 64, "ninf_lead40", 236),
    (8, 2, 64, 500, 128, "ninf_splits", 436),
    (4, 1, 40, 140, 40, "ninf_one_key", 100),
]


def _inputs(Hq, Hkv, Tq, Tk, d, row_scales=False):
    """q [Hq, Tq, d], k / v [Hkv, Tk, d] fp16.  row_scales: query rows spread over three decades (|q| stays below 1e3, well inside
    fp16) and key rows whose norm grows along the sequence, so the rows' maxima keep moving to later key tiles."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(Hq * 7919 + Tq * 31 + Tk + d)
    q = torch.randn(Hq, Tq, d, device="cuda", generator=g)
    k = torch.randn(Hkv, Tk, d, device="cuda", generator=g)
    v = torch.randn(Hkv, Tk, d, device="cuda", generator=g)
    if row_scales:
        q *= torch.logspace(-1, 2, Tq, device="cuda")[torch.randperm(Tq, device="cuda", generator=g)].view(1, Tq, 1)
        k *= torch.linspace(0.25, 2.0, Tk, device="cuda").view(1, Tk, 1)
    return q.half(), k.half(), v.half()


def _flash(K, q, k, v, mask, scale):
    import torch
    Hq, Tq, d = q.shape
    Hkv, Tk, _ = k.shape
    o = torch.full((Hq, Tq, d), float("nan"), device="cuda", dtype=torch.half)
    rc = K.osb_sdpa_flash(q.data_ptr(), k.data_ptr(), v.data_ptr(), mask.data_ptr() if mask is not None else None, o.data_ptr(),
                          Hq, Hkv, Tq, Tk, d, scale, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    return o


def _check(o, q, k, v, mask, scale):
    """softmax(Q K^T s + mask) V in fp64 on the fp16-rounded operands.  P is rounded to fp16 before the second MMA, so
    |err| <= 2^-8 sum p|v| + 2^-9 |ref| + 1e-4 (the bar of test_flash_attention); every output finite."""
    import torch
    G = q.shape[0] // k.shape[0]
    kk = k.double().repeat_interleave(G, 0)
    vv = v.double().repeat_interleave(G, 0)
    s = q.double() @ kk.transpose(1, 2) * scale
    P = torch.softmax(s + mask.double() if mask is not None else s, dim=-1)
    ref = P @ vv
    absref = P @ vv.abs()
    assert bool(torch.isfinite(o).all()), f"{int((~torch.isfinite(o)).sum())} / {o.numel()} outputs not finite"
    err = (o.double() - ref).abs()
    tol = absref * 2.0 ** -8 + ref.abs() * 2.0 ** -9 + 1e-4
    assert not (err > tol).any(), f"max err {float(err.max()):.4g}, ref max {float(ref.abs().max()):.4g}, bad {(err > tol).sum().item()}"


@pytest.mark.gpu
@pytest.mark.parametrize("Hq,Hkv,Tq,Tk,d,kind,past", SDPA_CASES + SDPA_NEG_INF_CASES)
def test_sdpa_flash_matches_fp64(K, Hq, Hkv, Tq, Tk, d, kind, past):
    """The bar of _check; a second launch gives the same bits."""
    import torch
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d)
    mask = _mask(kind, Tq, Tk, past)
    scale = float(np.float32(1.0 / d ** 0.5))
    assert K.osb_sdpa_flash_ok(Hq, Hkv, Tq, Tk, d, d, F16) == 1
    a = _flash(K, q, k, v, mask, scale)
    b = _flash(K, q, k, v, mask, scale)
    assert torch.equal(a, b), "second launch differs"
    _check(a, q, k, v, mask, scale)


@pytest.mark.gpu
@pytest.mark.parametrize("Hq,Hkv,Tq,Tk,d,past", [(32, 4, 512, 512, 64, 0), (8, 2, 333, 777, 128, 444), (4, 4, 300, 300, 40, 0)])
def test_sdpa_flash_running_max(K, Hq, Hkv, Tq, Tk, d, past):
    """Rows of very different scale under a causal mask: a kernel that kept the first tile's maximum or skipped the rescaling of O fails."""
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d, row_scales=True)
    mask = _mask("causal", Tq, Tk, past)
    scale = float(np.float32(1.0 / d ** 0.5))
    _check(_flash(K, q, k, v, mask, scale), q, k, v, mask, scale)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 128])
def test_sdpa_flash_leading_neg_inf_tiles(K, d):
    """-inf over the first 192 keys of every row (whole key tiles) and on the causally masked keys, in rows that have finite keys later:
    those tiles must leave the running maximum, the sums and O untouched instead of making them NaN."""
    Hq, Hkv, Tq, Tk, past = 8, 2, 200, 456, 256
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d)
    scale = float(np.float32(1.0 / d ** 0.5))
    mask = _mask("causal", Tq, Tk, past)
    mask[mask < 0] = float("-inf")
    mask[:, :192] = float("-inf")
    _check(_flash(K, q, k, v, mask, scale), q, k, v, mask, scale)


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [-0.125, 0.9, 1e-3])
def test_sdpa_flash_any_scale(K, scale):
    """Any finite scale, negative included: the running maximum is taken over the masked, scaled logits."""
    Hq, Hkv, Tq, Tk, d = 8, 2, 130, 200, 64
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d)
    mask = _mask("causal", Tq, Tk, Tk - Tq)
    _check(_flash(K, q, k, v, mask, scale), q, k, v, mask, scale)


@pytest.mark.gpu
def test_sdpa_flash_no_mask(K):
    """A null mask is softmax(Q K^T * scale) V."""
    Hq, Hkv, Tq, Tk, d = 4, 2, 100, 170, 64
    q, k, v = _inputs(Hq, Hkv, Tq, Tk, d)
    scale = float(np.float32(1.0 / d ** 0.5))
    _check(_flash(K, q, k, v, None, scale), q, k, v, None, scale)


@pytest.mark.gpu
def test_sdpa_flash_refuses_misaligned_pointers(K):
    """q / k / v / out off 16-byte alignment and a mask off 4-byte alignment are refused before anything is enqueued: the launch count
    stays and the output stays as it was.  A mask 4 bytes past a 16-byte boundary is taken."""
    import torch
    Hq, Hkv, Tq, Tk, d = 4, 2, 64, 64, 64
    buf = torch.zeros(Hq * Tq * d + 64, device="cuda", dtype=torch.half)
    mask = torch.zeros(Tq * Tk + 8, device="cuda", dtype=torch.half)
    out = torch.full((Hq * Tq * d + 16,), 7.0, device="cuda", dtype=torch.half)
    p = buf.data_ptr()

    def refused(qoff=0, koff=0, voff=0, ooff=0, moff=0):          # byte offsets
        n0 = K.osb_launch_count()
        rc = K.osb_sdpa_flash(p + qoff, p + koff, p + voff, mask.data_ptr() + moff, out.data_ptr() + ooff, Hq, Hkv, Tq, Tk, d, 0.125, _stream())
        torch.cuda.synchronize()
        return rc != 0 and K.osb_launch_count() == n0
    assert refused(qoff=8) and refused(koff=8) and refused(voff=2) and refused(ooff=8)
    assert refused(moff=2)
    assert bool((out == 7.0).all())
    assert not refused(moff=4)


@pytest.mark.gpu
def test_sdpa_flash_scope(K):
    """fp16, d % 8 == 0 with 8 <= d <= 128, dv == d, Hq a multiple of Hkv; anything else is refused, never computed."""
    assert K.osb_sdpa_flash_ok(32, 4, 2048, 2048, 64, 64, F16) == 1
    assert K.osb_sdpa_flash_ok(32, 8, 1, 1, 128, 128, F16) == 1
    assert K.osb_sdpa_flash_ok(32, 4, 64, 64, 136, 136, F16) == 0
    assert K.osb_sdpa_flash_ok(32, 4, 64, 64, 60, 60, F16) == 0
    assert K.osb_sdpa_flash_ok(32, 4, 64, 64, 64, 32, F16) == 0
    assert K.osb_sdpa_flash_ok(32, 5, 64, 64, 64, 64, F16) == 0
    assert K.osb_sdpa_flash_ok(32, 4, 64, 64, 64, 64, 3) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("heads,T,D", [(4, 33, 64), (2, 40, 128), (1, 7, 16)])
def test_rope_per_position_tables(K, heads, T, D):
    """Rotary over T positions: x [heads, T, D] with cos / sin [T, D] broadcast over the heads (table row = x row % T)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(heads * T * D)
    x = torch.randn(heads, T, D, device="cuda", generator=g).half()
    ang = torch.rand(T, D, device="cuda", generator=g) * 6.28
    cs, sn = torch.cos(ang).half(), torch.sin(ang).half()
    y = torch.empty_like(x)
    assert K.osb_rope(x.data_ptr(), cs.data_ptr(), sn.data_ptr(), y.data_ptr(), F16, heads * T, D, T, _stream()) == 0
    torch.cuda.synchronize()
    rot = torch.cat([-x[..., D // 2:], x[..., :D // 2]], -1)
    ref = (x * cs).half() + (rot * sn).half()
    assert float((y.float() - ref.float()).abs().max()) <= 2e-3 * max(1.0, float(ref.abs().max()))


# ---- the prefill graph against the reference ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("turn", ["first", "later"])
@pytest.mark.parametrize("cfgkw", [MID64, MID128], ids=["d64", "d128"])
def test_llama_prefill_parity(engine_lib, oracle_lib, workdir, cfgkw, turn):
    """Prefill of 40 tokens into an empty cache and of 33 tokens after 300 cached positions (5:40 padded): logits of every new
    token and the grown caches, streamed, resident and with the flash route off, against ONE reference run."""
    cfg, d, inputs, dyn = _prefill_case(workdir, cfgkw, turn)
    kw = dict(extra_outputs=("opkv0", "opkv3"), upcast=UPCAST)
    ref = reference_outputs(oracle_lib, d, inputs, OPTS32 + dyn, extra_outputs=("opkv0", "opkv3"))     # fp32 arithmetic, same blobs
    ref16 = reference_outputs(oracle_lib, d, inputs, OPTS16 + dyn, **kw)
    base_err = report(ref16["logits"], ref["logits"])["rel_to_max"]
    for b200 in ((), (("b200_resident_weights", 1),), (("b200_flash_attention", 0),)):
        got, _ = run_model(engine_lib, d, inputs, OPTS16 + dyn, wp="ram+nocache", b200_options=b200, runs=2 if b200 else 1, **kw)
        for n in ("logits", "opkv0", "opkv3"):
            assert got[n].shape == ref[n].shape, (n, b200)
            assert report(got[n], ref16[n])["rel_to_max"] <= 3e-2, (n, b200, report(got[n], ref16[n]))
        # no further from the fp32-arithmetic result than the reference's own fp16 mode (x2 + slack)
        assert report(got["logits"], ref["logits"])["rel_to_max"] <= 2 * base_err + 2e-3, (b200, report(got["logits"], ref["logits"]), base_err)


@pytest.mark.gpu
@pytest.mark.parametrize("cfgkw", [MID64, MID128], ids=["d64", "d128"])
def test_prefill_attention_takes_the_flash_route(engine_lib, workdir, cfgkw):
    """One tensor-core attention launch per layer: the tensor-core launches of one prefill run (stats()["tc_launches"]; the launch
    counters restart with every run) with b200_flash_attention on, minus those with it off, are the layer count."""
    from onnxstream_b200.model import Model
    cfg, d, inputs, dyn = _prefill_case(workdir, cfgkw, "later")

    def tc_launches(flash):
        m = Model(engine_lib, 0, "ram+nocache")
        for o in OPTS16 + dyn:
            m.set_option(o, True)
        m.lib.model_set_option(m.h, b"b200_flash_attention", int(flash))
        for p in UPCAST:
            m.add_upcast_pattern(p)
        m.read_file(d + "model.txt")
        for _ in range(2):                                  # the second run is the counted one
            m.clear_tensors()
            for k, v in inputs.items():
                m.add_tensor(k, v)
            m.run()
        return int(m.stats()["tc_launches"])

    on, off = tc_launches(True), tc_launches(False)
    assert on - off == cfg.layers, (on, off)


@pytest.mark.gpu
def test_prefill_then_decode(engine_lib, oracle_lib, workdir):
    """The first turn's prefill, then one decode step on the cache it produced: each side (engine, reference) feeds its own prefill
    caches back in, and the decode logits must agree."""
    cfg, d, inputs, dyn = _prefill_case(workdir, MID64, "first")
    T = TURNS["first"][0]
    kv = tuple(f"opkv{i}" for i in range(2 * cfg.layers))
    ref_pf = reference_outputs(oracle_lib, d, inputs, OPTS16 + dyn, whole=True, extra_outputs=kv, upcast=UPCAST)
    dcfg = emit.LlamaConfig(past=T, **MID64)
    dd = os.path.join(workdir, "prefill_then_decode") + "/"
    emit.emit_llama_decode(dd, dcfg, "float16")
    step = emit.llama_inputs(dcfg, seed=1)
    ref_in = dict(step)
    for i in range(2 * cfg.layers):
        ref_in[f"pkv{i}"] = np.ascontiguousarray(ref_pf[f"opkv{i}"], np.float32)
    ref = reference_outputs(oracle_lib, dd, ref_in, OPTS16, upcast=UPCAST)

    got_pf = run_model(engine_lib, d, inputs, OPTS16 + dyn, extra_outputs=kv, upcast=UPCAST)[0]
    got_in = dict(step)
    for i in range(2 * cfg.layers):
        assert got_pf[f"opkv{i}"].shape == ref_in[f"pkv{i}"].shape
        got_in[f"pkv{i}"] = np.ascontiguousarray(got_pf[f"opkv{i}"], np.float32)
    got = run_model(engine_lib, dd, got_in, OPTS16, upcast=UPCAST)[0]
    assert got["logits"].shape == (1, 1, cfg.vocab)
    assert report(got["logits"], ref["logits"])["rel_to_max"] <= 3e-2, report(got["logits"], ref["logits"])


# ---- CPU -----------------------------------------------------------------------------------------------------------------

def test_prefill_plan_has_one_attention_and_two_rotary_steps_per_layer(engine_lib, workdir):
    from onnxstream_b200.model import plan_summary
    cfg, d, _, _ = _prefill_case(workdir, MID64, "later")
    last = plan_summary(open(d + "model.txt").read(), use_scaled_dp_attn_op=True, library_path=engine_lib).splitlines()[-1]
    for kind, n in (("SDPA", cfg.layers), ("ROPE", 2 * cfg.layers)):
        assert re.search(rf"\b{kind}={n}\b", last), last


def test_decode_model_text_unchanged():
    """new_tokens = 1 must emit the decode step byte for byte as before (stored reference outputs are keyed by the text)."""
    cfg = emit.LlamaConfig.tiny()
    for wdtype, sha in (("float32", "4977ead5d622270cfaf7ecbf066976c8d383de13"), ("float16", "e00637802a8d4f50bfe5d549f2cf804437d9d1d8")):
        assert hashlib.sha1(emit.emit_llama_decode(None, cfg, wdtype).text().encode()).hexdigest() == sha, wdtype


@pytest.mark.parametrize("T,past,masked", [(12, 0, None), (7, 9, (2, 4))])
def test_prefill_restatement_matches_reference(oracle_lib, workdir, T, past, masked):
    """The numpy restatement of the prefill graph (causal AND padding mask, rotary over T positions, grouped-KV attention) equals the
    reference in fp32: pins the mask construction independently of the engine."""
    cfg = emit.LlamaConfig.tiny()
    cfg.past = past
    d = os.path.join(workdir, f"prefill_np_{T}_{past}") + "/"
    emit.emit_llama_decode(d, cfg, "float32", new_tokens=T)
    inputs = emit.llama_inputs(cfg, new_tokens=T)
    if masked:
        inputs["attention_5F_mask"][0, masked[0]:masked[1]] = 0
    opts = OPTS32 + (DYN if past == 0 else ())
    ref = reference_outputs(oracle_lib, d, inputs, opts, extra_outputs=("opkv1",))
    got = NumpyOracle(d).run(inputs, extra_outputs=("opkv1",))
    assert got["logits"].shape == (1, T, cfg.vocab)
    for n in ("logits", "opkv1"):
        assert report(got[n], ref[n])["rel_to_max"] <= 5e-5, n
