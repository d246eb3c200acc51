"""Every fusion group of the planner (plan.cpp: Planner::mha ... Planner::conv_add) and its executor (engine_run.cpp: fused_*), one tiny
graph per spelling, against an fp64 op-by-op run of the same graph (oracle/np_oracle.py: NumpyOracle, fp32 storage between ops).

The whole-model tests spell each pattern one way (emit.py) and hold it to a whole-model bar.  Here each row builds only the chain
under test, written with GraphBuilder.node so that operand slots, constants, attributes and op names are the row's choice, and asserts:

  plan      (no GPU) plan_summary claims the chain as the expected step kinds and op counts, or, for a structural near miss, leaves it
            to single ops;
  numbers   the engine with b200_fuse_nodes 1 and 0, in fp32 arithmetic and with use_fp16_arithmetic, within the row's bar of the fp64
            oracle (max |err| / max |ref|, BARS below).  The op-by-op run must meet the same bar, so the bar is not fitted to the fused
            path.  In fp16 the fused run's rms error may also be no larger than SLACK times the op-by-op run's, plus FLOOR rms of the
            reference;
  fallback  a value near miss (a constant or Slice bound the executor checks at run time) is claimed by the planner but must run op by
            op: its output equals the b200_fuse_nodes 0 run bit for bit (on a graph that is only the chain both paths run the same
            single-op handlers).

Every row runs twice on one Model, with new inputs the second time, so state carried across runs (the SiLU result cache, the K / V
pre-pass of a cross-attention block) shows up as a wrong second result.  Rows with an intermediate also run with it requested as an
extra output: the planner must then leave the group alone (stats()["ops_fused_away"] counts the ops of the planned groups), and the
intermediate and the output must both match the oracle."""
import math
import os
import sys
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import pytest

from onnxstream_b200 import emit
from onnxstream_b200.model import Model, plan_summary

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
from np_oracle import NumpyOracle  # noqa: E402

I64_MAX = np.iinfo(np.int64).max

# Bars, as max |engine - fp64| / max |fp64|, per kind of group: (fp32 arithmetic, fp16 arithmetic against the fp32-storage oracle).
BARS = {
    # one elementwise pass (GELU, GEGLU gate, SiLU, RoPE): a few fp32 ulps of a value of the order of the maximum; in fp16 the input's
    # and the output's rounding (2^-11 each) through a slope of at most ~1.1, plus the fp16 arithmetic of the op-by-op run
    "elementwise": (2e-6, 2.5e-3),
    # a row or group reduction and a division by its deviation (LayerNorm, RMSNorm, GroupNorm): fp32 sums of up to ~1e4 terms; fp16
    # storage of x - mean and of the normalised value (gamma ~ 1 +- 0.25 keeps the output of the order of its maximum)
    "norm": (2e-6, 5e-3),
    # mean 1e3, std 1 rows (fp32 only): the oracle's mean is rounded to fp32 storage (ulp(1e3) = 6.1e-5 against a unit deviation),
    # and so is the kernel's
    "norm_cancel": (1.5e-4, None),
    # GEMM / GEMV / conv epilogues (K <= 288 with unit-variance operands): fp32 accumulation on the tensor cores through the bf16
    # triple split; in fp16 the operand roundings add up over K and the output is rounded once more
    "gemm": (1e-5, 5e-3),
    # attention: two GEMMs and a softmax; in fp16 the probabilities are rounded before the second GEMM in the op-by-op run
    "attention": (3e-5, 1e-2),
}
SLACK, FLOOR = 1.5, 2.5e-4


@dataclass
class Graph:
    outs: List[str]
    inputs: Callable[[np.random.Generator], Dict[str, np.ndarray]]
    mid: Optional[str] = None          # an intermediate of the group (requested as an extra output in test_intermediate)


@dataclass
class Case:
    id: str
    build: Callable[[emit.GraphBuilder], Graph]
    plan: Tuple[Tuple[str, int], ...]  # the fused steps the planner makes, in order (empty: every op runs by itself)
    bar: str
    fallback: bool = False             # claimed, but the executor must run the group op by op
    wdtype: str = "float32"
    modes: Tuple[str, ...] = ("f32", "f16")
    b200: Tuple[Tuple[str, int], ...] = ()
    sdpa: bool = False
    mid_fused_away: Optional[int] = None   # ops fused away when the intermediate is requested
    upcast: Optional[Tuple[str, int]] = None   # (upcast pattern, ops fused away with it under fp16 arithmetic)
    unfused_sdpa: bool = True          # the yardstick run may switch the ScaledDotProductAttention rewrite off (equal head counts)
    bit_equal_f32: bool = False        # fp32: the fused output equals the op-by-op one bit for bit (RoPE keeps the per-op roundings)


def _normal(shape, mean=0.0, std=1.0):
    return lambda r: (r.standard_normal(shape) * std + mean).astype(np.float32)


def _feeds(**gens):
    return lambda r: {k: f(r) for k, f in gens.items()}


# ---------------------------------------------------------------------------------------------------------------- LayerNorm (9 ops)
def layernorm(rows, cols, eps=1e-5, mean=0.0, std=1.0, pow_e=2.0, gamma_slot=1, axes="-1", skewed=False):
    """ReduceMean, Sub, Pow, ReduceMean, Add(eps), Sqrt, Div, Mul(gamma), Add(beta) over the last axis of x [rows, cols]."""
    def build(g):
        x = g.input("x", (rows, cols))
        red = (rows, 1)
        m = g.node("ReduceMean", [x], [red], [("axes", axes), ("keepdims", "1")])
        d = g.node("Sub", [x, m], [x.shape], out_names=["ln_d"])
        p = g.node("Pow", [d, g.scalar(pow_e)], [x.shape])
        v = g.node("ReduceMean", [p], [red], [("axes", axes), ("keepdims", "1")])
        ve = g.node("Add", [v, g.scalar(eps)], [red])
        sd = g.node("Sqrt", [ve], [red])
        n = g.node("Div", [d, sd], [x.shape])
        gam = g.const(g.randn((cols,), std=0.25, mean=1.0))
        mm = g.node("Mul", [n, gam] if gamma_slot == 1 else [gam, n], [x.shape])
        g.node("Add", [mm, g.const(g.randn((cols,), std=0.25))], [x.shape], out_names=["y"])
        # Pow 3 takes the mean of signed cubes: exponential rows (skewness 2) keep it positive
        gen = (lambda r: (r.exponential(1.0, (rows, cols)) * std + mean).astype(np.float32)) if skewed else _normal((rows, cols), mean, std)
        return Graph(["y"], _feeds(x=gen), "ln_d")
    return build


# small-deviation rows (std 3e-3, variance 1e-5) make the output depend on eps at the percent level: a kernel fed another eps fails
LN = [
    Case("ln_eps1e-5_warp", layernorm(64, 320, 1e-5, std=3e-3), (("LAYERNORM", 9),), "norm", mid_fused_away=0),
    Case("ln_eps1e-6_warp_1280", layernorm(96, 1280, 1e-6, std=3e-3), (("LAYERNORM", 9),), "norm"),
    Case("ln_eps1e-12_block", layernorm(5, 320, 1e-12, std=3e-3), (("LAYERNORM", 9),), "norm"),
    Case("ln_block_odd_cols", layernorm(70, 77, 1e-5), (("LAYERNORM", 9),), "norm"),
    Case("ln_block_wide", layernorm(64, 1536, 1e-6, std=3e-3), (("LAYERNORM", 9),), "norm"),
    Case("ln_mean1e3_warp", layernorm(64, 640, 1e-5, mean=1e3), (("LAYERNORM", 9),), "norm_cancel", modes=("f32",)),
    Case("ln_mean1e3_block", layernorm(3, 2048, 1e-5, mean=1e3), (("LAYERNORM", 9),), "norm_cancel", modes=("f32",)),
    Case("ln_pow3_fallback", layernorm(64, 256, 1.0, pow_e=3.0, skewed=True), (("LAYERNORM", 9),), "norm", fallback=True),
    Case("ln_gamma_slot0", layernorm(64, 256, gamma_slot=0), (), "norm"),
    Case("ln_axes_positive", layernorm(64, 256, axes="1"), (), "norm"),
]


# ---------------------------------------------------------------------------------------------------------------- RMSNorm (7 ops)
def rmsnorm(rows, cols, eps=1e-6, x_slot=0, w_slot=0, two=2.0, one=1.0, positive=False, tag=""):
    """Pow(x, 2), ReduceMean, Add(eps), Sqrt, Div(1, .), Mul(x, .), Mul(w, .); op names carry `tag` on the first four ops only."""
    def build(g):
        x = g.input("x", (rows, cols))
        red = (rows, 1)
        p = g.node("Pow", [x, g.scalar(two)], [x.shape], name=f"{tag}Pow_1")
        m = g.node("ReduceMean", [p], [red], [("axes", "-1"), ("keepdims", "1")], name=f"{tag}ReduceMean_1")
        a = g.node("Add", [m, g.scalar(eps)], [red], name=f"{tag}Add_1")
        s = g.node("Sqrt", [a], [red], name=f"{tag}Sqrt_1", out_names=["rms_s"])
        r = g.node("Div", [g.scalar(one), s], [red], name="Div_1")
        n = g.node("Mul", [x, r] if x_slot == 0 else [r, x], [x.shape], name="Mul_1")
        w = g.const(g.randn((cols,), std=0.25, mean=1.0))
        g.node("Mul", [w, n] if w_slot == 0 else [n, w], [x.shape], name="Mul_2", out_names=["y"])
        gen = (lambda r_: (np.abs(r_.standard_normal((rows, cols))) + 0.1).astype(np.float32)) if positive else _normal((rows, cols))
        return Graph(["y"], _feeds(x=gen), "rms_s")
    return build


RMS = [
    Case("rms_w0_x0_block", rmsnorm(1, 512), (("RMSNORM", 7),), "norm", mid_fused_away=0),
    Case("rms_w1_x1_warp", rmsnorm(9, 64, w_slot=1, x_slot=1), (("RMSNORM", 7),), "norm"),
    Case("rms_w1_x0_block", rmsnorm(4, 1024, w_slot=1), (("RMSNORM", 7),), "norm"),
    Case("rms_f16_weights", rmsnorm(9, 64), (("RMSNORM", 7),), "norm", wdtype="float16"),
    Case("rms_pow3_fallback", rmsnorm(9, 64, two=3.0, positive=True), (("RMSNORM", 7),), "norm", fallback=True),
    Case("rms_div2_fallback", rmsnorm(9, 64, one=2.0), (("RMSNORM", 7),), "norm", fallback=True),
    # fp16 arithmetic with an upcast pattern naming only the first four ops: two arithmetic classes in one chain, not a group
    Case("rms_partial_upcast", rmsnorm(9, 64, tag="_2F_input_5F_layernorm_2F_"), (("RMSNORM", 7),), "norm", modes=("f16",),
         upcast=("_2F_input_5F_layernorm_2F_", 0)),
]


# ---------------------------------------------------------------------------------------------------------------- RoPE (7 ops)
def rope(xshape, tshape, s1=None, s2=None, axis="-1", odd=False):
    """Slice(x, first half), Slice(x, second half), Neg, Concat(-x2, x1), Mul(x, cos), Mul(rot, sin), Add.  s1 / s2: (starts, ends, axes)
    of the two Slices (default: the two halves of the last axis)."""
    D = xshape[-1]
    h = D // 2

    def build(g):
        x = g.input("x", xshape)
        a = s1 or ([0], [h], [-1])
        b = s2 or ([h], [D], [-1])

        def sl(spec):
            st, en, ax = spec
            shp = list(xshape)
            for s_, e_, a_ in zip(st, en, ax):
                n = xshape[a_]
                s_, e_ = (s_ + n if s_ < 0 else s_), min(e_ + n if e_ < 0 else e_, n)
                shp[a_] = e_ - s_
            return g.node("Slice", [x, g.i64(st), g.i64(en), g.i64(ax), g.i64([1] * len(st))], [tuple(shp)])
        x1, x2 = sl(a), sl(b)
        ng = g.node("Neg", [x2], [x2.shape])
        cshape = list(xshape)
        cshape[-1] = ng.shape[-1] + x1.shape[-1]
        rot = g.node("Concat", [ng, x1], [tuple(cshape)], [("axis", axis)], out_names=["rot"])
        cs, sn = g.input("cs", tshape), g.input("sn", tshape)
        m1 = g.node("Mul", [x, cs], [xshape])
        m2 = g.node("Mul", [rot, sn], [xshape])
        g.node("Add", [m1, m2], [xshape], out_names=["y"])
        ang = lambda r: r.uniform(0, 2 * np.pi, tshape)
        return Graph(["y"], lambda r: (lambda t: {"x": _normal(xshape)(r), "cs": np.cos(t).astype(np.float32), "sn": np.sin(t).astype(np.float32)})(ang(r)), "rot")
    return build


ROPE = [
    Case("rope_one_row", rope((4, 1, 64), (64,)), (("ROPE", 7),), "elementwise", bit_equal_f32=True, mid_fused_away=0),
    Case("rope_table_TD", rope((1, 4, 16, 64), (16, 64)), (("ROPE", 7),), "elementwise", bit_equal_f32=True),
    Case("rope_table_11TD_end_max", rope((1, 2, 9, 32), (1, 1, 9, 32), s2=([16], [I64_MAX], [-1])), (("ROPE", 7),), "elementwise", bit_equal_f32=True),
    Case("rope_axis_rank_minus_1", rope((1, 2, 9, 32), (9, 32), s1=([0], [16], [3]), s2=([16], [32], [3]), axis="3"), (("ROPE", 7),), "elementwise", bit_equal_f32=True),
    Case("rope_slices_swapped", rope((1, 2, 9, 32), (9, 32), s1=([16], [32], [-1]), s2=([0], [16], [-1])), (("ROPE", 7),), "elementwise", fallback=True),
    Case("rope_negative_start", rope((1, 2, 9, 32), (9, 32), s2=([-16], [32], [-1])), (("ROPE", 7),), "elementwise", fallback=True),
    # the second Slice also cuts (in full) another axis: two axes, not one
    Case("rope_slice_two_axes", rope((1, 2, 9, 32), (9, 32), s2=([0, 16], [9, 32], [2, 3])), (("ROPE", 7),), "elementwise", fallback=True),
    Case("rope_odd_D", rope((1, 2, 9, 33), (9, 33), s1=([0], [16], [-1]), s2=([16], [33], [-1])), (), "elementwise"),
]


# ---------------------------------------------------------------------------------------------------------------- GELU (5) / + Mul (6)
def gelu(shape, c0=math.sqrt(2.0), c1=1.0, c2=0.5, gate=None):
    """Div(x, c0), Erf, Add(c1), Mul(x, .), Mul(., c2) [, Mul(a, gelu)] with a of shape `gate`."""
    def build(g):
        x = g.input("x", shape)
        d = g.node("Div", [x, g.scalar(c0)], [shape])
        e = g.node("Erf", [d], [shape], out_names=["gelu_e"])
        a = g.node("Add", [e, g.scalar(c1)], [shape])
        m = g.node("Mul", [x, a], [shape])
        y = g.node("Mul", [m, g.scalar(c2)], [shape], out_names=None if gate else ["y"])
        gens = dict(x=_normal(shape, std=2.0))
        if gate:
            av = g.input("a", gate)
            g.node("Mul", [av, y], [shape], out_names=["y"])
            gens["a"] = _normal(gate)
        return Graph(["y"], _feeds(**gens), "gelu_e")
    return build


GELU = [
    Case("gelu5", gelu((33, 96)), (("GELU", 5),), "elementwise", mid_fused_away=0),
    Case("gelu_mul6", gelu((33, 96), gate=(33, 96)), (("GELU", 6),), "elementwise", mid_fused_away=0),
    Case("gelu_div2_fallback", gelu((33, 96), c0=2.0), (("GELU", 5),), "elementwise", fallback=True),
    Case("gelu_add05_fallback", gelu((33, 96), c1=0.5), (("GELU", 5),), "elementwise", fallback=True),
    Case("gelu_mul1_fallback", gelu((33, 96), gate=(33, 96), c2=1.0), (("GELU", 6),), "elementwise", fallback=True),
    Case("gelu_broadcast_gate", gelu((33, 96), gate=(1, 96)), (("GELU", 5),), "elementwise"),
]


@pytest.mark.gpu
def test_gelu_divisor_within_tolerance(engine_lib, cuda, tmp_path):
    """fused_gelu accepts a divisor within 1e-3 of sqrt(2) and then computes the exact erf GELU.  With Div 1.4142 the graph as written
    differs from the exact GELU by 0.5 x erf'(z) z (1 - 1.4142 / sqrt 2) with z = x / sqrt 2, at most 0.5 sqrt(2) e^-1 (2 / sqrt pi) 9.6e-6
    = 2.8e-6 for any x, under 5e-7 of max|y| for these inputs (std 2, max|x| ~ 7): the fused output must stay within 2e-6 of the
    oracle's result for the graph as written (fp32), the op-by-op run within the elementwise bar."""
    _run_numbers(engine_lib, tmp_path, Case("gelu_div_1_4142", gelu((33, 96), c0=1.4142), (("GELU", 5),), "elementwise"), "f32",
                 fused_bar=2e-6)


# ---------------------------------------------------------------------------------------------------------------- GEGLU (8 / 10)
def geglu(rows, inner, lead=False, K=64, a_spec=None, b_spec=None, bias_slot=0):
    """[MatMul(x, W[K, 2 inner]), Add(bias)] then Slice(h, 0:inner), Slice(h, inner:2 inner) on the last axis, erf GELU of the second,
    Mul(first, gelu)."""
    n2 = 2 * inner

    def build(g):
        if lead:
            x = g.input("x", (1, rows, K))
            mm = g.node("MatMul", [x, g.const(g.randn((K, n2), std=1.0 / math.sqrt(K)))], [(1, rows, n2)])
            b = g.const(g.randn((n2,), std=0.25))
            h = g.node("Add", [b, mm] if bias_slot == 0 else [mm, b], [(1, rows, n2)], out_names=["geglu_h"])
            gens = dict(x=_normal((1, rows, K)))
        else:
            h = g.input("h", (1, rows, n2))
            gens = dict(h=_normal((1, rows, n2), std=2.0))
        a_st, a_en = a_spec or ([0], [inner])
        b_st, b_en = b_spec or ([inner], [n2])
        a = g.node("Slice", [h, g.i64(a_st), g.i64(a_en), g.i64([-1]), g.i64([1])], [(1, rows, inner)])
        gt = g.node("Slice", [h, g.i64(b_st), g.i64(b_en), g.i64([-1]), g.i64([1])], [(1, rows, inner)])
        shp = gt.shape
        d = g.node("Div", [gt, g.scalar(math.sqrt(2.0))], [shp])
        e = g.node("Erf", [d], [shp])
        ad = g.node("Add", [e, g.scalar(1.0)], [shp])
        m = g.node("Mul", [gt, ad], [shp])
        y = g.node("Mul", [m, g.scalar(0.5)], [shp])
        g.node("Mul", [a, y], [shp], out_names=["y"])
        return Graph(["y"], _feeds(**gens), "geglu_h" if lead else None)
    return build


GEGLU = [
    Case("geglu8", geglu(33, 96), (("GEGLU", 8),), "elementwise"),
    Case("geglu8_negative_start_end_max", geglu(33, 96, b_spec=([-96], [I64_MAX])), (("GEGLU", 8),), "elementwise"),
    Case("geglu8_not_halves_fallback", geglu(33, 96, a_spec=([8], [104])), (("GEGLU", 8),), "elementwise", fallback=True),
    Case("geglu8_swapped_fallback", geglu(33, 96, a_spec=([96], [192]), b_spec=([0], [96])), (("GEGLU", 8),), "elementwise", fallback=True),
    # fp16: inner % 64 == 0 takes the gate in the tensor-core GEMM epilogue (osb_tc_gemm_geglu), inner % 64 != 0 the GEMM then the gate
    # pass; fp32 arithmetic: the GEMM then the gate pass
    Case("geglu10_tc_epilogue", geglu(96, 128, lead=True), (("GEGLU", 10),), "gemm", mid_fused_away=8),
    Case("geglu10_inner_96", geglu(40, 96, lead=True, bias_slot=1), (("GEGLU", 10),), "gemm", mid_fused_away=8),
    Case("geglu10_swapped_fallback", geglu(40, 64, lead=True, a_spec=([64], [128]), b_spec=([0], [64])), (("GEGLU", 10),), "gemm", fallback=True),
]


# ---------------------------------------------------------------------------------------------------------------- SiLU (2)
def silu(shape, twice=False, swapped=False):
    def build(g):
        x = g.input("x", shape)
        outs = []
        for k in range(2 if twice else 1):
            s = g.node("Sigmoid", [x], [shape])
            outs.append(f"y{k}")
            g.node("Mul", [s, x] if swapped else [x, s], [shape], out_names=[outs[-1]])
        return Graph(outs, _feeds(x=_normal(shape, std=3.0)))
    return build


SILU = [
    Case("silu", silu((8, 320)), (("SILU", 2),), "elementwise"),
    Case("silu_large", silu((1, 320, 16, 16)), (("SILU", 2),), "elementwise"),
    Case("silu_twice_same_input", silu((8, 320), twice=True), (("SILU", 2), ("SILU", 2)), "elementwise"),
    # Mul(Sigmoid(x), x): not claimed (Planner::silu wants x in slot 0, as the diffusers export writes it)
    Case("silu_sigmoid_first", silu((8, 320), swapped=True), (), "elementwise"),
]


# ---------------------------------------------------------------------------------------------------------------- Linear (2 / 3)
def linear(rows, K, N, bias_slot=0, res=None, res_slot=1, bias=True):
    """MatMul(x [rows, K], W[K, N]) [-> Add(bias)] [-> Add(residual)]; res: the residual's shape (None: no residual Add)."""
    def build(g):
        x = g.input("x", (rows, K))
        y = g.node("MatMul", [x, g.const(g.randn((K, N), std=1.0 / math.sqrt(K)))], [(rows, N)], out_names=["lin_mm"])
        gens = dict(x=_normal((rows, K)))
        last = res is None
        if bias:
            b = g.const(g.randn((N,), std=0.25))
            y = g.node("Add", [b, y] if bias_slot == 0 else [y, b], [(rows, N)], out_names=["y"] if last else None)
        if res is not None:
            r = g.input("r", res)
            gens["r"] = _normal(res, mean=0.5)
            g.node("Add", [y, r] if res_slot == 1 else [r, y], [(rows, N)], out_names=["y"])
        return Graph(["y"], _feeds(**gens), "lin_mm")
    return build


LINEAR = [
    Case("linear_bias0_gemm", linear(300, 96, 128), (("LINEAR", 2),), "gemm", mid_fused_away=0),
    Case("linear_bias1_gemv", linear(1, 256, 256, bias_slot=1), (("LINEAR", 2),), "gemm"),
    Case("linear_bias_res1_gemm", linear(300, 96, 128, res=(300, 128)), (("LINEAR", 3),), "gemm", mid_fused_away=0),
    Case("linear_bias_res0_gemv", linear(1, 256, 256, bias_slot=1, res=(1, 256), res_slot=0), (("LINEAR", 3),), "gemm"),
    Case("linear_res_only_gemm", linear(300, 96, 128, bias=False, res=(300, 128), res_slot=0), (("LINEAR", 2),), "gemm", mid_fused_away=0),
    Case("linear_res_only_gemv", linear(1, 256, 256, bias=False, res=(1, 256)), (("LINEAR", 2),), "gemm"),
    Case("linear_f16w_gemm", linear(300, 96, 128, res=(300, 128)), (("LINEAR", 3),), "gemm", wdtype="float16"),
    Case("linear_f16w_gemv", linear(1, 256, 256, bias=False, res=(1, 256)), (("LINEAR", 2),), "gemm", wdtype="float16"),
    # a [1, N] residual broadcast over the rows: not an epilogue residual (the bias Add still is)
    Case("linear_broadcast_residual", linear(300, 96, 128, res=(1, 128)), (("LINEAR", 2),), "gemm"),
]


# ---------------------------------------------------------------------------------------------------------------- Conv + Add
def conv_add(C=32, H=12, res_slot=1, self_res=False, addend=None):
    def build(g):
        x = g.input("x", (1, C, H, H))
        wt = g.const(g.randn((C, C, 3, 3), std=1.0 / math.sqrt(9 * C)), conv_weight=True)
        c = g.node("Conv", [x, wt, g.const(g.randn((C,), std=0.25), quantizable=False)], [(1, C, H, H)],
                   [("dilations", "1,1"), ("group", "1"), ("kernel_shape", "3,3"), ("pads", "1,1,1,1"), ("strides", "1,1")], out_names=["conv_y"])
        gens = dict(x=_normal((1, C, H, H)))
        if self_res:
            r = x
        else:
            r = g.input("r", addend or (1, C, H, H))
            gens["r"] = _normal(addend or (1, C, H, H), mean=0.5)
        g.node("Add", [c, r] if res_slot == 1 else [r, c], [(1, C, H, H)], out_names=["y"])
        return Graph(["y"], _feeds(**gens), "conv_y")
    return build


CONV = []
for _nhwc in (0, 1):
    CONV += [
        Case(f"conv_add_res1_nhwc{_nhwc}", conv_add(), (("CONV_ADD", 2),), "gemm", b200=(("b200_keep_nhwc", _nhwc),), mid_fused_away=0),
        Case(f"conv_add_res0_nhwc{_nhwc}", conv_add(res_slot=0), (("CONV_ADD", 2),), "gemm", b200=(("b200_keep_nhwc", _nhwc),)),
        Case(f"conv_add_self_nhwc{_nhwc}", conv_add(self_res=True, res_slot=0), (("CONV_ADD", 2),), "gemm", b200=(("b200_keep_nhwc", _nhwc),)),
        Case(f"conv_add_channel_addend_nhwc{_nhwc}", conv_add(addend=(1, 32, 1, 1)), (), "gemm", b200=(("b200_keep_nhwc", _nhwc),)),
    ]


# ---------------------------------------------------------------------------------------------------------------- GroupNorm (5 / 7)
def groupnorm(C, G, H=8, eps=1e-5, tail=None, gs=1.0, gb=0.0):
    """Reshape, InstanceNormalization(scale gs, bias gb), Reshape, Mul(gamma), Add(beta) [+ Sigmoid, Mul]: tail "silu" (Mul(y, s)) or
    "sigmoid_first" (Mul(s, y))."""
    def build(g):
        x = g.input("x", (1, C, H, H))
        r = g.node("Reshape", [x, g.i64([0, G, -1])], [(1, G, C // G * H * H)])
        n = g.node("InstanceNormalization", [r, g.const(np.full(G, gs, np.float32), quantizable=False), g.const(np.full(G, gb, np.float32), quantizable=False)],
                   [r.shape], [("epsilon", repr(float(eps)))])
        r2 = g.node("Reshape", [n, g.i64([1, C, H, H])], [(1, C, H, H)])
        m = g.node("Mul", [r2, g.const(g.randn((C, 1, 1), std=0.25, mean=1.0))], [(1, C, H, H)])
        y = g.node("Add", [m, g.const(g.randn((C, 1, 1), std=0.25))], [(1, C, H, H)], out_names=None if tail else ["y"])
        if tail:
            s = g.node("Sigmoid", [y], [y.shape])
            g.node("Mul", [y, s] if tail == "silu" else [s, y], [y.shape], out_names=["y"])
        return Graph(["y"], _feeds(x=_normal((1, C, H, H), mean=0.5)))
    return build


GN = []
for _nhwc in (0, 1):
    _o = (("b200_keep_nhwc", _nhwc),)
    GN += [
        Case(f"gn_G8_nhwc{_nhwc}", groupnorm(64, 8), (("GROUPNORM", 5),), "norm", b200=_o),
        Case(f"gn_G32_eps1e-6_silu_nhwc{_nhwc}", groupnorm(128, 32, eps=1e-6, tail="silu"), (("GROUPNORM", 7),), "norm", b200=_o),
        Case(f"gn_G64_silu_nhwc{_nhwc}", groupnorm(256, 64, tail="silu"), (("GROUPNORM", 7),), "norm", b200=_o),
        Case(f"gn_G128_nhwc{_nhwc}", groupnorm(256, 128), (), "norm", b200=_o),
        Case(f"gn_instnorm_scale_fallback_nhwc{_nhwc}", groupnorm(64, 8, gs=1.5), (("GROUPNORM", 5),), "norm", fallback=True, b200=_o),
        Case(f"gn_instnorm_bias_fallback_nhwc{_nhwc}", groupnorm(64, 8, gb=0.25, tail="silu"), (("GROUPNORM", 7),), "norm", fallback=True, b200=_o),
        Case(f"gn_sigmoid_first_tail_nhwc{_nhwc}", groupnorm(64, 8, tail="sigmoid_first"), (("GROUPNORM", 5),), "norm", b200=_o),
    ]


# ---------------------------------------------------------------------------------------------------------------- attention (3 / 4)
def attention(h, T, Tk, d, scale=None, scale_slot=1, lead1=False):
    """MatMul(q, kt) [-> Mul(s, scale)] -> Softmax(-1) -> MatMul(p, v), with K pre-transposed: q [h, T, d], kt [h, d, Tk], v [h, Tk, d]
    (a leading 1 with lead1)."""
    pre = (1,) if lead1 else ()

    def build(g):
        q, kt, v = g.input("q", pre + (h, T, d)), g.input("kt", pre + (h, d, Tk)), g.input("v", pre + (h, Tk, d))
        s = g.node("MatMul", [q, kt], [pre + (h, T, Tk)], out_names=["att_s"])
        if scale is not None:
            c = g.scalar(scale)
            s = g.node("Mul", [s, c] if scale_slot == 1 else [c, s], [s.shape])
        p = g.node("Softmax", [s], [s.shape], [("axis", "-1")])
        g.node("MatMul", [p, v], [pre + (h, T, d)], out_names=["y"])
        return Graph(["y"], _feeds(q=_normal(q.shape), kt=_normal(kt.shape), v=_normal(v.shape)), "att_s")
    return build


ATT = [
    Case("att4_3d", attention(4, 40, 77, 64, scale=0.125), (("ATTENTION", 4),), "attention", mid_fused_away=0),
    Case("att3_3d", attention(2, 33, 40, 40), (("ATTENTION", 3),), "attention"),
    Case("att4_lead1_Tk77", attention(2, 64, 77, 40, scale=1 / math.sqrt(40), lead1=True), (("ATTENTION", 4),), "attention"),
    Case("att3_lead1", attention(2, 16, 24, 64, lead1=True), (("ATTENTION", 3),), "attention"),
    Case("att_scale_slot0", attention(2, 33, 40, 40, scale=0.125, scale_slot=0), (), "attention"),
]


# ---------------------------------------------------------------------------------------------------------------- multi-head attention (20)
def mha(T, heads, d, ctx=None, q_perm="0,2,1,3"):
    """The diffusers export of Attention without its output projection (emit.GraphBuilder.attention): bias-free q / k / v projections,
    the Reshape / Transpose / Reshape head split (K transposed), MatMul, Mul(1/sqrt d), Softmax, MatMul and the head merge.  ctx: (Tk, Cc)
    of a cross-attention context (None: self-attention on x).  q_perm: the perm of the query's head-split Transpose."""
    C = heads * d

    def build(g):
        x = g.input("x", (1, T, C))
        c = g.input("ctx", (1,) + ctx) if ctx else x
        Tk = c.shape[1]

        def split(t, tt, transpose_k=False, perm="0,2,1,3"):
            r = g.node("Reshape", [t, g.i64([1, tt, heads, d])], [(1, tt, heads, d)])
            p = g.node("Transpose", [r], [(1, heads, tt, d) if perm == "0,2,1,3" else (1, tt, heads, d)], [("perm", perm)])
            r2 = g.node("Reshape", [p, g.i64([heads, tt, d])], [(heads, tt, d)])
            return g.node("Transpose", [r2], [(heads, d, tt)], [("perm", "0,2,1")]) if transpose_k else r2
        w = lambda k: g.const(g.randn((k, C), std=1.0 / math.sqrt(k)))
        q = split(g.node("MatMul", [x, w(C)], [(1, T, C)]), T, perm=q_perm)
        k = split(g.node("MatMul", [c, w(c.shape[2])], [(1, Tk, C)]), Tk, transpose_k=True)
        v = split(g.node("MatMul", [c, w(c.shape[2])], [(1, Tk, C)]), Tk)
        s = g.node("MatMul", [q, k], [(heads, T, Tk)])
        s = g.node("Mul", [s, g.scalar(1.0 / math.sqrt(d))], [s.shape])
        p = g.node("Softmax", [s], [s.shape], [("axis", "-1")])
        o = g.node("MatMul", [p, v], [(heads, T, d)])
        o = g.node("Reshape", [o, g.i64([1, heads, T, d])], [(1, heads, T, d)])
        o = g.node("Transpose", [o], [(1, T, heads, d)], [("perm", "0,2,1,3")])
        g.node("Reshape", [o, g.i64([1, T, C])], [(1, T, C)], out_names=["y"])
        gens = dict(x=_normal((1, T, C)))
        if ctx:
            gens["ctx"] = _normal((1,) + ctx)
        return Graph(["y"], _feeds(**gens))
    return build


# fp16 with T < 64 takes the padded-GEMM route of fused_mha, T >= 64 the flash kernel; fp32 takes the f32x flash kernel
MHA = [
    Case("mha_self_d40_T16", mha(16, 2, 40), (("MHA", 20),), "attention"),
    Case("mha_self_d64_T64", mha(64, 2, 64), (("MHA", 20),), "attention"),
    Case("mha_cross_d40_T64_Tk77", mha(64, 2, 40, ctx=(77, 48)), (("MHA", 20),), "attention"),
    Case("mha_cross_d64_T16_Tk77", mha(16, 2, 64, ctx=(77, 48)), (("MHA", 20),), "attention"),
    # not the head split: the projections and reshapes run by themselves, the attention core is still the 4-op group
    Case("mha_query_perm_identity", mha(16, 2, 40, q_perm="0,1,2,3"), (("ATTENTION", 4),), "attention"),
]


# ---------------------------------------------------------------------------------------------------------------- SDPA (6)
def sdpa(Hq, Hkv, Tq, Tk, D, mask4=False):
    """Transpose(K, 0,1,3,2), MatMul(q, kt), Div(s), Add(mask), Softmax(-1), MatMul(p, v) -- the chain the reference rewrites into
    ScaledDotProductAttention under use_scaled_dp_attn_op.  Neither Planner::sdpa nor the reference's rewrite checks the Transpose's perm,
    so only 0,1,3,2 is spelled here."""
    mshape = (1, 1, Tq, Tk) if mask4 else (Tq, Tk)

    def build(g):
        q, k, v = g.input("q", (1, Hq, Tq, D)), g.input("k", (1, Hkv, Tk, D)), g.input("v", (1, Hkv, Tk, D))
        m = g.input("mask", mshape)
        kt = g.node("Transpose", [k], [(1, Hkv, D, Tk)], [("perm", "0,1,3,2")])
        s = g.node("MatMul", [q, kt], [(1, Hq, Tq, Tk)])
        s = g.node("Div", [s, g.scalar(math.sqrt(D))], [s.shape])
        s = g.node("Add", [s, m], [s.shape])
        p = g.node("Softmax", [s], [s.shape], [("axis", "-1")])
        g.node("MatMul", [p, v], [(1, Hq, Tq, D)], out_names=["y"])

        def mask(r):
            keep = (np.arange(Tk)[None, :] <= (Tk - Tq) + np.arange(Tq)[:, None]) & (r.random((Tq, Tk)) > 0.1)
            keep[:, 0] = True
            return np.where(keep, 0.0, -65504.0).astype(np.float32).reshape(mshape)
        return Graph(["y"], _feeds(q=_normal(q.shape), k=_normal(k.shape), v=_normal(v.shape), mask=mask))
    return build


SDPA = [
    Case("sdpa_Tq1_grouped", sdpa(4, 2, 1, 40, 64), (("SDPA", 6),), "attention", sdpa=True, unfused_sdpa=False),
    Case("sdpa_Tq33_grouped", sdpa(4, 2, 33, 57, 64), (("SDPA", 6),), "attention", sdpa=True, unfused_sdpa=False),
    Case("sdpa_Tq33_mask4", sdpa(2, 2, 33, 40, 32, mask4=True), (("SDPA", 6),), "attention", sdpa=True),
    Case("sdpa_Tq1_mask4", sdpa(2, 2, 1, 40, 32, mask4=True), (("SDPA", 6),), "attention", sdpa=True),
]


# ---------------------------------------------------------------------------------------------------------------- grouped GEMV / SwiGLU
def gemv(rows, n, K=64, N=256, trailing_add=False, mixed=False):
    """n MatMuls of one activation x [rows, K] (q / k / v projections); trailing_add: an Add of a bias after the last one."""
    def build(g):
        x = g.input("x", (rows, K))
        outs = []
        for k in range(n):
            w = g.const(g.randn((K, N), std=1.0 / math.sqrt(K)), force_dtype="float32" if (mixed and k == n - 1) else None)
            y = g.node("MatMul", [x, w], [(rows, N)], out_names=[f"y{k}"] if not (trailing_add and k == n - 1) else None)
            if trailing_add and k == n - 1:
                g.node("Add", [y, g.const(g.randn((N,), std=0.25), force_dtype="float32")], [(rows, N)], out_names=[f"y{k}"])
            outs.append(f"y{k}")
        return Graph(outs, _feeds(x=_normal((rows, K))))
    return build


def swiglu(rows, K=64, N=256, silu_slot=0, gate_slot=0):
    """MatMul(x, Wg) -> Sigmoid -> Mul(g, s) -> MatMul(x, Wu) -> Mul(silu, u); *_slot 1 swaps the operands of that Mul."""
    def build(g):
        x = g.input("x", (rows, K))
        gt = g.node("MatMul", [x, g.const(g.randn((K, N), std=1.0 / math.sqrt(K)))], [(rows, N)])
        s = g.node("Sigmoid", [gt], [(rows, N)])
        sl = g.node("Mul", [gt, s] if silu_slot == 0 else [s, gt], [(rows, N)])
        up = g.node("MatMul", [x, g.const(g.randn((K, N), std=1.0 / math.sqrt(K)))], [(rows, N)])
        g.node("Mul", [sl, up] if gate_slot == 0 else [up, sl], [(rows, N)], out_names=["y"])
        return Graph(["y"], _feeds(x=_normal((rows, K), std=2.0)))
    return build


GEMV = [
    Case("gemv2_rows8", gemv(8, 2), (("GEMV_GROUP", 2),), "gemm"),
    Case("gemv3_rows1", gemv(1, 3), (("GEMV_GROUP", 3),), "gemm"),
    Case("gemv3_trailing_add", gemv(2, 3, trailing_add=True), (("GEMV_GROUP", 2), ("LINEAR", 2)), "gemm"),
    Case("gemv3_u8", gemv(1, 3), (("GEMV_GROUP", 3),), "gemm", wdtype="uint8"),
    Case("gemv2_u8_rows8", gemv(8, 2), (("GEMV_GROUP", 2),), "gemm", wdtype="uint8"),
    Case("gemv3_f16w", gemv(4, 3), (("GEMV_GROUP", 3),), "gemm", wdtype="float16"),
    Case("gemv_rows9", gemv(9, 3), (), "gemm"),
    # two uint8 MatMuls then a float one: the first two still group
    Case("gemv_mixed_u8_float", gemv(1, 3, mixed=True), (("GEMV_GROUP", 2),), "gemm", wdtype="uint8"),
    Case("gemv_mixed_u8_float_pair", gemv(1, 2, mixed=True), (), "gemm", wdtype="uint8"),
    Case("swiglu_00", swiglu(1), (("SWIGLU", 5),), "gemm"),
    Case("swiglu_11", swiglu(4, silu_slot=1, gate_slot=1), (("SWIGLU", 5),), "gemm"),
    Case("swiglu_10_u8", swiglu(1, silu_slot=1), (("SWIGLU", 5),), "gemm", wdtype="uint8"),
    Case("swiglu_01_f16w", swiglu(8, gate_slot=1), (("SWIGLU", 5),), "gemm", wdtype="float16"),
    # rows 9: no grouped GEMV; the SiLU is still its own group
    Case("swiglu_rows9", swiglu(9), (("SILU", 2),), "gemm"),
]

CASES = LN + RMS + ROPE + GELU + GEGLU + SILU + LINEAR + CONV + GN + ATT + MHA + SDPA + GEMV
IDS = [c.id for c in CASES]
assert len(set(IDS)) == len(IDS)


# ---------------------------------------------------------------------------------------------------------------- runners
def _emit(case, d):
    g = emit.GraphBuilder(d, case.wdtype, seed=len(case.id))
    spec = case.build(g)
    g.finish()
    return spec


def _fused_steps(text, fp16, sdpa, lib):
    rep = plan_summary(text, fp16_arithmetic=fp16, use_scaled_dp_attn_op=sdpa, library_path=lib)
    steps = [l.split(" ") for l in rep.splitlines() if l and not l.startswith("#")]
    return tuple((s[0], int(s[1])) for s in steps if s[0] != "SINGLE")


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_plan(engine_lib, case, tmp_path):
    """The planner (host code, no GPU) claims exactly the expected groups, in fp32 and fp16 arithmetic alike."""
    d = str(tmp_path) + "/"
    _emit(case, d)
    text = open(d + "model.txt").read()
    for fp16 in (False, True):
        got = _fused_steps(text, fp16, case.sdpa, engine_lib)
        assert got == case.plan, (case.id, "fp16" if fp16 else "fp32", got)


@pytest.fixture(scope="module")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _engine(lib, d, feeds, names, fp16, fuse, case, extra=(), upcast=None, sdpa=None):
    """Run the model once per input set on one Model; returns the named tensors of each run and ops_fused_away."""
    m = Model(lib, 4, "nocache")
    try:
        if fp16:
            m.set_option("use_fp16_arithmetic", True)
        if case.sdpa if sdpa is None else sdpa:
            m.set_option("use_scaled_dp_attn_op", True)
        m.lib.model_set_option(m.h, b"b200_fuse_nodes", int(fuse))
        for k, v in case.b200:
            m.lib.model_set_option(m.h, k.encode(), int(v))
        if upcast:
            m.add_upcast_pattern(upcast)
        for e in extra:
            m.add_extra_output(e)
        m.read_file(d + "model.txt")
        runs = []
        for f in feeds:
            m.clear_tensors()
            for k, v in f.items():
                m.add_tensor(k, v)
            m.run()
            runs.append({n: np.array(m.get_tensor(n), np.float64) for n in names})
        return runs, int(m.stats()["ops_fused_away"])
    finally:
        m.close()


def _err(got, ref):
    d = np.abs(got - ref)
    scale = max(float(np.abs(ref).max()), 1e-30)
    return float(d.max()) / scale, float(np.sqrt((d ** 2).mean())), float(np.sqrt((ref ** 2).mean()))


def _within(got, ref, bar, what):
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    rel, rms, _ = _err(got, ref)
    assert rel <= bar, f"{what}: max|err| / max|ref| = {rel:.3e} > {bar:.1e}"
    return rms


def _run_numbers(lib, tmp_path, case, mode, fused_bar=None, extra=(), upcast=None):
    d = str(tmp_path) + "/"
    spec = _emit(case, d)
    fp16 = mode == "f16"
    bar = BARS[case.bar][1 if fp16 else 0]
    feeds = [spec.inputs(np.random.default_rng(s)) for s in (1, 2)]
    names = list(spec.outs) + list(extra)
    oracle = NumpyOracle(d, fp16=False)
    refs = [oracle.run(f, extra_outputs=extra) for f in feeds]
    fused, fused_away = _engine(lib, d, feeds, names, fp16, 1, case, extra, upcast)
    unfused_sdpa = case.sdpa and not case.unfused_sdpa
    plain, _ = _engine(lib, d, feeds, names, fp16, 0, case, extra, upcast, sdpa=unfused_sdpa if case.sdpa else None)
    for r in range(len(feeds)):
        for n in names:
            ref = np.asarray(refs[r][n], np.float64)
            what = f"{case.id} {mode} run {r + 1} {n}"
            e_fused = _within(fused[r][n], ref, fused_bar or bar, what + " fused")
            e_plain = _within(plain[r][n], ref, bar, what + " op by op")
            if case.fallback or (case.bit_equal_f32 and not fp16):
                assert np.array_equal(fused[r][n], plain[r][n]), f"{what}: the fused step is not bit-identical to the op-by-op run " \
                    f"(max |diff| {np.abs(fused[r][n] - plain[r][n]).max():.3e})"
            elif fp16:
                ref_rms = _err(ref, ref)[2]
                assert e_fused <= SLACK * e_plain + FLOOR * ref_rms, f"{what}: fused rms err {e_fused:.3e} > {SLACK} x op-by-op {e_plain:.3e} + floor"
    return fused_away


def _ops_fused_away(case):
    return sum(n - 1 for _, n in case.plan)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f32", "f16"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_numbers(engine_lib, cuda, case, mode, tmp_path):
    """fuse_nodes 1 and 0 against the fp64 oracle on two input sets (one Model); fallback rows bit-identical to the op-by-op run."""
    if mode not in case.modes:
        pytest.skip(f"{case.id}: {mode} is not meaningful for this row")
    upcast = case.upcast[0] if case.upcast and mode == "f16" else None
    fused_away = _run_numbers(engine_lib, tmp_path, case, mode, upcast=upcast)
    want = case.upcast[1] if upcast else _ops_fused_away(case)
    assert fused_away == want, f"{case.id} {mode}: {fused_away} ops in planned groups, expected {want}"


MID_CASES = [c for c in CASES if c.mid_fused_away is not None]


@pytest.mark.gpu
@pytest.mark.parametrize("case", MID_CASES, ids=[c.id for c in MID_CASES])
def test_intermediate(engine_lib, cuda, case, tmp_path):
    """An intermediate of the group requested as an extra output: the planner leaves the group (or its part that would hide the
    intermediate) alone, and the intermediate and the output both match the oracle, in fp32 and fp16 arithmetic."""
    g = emit.GraphBuilder(None, case.wdtype, seed=len(case.id))
    mid = case.build(g).mid
    assert mid
    for mode in case.modes:
        fused_away = _run_numbers(engine_lib, tmp_path / mode, case, mode, extra=(mid,))
        assert fused_away == case.mid_fused_away, f"{case.id} {mode}: {fused_away} ops in planned groups with {mid} requested"
