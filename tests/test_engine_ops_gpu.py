"""The engine's single-op layout, shape and index handlers (engine_run.cpp: op_reshape_like ... op_misc_host), one tiny graph per
spelling, against the fp64 op-by-op oracle (oracle/np_oracle.py: NumpyOracle).

These handlers decide the output shape, view or copy, the strides and offsets of the copy, whether a channel-last (NHWC) input stays
channel-last, and which scale a uint8 result carries, before any kernel runs.  Each row builds only the op under test, written with
GraphBuilder.node, and feeds it from two producers:

  plain     a graph input;
  nhwc      a 1x1 or 3x3 Conv of a graph input with b200_keep_nhwc 1 (rows whose source is 4-D with batch 1), requested as an extra
            output so the test sees the exact values the op consumed.

and asserts, in fp32 arithmetic, use_fp16_arithmetic and (ops of op_takes_u8) use_uint8_arithmetic:

  exact     the engine's output equals the oracle's op applied to the producer's own output, bit for bit: the producer values are the
            fp32 input, its fp16 rounding, its uint8 quantisation by the percentile rule at the engine's 4 threads (dequantised), or
            the Conv output the engine returned.  A uint8 result the engine re-quantises (Concat of sources with different scales) is
            the same rule applied to the float result, and within one output step of it;
  bar       the whole row (producer included) within an fp32 / fp16 bar of the fp64 oracle, so a wrong producer cannot hide;
  arithmetic  Softmax and ReduceMean within a bar of fp64 instead of bit-exact; a non-last-axis Softmax equals the last-axis Softmax
            of the transposed input bit for bit.

Every row runs twice on one Model with new inputs the second time.  Rows whose index or shape input is a graph input also run four
times with resident weights and CUDA graphs: outputs must follow the new values whether the graph replays (Gather indices) or capture
falls back to eager runs (host-evaluated Where, Trilu, Cast float -> int).  REFUSALS must raise OnnxStreamError, never return numbers."""
import os
import sys
from dataclasses import dataclass
from typing import Callable, Dict, List, Tuple

import numpy as np
import pytest

from onnxstream_b200 import emit
from onnxstream_b200.model import Model, OnnxStreamError

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
from np_oracle import NumpyOracle, qu8_dequantize, qu8_percentiles, qu8_quantize, qu8_range_to_scale  # noqa: E402

I64_MAX = np.iinfo(np.int64).max
THREADS = 4     # the engine's (and the reference's) percentile chunking follows the Model's thread count

# Bars, as max |engine - fp64| / max |fp64|, of a whole row (producer included): (fp32 arithmetic, fp16 arithmetic).  Movement: a plain
# producer is exact in fp32 and rounded once to fp16 (2^-11); the Conv producer adds its fp32 tensor-core (bf16 triple split) or fp16
# error over K <= 9 x 9 unit-variance terms.  Softmax: the logits' absolute error (of the order of the bar times max|x| ~ 4) moves the
# probabilities by as much relative to themselves.  ReduceMean: a mean of up to 33 terms, of the order of a third of max|x|.
# Truncation to int64 has no bar against fp64 in fp16: a value rounded to fp16 across an integer truncates one unit lower or higher.
BARS = {"move": (1e-5, 5e-3), "trunc": (1e-5, None), "softmax": (1e-4, 2e-2), "reduce": (1e-4, 1e-2)}
U8_SOFTMAX_STEPS = 2.5      # uint8 Softmax (output scale 2^-8) against fp64 on the same dequantised input, in output steps


@dataclass
class Spec:
    outs: List[str]
    feeds: Callable[[np.random.Generator], Dict[str, np.ndarray]]
    equal: Tuple[Tuple[str, str], ...] = ()     # output pairs that must be bit-identical


@dataclass
class Row:
    id: str
    build: Callable                      # build(g, src) -> Spec; src(name, shape) is the producer of a float source
    kind: str = "move"                   # "move" (exact), "trunc" (exact on the producer's values only), "softmax", "reduce"
    modes: Tuple[str, ...] = ("f32", "f16", "u8")
    nhwc: int = 0                        # kernel size of the NHWC Conv producer (0: 4-D batch-1 sources absent, plain only)
    graph: bool = False                  # an index / shape / mask input is a graph input: also the CUDA-graph runs
    replays: bool = False                # ... and the captured graph must replay (device-mirror indices)
    requant_u8: bool = False             # uint8: the result is re-quantised (sources with different scales)
    dynamic: bool = False                # support_dynamic_shapes: the model text declares a zero-length source


def _normal(shape, mean=0.0, std=1.0):
    return lambda r: (r.standard_normal(shape) * std + mean).astype(np.float32)


def _eighths(shape):
    """Small multiples of 1/8: exact in fp16, so an fp16-arithmetic binary op on them rounds like fp64 then fp16."""
    return lambda r: (np.round(r.standard_normal(shape) * 8) / 8).astype(np.float32)


def _feeds(**gens):
    return lambda r: {k: f(r) for k, f in gens.items()}


def _const_eighths(g, shape):
    return g.const((np.round(g.randn(shape) * 8) / 8).astype(np.float32), quantizable=False)


# ---------------------------------------------------------------------------------------------------------------- row builders
def unary(op, shape, out_shape, ins=(), attrs=None, gen=None):
    """op(src x [, constant int64 inputs]) -> y."""
    def build(g, src):
        x = src("x", shape)
        g.node(op, [x] + [g.i64(v) if v is not None else None for v in ins], [out_shape], attrs, out_names=["y"])
        return Spec(["y"], _feeds(x=gen or _normal(shape)))
    return build


def concat(shapes, axis, names=None, gens=None):
    """Concat of sources `names` (default x0, x1, ...; a name given twice is one source read twice) of the given shapes."""
    names = names or [f"x{k}" for k in range(len(shapes))]

    def build(g, src):
        made = {}
        for n, s in zip(names, shapes):
            if n not in made:
                made[n] = src(n, s)
        xs = [made[n] for n in names]
        ax = axis % len(shapes[0])
        out = list(shapes[0]); out[ax] = sum(s[ax] for s in shapes)
        g.node("Concat", xs, [tuple(out)], [("axis", str(axis))], out_names=["y"])
        first = {n: k for k, n in reversed(list(enumerate(names)))}
        return Spec(["y"], _feeds(**{n: (gens[k] if gens else _normal(shapes[k])) for n, k in first.items()}))
    return build


def split(shape, axis, sizes, explicit):
    def build(g, src):
        x = src("x", shape)
        outs = []
        for k, s in enumerate(sizes):
            o = list(shape); o[axis] = s; outs.append(tuple(o))
        names = [f"y{k}" for k in range(len(sizes))]
        g.node("Split", [x, g.i64(sizes)] if explicit else [x], outs, [("axis", str(axis))], out_names=names)
        return Spec(names, _feeds(x=_normal(shape)))
    return build


def slice_(shape, starts, ends, axes):
    def build(g, src):
        x = src("x", shape)
        out = list(shape)
        for s, e, a in zip(starts, ends, axes):
            n = shape[a]
            s = min(max(s + n if s < 0 else s, 0), n)
            e = min(max(e + n if e < 0 else e, 0), n)
            out[a] = max(e - s, 0)
        g.node("Slice", [x, g.i64(starts), g.i64(ends), g.i64(axes), g.i64([1] * len(axes))], [tuple(out)], out_names=["y"])
        return Spec(["y"], _feeds(x=_normal(shape)))
    return build


def resize(shape, sy, sx, by_sizes):
    """Nearest / asymmetric / floor.  By sizes, the scales input is given too (with the same values) for the oracle, which reads scales;
    the engine takes sizes whenever the fourth input is present."""
    def build(g, src):
        x = src("x", shape)
        out = (shape[0], shape[1], shape[2] * sy, shape[3] * sx)
        sc = g.const(np.array([1, 1, sy, sx], np.float32), quantizable=False)
        ins = [x, None, sc] + ([g.i64(out)] if by_sizes else [])
        g.node("Resize", ins, [out], [("coordinate_transformation_mode", "asymmetric"), ("mode", "nearest"), ("nearest_mode", "floor")],
               out_names=["y"])
        return Spec(["y"], _feeds(x=_normal(shape)))
    return build


def softmax(shape, axis):
    """Softmax(x, axis) beside Transpose(axis last) -> Softmax(-1) -> Transpose back: the two must agree bit for bit."""
    def build(g, src):
        x = src("x", shape)
        nd = len(shape)
        ax = axis % nd
        perm = [i for i in range(nd) if i != ax] + [ax]
        inv = list(np.argsort(perm))
        g.node("Softmax", [x], [shape], [("axis", str(axis))], out_names=["y"])
        t = g.node("Transpose", [x], [tuple(shape[p] for p in perm)], [("perm", ",".join(map(str, perm)))])
        s = g.node("Softmax", [t], [t.shape], [("axis", "-1")])
        g.node("Transpose", [s], [shape], [("perm", ",".join(map(str, inv)))], out_names=["yt"])
        return Spec(["y", "yt"], _feeds(x=_normal(shape, std=2.0)), equal=(("y", "yt"),))
    return build


def reduce_mean(shape, axes, keepdims):
    def build(g, src):
        x = src("x", shape)
        out = list(shape)
        if keepdims: out[-1] = 1
        else: out.pop()
        g.node("ReduceMean", [x], [tuple(out)], [("axes", axes), ("keepdims", str(keepdims))], out_names=["y"])
        return Spec(["y"], _feeds(x=_normal(shape, mean=0.5)))
    return build


def gather(shape, idx_shape, idx, graph_idx):
    """Gather(data, indices) on axis 0; indices a constant (host-index path) or an int64 graph input (device-mirror path) drawn from
    [-rows, rows), negatives included."""
    rows = shape[0]

    def build(g, src):
        x = src("x", shape)
        i = g.input("idx", idx_shape) if graph_idx else g.i64(np.asarray(idx, np.int64).reshape(idx_shape))
        g.node("Gather", [x, i], [tuple(idx_shape) + tuple(shape[1:])], [("axis", "0")], out_names=["y"])
        gens = dict(x=_normal(shape))
        if graph_idx:
            gens["idx"] = lambda r: r.integers(-rows, rows, idx_shape).astype(np.int64)
        return Spec(["y"], _feeds(**gens))
    return build


def expand(shape, target, i64=False):
    def build(g, src):
        out = tuple(np.broadcast_shapes(shape, tuple(target)))
        if i64:
            x = g.input("xi", shape)
            g.node("Expand", [x, g.i64(target)], [out], out_names=["y"])
            return Spec(["y"], _feeds(xi=lambda r: r.integers(-50, 50, shape).astype(np.int64)))
        x = src("x", shape)
        g.node("Expand", [x, g.i64(target)], [out], out_names=["y"])
        return Spec(["y"], _feeds(x=_normal(shape)))
    return build


def binary_per_channel(op, shape, cshape, const_slot):
    """op(x, per-channel constant): the NHWC per-channel path of Impl::binary when x is channel-last."""
    def build(g, src):
        x = src("x", shape)
        c = _const_eighths(g, cshape)
        g.node(op, [x, c] if const_slot == 1 else [c, x], [shape], out_names=["y"])
        return Spec(["y"], _feeds(x=_eighths(shape)))
    return build


def maxpool(shape, k, pad, stride):
    def build(g, src):
        x = src("x", shape)
        ho, wo = (shape[2] + 2 * pad - k) // stride + 1, (shape[3] + 2 * pad - k) // stride + 1
        g.node("MaxPool", [x], [(1, shape[1], ho, wo)], [("ceil_mode", "0"), ("dilations", "1,1"), ("kernel_shape", f"{k},{k}"),
                                                          ("pads", f"{pad},{pad},{pad},{pad}"), ("strides", f"{stride},{stride}")], out_names=["y"])
        return Spec(["y"], _feeds(x=_normal(shape)))
    return build


def where(cshape, xshape, yshape, scalar=None):
    """Where(cond, x, y): cond an int64 graph input; x a float source; y a float graph input of yshape, or the scalar constant `scalar`."""
    def build(g, src):
        c = g.input("cond", cshape)
        x = src("x", xshape)
        y = g.scalar(scalar) if scalar is not None else g.input("z", yshape)
        out = tuple(np.broadcast_shapes(cshape, xshape, () if scalar is not None else yshape))
        g.node("Where", [c, x, y], [out], out_names=["y"])
        gens = dict(cond=lambda r: (r.random(cshape) > 0.4).astype(np.int64), x=_normal(xshape))
        if scalar is None:
            gens["z"] = _normal(yshape, mean=5.0)
        return Spec(["y"], _feeds(**gens))
    return build


def compare(op, ashape, bshape, b_const=False):
    """op(a, b) on int64 graph inputs (b a constant with b_const) -> int64 0 / 1, numpy broadcasting."""
    def build(g, src):
        a = g.input("ai", ashape)
        b = g.i64(np.arange(-2, -2 + int(np.prod(bshape)), dtype=np.int64).reshape(bshape)) if b_const else g.input("bi", bshape)
        g.node(op, [a, b], [tuple(np.broadcast_shapes(ashape, bshape))], out_names=["y"])
        gens = dict(ai=lambda r: r.integers(-2, 3, ashape).astype(np.int64))
        if not b_const:
            gens["bi"] = lambda r: r.integers(-2, 3, bshape).astype(np.int64)
        return Spec(["y"], _feeds(**gens))
    return build


def where_i64(cshape, xshape, yshape, y_scalar=None):
    """Where(cond, x, y) with int64 branches: x an int64 graph input, y one too or the scalar constant y_scalar."""
    def build(g, src):
        c, x = g.input("cond", cshape), g.input("xi", xshape)
        y = g.i64(np.asarray(y_scalar, np.int64)) if y_scalar is not None else g.input("yi", yshape)
        g.node("Where", [c, x, y], [tuple(np.broadcast_shapes(cshape, xshape, () if y_scalar is not None else yshape))], out_names=["y"])
        gens = dict(cond=lambda r: (r.random(cshape) > 0.4).astype(np.int64), xi=lambda r: r.integers(-50, 50, xshape).astype(np.int64))
        if y_scalar is None:
            gens["yi"] = lambda r: r.integers(100, 150, yshape).astype(np.int64)
        return Spec(["y"], _feeds(**gens))
    return build


def trilu(shape, k):
    """Upper triangle of a float graph input (read on the host) with a constant scalar k."""
    def build(g, src):
        x = src("x", shape)
        g.node("Trilu", [x, g.i64(np.asarray(k, np.int64))], [shape], [("upper", "1")], out_names=["y"])
        return Spec(["y"], _feeds(x=_normal(shape)))
    return build


def cast_f2i(shape):
    """Cast float -> int64 (truncation toward zero, negatives included) -> float."""
    def build(g, src):
        x = src("x", shape)
        i = g.node("Cast", [x], [shape], [("to", "7")])
        g.node("Cast", [i], [shape], [("to", "1")], out_names=["y"])
        return Spec(["y"], _feeds(x=_normal(shape, std=6.0)))
    return build


ROWS = [
    # Reshape / Unsqueeze / Squeeze / Flatten: zero-copy relabels of the plain layout (an NHWC source goes through to_plain first)
    Row("reshape_0_neg1", unary("Reshape", (1, 7, 9, 11), (1, 63, 11), ins=([0, -1, 11],)), nhwc=1),
    Row("reshape_neg1_lead", unary("Reshape", (1, 7, 9, 11), (77, 9), ins=([-1, 9],)), nhwc=3),
    Row("unsqueeze_neg_axes", unary("Unsqueeze", (7, 33), (1, 7, 33, 1), ins=([-1, 0],))),
    Row("squeeze_neg_axis", unary("Squeeze", (1, 7, 1, 9), (1, 7, 9), ins=([-2],)), nhwc=1),
    Row("squeeze_all_units", unary("Squeeze", (1, 7, 1, 9), (7, 9)), nhwc=1),
    Row("flatten_axis2", unary("Flatten", (1, 5, 7, 9), (5, 63), attrs=[("axis", "2")]), nhwc=3),
    Row("flatten_axis_neg1", unary("Flatten", (1, 5, 7, 9), (35, 9), attrs=[("axis", "-1")]), nhwc=1),
    # Transpose: the channel-last relabels, the unit-axis view, the batched 2-D kernel (and its strided fallback above 65535), the
    # general strided copy
    Row("transpose_0231", unary("Transpose", (1, 5, 7, 9), (1, 7, 9, 5), attrs=[("perm", "0,2,3,1")]), nhwc=1),
    Row("transpose_0312", unary("Transpose", (1, 7, 9, 5), (1, 5, 7, 9), attrs=[("perm", "0,3,1,2")]), nhwc=3),
    Row("transpose_unit_axes_view", unary("Transpose", (1, 1, 7, 33), (1, 7, 1, 33), attrs=[("perm", "0,2,1,3")]), nhwc=1),
    Row("transpose_unit_axes_moved", unary("Transpose", (1, 7, 1, 33), (33, 1, 1, 7), attrs=[("perm", "3,0,2,1")]), nhwc=1),
    Row("transpose_last2_batched", unary("Transpose", (3, 7, 33), (3, 33, 7), attrs=[("perm", "0,2,1")])),
    Row("transpose_last2_batch_65537", unary("Transpose", (65537, 2, 3), (65537, 3, 2), attrs=[("perm", "0,2,1")])),
    Row("transpose_general_4d", unary("Transpose", (3, 5, 7, 9), (9, 5, 3, 7), attrs=[("perm", "3,1,0,2")])),
    Row("transpose_0213_nchw", unary("Transpose", (1, 5, 7, 9), (1, 7, 5, 9), attrs=[("perm", "0,2,1,3")]), nhwc=3),
    # Concat: the NHWC channel path, osb_concat2 and its strided fallback (parts not 16-byte granular), three sources, and uint8 sources
    # with one or with different scales.  (A zero-length source cannot be declared in model text: dimension 0 is refused by the parser.)
    Row("concat_channels", concat([(1, 5, 7, 9), (1, 3, 7, 9)], 1), nhwc=1, requant_u8=True),
    Row("concat_axis_neg1_odd", concat([(3, 7, 5), (3, 7, 3)], -1), requant_u8=True),
    Row("concat_axis1_granular", concat([(2, 8, 33), (2, 4, 33)], 1), requant_u8=True),
    Row("concat_three", concat([(7, 3), (7, 5), (7, 1)], 1), requant_u8=True),
    Row("concat_same_source", concat([(1, 5, 7, 9), (1, 5, 7, 9)], 3, names=["x0", "x0"]), nhwc=1),
    # a zero-length source (the first turn's KV cache, declared with support_dynamic_shapes): the empty-source shortcut with the empty
    # source first and second, and three sources with one empty; under uint8 the empty source stays float (it has no range), and only
    # the non-empty sources decide whether the bytes are copied (one source read twice: one scale) or re-quantised
    Row("concat_empty_first", concat([(1, 2, 0, 9), (1, 2, 7, 9)], 2), dynamic=True),
    Row("concat_empty_second", concat([(1, 2, 7, 9), (1, 2, 0, 9)], -2), dynamic=True),
    Row("concat_three_empty_middle", concat([(7, 3), (7, 0), (7, 5)], 1), dynamic=True, requant_u8=True),
    Row("concat_three_empty_first_one_scale", concat([(0, 33), (3, 33), (3, 33)], 0, names=["e", "x0", "x0"]), dynamic=True),
    Row("concat_u8_scales_differ", concat([(7, 33), (7, 33)], 0, gens=[_normal((7, 33)), _normal((7, 33), mean=3.0, std=8.0)]), requant_u8=True),
    # Split with default and explicit sizes
    Row("split_default_3", split((1, 9, 7, 5), 1, [3, 3, 3], explicit=False), nhwc=1),
    Row("split_sizes_neg_axis", split((1, 7, 9, 11), -1, [2, 4, 5], explicit=True), nhwc=3),
    Row("split_sizes_axis0", split((7, 33), 0, [1, 6], explicit=True)),
    # Slice: negative starts and ends, clamped ends (INT64_MAX included), several negative axes
    Row("slice_neg_start_end", slice_((1, 7, 9, 33), [-5], [-1], [3]), nhwc=1),
    Row("slice_end_int64_max", slice_((1, 7, 9, 33), [2], [I64_MAX], [1]), nhwc=3),
    Row("slice_clamped", slice_((1, 7, 9, 33), [-100], [100], [-2]), nhwc=1),
    Row("slice_neg_axes", slice_((1, 7, 9, 33), [1, -6, 2], [-1, I64_MAX, 7], [-3, -1, -2]), nhwc=1),
    Row("slice_3d", slice_((7, 9, 33), [3], [8], [1])),
    # Resize by scales and by sizes, unequal row and column factors
    Row("resize_scales_2x3", resize((1, 5, 7, 9), 2, 3, by_sizes=False), nhwc=1),
    Row("resize_sizes_3x2", resize((1, 5, 7, 9), 3, 2, by_sizes=True), nhwc=3),
    # Softmax on a non-last axis (the transposing path), float and uint8
    Row("softmax_axis1", softmax((1, 7, 9, 11), 1), kind="softmax", nhwc=1),
    Row("softmax_axis0_3d", softmax((7, 5, 33), 0), kind="softmax"),
    Row("softmax_axis_neg2", softmax((3, 33, 7), -2), kind="softmax"),
    # Gather on axis 0 with negative indices: constant indices (host path) and an int64 graph input (device mirror)
    Row("gather_const_idx", gather((33, 7), (2, 3), [[3, -1, 0], [-33, 32, 5]], graph_idx=False)),
    Row("gather_input_idx", gather((33, 7, 5), (5,), None, graph_idx=True), graph=True, replays=True),
    # Expand: stride-0 broadcast dimensions collapsed by strided(); fp32 / fp16 / uint8 data, and int64 on the host
    Row("expand_lead_and_inner", expand((7, 1, 9), [2, 7, 11, 9])),
    Row("expand_rank_up", expand((1, 33), [7, 1, 33])),
    Row("expand_i64", expand((3, 1), [3, 5], i64=True), modes=("f32",)),
    # ReduceMean over the last axis, keepdims 1 and 0
    Row("reducemean_keep1", reduce_mean((7, 33), "-1", 1), kind="reduce", modes=("f32", "f16")),
    Row("reducemean_keep0", reduce_mean((1, 5, 7, 9), "3", 0), kind="reduce", modes=("f32", "f16"), nhwc=1),
    # Cast float -> int64 truncates toward zero, negatives included
    Row("cast_float_to_int", cast_f2i((7, 9)), kind="trunc", modes=("f32", "f16"), graph=True),
    # Where with a broadcast condition (the [1, 1, T, T] causal mask against [1, H, T, T]), a scalar branch, and all three broadcasting
    Row("where_causal_mask_scalar", where((1, 1, 7, 7), (1, 3, 7, 7), None, scalar=-1e4), modes=("f32", "f16"), nhwc=1, graph=True),
    Row("where_all_broadcast", where((3, 1), (1, 5), (3, 5)), modes=("f32", "f16"), graph=True),
    # Where with int64 branches: a broadcast (causal) condition, and a scalar branch broadcast against both others
    Row("where_i64_causal_mask", where_i64((1, 1, 4, 4), (1, 3, 4, 4), (1, 3, 4, 4)), modes=("f32", "f16")),
    Row("where_i64_scalar_branch", where_i64((3, 1), (1, 5), None, y_scalar=-7), modes=("f32", "f16")),
    Row("trilu_k1", trilu((7, 9), 1), modes=("f32", "f16"), graph=True),
    Row("trilu_k_neg2", trilu((9, 7), -2), modes=("f32", "f16"), graph=True),
    # the NHWC per-channel paths of the binary ops, and MaxPool (channel-last by construction)
    Row("add_per_channel_c11", binary_per_channel("Add", (1, 5, 7, 9), (5, 1, 1), 1), modes=("f32", "f16"), nhwc=1),
    Row("mul_per_channel_1c11_slot0", binary_per_channel("Mul", (1, 5, 7, 9), (1, 5, 1, 1), 0), modes=("f32", "f16"), nhwc=3),
    Row("maxpool_3x3_s2", maxpool((1, 5, 9, 11), 3, 1, 2), modes=("f32", "f16"), nhwc=1),
]
# the int64 compare ops, each on an outer product [n,1] x [m], [1,3] x [3,1], a rank-raising single element [1,1,1] x [5], a scalar
# constant and equal shapes
for _op in ("Less", "Greater", "Equal", "And"):
    _o = _op.lower()
    ROWS += [
        Row(f"{_o}_outer_n1_m", compare(_op, (5, 1), (7,)), modes=("f32", "f16")),
        Row(f"{_o}_13_vs_31", compare(_op, (1, 3), (3, 1)), modes=("f32", "f16")),
        Row(f"{_o}_111_vs_5", compare(_op, (1, 1, 1), (5,)), modes=("f32", "f16")),
        Row(f"{_o}_scalar_const", compare(_op, (2, 3), (), b_const=True), modes=("f32", "f16")),
        Row(f"{_o}_equal_shapes", compare(_op, (3, 5), (3, 5)), modes=("f32", "f16")),
    ]
IDS = [r.id for r in ROWS]
assert len(set(IDS)) == len(IDS)


# ---------------------------------------------------------------------------------------------------------------- graphs and references
def _emit(row, d, producer):
    """Write the row's graph to directory d.  producer "plain": sources are graph inputs; "nhwc": each source is Conv(<name>_in) named
    <name>.  Returns (spec, source names)."""
    g = emit.GraphBuilder(d, "float32", seed=len(row.id))
    srcs = []

    def src(name, shape):
        srcs.append(name)
        if producer == "plain":
            return g.input(name, shape)
        x = g.input(name + "_in", shape)
        k, c = row.nhwc, shape[1]
        r = np.random.default_rng(len(srcs))   # not the builder's generator: the row's own constants match its plain graph
        w = g.const((r.standard_normal((c, c, k, k)) / np.sqrt(c * k * k)).astype(np.float32), conv_weight=True)
        b = g.const((r.standard_normal(c) * 0.25).astype(np.float32), quantizable=False)
        return g.node("Conv", [x, w, b], [shape], [("dilations", "1,1"), ("group", "1"), ("kernel_shape", f"{k},{k}"),
                                                  ("pads", ",".join([str(k // 2)] * 4)), ("strides", "1,1")], out_names=[name])
    spec = row.build(g, src)
    g.finish()
    return spec, list(dict.fromkeys(srcs))


def _feeds_for(spec, srcs, producer, seed):
    f = spec.feeds(np.random.default_rng(seed))
    if producer == "nhwc":
        f = {(k + "_in" if k in srcs else k): v for k, v in f.items()}
    return f


def _qu8_roundtrip(x):
    """x quantised by the engine's percentile rule (at THREADS) and dequantised; None when the tensor has no usable range (it then
    stays float)."""
    rng = qu8_percentiles(np.asarray(x, np.float32), threads=THREADS)
    if rng is None:
        return None
    scale, zp = qu8_range_to_scale(*rng)
    return qu8_dequantize(qu8_quantize(x, scale, zp), scale, zp), scale


def _round_mode(a, mode):
    a = np.asarray(a)
    if a.dtype == np.int64:
        return a
    return a.astype(np.float16).astype(np.float32) if mode == "f16" else a.astype(np.float32)


def _engine(lib, d, feed_list, names, mode, producer, extra=(), b200=(), wp="nocache", dynamic=False):
    """Run the graph once per input set on one Model; returns the named tensors of each run and the Model's stats."""
    m = Model(lib, THREADS, wp)
    try:
        if mode == "f16":
            m.set_option("use_fp16_arithmetic", True)
        elif mode == "u8":
            m.set_option("use_uint8_arithmetic", True)
        if dynamic:
            m.set_option("support_dynamic_shapes", True)
        m.lib.model_set_option(m.h, b"b200_keep_nhwc", 1)
        for k, v in b200:
            m.lib.model_set_option(m.h, k.encode(), int(v))
        for e in extra:
            m.add_extra_output(e)
        m.read_file(d + "model.txt")
        runs = []
        for f in feed_list:
            m.clear_tensors()
            for k, v in f.items():
                m.add_tensor(k, v)
            m.run()
            out = {}
            for n in list(names) + list(extra):
                t = m.get_tensor(n)
                out[n] = m.get_tensor_i64(n) if t is None else t
            runs.append(out)
        return runs, m.stats()
    finally:
        m.close()


def _rel(got, ref):
    d = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64))
    return float(d.max()) / max(float(np.abs(ref).max()), 1e-30) if d.size else 0.0


# ---------------------------------------------------------------------------------------------------------------- tests
def _cases():
    out = []
    for r in ROWS:
        for mode in r.modes:
            for producer in ("plain", "nhwc") if r.nhwc else ("plain",):
                if producer == "nhwc" and mode == "u8":
                    continue    # a uint8 Conv needs uint8 weights and calibrated output ranges: the plain producer covers uint8
                out.append(pytest.param(r, mode, producer, id=f"{r.id}-{mode}-{producer}"))
    return out


@pytest.fixture(scope="module")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def test_rows_emit_and_oracle_shapes(tmp_path):
    """(no GPU) Every row's graphs are well formed: the fp64 oracle runs them and every output has the shape the graph declares."""
    for r in ROWS:
        for producer in ("plain", "nhwc") if r.nhwc else ("plain",):
            d = str(tmp_path / r.id / producer) + "/"
            spec, srcs = _emit(r, d, producer)
            ref = NumpyOracle(d).run(_feeds_for(spec, srcs, producer, 1))
            for n in spec.outs:
                assert n in ref, (r.id, producer, n)


@pytest.mark.gpu
@pytest.mark.parametrize("row,mode,producer", _cases())
def test_op(engine_lib, cuda, row, mode, producer, tmp_path):
    d = str(tmp_path / producer) + "/"
    spec, srcs = _emit(row, d, producer)
    dp = d
    if producer == "nhwc":
        dp = str(tmp_path / "plain") + "/"
        _emit(row, dp, "plain")
    feed_list = [_feeds_for(spec, srcs, producer, s) for s in (1, 2)]
    extra = tuple(srcs) if producer == "nhwc" else ()
    runs, _ = _engine(engine_lib, d, feed_list, spec.outs, mode, producer, extra, dynamic=row.dynamic)
    full = NumpyOracle(d)
    for k, (f, got) in enumerate(zip(feed_list, runs)):
        what = f"{row.id} {mode} {producer} run {k + 1}"
        # the producer values the op consumed, then the oracle's op on exactly those
        p = dict(f)
        u8_scales = {}
        for s in srcs:
            if producer == "nhwc":
                p.pop(s + "_in")
                p[s] = np.asarray(got[s], np.float32)
            elif mode == "u8":
                q = _qu8_roundtrip(f[s])
                if q is not None:
                    p[s], u8_scales[s] = q
            else:
                p[s] = _round_mode(f[s], mode)
        on_p = NumpyOracle(dp).run(p)
        whole = full.run(f)
        for n in spec.outs:
            g_, e = np.asarray(got[n]), np.asarray(on_p[n])
            assert g_.shape == e.shape, (what, n, g_.shape, e.shape)
            if row.kind == "move" and mode == "u8" and row.requant_u8 and len(set(u8_scales.values())) > 1:
                # sources at different scales: the float concatenation re-quantised by the percentile rule, within one output step
                want = _qu8_roundtrip(e)
                assert want is not None
                want, step = want
                err = np.abs(g_.astype(np.float64) - e.astype(np.float64))
                lo, hi = qu8_percentiles(e, threads=THREADS)
                inside = (e >= lo) & (e <= hi)
                assert float(err[inside].max()) <= step, f"{what} {n}: {float(err[inside].max()):.4g} off the fp64 concatenation, " \
                    f"above one output step {step:.4g}"
                bad = int((g_ != want).sum())
                assert bad == 0, f"{what} {n}: {bad} of {want.size} values differ from the re-quantised concatenation"
            elif row.kind in ("move", "trunc"):
                want = _round_mode(e, mode) if mode == "f16" else e
                bad = int((g_ != want).sum()) if g_.size else 0
                assert bad == 0, f"{what} {n}: {bad} of {g_.size} values differ from the op applied to the producer's output " \
                    f"(max |diff| {float(np.abs(g_.astype(np.float64) - want).max()):.4g})"
            elif mode == "u8":
                err = float(np.abs(g_.astype(np.float64) - e).max())
                assert err <= U8_SOFTMAX_STEPS / 256, f"{what} {n}: {err:.4g} off fp64 on the dequantised input"
            else:
                rel = _rel(g_, e)
                bar = BARS[row.kind][1 if mode == "f16" else 0]
                assert np.isfinite(g_).all() and rel <= bar, f"{what} {n}: {rel:.3e} > {bar:.1e} against fp64 on the producer's output"
            bar = BARS[row.kind][1 if mode == "f16" else 0]
            if mode != "u8" and g_.dtype != np.int64 and bar is not None:
                rel = _rel(g_, whole[n])
                assert rel <= bar, f"{what} {n}: the whole row is {rel:.3e} > {bar:.1e} off the fp64 oracle"
        for a, b in spec.equal:
            assert np.array_equal(got[a], got[b]), f"{what}: {a} and {b} differ (max {float(np.abs(got[a] - got[b]).max()):.4g})"


GRAPH_ROWS = [r for r in ROWS if r.graph]


@pytest.mark.gpu
@pytest.mark.parametrize("row", GRAPH_ROWS, ids=[r.id for r in GRAPH_ROWS])
def test_cuda_graph_follows_inputs(engine_lib, cuda, row, tmp_path):
    """Resident weights + CUDA graphs, four runs with new values each time (fp32): every output equals the oracle's on that run's
    inputs, whether the graph replays or the capture falls back to eager runs."""
    d = str(tmp_path) + "/"
    spec, srcs = _emit(row, d, "plain")
    feed_list = [_feeds_for(spec, srcs, "plain", s) for s in (1, 2, 3, 4)]
    runs, st = _engine(engine_lib, d, feed_list, spec.outs, "f32", "plain",
                       b200=(("b200_resident_weights", 1), ("b200_cuda_graph", 1)), wp="ram+nocache", dynamic=row.dynamic)
    oracle = NumpyOracle(d)
    for k, (f, got) in enumerate(zip(feed_list, runs)):
        ref = oracle.run(f)
        for n in spec.outs:
            assert np.array_equal(np.asarray(got[n]), ref[n]), f"{row.id} run {k + 1} {n}: the output does not follow the new inputs"
    if row.replays:
        assert st["graph_replays"] >= 1, f"{row.id}: the captured graph never replayed"


REFUSALS = [
    ("slice_step_2", lambda g: g.node("Slice", [g.input("x", (7, 9)), g.i64([0]), g.i64([9]), g.i64([1]), g.i64([2])], [(7, 5)]),
     {"x": (7, 9)}, "steps != 1"),
    ("gather_axis_1", lambda g: g.node("Gather", [g.input("x", (7, 9)), g.i64([1, 2])], [(7, 2)], [("axis", "1")]), {"x": (7, 9)}, "axis != 0"),
    ("resize_scale_1_5", lambda g: g.node("Resize", [g.input("x", (1, 3, 4, 4)), None, g.const(np.array([1, 1, 1.5, 1.5], np.float32), quantizable=False)],
                                          [(1, 3, 6, 6)], [("coordinate_transformation_mode", "asymmetric"), ("mode", "nearest"), ("nearest_mode", "floor")]),
     {"x": (1, 3, 4, 4)}, "non-integer resize"),
    ("transpose_int64", lambda g: g.node("Transpose", [g.input("xi", (3, 5))], [(5, 3)], [("perm", "1,0")]), {"xi": (3, 5)}, "int64 transpose"),
    ("where_not_broadcastable", lambda g: g.node("Where", [g.input("cond", (3, 4)), g.input("x", (3, 5)), g.scalar(0.0)], [(3, 5)]),
     {"cond": (3, 4), "x": (3, 5)}, "not broadcastable"),
    ("less_not_broadcastable", lambda g: g.node("Less", [g.input("xi", (3, 4)), g.input("yi", (2, 4))], [(3, 4)]), {"xi": (3, 4), "yi": (2, 4)}, "not broadcastable"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,build,inputs,message", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refused(engine_lib, cuda, name, build, inputs, message, tmp_path):
    """Spellings the engine does not implement raise OnnxStreamError from the handler's own check (its message), never numbers."""
    d = str(tmp_path) + "/"
    g = emit.GraphBuilder(d, "float32", seed=0)
    out = build(g)
    g.mark_output(out)
    g.finish()
    r = np.random.default_rng(0)
    m = Model(engine_lib, THREADS, "nocache")
    try:
        m.read_file(d + "model.txt")
        for k, shp in inputs.items():
            v = r.integers(0, 2, shp).astype(np.int64) if k in ("cond", "xi", "yi") else r.standard_normal(shp).astype(np.float32)
            m.add_tensor(k, v)
        with pytest.raises(OnnxStreamError, match=message):
            m.run()
    finally:
        m.close()
