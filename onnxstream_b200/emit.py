"""Synthetic model emitter: writes OnnxStream model directories (``model.txt`` + raw ``.bin`` blobs).

No SD / SDXL / TinyLlama checkpoints exist offline (the reference downloads them at run time,
src/sd.cpp:3030-3199, src/llm.cpp:147-221), so every BASELINE.json config runs on a seeded synthetic graph of
the same architecture.  The on-disk format follows the reference's parser (src/onnxstream.cpp:2445-2616) and
converter (onnx2txt/onnx2txt.ipynb cell 1): one op per line ``Name:Type*input:T;T*output:T*attr:val;attr:val``;
a tensor is ``name(shape)`` or, for a static weight, ``file(dtype:shape)``; Conv weights are listed as
``X_nchw.bin(dtype:O,I,kh,kw)`` while the blob on disk is ``X_nhwc.bin`` in OHWI order
(src/onnxstream.cpp:2666-2692); uint8 weights carry ``uint8[scale,zero_point]`` produced by the onnx2txt
percentile rule (cell 1 lines 25-58).  Graph patterns (GroupNorm as Reshape/InstanceNormalization/Reshape/Mul/Add,
SiLU as Sigmoid/Mul, LayerNorm and erf-GELU as primitive chains, attention as MatMul/Mul/Softmax/MatMul with K
pre-transposed) are the diffusers-export patterns the reference's fusion matcher expects
(src/onnxstream.cpp:3576-3633).
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np


@dataclass
class T:
    """A tensor reference inside the emitted graph."""
    name: str
    shape: Tuple[int, ...]
    wtype: Optional[str] = None  # dtype prefix for static weights ("float32", "float16", "int64", "uint8[s,z]")

    def text(self) -> str:
        dims = ",".join(str(d) for d in self.shape)
        return f"{self.name}({self.wtype}:{dims})" if self.wtype else f"{self.name}({dims})"


def quantize_uint8(a: np.ndarray, from_left: float = 0.001, from_right: float = 0.001):
    """onnx2txt.ipynb cell 1 `quantize`: percentile range -> (uint8 array, scale, zero_point); None if not quantisable."""
    flat = a.astype(np.float32).ravel()
    s = flat[np.isfinite(flat)]
    if len(s) == 1 and flat.size == 1:
        scale = abs(float(flat[0]))
        zero = 0 if flat[0] >= 0 else 2
        return np.array([1], dtype=np.uint8).reshape(a.shape), scale, zero
    if len(s) >= 2:
        s = np.sort(s)
        left = float(s[int(len(s) * from_left)])
        right = float(s[int(len(s) * from_right * -1 - 1)])
        del s
        if left > 0 and right > 0:
            left = 0.0
        elif left < 0 and right < 0:
            right = 0.0
        if right > left:
            scale = (right - left) / 255.0
            zero = min(int(abs(left) / scale), 255)
            # clip(a / scale + zero, 0, 255) in float64, truncated to uint8 -- in place: fresh multi-GB temporaries per step made the
            # SDXL-size emission page-fault bound
            x = a.astype(np.float64)
            x /= scale
            x += zero
            np.clip(x, 0, 255, out=x)
            return x.astype(np.uint8), scale, zero
    return None


class GraphBuilder:
    """Accumulates ops + weight blobs and writes them in OnnxStream's text format."""

    def __init__(self, out_dir: Optional[str], wdtype: str = "float32", seed: int = 0, keep_in_memory: bool = False):
        assert wdtype in ("float32", "float16", "uint8")
        self.out_dir = out_dir
        self.wdtype = wdtype
        self.rng = np.random.default_rng(seed)
        self.lines: List[str] = []
        self.n = 0
        self.keep = keep_in_memory or out_dir is None
        self.blobs: Dict[str, Tuple[str, np.ndarray]] = {}  # file name -> (dtype string, array) when keep
        self.inputs: List[T] = []
        self.outputs: List[T] = []
        self.weight_bytes = 0
        self.weight_params = 0
        self.flops = 0  # 2*MACs over Conv/MatMul/Gemm/attention, for the roofline bookkeeping
        if out_dir:
            os.makedirs(out_dir, exist_ok=True)

    # ---- naming -------------------------------------------------------------------------------------
    def _uid(self, prefix: str) -> str:
        self.n += 1
        return f"{prefix}{self.n}"

    # ---- tensors ------------------------------------------------------------------------------------
    def input(self, name: str, shape: Sequence[int]) -> T:
        t = T(name, tuple(shape))
        self.inputs.append(t)
        return t

    def _save(self, fname: str, dtype: str, arr: np.ndarray):
        arr = np.ascontiguousarray(arr)
        self.weight_bytes += arr.nbytes
        self.weight_params += arr.size
        if self.keep:
            self.blobs[fname] = (dtype.split("[")[0], arr)
        if self.out_dir:
            arr.tofile(os.path.join(self.out_dir, fname))

    def const(self, arr: np.ndarray, name: Optional[str] = None, conv_weight: bool = False, quantizable: bool = True,
              force_dtype: Optional[str] = None) -> T:
        """Register a static weight. `arr` is int64 or float32 in ONNX layout (Conv: OIHW)."""
        base = name or self._uid("w")
        arr = np.asarray(arr)
        logical_shape = tuple(arr.shape)
        if arr.dtype == np.int64:
            dt, data = "int64", arr
        else:
            arr = arr.astype(np.float32)
            want = force_dtype or self.wdtype
            if want == "uint8" and quantizable:
                q = quantize_uint8(arr)
                if q is None:
                    dt, data = "float32", arr
                else:
                    data, scale, zero = q
                    dt = f"uint8[{scale!r},{zero}]"
            elif want == "float16":
                dt, data = "float16", arr.astype(np.float16)
            else:
                dt, data = "float32", arr
        if conv_weight:
            if data.ndim == 3:
                data = data[..., None]
            self._save(base + "_nhwc.bin", dt, np.transpose(data, (0, 2, 3, 1)))
            return T(base + "_nchw.bin", logical_shape, dt)
        self._save(base + ".bin", dt, data)
        return T(base + ".bin", logical_shape, dt)

    def randn(self, shape: Sequence[int], std: float = 1.0, mean: float = 0.0) -> np.ndarray:
        a = self.rng.standard_normal(tuple(shape), dtype=np.float32)
        if std != 1.0:
            a *= np.float32(std)
        if mean != 0.0:
            a += np.float32(mean)
        return a

    # ---- ops ----------------------------------------------------------------------------------------
    def node(self, op_type: str, inputs: Sequence[Optional[T]], out_shapes: Sequence[Sequence[int]],
             attrs: Optional[Sequence[Tuple[str, str]]] = None, name: Optional[str] = None,
             out_names: Optional[Sequence[str]] = None):
        op_name = name or self._uid(op_type + "_")
        outs = [T(out_names[i] if out_names else self._uid("t"), tuple(s)) for i, s in enumerate(out_shapes)]
        line = f"{op_name}:{op_type}*input:" + ";".join(i.text() if i is not None else "" for i in inputs)
        line += "*output:" + ";".join(o.text() for o in outs)
        if attrs:
            line += "*" + ";".join(f"{k}:{v}" for k, v in attrs)
        self.lines.append(line)
        return outs[0] if len(outs) == 1 else outs

    def mark_output(self, t: T):
        self.outputs.append(t)

    def text(self) -> str:
        return "\n".join(self.lines) + "\n"

    def finish(self) -> str:
        txt = self.text()
        if self.out_dir:
            with open(os.path.join(self.out_dir, "model.txt"), "w") as f:
                f.write(txt)
        return txt

    # ---- composite layers (diffusers-export patterns) -----------------------------------------------
    def i64(self, vals: Sequence[int]) -> T:
        return self.const(np.asarray(vals, dtype=np.int64))

    def scalar(self, v: float) -> T:
        return self.const(np.asarray(v, dtype=np.float32))

    def conv(self, x: T, cout: int, k: int, stride: int = 1, pad: Optional[int] = None, bias: bool = True, name=None) -> T:
        _, cin, h, w = x.shape
        pad = (k // 2) if pad is None else pad
        wt = self.const(self.randn((cout, cin, k, k), std=1.0 / math.sqrt(cin * k * k)), conv_weight=True)
        ins = [x, wt]
        if bias:
            ins.append(self.const(self.randn((cout,), std=0.02), quantizable=False))
        ho = (h + 2 * pad - k) // stride + 1
        wo = (w + 2 * pad - k) // stride + 1
        self.flops += 2 * ho * wo * cout * cin * k * k
        return self.node("Conv", ins, [(1, cout, ho, wo)],
                         [("dilations", "1,1"), ("group", "1"), ("kernel_shape", f"{k},{k}"),
                          ("pads", f"{pad},{pad},{pad},{pad}"), ("strides", f"{stride},{stride}")], name=name)

    def group_norm(self, x: T, groups: int = 32, eps: float = 1e-5) -> T:
        _, c, h, w = x.shape
        r = self.node("Reshape", [x, self.i64([0, groups, -1])], [(1, groups, c // groups * h * w)])
        n = self.node("InstanceNormalization",
                      [r, self.const(np.ones(groups, np.float32), quantizable=False), self.const(np.zeros(groups, np.float32), quantizable=False)],
                      [r.shape], [("epsilon", repr(float(eps)))])
        r2 = self.node("Reshape", [n, self.i64([1, c, h, w])], [(1, c, h, w)])
        m = self.node("Mul", [r2, self.const(self.randn((c, 1, 1), std=0.02, mean=1.0))], [(1, c, h, w)])
        return self.node("Add", [m, self.const(self.randn((c, 1, 1), std=0.02))], [(1, c, h, w)])

    def silu(self, x: T) -> T:
        s = self.node("Sigmoid", [x], [x.shape])
        return self.node("Mul", [x, s], [x.shape])

    def linear(self, x: T, nout: int, bias: bool = True, std: Optional[float] = None, name=None) -> T:
        """x [..., K] @ W[K, nout] (+ b) exported as MatMul (+ Add(bias, y))."""
        k = x.shape[-1]
        w = self.const(self.randn((k, nout), std=std if std is not None else 1.0 / math.sqrt(k)))
        out_shape = tuple(x.shape[:-1]) + (nout,)
        self.flops += 2 * int(np.prod(x.shape[:-1])) * k * nout
        y = self.node("MatMul", [x, w], [out_shape], name=name)
        if bias:
            y = self.node("Add", [self.const(self.randn((nout,), std=0.02)), y], [out_shape])
        return y

    def gemm(self, x: T, nout: int) -> T:
        """[1,K] x [K,N] + [N]; transB already folded by the converter (cell 1 lines 129-141)."""
        k = x.shape[-1]
        w = self.const(self.randn((k, nout), std=1.0 / math.sqrt(k)), name=self._uid("w") + "_transposed")
        b = self.const(self.randn((nout,), std=0.02))
        self.flops += 2 * x.shape[0] * k * nout
        return self.node("Gemm", [x, w, b], [(x.shape[0], nout)])

    def layer_norm(self, x: T, eps: float = 1e-5) -> T:
        c = x.shape[-1]
        red = tuple(x.shape[:-1]) + (1,)
        mean = self.node("ReduceMean", [x], [red], [("axes", "-1"), ("keepdims", "1")])
        d = self.node("Sub", [x, mean], [x.shape])
        p = self.node("Pow", [d, self.scalar(2.0)], [x.shape])
        var = self.node("ReduceMean", [p], [red], [("axes", "-1"), ("keepdims", "1")])
        ve = self.node("Add", [var, self.scalar(eps)], [red])
        sd = self.node("Sqrt", [ve], [red])
        nrm = self.node("Div", [d, sd], [x.shape])
        m = self.node("Mul", [nrm, self.const(self.randn((c,), std=0.02, mean=1.0))], [x.shape])
        return self.node("Add", [m, self.const(self.randn((c,), std=0.02))], [x.shape])

    def gelu(self, x: T) -> T:
        d = self.node("Div", [x, self.scalar(math.sqrt(2.0))], [x.shape])
        e = self.node("Erf", [d], [x.shape])
        a = self.node("Add", [e, self.scalar(1.0)], [x.shape])
        m = self.node("Mul", [x, a], [x.shape])
        return self.node("Mul", [m, self.scalar(0.5)], [x.shape])

    def split_heads(self, x: T, heads: int, transpose_k: bool = False) -> T:
        """[1,T,C] -> [heads,T,d] (or [heads,d,T] for K, transposed before the MatMul)."""
        _, t, c = x.shape
        d = c // heads
        r = self.node("Reshape", [x, self.i64([1, t, heads, d])], [(1, t, heads, d)])
        p = self.node("Transpose", [r], [(1, heads, t, d)], [("perm", "0,2,1,3")])
        r2 = self.node("Reshape", [p, self.i64([heads, t, d])], [(heads, t, d)])
        if transpose_k:
            r2 = self.node("Transpose", [r2], [(heads, d, t)], [("perm", "0,2,1")])
        return r2

    def attention(self, x: T, ctx: T, heads: int, scale: Optional[float] = None) -> T:
        """diffusers Attention: q from x, k/v from ctx; MatMul -> Mul(scale, default 1 / sqrt(d)) -> Softmax -> MatMul; out proj with bias."""
        _, t, c = x.shape
        tk = ctx.shape[1]
        d = c // heads
        q = self.split_heads(self.linear(x, c, bias=False), heads)
        k = self.split_heads(self.linear(ctx, c, bias=False), heads, transpose_k=True)
        v = self.split_heads(self.linear(ctx, c, bias=False), heads)
        s = self.node("MatMul", [q, k], [(heads, t, tk)])
        s = self.node("Mul", [s, self.scalar(1.0 / math.sqrt(d) if scale is None else scale)], [(heads, t, tk)])
        p = self.node("Softmax", [s], [(heads, t, tk)], [("axis", "-1")])
        o = self.node("MatMul", [p, v], [(heads, t, d)])
        self.flops += 4 * heads * t * tk * d
        o = self.node("Reshape", [o, self.i64([1, heads, t, d])], [(1, heads, t, d)])
        o = self.node("Transpose", [o], [(1, t, heads, d)], [("perm", "0,2,1,3")])
        o = self.node("Reshape", [o, self.i64([1, t, c])], [(1, t, c)])
        return self.linear(o, c, bias=True)

    def geglu_ff(self, x: T, mult: int = 4) -> T:
        _, t, c = x.shape
        inner = c * mult
        g = self.linear(x, inner * 2, bias=True)
        a = self.node("Slice", [g, self.i64([0]), self.i64([inner]), self.i64([-1]), self.i64([1])], [(1, t, inner)])
        gate = self.node("Slice", [g, self.i64([inner]), self.i64([inner * 2]), self.i64([-1]), self.i64([1])], [(1, t, inner)])
        y = self.node("Mul", [a, self.gelu(gate)], [(1, t, inner)])
        return self.linear(y, c, bias=True)

    def transformer_block(self, h: T, ctx: T, heads: int) -> T:
        n1 = self.layer_norm(h)
        h = self.node("Add", [self.attention(n1, n1, heads), h], [h.shape])
        n2 = self.layer_norm(h)
        h = self.node("Add", [self.attention(n2, ctx, heads), h], [h.shape])
        n3 = self.layer_norm(h)
        return self.node("Add", [self.geglu_ff(n3), h], [h.shape])

    def spatial_transformer(self, x: T, ctx: T, heads: int, depth: int = 1, linear_proj: bool = False) -> T:
        _, c, hh, ww = x.shape
        res = x
        h = self.group_norm(x, eps=1e-6)
        if not linear_proj:
            h = self.conv(h, c, 1)
        h = self.node("Transpose", [h], [(1, hh, ww, c)], [("perm", "0,2,3,1")])
        h = self.node("Reshape", [h, self.i64([1, hh * ww, c])], [(1, hh * ww, c)])
        if linear_proj:
            h = self.linear(h, c, bias=True)
        for _ in range(depth):
            h = self.transformer_block(h, ctx, heads)
        if linear_proj:
            h = self.linear(h, c, bias=True)
        h = self.node("Reshape", [h, self.i64([1, hh, ww, c])], [(1, hh, ww, c)])
        h = self.node("Transpose", [h], [(1, c, hh, ww)], [("perm", "0,3,1,2")])
        if not linear_proj:
            h = self.conv(h, c, 1)
        return self.node("Add", [h, res], [x.shape])

    def resnet(self, x: T, temb: Optional[T], cout: int, groups: int = 32, eps: float = 1e-5) -> T:
        _, cin, hh, ww = x.shape
        h = self.conv(self.silu(self.group_norm(x, groups, eps)), cout, 3)
        if temb is not None:
            t = self.gemm(self.silu(temb), cout)
            t = self.node("Unsqueeze", [t, self.i64([2])], [(1, cout, 1)])
            t = self.node("Unsqueeze", [t, self.i64([3])], [(1, cout, 1, 1)])
            h = self.node("Add", [h, t], [h.shape])
        h = self.conv(self.silu(self.group_norm(h, groups, eps)), cout, 3)
        if cin != cout:
            x = self.conv(x, cout, 1)
        return self.node("Add", [x, h], [h.shape])

    def upsample2x(self, x: T) -> T:
        _, c, hh, ww = x.shape
        scales = self.const(np.asarray([1, 1, 2, 2], np.float32), quantizable=False)
        r = self.node("Resize", [x, None, scales], [(1, c, hh * 2, ww * 2)],
                      [("coordinate_transformation_mode", "asymmetric"), ("cubic_coeff_a", "-0.75"),
                       ("mode", "nearest"), ("nearest_mode", "floor")])
        return self.conv(r, c, 3)

    def timestep_embedding(self, timestep: T, dim: int, flip_sin_to_cos: bool = True) -> T:
        """[N] -> [N, dim] sinusoid: Unsqueeze, Mul(freqs), Sin/Cos, Concat."""
        n = timestep.shape[0]
        half = dim // 2
        freqs = np.exp(-math.log(10000.0) * np.arange(half, dtype=np.float32) / half).astype(np.float32)
        t = self.node("Unsqueeze", [timestep, self.i64([1])], [(n, 1)])
        a = self.node("Mul", [t, self.const(freqs.reshape(1, half), quantizable=False, force_dtype="float32" if self.wdtype == "uint8" else None)], [(n, half)])
        s = self.node("Sin", [a], [(n, half)])
        c = self.node("Cos", [a], [(n, half)])
        parts = [c, s] if flip_sin_to_cos else [s, c]
        return self.node("Concat", parts, [(n, dim)], [("axis", "-1")])


# ======================================================================================================
# Architectures
# ======================================================================================================

@dataclass
class UNetConfig:
    """SD1.5 defaults (SURVEY Appendix C.1). `tiny()` keeps the topology and shrinks every dimension."""
    latent: int = 64
    in_ch: int = 4
    block_ch: Tuple[int, ...] = (320, 640, 1280, 1280)
    attn_levels: Tuple[bool, ...] = (True, True, True, False)
    layers_per_block: int = 2
    heads: Optional[int] = 8            # SD1.5: 8 heads everywhere; SDXL: None -> head_dim 64
    head_dim: Optional[int] = None
    depth: Tuple[int, ...] = (1, 1, 1, 0)  # transformer layers per attention block
    mid_depth: int = 1
    ctx_len: int = 77
    ctx_dim: int = 768
    linear_proj: bool = False
    groups: int = 32
    sdxl_addition: bool = False         # time_ids/text_embeds add-embedding (SDXL, src/sd.cpp:1488-1516)
    add_time_dim: int = 256
    text_embed_dim: int = 1280

    @staticmethod
    def sd15(latent: int = 64) -> "UNetConfig":
        return UNetConfig(latent=latent)

    @staticmethod
    def sdxl(latent: int = 128) -> "UNetConfig":
        return UNetConfig(latent=latent, block_ch=(320, 640, 1280), attn_levels=(False, True, True), heads=None, head_dim=64,
                          depth=(0, 2, 10), mid_depth=10, ctx_dim=2048, linear_proj=True, sdxl_addition=True)

    @staticmethod
    def tiny(latent: int = 16, sdxl: bool = False) -> "UNetConfig":
        if sdxl:
            return UNetConfig(latent=latent, block_ch=(32, 64, 64), attn_levels=(False, True, True), heads=None, head_dim=16,
                              depth=(0, 1, 2), mid_depth=2, ctx_len=7, ctx_dim=48, linear_proj=True, sdxl_addition=True,
                              groups=8, add_time_dim=8, text_embed_dim=40)
        return UNetConfig(latent=latent, block_ch=(32, 64, 64), attn_levels=(True, True, False), heads=4,
                          depth=(1, 1, 0), mid_depth=1, ctx_len=7, ctx_dim=48, groups=8)


def emit_unet(out_dir: Optional[str], cfg: UNetConfig, wdtype: str = "float32", seed: int = 0, keep_in_memory: bool = False) -> GraphBuilder:
    """SD1.5 / SDXL UNet-shaped graph. Inputs as pushed by sd.cpp (src/sd.cpp:1461-1516, names are the mangled ones)."""
    g = GraphBuilder(out_dir, wdtype, seed, keep_in_memory)
    L = cfg.latent
    x = g.input("sample", (1, cfg.in_ch, L, L))
    ts = g.input("timestep", (1,))
    ctx = g.input("encoder_5F_hidden_5F_states", (1, cfg.ctx_len, cfg.ctx_dim))
    c0 = cfg.block_ch[0]
    temb_dim = c0 * 4
    groups = cfg.groups

    def nheads(c):
        return cfg.heads if cfg.heads else c // cfg.head_dim

    temb = g.timestep_embedding(ts, c0)
    temb = g.gemm(temb, temb_dim)
    temb = g.silu(temb)
    temb = g.gemm(temb, temb_dim)
    if cfg.sdxl_addition:
        text_embeds = g.input("text_5F_embeds", (1, cfg.text_embed_dim))
        time_ids = g.input("time_5F_ids", (1, 6))
        tid = g.node("Reshape", [time_ids, g.i64([-1])], [(6,)])
        te = g.timestep_embedding(tid, cfg.add_time_dim)
        te = g.node("Reshape", [te, g.i64([1, -1])], [(1, 6 * cfg.add_time_dim)])
        add = g.node("Concat", [text_embeds, te], [(1, cfg.text_embed_dim + 6 * cfg.add_time_dim)], [("axis", "-1")])
        add = g.gemm(add, temb_dim)
        add = g.silu(add)
        add = g.gemm(add, temb_dim)
        temb = g.node("Add", [temb, add], [temb.shape])

    h = g.conv(x, c0, 3)
    skips = [h]
    nlev = len(cfg.block_ch)
    for lvl, c in enumerate(cfg.block_ch):
        for _ in range(cfg.layers_per_block):
            h = g.resnet(h, temb, c, groups)
            if cfg.attn_levels[lvl]:
                h = g.spatial_transformer(h, ctx, nheads(c), cfg.depth[lvl], cfg.linear_proj)
            skips.append(h)
        if lvl != nlev - 1:
            h = g.conv(h, c, 3, stride=2, pad=1)
            skips.append(h)
    cm = cfg.block_ch[-1]
    h = g.resnet(h, temb, cm, groups)
    if cfg.mid_depth > 0:
        h = g.spatial_transformer(h, ctx, nheads(cm), cfg.mid_depth, cfg.linear_proj)
    h = g.resnet(h, temb, cm, groups)
    for lvl in reversed(range(nlev)):
        c = cfg.block_ch[lvl]
        for i in range(cfg.layers_per_block + 1):
            s = skips.pop()
            h = g.node("Concat", [h, s], [(1, h.shape[1] + s.shape[1], h.shape[2], h.shape[3])], [("axis", "1")])
            h = g.resnet(h, temb, c, groups)
            if cfg.attn_levels[lvl]:
                h = g.spatial_transformer(h, ctx, nheads(c), cfg.depth[lvl], cfg.linear_proj)
        if lvl != 0:
            h = g.upsample2x(h)
    h = g.silu(g.group_norm(h, groups))
    out = g.conv(h, cfg.in_ch, 3, name="conv_out")
    # give the graph output the name sd.cpp reads back (src/sd.cpp:1521)
    g.lines[-1] = g.lines[-1].replace(out.text(), T("out_5F_sample", out.shape).text())
    g.mark_output(T("out_5F_sample", out.shape))
    g.finish()
    return g


@dataclass
class VAEConfig:
    latent: int = 64
    block_ch: Tuple[int, ...] = (512, 512, 256, 128)   # decoder up-block widths, deepest first (SURVEY C.4)
    layers_per_block: int = 3
    groups: int = 32
    mid_attention: bool = True

    @staticmethod
    def tiny(latent: int = 8) -> "VAEConfig":
        return VAEConfig(latent=latent, block_ch=(32, 32, 16), layers_per_block=2, groups=8)


def emit_vae_decoder(out_dir: Optional[str], cfg: VAEConfig, wdtype: str = "float32", seed: int = 1, keep_in_memory: bool = False) -> GraphBuilder:
    """SD1.5 VAE-decoder-shaped graph; input `input_2E_1` (1,4,L,L) as pushed by sd.cpp (src/sd.cpp:1196-1206)."""
    g = GraphBuilder(out_dir, wdtype, seed, keep_in_memory)
    L = cfg.latent
    x = g.input("input_2E_1", (1, 4, L, L))
    h = g.conv(x, 4, 1)                     # post_quant_conv
    c = cfg.block_ch[0]
    h = g.conv(h, c, 3)
    h = g.resnet(h, None, c, cfg.groups, 1e-6)
    if cfg.mid_attention:                   # single-head attention over HW tokens, Linear q/k/v/out with bias
        res = h
        n = g.group_norm(h, cfg.groups, 1e-6)
        n = g.node("Reshape", [n, g.i64([1, c, L * L])], [(1, c, L * L)])
        n = g.node("Transpose", [n], [(1, L * L, c)], [("perm", "0,2,1")])
        q = g.linear(n, c)
        k = g.linear(n, c)
        v = g.linear(n, c)
        kt = g.node("Transpose", [k], [(1, c, L * L)], [("perm", "0,2,1")])
        s = g.node("MatMul", [q, kt], [(1, L * L, L * L)])
        s = g.node("Mul", [s, g.scalar(1.0 / math.sqrt(c))], [s.shape])
        p = g.node("Softmax", [s], [s.shape], [("axis", "-1")])
        o = g.node("MatMul", [p, v], [(1, L * L, c)])
        g.flops += 4 * L * L * L * L * c
        o = g.linear(o, c)
        o = g.node("Transpose", [o], [(1, c, L * L)], [("perm", "0,2,1")])
        o = g.node("Reshape", [o, g.i64([1, c, L, L])], [(1, c, L, L)])
        h = g.node("Add", [o, res], [res.shape])
    h = g.resnet(h, None, c, cfg.groups, 1e-6)
    for i, c in enumerate(cfg.block_ch):
        for _ in range(cfg.layers_per_block):
            h = g.resnet(h, None, c, cfg.groups, 1e-6)
        if i != len(cfg.block_ch) - 1:
            h = g.upsample2x(h)
    h = g.silu(g.group_norm(h, cfg.groups, 1e-6))
    out = g.conv(h, 3, 3)
    g.lines[-1] = g.lines[-1].replace(out.text(), T("outsample", out.shape).text())
    g.mark_output(T("outsample", out.shape))
    g.finish()
    return g


@dataclass
class CLIPConfig:
    vocab: int = 49408
    tokens: int = 77
    width: int = 768
    heads: int = 12
    layers: int = 12

    @staticmethod
    def tiny() -> "CLIPConfig":
        return CLIPConfig(vocab=100, tokens=7, width=32, heads=4, layers=2)


def emit_text_encoder(out_dir: Optional[str], cfg: CLIPConfig, wdtype: str = "float32", seed: int = 2, keep_in_memory: bool = False) -> GraphBuilder:
    """CLIP-text-encoder-shaped graph: int64 (1,77) token ids -> (1,77,width). Causal mask added as a constant."""
    g = GraphBuilder(out_dir, wdtype, seed, keep_in_memory)
    ids = g.input("input_5F_ids", (1, cfg.tokens))
    T_, C, H = cfg.tokens, cfg.width, cfg.heads
    d = C // H
    emb = g.const(g.randn((cfg.vocab, C), std=0.02))
    h = g.node("Gather", [emb, ids], [(1, T_, C)], [("axis", "0")])
    pos = g.const(g.randn((1, T_, C), std=0.02))
    h = g.node("Add", [h, pos], [(1, T_, C)])
    mask = np.triu(np.full((T_, T_), -3.4028234663852886e+38, np.float32), k=1).reshape(1, 1, T_, T_)
    mask_t = g.const(mask, quantizable=False, force_dtype="float32")
    for _ in range(cfg.layers):
        n = g.layer_norm(h)
        q = g.node("Mul", [g.linear(n, C), g.scalar(1.0 / math.sqrt(d))], [(1, T_, C)])
        k = g.linear(n, C)
        v = g.linear(n, C)

        def heads4(t, kt=False):
            r = g.node("Reshape", [t, g.i64([1, T_, H, d])], [(1, T_, H, d)])
            r = g.node("Transpose", [r], [(1, H, T_, d)], [("perm", "0,2,1,3")])
            if kt:
                r = g.node("Transpose", [r], [(1, H, d, T_)], [("perm", "0,1,3,2")])
            return r
        s = g.node("MatMul", [heads4(q), heads4(k, True)], [(1, H, T_, T_)])
        s = g.node("Add", [s, mask_t], [(1, H, T_, T_)])
        p = g.node("Softmax", [s], [(1, H, T_, T_)], [("axis", "-1")])
        o = g.node("MatMul", [p, heads4(v)], [(1, H, T_, d)])
        g.flops += 4 * H * T_ * T_ * d
        o = g.node("Transpose", [o], [(1, T_, H, d)], [("perm", "0,2,1,3")])
        o = g.node("Reshape", [o, g.i64([1, T_, C])], [(1, T_, C)])
        h = g.node("Add", [h, g.linear(o, C)], [(1, T_, C)])
        n = g.layer_norm(h)
        f = g.linear(n, C * 4)
        # quick-GELU: x * sigmoid(1.702 x)
        sg = g.node("Sigmoid", [g.node("Mul", [f, g.scalar(1.702)], [f.shape])], [f.shape])
        f = g.node("Mul", [f, sg], [f.shape])
        h = g.node("Add", [h, g.linear(f, C)], [(1, T_, C)])
    out = g.layer_norm(h)
    g.lines[-1] = g.lines[-1].replace(out.text(), T("last_5F_hidden_5F_state", out.shape).text())
    g.mark_output(T("last_5F_hidden_5F_state", out.shape))
    g.finish()
    return g


def unet_inputs(cfg: UNetConfig, seed: int = 0) -> Dict[str, np.ndarray]:
    """Seeded synthetic inputs of the shapes sd.cpp pushes (SURVEY section 8d)."""
    rng = np.random.default_rng(1000 + seed)
    d = {
        "sample": rng.standard_normal((1, cfg.in_ch, cfg.latent, cfg.latent), dtype=np.float32),
        "timestep": np.asarray([500.0], np.float32),
        "encoder_5F_hidden_5F_states": rng.standard_normal((1, cfg.ctx_len, cfg.ctx_dim), dtype=np.float32),
    }
    if cfg.sdxl_addition:
        px = float(cfg.latent * 8)
        d["text_5F_embeds"] = rng.standard_normal((1, cfg.text_embed_dim), dtype=np.float32)
        d["time_5F_ids"] = np.asarray([[px, px, 0, 0, px, px]], np.float32)
    return d


@dataclass
class LlamaConfig:
    """TinyLlama-1.1B defaults (SURVEY Appendix C.3); `tiny()` shrinks every dimension, topology unchanged."""
    vocab: int = 32003
    hidden: int = 2048
    heads: int = 32
    kv_heads: int = 4
    head_dim: int = 64
    mlp: int = 5632
    layers: int = 22
    past: int = 2047          # cached positions; the decode step adds one token
    max_pos: int = 2048
    eps: float = 1e-5

    @staticmethod
    def tiny() -> "LlamaConfig":
        return LlamaConfig(vocab=50, hidden=64, heads=4, kv_heads=2, head_dim=16, mlp=128, layers=2, past=15, max_pos=32)


def emit_llama_decode(out_dir: Optional[str], cfg: LlamaConfig, wdtype: str = "float32", seed: int = 4, keep_in_memory: bool = False,
                      new_tokens: int = 1) -> GraphBuilder:
    """Llama-style step with a KV cache, as llm.cpp drives it (src/llm.cpp:396-440, 472-480): `new_tokens` = 1 is the single-token
    decode step, more is the prefill of a prompt of that many tokens.  Inputs input_ids (1,T) int64, position_ids (1,T) int64,
    attention_mask (1,past+T) int64, pkv{2l},pkv{2l+1} (1,kv_heads,past,d); outputs logits (1,T,vocab) and opkv* (the grown
    cache).  Attention uses the Transpose/MatMul/Div/Add/Softmax/MatMul chain that the reference rewrites into
    ScaledDotProductAttention (src/onnxstream.cpp:3643-3695), with grouped KV heads.  With T > 1 the additive mask is causal and
    padding at once: keep[t, j] = (j <= past + t) * attention_mask[j], mask = (1 - keep) * -65504.  past = 0 (the first turn) writes
    the caches as (1,kv_heads,0,d), which the reader accepts with support_dynamic_shapes, as llm.cpp sets it (src/llm.cpp:376).
    RMSNorm ops carry `/input_layernorm/`, `/post_attention_layernorm/`, `/norm/` in their names so that m_requires_upcast can
    keep them in fp32 (src/llm.cpp:385-389).  The text for new_tokens = 1 is the same as before the parameter existed."""
    g = GraphBuilder(out_dir, wdtype, seed, keep_in_memory)
    NT = new_tokens
    assert NT >= 1
    H, NH, KV, D, TT = cfg.hidden, cfg.heads, cfg.kv_heads, cfg.head_dim, cfg.past + NT
    ids = g.input("input_5F_ids", (1, NT))
    pos = g.input("position_5F_ids", (1, NT))
    am = g.input("attention_5F_mask", (1, TT))
    emb = g.const(g.randn((cfg.vocab, H), std=0.05))
    h = g.node("Gather", [emb, ids], [(1, NT, H)], [("axis", "0")])
    # rotary tables, gathered at position_ids
    inv = 1.0 / (10000.0 ** (np.arange(0, D, 2, dtype=np.float64) / D))
    fr = np.outer(np.arange(cfg.max_pos), inv)
    tab = np.concatenate([fr, fr], axis=-1)
    cos_t = g.const(np.cos(tab).astype(np.float32), quantizable=False)
    sin_t = g.const(np.sin(tab).astype(np.float32), quantizable=False)
    cos = g.node("Unsqueeze", [g.node("Gather", [cos_t, pos], [(1, NT, D)], [("axis", "0")]), g.i64([1])], [(1, 1, NT, D)])
    sin = g.node("Unsqueeze", [g.node("Gather", [sin_t, pos], [(1, NT, D)], [("axis", "0")]), g.i64([1])], [(1, 1, NT, D)])
    if NT == 1:
        # additive mask from the int64 attention mask: (1 - m) * -65504 -> [1,1,1,T]
        mf = g.node("Cast", [am], [(1, TT)], [("to", "1")])
        mf = g.node("Sub", [g.scalar(1.0), mf], [(1, TT)])
        mf = g.node("Mul", [mf, g.scalar(-65504.0)], [(1, TT)])
        mf = g.node("Unsqueeze", [mf, g.i64([1])], [(1, 1, TT)])
        mask = g.node("Unsqueeze", [mf, g.i64([2])], [(1, 1, 1, TT)])
    else:
        # causal AND padding in one 0/1 product, then ONE -65504 (two added -65504 masks would overflow to -inf in fp16)
        causal = (np.arange(TT)[None, :] <= cfg.past + np.arange(NT)[:, None]).astype(np.float32)
        mf = g.node("Cast", [am], [(1, TT)], [("to", "1")])
        keep = g.node("Mul", [g.const(causal, quantizable=False), mf], [(NT, TT)])
        mf = g.node("Sub", [g.scalar(1.0), keep], [(NT, TT)])
        mf = g.node("Mul", [mf, g.scalar(-65504.0)], [(NT, TT)])
        mf = g.node("Unsqueeze", [mf, g.i64([0])], [(1, NT, TT)])
        mask = g.node("Unsqueeze", [mf, g.i64([1])], [(1, 1, NT, TT)])

    def rms(x, tag):
        p = g.node("Pow", [x, g.scalar(2.0)], [x.shape], name=g._uid(f"{tag}_Pow_"))
        m = g.node("ReduceMean", [p], [x.shape[:-1] + (1,)], [("axes", "-1"), ("keepdims", "1")], name=g._uid(f"{tag}_ReduceMean_"))
        a = g.node("Add", [m, g.scalar(cfg.eps)], [m.shape], name=g._uid(f"{tag}_Add_"))
        s = g.node("Sqrt", [a], [m.shape], name=g._uid(f"{tag}_Sqrt_"))
        r = g.node("Div", [g.scalar(1.0), s], [m.shape], name=g._uid(f"{tag}_Div_"))
        n = g.node("Mul", [x, r], [x.shape], name=g._uid(f"{tag}_Mul_"))
        return g.node("Mul", [g.const(g.randn((H,), std=0.02, mean=1.0)), n], [x.shape], name=g._uid(f"{tag}_Mul_"))

    def rope(x, nh):
        x1 = g.node("Slice", [x, g.i64([0]), g.i64([D // 2]), g.i64([3]), g.i64([1])], [(1, nh, NT, D // 2)])
        x2 = g.node("Slice", [x, g.i64([D // 2]), g.i64([D]), g.i64([3]), g.i64([1])], [(1, nh, NT, D // 2)])
        rot = g.node("Concat", [g.node("Neg", [x2], [x2.shape]), x1], [(1, nh, NT, D)], [("axis", "-1")])
        return g.node("Add", [g.node("Mul", [x, cos], [x.shape]), g.node("Mul", [rot, sin], [x.shape])], [x.shape])

    for l in range(cfg.layers):
        pk = g.input(f"pkv{2 * l}", (1, KV, cfg.past, D))
        pv = g.input(f"pkv{2 * l + 1}", (1, KV, cfg.past, D))
        n = rms(h, f"_2F_model_2F_layers_2E_{l}_2F_input_5F_layernorm_2F_")
        q = g.linear(n, NH * D, bias=False)
        k = g.linear(n, KV * D, bias=False)
        v = g.linear(n, KV * D, bias=False)
        q = g.node("Transpose", [g.node("Reshape", [q, g.i64([1, NT, NH, D])], [(1, NT, NH, D)])], [(1, NH, NT, D)], [("perm", "0,2,1,3")])
        k = g.node("Transpose", [g.node("Reshape", [k, g.i64([1, NT, KV, D])], [(1, NT, KV, D)])], [(1, KV, NT, D)], [("perm", "0,2,1,3")])
        v = g.node("Transpose", [g.node("Reshape", [v, g.i64([1, NT, KV, D])], [(1, NT, KV, D)])], [(1, KV, NT, D)], [("perm", "0,2,1,3")])
        q, k = rope(q, NH), rope(k, KV)
        kc = g.node("Concat", [pk, k], [(1, KV, TT, D)], [("axis", "2")], out_names=[f"opkv{2 * l}"])
        vc = g.node("Concat", [pv, v], [(1, KV, TT, D)], [("axis", "2")], out_names=[f"opkv{2 * l + 1}"])
        g.mark_output(kc); g.mark_output(vc)
        kt = g.node("Transpose", [kc], [(1, KV, D, TT)], [("perm", "0,1,3,2")])
        s = g.node("MatMul", [q, kt], [(1, NH, NT, TT)])
        s = g.node("Div", [s, g.scalar(math.sqrt(D))], [(1, NH, NT, TT)])
        s = g.node("Add", [s, mask], [(1, NH, NT, TT)])
        p = g.node("Softmax", [s], [(1, NH, NT, TT)], [("axis", "-1")])
        o = g.node("MatMul", [p, vc], [(1, NH, NT, D)])
        g.flops += 4 * NH * NT * TT * D
        o = g.node("Reshape", [g.node("Transpose", [o], [(1, NT, NH, D)], [("perm", "0,2,1,3")]), g.i64([1, NT, NH * D])], [(1, NT, NH * D)])
        h = g.node("Add", [h, g.linear(o, H, bias=False)], [(1, NT, H)])
        n = rms(h, f"_2F_model_2F_layers_2E_{l}_2F_post_5F_attention_5F_layernorm_2F_")
        gate = g.silu(g.linear(n, cfg.mlp, bias=False))
        up = g.linear(n, cfg.mlp, bias=False)
        h = g.node("Add", [h, g.linear(g.node("Mul", [gate, up], [(1, NT, cfg.mlp)]), H, bias=False)], [(1, NT, H)])
    n = rms(h, "_2F_model_2F_norm_2F_")
    out = g.linear(n, cfg.vocab, bias=False)
    g.lines[-1] = g.lines[-1].replace(out.text(), T("logits", out.shape).text())
    g.mark_output(T("logits", out.shape))
    g.finish()
    return g


def llama_inputs(cfg: LlamaConfig, seed: int = 0, new_tokens: int = 1) -> Dict[str, np.ndarray]:
    """Seeded inputs of emit_llama_decode(cfg, new_tokens=...): token ids, positions past..past+T-1, an all-ones mask and a random cache."""
    rng = np.random.default_rng(2000 + seed)
    d = {"input_5F_ids": rng.integers(0, cfg.vocab, (1, new_tokens)).astype(np.int64),
         "position_5F_ids": np.arange(cfg.past, cfg.past + new_tokens, dtype=np.int64).reshape(1, new_tokens),
         "attention_5F_mask": np.ones((1, cfg.past + new_tokens), np.int64)}
    for l in range(cfg.layers):
        d[f"pkv{2 * l}"] = rng.standard_normal((1, cfg.kv_heads, cfg.past, cfg.head_dim), dtype=np.float32)
        d[f"pkv{2 * l + 1}"] = rng.standard_normal((1, cfg.kv_heads, cfg.past, cfg.head_dim), dtype=np.float32)
    return d
