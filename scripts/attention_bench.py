#!/usr/bin/env python
"""scripts/attention_bench.py -- the SD 1.5 UNet attentions on the GPU: the fused flash kernel (osb_flash_attention) against the
three-kernel path (QK^T GEMM -> scaled softmax -> PV GEMM through an fp16 score buffer) at the shapes of one UNet step, and, with
--trace, attention's share of one eager UNet step from a torch.profiler trace.

Prints ONE JSON line: the card (name, power limit, max SM clock, read with an nvidia-smi query), then
  kernel: per shape (8 heads; T x Tk at the 64^2 / 32^2 / 16^2 / 8^2 levels, self- and cross-attention with the 77-token context;
          d = 40 / 80 / 160 as the level has it), ms per call (CUDA events over --iters calls after warm-up) for
            flash  : osb_flash_attention, where osb_flash_attention_ok accepts the shape (else null)
            chain  : osb_gemm_ld(QK^T, Tk padded to a multiple of 8) -> osb_softmax_scaled_ld -> osb_gemm_ld(PV)
          TFLOP/s as 4*h*T*Tk*d / t, and the share of two floors taken from the shape: ex2 (one MUFU.EX2 per score at 16 per clock
          per SM, 132 SMs, the card's max SM clock) and MMA (the data sheet's 989 TFLOP/s dense fp16 on the padded shapes the kernel
          runs: keys rounded up to its key tile, QK^T contracted over its k-steps of 16, PV n = d rounded up to 64; FLASH_TILES).
          max|flash - chain| on the same inputs.
  vae   : (--vae, instead of kernel) the VAE decoder's mid-block attention, one head at d = 512 with K pre-transposed [d, Tk] as the
          graph has it, at T = Tk = 1024 (32^2 latent) ... 4096 (64^2) and 16384 (128^2), ms per call for
            flash  : osb_flash_attention_wide
            chain  : attention_core's chain: osb_gemm(QK^T) -> osb_softmax_scaled -> osb_gemm(PV) through an fp16 [T, Tk] buffer
          TFLOP/s as 4*T*Tk*d / t; flash_mma_tflops counts the MMA work the kernel issues (Q K^T once per 256-column slice of V, so
          2*T*Tk*d*(slices + 1)); the score buffer the chain allocates; max|flash - chain|.
          tiled: the SD VAE decoder (emit.VAEConfig(), 32 x 32 latent tiles: T = 1024 per tile, the shape where the kernel alone is
          slower than the chain) decoding a 64 x 64 latent as 9 batch siblings of one run (tiled_vae.py), b200_flash_attention on and
          off alternated; device ms per run (last_gpu_ms), median of --tiled-runs runs after 2 warm-up runs each.
  vae --f32: the same shapes in fp32, ms per call for
            flash  : osb_flash_attention_wide_f32x (bf16 triple split; the three plane-split launches included)
            chain  : the fp32 chain: osb_gemm(QK^T) -> osb_softmax_scaled -> osb_gemm(PV) on the CUDA cores through an fp32 [T, Tk]
                     buffer
          TFLOP/s of algorithmic fp32 work (4*T*Tk*d / t); flash_mma_tflops counts the bf16 MMA work the kernel issues (six products in
          Q K^T once per slice and in P V: 6*2*T*Tk*d*(slices + 1)); the chain's score bytes; max|flash - chain|.
          tiled: the SD VAE decoder as above with fp16 weights and fp32 arithmetic (no options: SDXL's default decode).
          whole: the same decoder built for 64 x 64 and 128 x 128 latents decoding untiled, on and off alternated, median device ms of
          --tiled-runs runs after one warm-up run each, and each setting's activation high-water.
  trace : (--trace DIR) per-kernel-name GPU time of one eager SD 1.5 UNet step (64x64 latent, fp16, resident weights, no CUDA graph)
          and the attention share: flash_attention_kernel, softmax_scaled_* and the tensor-core GEMM launched right before and right
          after each softmax (the QK^T / PV pair) over all kernel and memset time.  The chrome trace is written to DIR.
  f32   : (--f32) the fp32 attentions instead of the fp16 ones: the SD 1.5 shapes above and SDXL's d = 64 (10 heads at 64^2 with the
          77-token context, 20 heads at 32^2), ms per call for
            flash  : osb_flash_attention_f32x (bf16 triple split; the plane split launch included)
            chain  : the fp32 chain: osb_gemm_ld(QK^T) -> osb_softmax_scaled_ld -> osb_gemm_ld(PV) on the CUDA cores through an fp32
                     [h, T, Tk padded to 8] score buffer
          TFLOP/s of algorithmic fp32 work (4*h*T*Tk*d / t), the score buffer the chain allocates, max|flash - chain|.  With --trace
          the traced step is the fp32 UNet (fp32 weights and arithmetic).
OSB_ENGINE_LIB selects the engine library (build variants).  Needs a CUDA device; everything else it writes goes to a temporary
directory.
"""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onnxstream_b200 import emit  # noqa: E402
from onnxstream_b200.model import ENGINE_LIB, Model  # noqa: E402

F16, F32 = 2, 3
HEADS = 8
SHAPES = [
    # name, T, Tk, d
    ("64sq_self", 4096, 4096, 40), ("64sq_cross", 4096, 77, 40),
    ("32sq_self", 1024, 1024, 80), ("32sq_cross", 1024, 77, 80),
    ("16sq_self", 256, 256, 160), ("16sq_cross", 256, 77, 160),
    ("8sq_self", 64, 64, 160), ("8sq_cross", 64, 77, 160),
]
SMS, EX2_PER_CLK, MMA_PEAK = 132, 16, 989e12
# osb_flash_attention's instantiations (attention_wgmma.cu): largest d -> (keys per tile, QK^T contraction, PV n)
FLASH_TILES = [(48, 128, 48, 64), (64, 128, 64, 64), (80, 64, 80, 128), (128, 64, 128, 128), (160, 32, 160, 192)]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def kernel_level(iters, warmup, clock_hz):
    import torch
    lib = ctypes.CDLL(ENGINE_LIB)
    vp, i64, cf, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int
    lib.osb_flash_attention.argtypes = [vp, i64, vp, i64, vp, i64, vp, i64, i64, i64, i64, i64, cf, vp]
    lib.osb_flash_attention_ok.argtypes = [i64, i64, i64, ci]
    lib.osb_gemm_ld.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_softmax_scaled_ld.argtypes = [vp, vp, ci, i64, i64, i64, cf, vp, i64, vp]
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = []
    for name, T, Tk, d in SHAPES:
        h, C = HEADS, HEADS * d
        Tkp = (Tk + 7) // 8 * 8
        g = torch.Generator(device="cuda").manual_seed(T * 7 + Tk + d)
        q = torch.randn(T, C, device="cuda", generator=g).half()
        k = torch.zeros(Tkp, C, device="cuda", dtype=torch.half); k[:Tk] = torch.randn(Tk, C, device="cuda", generator=g).half()
        v = torch.zeros(Tkp, C, device="cuda", dtype=torch.half); v[:Tk] = torch.randn(Tk, C, device="cuda", generator=g).half()
        S = torch.empty(h, T, Tkp, device="cuda", dtype=torch.half)
        o_flash = torch.zeros(T, C, device="cuda", dtype=torch.half)
        o_chain = torch.zeros(T, C, device="cuda", dtype=torch.half)
        scale = float(torch.tensor(1.0 / d ** 0.5).half())

        def flash():
            assert lib.osb_flash_attention(q.data_ptr(), C, k.data_ptr(), C, v.data_ptr(), C, o_flash.data_ptr(), C, h, T, Tk, d, scale, stream) == 0

        def chain():
            assert lib.osb_gemm_ld(q.data_ptr(), C, k.data_ptr(), C, S.data_ptr(), Tkp, None, None, h, T, Tkp, d, d, d, T * Tkp, 1, F16, 0, stream) == 0
            assert lib.osb_softmax_scaled_ld(S.data_ptr(), S.data_ptr(), F16, h * T, Tk, Tkp, scale, None, 1, stream) == 0
            assert lib.osb_gemm_ld(S.data_ptr(), Tkp, v.data_ptr(), C, o_chain.data_ptr(), C, None, None, h, T, d, Tkp, T * Tkp, d, d, 0, F16, 0, stream) == 0

        def timed(fn):
            for _ in range(warmup):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / iters

        has_flash = bool(lib.osb_flash_attention_ok(T, Tk, d, F16))
        t_flash = timed(flash) if has_flash else None
        t_chain = timed(chain)
        flop = 4.0 * h * T * Tk * d
        bk, kqk, npv = next((bk, kqk, npv) for dmax, bk, kqk, npv in FLASH_TILES if d <= dmax)
        mma_flop = 2.0 * h * T * (-(-Tk // bk) * bk) * (kqk + npv)
        ex2_s = h * T * Tk / (SMS * EX2_PER_CLK * clock_hz)
        mma_s = mma_flop / MMA_PEAK
        row = {"shape": name, "h": h, "T": T, "Tk": Tk, "d": d, "flash_ms": None if t_flash is None else round(t_flash, 4),
               "chain_ms": round(t_chain, 4), "chain_tflops": round(flop / t_chain / 1e9, 2),
               "ex2_floor_us": round(ex2_s * 1e6, 2), "mma_floor_us": round(mma_s * 1e6, 2)}
        if t_flash is not None:
            row.update({"flash_tflops": round(flop / t_flash / 1e9, 2), "flash_vs_chain": round(t_chain / t_flash, 2),
                        "flash_ex2_floor_share": round(ex2_s * 1e3 / t_flash, 3), "flash_mma_floor_share": round(mma_s * 1e3 / t_flash, 3),
                        "max_abs_diff": float((o_flash.float() - o_chain.float()).abs().max())})
        out.append(row)
        del q, k, v, S, o_flash, o_chain
        torch.cuda.empty_cache()
    return out


# (name, heads, T, Tk, d): the SD 1.5 levels (8 heads) and SDXL's d = 64 levels
F32_SHAPES = [(n, HEADS, T, Tk, d) for n, T, Tk, d in SHAPES] + [("xl_64sq_cross", 10, 4096, 77, 64), ("xl_32sq_self", 20, 1024, 1024, 64)]


def kernel_level_f32(iters, warmup):
    import torch
    lib = ctypes.CDLL(ENGINE_LIB)
    vp, i64, cf, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int
    lib.osb_flash_attention_f32x.argtypes = [vp, i64, vp, i64, vp, i64, vp, i64, i64, i64, i64, i64, cf, vp, vp]
    lib.osb_gemm_ld.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_softmax_scaled_ld.argtypes = [vp, vp, ci, i64, i64, i64, cf, vp, i64, vp]
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = []
    for name, h, T, Tk, d in F32_SHAPES:
        C = h * d
        Tkp = (Tk + 7) // 8 * 8
        g = torch.Generator(device="cuda").manual_seed(T * 7 + Tk + d)
        q = torch.randn(T, C, device="cuda", generator=g)
        k = torch.zeros(Tkp, C, device="cuda"); k[:Tk] = torch.randn(Tk, C, device="cuda", generator=g)
        v = torch.zeros(Tkp, C, device="cuda"); v[:Tk] = torch.randn(Tk, C, device="cuda", generator=g)
        S = torch.empty(h, T, Tkp, device="cuda")
        planes = torch.empty(3 * (T + 2 * Tk) * C, device="cuda", dtype=torch.bfloat16)
        o_flash = torch.zeros(T, C, device="cuda")
        o_chain = torch.zeros(T, C, device="cuda")
        scale = 1.0 / d ** 0.5

        def flash():
            assert lib.osb_flash_attention_f32x(q.data_ptr(), C, k.data_ptr(), C, v.data_ptr(), C, o_flash.data_ptr(), C, h, T, Tk, d, scale,
                                                planes.data_ptr(), stream) == 0

        def chain():
            assert lib.osb_gemm_ld(q.data_ptr(), C, k.data_ptr(), C, S.data_ptr(), Tkp, None, None, h, T, Tkp, d, d, d, T * Tkp, 1, F32, 0, stream) == 0
            assert lib.osb_softmax_scaled_ld(S.data_ptr(), S.data_ptr(), F32, h * T, Tk, Tkp, scale, None, 1, stream) == 0
            assert lib.osb_gemm_ld(S.data_ptr(), Tkp, v.data_ptr(), C, o_chain.data_ptr(), C, None, None, h, T, d, Tkp, T * Tkp, d, d, 0, F32, 0, stream) == 0

        def timed(fn):
            for _ in range(warmup):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / iters

        t_flash, t_chain = timed(flash), timed(chain)
        flop = 4.0 * h * T * Tk * d
        out.append({"shape": name, "h": h, "T": T, "Tk": Tk, "d": d, "flash_ms": round(t_flash, 4), "chain_ms": round(t_chain, 4),
                    "flash_tflops": round(flop / t_flash / 1e9, 2), "chain_tflops": round(flop / t_chain / 1e9, 2),
                    "flash_vs_chain": round(t_chain / t_flash, 2), "score_buffer_mb": round(h * T * Tkp * 4 / 2 ** 20, 1),
                    "max_abs_diff": float((o_flash - o_chain).abs().max())})
        del q, k, v, S, planes, o_flash, o_chain
        torch.cuda.empty_cache()
    return out


VAE_SHAPES = [("vae_32sq", 1024), ("vae_40sq", 1600), ("vae_48sq", 2304), ("vae_56sq", 3136), ("vae_64sq", 4096), ("vae_128sq", 16384)]


def vae_level(iters, warmup):
    import torch
    lib = ctypes.CDLL(ENGINE_LIB)
    vp, i64, cf, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int
    lib.osb_flash_attention_wide.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, cf, ci, ci, vp]
    lib.osb_gemm.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_softmax_scaled.argtypes = [vp, vp, ci, i64, i64, cf, vp, i64, vp]
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    d, out = 512, []
    for name, T in VAE_SHAPES:
        Tk = T
        g = torch.Generator(device="cuda").manual_seed(T + d)
        q = torch.randn(T, d, device="cuda", generator=g).half()
        kt = torch.randn(d, Tk, device="cuda", generator=g).half()
        v = torch.randn(Tk, d, device="cuda", generator=g).half()
        S = torch.empty(T, Tk, device="cuda", dtype=torch.half)
        o_flash = torch.zeros(T, d, device="cuda", dtype=torch.half)
        o_chain = torch.zeros(T, d, device="cuda", dtype=torch.half)
        scale = float(torch.tensor(1.0 / d ** 0.5).half())

        def flash():
            assert lib.osb_flash_attention_wide(q.data_ptr(), kt.data_ptr(), v.data_ptr(), o_flash.data_ptr(), 1, T, Tk, d, scale, 1, F16, stream) == 0

        def chain():
            assert lib.osb_gemm(q.data_ptr(), kt.data_ptr(), S.data_ptr(), None, None, 1, T, Tk, d, T * d, Tk * d, T * Tk, 0, F16, 0, stream) == 0
            assert lib.osb_softmax_scaled(S.data_ptr(), S.data_ptr(), F16, T, Tk, scale, None, T, stream) == 0
            assert lib.osb_gemm(S.data_ptr(), v.data_ptr(), o_chain.data_ptr(), None, None, 1, T, d, Tk, T * Tk, Tk * d, T * d, 0, F16, 0, stream) == 0

        def timed(fn):
            for _ in range(warmup):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / iters

        t_flash, t_chain = timed(flash), timed(chain)
        flop = 4.0 * T * Tk * d
        slices = -(-d // 256)
        out.append({"shape": name, "h": 1, "T": T, "Tk": Tk, "d": d, "flash_ms": round(t_flash, 4), "chain_ms": round(t_chain, 4),
                    "flash_tflops": round(flop / t_flash / 1e9, 2), "chain_tflops": round(flop / t_chain / 1e9, 2),
                    "flash_mma_tflops": round(2.0 * T * Tk * d * (slices + 1) / t_flash / 1e9, 2), "flash_vs_chain": round(t_chain / t_flash, 2),
                    "chain_score_bytes": T * Tk * 2, "max_abs_diff": float((o_flash.float() - o_chain.float()).abs().max())})
        del q, kt, v, S, o_flash, o_chain
        torch.cuda.empty_cache()
    return out


def vae_level_f32(iters, warmup):
    import torch
    lib = ctypes.CDLL(ENGINE_LIB)
    vp, i64, cf, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int
    lib.osb_flash_attention_wide_f32x.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, cf, ci, vp, vp]
    lib.osb_gemm.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, i64, i64, i64, ci, ci, ci, vp]
    lib.osb_softmax_scaled.argtypes = [vp, vp, ci, i64, i64, cf, vp, i64, vp]
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    d, out = 512, []
    for name, T in VAE_SHAPES:
        Tk = T
        g = torch.Generator(device="cuda").manual_seed(T + d)
        q = torch.randn(T, d, device="cuda", generator=g)
        kt = torch.randn(d, Tk, device="cuda", generator=g)
        v = torch.randn(Tk, d, device="cuda", generator=g)
        S = torch.empty(T, Tk, device="cuda")
        planes = torch.empty(3 * (T + 2 * Tk) * d, device="cuda", dtype=torch.bfloat16)
        o_flash = torch.zeros(T, d, device="cuda")
        o_chain = torch.zeros(T, d, device="cuda")
        scale = 1.0 / d ** 0.5

        def flash():
            assert lib.osb_flash_attention_wide_f32x(q.data_ptr(), kt.data_ptr(), v.data_ptr(), o_flash.data_ptr(), 1, T, Tk, d, scale, 1,
                                                     planes.data_ptr(), stream) == 0

        def chain():
            assert lib.osb_gemm(q.data_ptr(), kt.data_ptr(), S.data_ptr(), None, None, 1, T, Tk, d, T * d, Tk * d, T * Tk, 0, F32, 0, stream) == 0
            assert lib.osb_softmax_scaled(S.data_ptr(), S.data_ptr(), F32, T, Tk, scale, None, T, stream) == 0
            assert lib.osb_gemm(S.data_ptr(), v.data_ptr(), o_chain.data_ptr(), None, None, 1, T, d, Tk, T * Tk, Tk * d, T * d, 0, F32, 0, stream) == 0

        def timed(fn):
            for _ in range(warmup):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / iters

        t_flash, t_chain = timed(flash), timed(chain)
        flop = 4.0 * T * Tk * d
        slices = -(-d // 256)
        out.append({"shape": name, "h": 1, "T": T, "Tk": Tk, "d": d, "flash_ms": round(t_flash, 4), "chain_ms": round(t_chain, 4),
                    "flash_tflops": round(flop / t_flash / 1e9, 2), "chain_tflops": round(flop / t_chain / 1e9, 2),
                    "flash_mma_tflops": round(6 * 2.0 * T * Tk * d * (slices + 1) / t_flash / 1e9, 2),
                    "flash_vs_chain": round(t_chain / t_flash, 2), "chain_score_bytes": T * Tk * 4,
                    "max_abs_diff": float((o_flash - o_chain).abs().max())})
        del q, kt, v, S, planes, o_flash, o_chain
        torch.cuda.empty_cache()
    return out


def _vae_models(d, f32):
    """The decoder in d on b200_flash_attention 1 and 0: fp16 arithmetic, or (f32) fp32 arithmetic on the fp16 weights."""
    models = {}
    for flash in (1, 0):
        m = Model(ENGINE_LIB, 0, "ram+nocache")
        for o in (() if f32 else ("use_fp16_arithmetic", "fuse_ops_in_attention")):
            m.set_option(o, True)
        m.lib.model_set_option(m.h, b"b200_resident_weights", 1)
        m.lib.model_set_option(m.h, b"b200_flash_attention", flash)
        m.read_file(d + "model.txt")
        models[flash] = m
    return models


def whole_level(runs):
    import numpy as np
    res = []
    for latent in (64, 128):
        d = tempfile.mkdtemp(prefix="osb200_attn_whole_") + "/"
        try:
            emit.emit_vae_decoder(d, emit.VAEConfig(latent=latent), "float16")
            x = np.random.default_rng(0).standard_normal((1, 4, latent, latent)).astype(np.float32)
            models = _vae_models(d, True)
            ms, imgs, hw = {1: [], 0: []}, {}, {}
            for i in range(runs + 1):
                for flash in (1, 0):
                    m = models[flash]
                    m.clear_tensors()
                    m.add_tensor("input_2E_1", x)
                    m.run()
                    if i == runs:
                        imgs[flash] = m.get_tensor("outsample")
                    if i >= 1:
                        ms[flash].append(m.stats()["last_gpu_ms"])
            for f, m in models.items():
                hw[f] = int(m.stats()["act_high_water_bytes"])
                m.close()
        finally:
            shutil.rmtree(d, ignore_errors=True)
        med = {f: float(np.median(v)) for f, v in ms.items()}
        res.append({"latent": latent, "T": latent * latent, "flash_ms": round(med[1], 3), "chain_ms": round(med[0], 3),
                    "flash_runs_ms": [round(x, 3) for x in ms[1]], "chain_runs_ms": [round(x, 3) for x in ms[0]],
                    "flash_act_high_water_mb": round(hw[1] / 2 ** 20, 1), "chain_act_high_water_mb": round(hw[0] / 2 ** 20, 1),
                    "max_abs_diff": float(np.abs(imgs[1] - imgs[0]).max())})
    return res


def tiled_level(runs, f32=False):
    import numpy as np
    from onnxstream_b200 import tiled_vae as tv
    d = tempfile.mkdtemp(prefix="osb200_attn_tiled_") + "/"
    try:
        emit.emit_vae_decoder(d, emit.VAEConfig(latent=32), "float16")
        latent = np.random.default_rng(0).standard_normal((1, 4, 64, 64)).astype(np.float32)
        models = _vae_models(d, f32)
        ms, imgs, tiles = {1: [], 0: []}, {}, 0
        for i in range(runs + 2):
            for flash in (1, 0):
                imgs[flash], tiles = tv.tiled_decode(models[flash], latent, "input_2E_1", "outsample")
                if i >= 2:
                    ms[flash].append(models[flash].stats()["last_gpu_ms"])
        launches = {f: int(models[f].stats()["kernel_launches"]) for f in (1, 0)}
        for m in models.values():
            m.close()
    finally:
        shutil.rmtree(d, ignore_errors=True)
    med = {f: float(np.median(v)) for f, v in ms.items()}
    return {"tiles": tiles, "tile_T": 1024, "flash_ms": round(med[1], 3), "chain_ms": round(med[0], 3), "flash_runs_ms": [round(x, 3) for x in ms[1]],
            "chain_runs_ms": [round(x, 3) for x in ms[0]], "launches_flash": launches[1], "launches_chain": launches[0],
            "max_abs_diff": float(np.abs(imgs[1] - imgs[0]).max())}


def trace_step(trace_dir, f32=False):
    """One eager SD 1.5 UNet step (fp16, or f32: fp32 weights and arithmetic) under torch.profiler (CUDA activities); per-kernel GPU time
    and attention's share of it."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    cfg = emit.UNetConfig.sd15(64)
    d = tempfile.mkdtemp(prefix="osb200_attn_trace_") + "/"
    try:
        emit.emit_unet(d, cfg, "float32" if f32 else "float16", seed=0)
        inputs = emit.unet_inputs(cfg)
        m = Model(ENGINE_LIB, 0, "ram+nocache")
        for o in (() if f32 else ("use_fp16_arithmetic", "fuse_ops_in_attention")):
            m.set_option(o, True)
        m.lib.model_set_option(m.h, b"b200_resident_weights", 1)
        m.lib.model_set_option(m.h, b"b200_cuda_graph", 0)
        m.read_file(d + "model.txt")

        def step():
            m.clear_tensors()
            for k, v in inputs.items():
                m.add_tensor(k, v)
            m.run()

        for _ in range(3):
            step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        gpu_ms = m.stats()["last_gpu_ms"]
        launches = int(m.stats()["kernel_launches"])
        m.close()
    finally:
        shutil.rmtree(d, ignore_errors=True)
    os.makedirs(trace_dir, exist_ok=True)
    path = os.path.join(trace_dir, "unet_step.pt.trace.json")
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset")]
    ev.sort(key=lambda e: e["ts"])
    attn = [False] * len(ev)
    for i, e in enumerate(ev):
        n = e["name"]
        if "flash_attention_kernel" in n or "flash_attention_f32x_kernel" in n or "f32x_split_kernel" in n:
            attn[i] = True
        elif "softmax_scaled" in n:
            attn[i] = True
            s = e["args"].get("stream")
            # the QK^T GEMM (and the pad memsets before it) and the PV GEMM on the same stream
            j = i - 1
            while j >= 0 and ev[j]["args"].get("stream") != s:
                j -= 1
            if j >= 0 and ("tc_gemm" in ev[j]["name"] or "igemm" in ev[j]["name"]):
                attn[j] = True
                j -= 1
                while j >= 0 and (ev[j]["args"].get("stream") != s or ev[j]["cat"] == "gpu_memset"):
                    if ev[j]["args"].get("stream") == s:
                        attn[j] = True
                    j -= 1
            j = i + 1
            while j < len(ev) and ev[j]["args"].get("stream") != s:
                j += 1
            if j < len(ev) and ("tc_gemm" in ev[j]["name"] or "igemm" in ev[j]["name"]):
                attn[j] = True
    total = sum(e["dur"] for e in ev)
    attn_us = sum(e["dur"] for e, a in zip(ev, attn) if a)
    by_name = {}
    for e in ev:
        k = e["name"].replace("(anonymous namespace)::", "").replace("void ", "").split("(")[0][:80]
        t = by_name.setdefault(k, [0, 0.0])
        t[0] += 1
        t[1] += e["dur"]
    top = sorted(by_name.items(), key=lambda kv: -kv[1][1])[:15]
    return {"step_gpu_ms": round(gpu_ms, 3), "engine_launches": launches, "traced_kernels_and_memsets": len(ev),
            "kernel_ms": round(total / 1e3, 3), "attention_ms": round(attn_us / 1e3, 3), "attention_calls": sum(attn),
            "attention_share_of_kernel_time": round(attn_us / total, 4) if total else None,
            "top": [{"name": k, "count": c, "ms": round(t / 1e3, 3)} for k, (c, t) in top], "trace": path}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=50, help="timed calls per path and shape")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--trace", default=None, metavar="DIR", help="also trace one eager UNet step and write the chrome trace to DIR")
    ap.add_argument("--skip-kernels", action="store_true")
    ap.add_argument("--vae", action="store_true", help="time the VAE's d = 512 attention shapes instead of the UNet's")
    ap.add_argument("--f32", action="store_true", help="time the fp32 attentions (and trace the fp32 UNet) instead of the fp16 ones")
    ap.add_argument("--tiled-runs", type=int, default=7, help="--vae: timed tiled decodes per setting (0 = skip)")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("attention_bench.py needs a CUDA device")
    c = card()
    res = {"card": c, "engine_lib": os.path.basename(ENGINE_LIB)}
    if a.vae:
        res["vae"] = vae_level_f32(a.iters, a.warmup) if a.f32 else vae_level(a.iters, a.warmup)
        if a.tiled_runs:
            res["tiled"] = tiled_level(a.tiled_runs, a.f32)
            if a.f32:
                res["whole"] = whole_level(a.tiled_runs)
    elif a.f32 and not a.skip_kernels:
        res["kernel"] = kernel_level_f32(a.iters, a.warmup)
    elif not a.skip_kernels:
        res["kernel"] = kernel_level(a.iters, a.warmup, float(c["max_sm_clock"].split()[0]) * 1e6)
    if a.trace:
        res["trace"] = trace_step(a.trace, a.f32)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
