// kernels_basic.cu -- bandwidth-bound node kernels for sm_90a: dtype conversion, unary / broadcasting binary
// elementwise, strided copies (transpose / concat / slice / expand / nearest resize), softmax, InstanceNorm,
// fused GroupNorm(+SiLU), fused LayerNorm, ReduceMean, row gather.  Each replaces an XnnPack method or an inline
// pthreadpool lambda of the reference's Model::run(); see include/onnxstream_b200_kernels.h for file:line citations.
//
// Design rules (HBM-bound work): 128-bit vectorised accesses where alignment allows, grid-stride loops sized as a
// multiple of the SM count, fp32 math on fp16 storage, every tensor read once and written once.

#include "common.cuh"
#include <cuda_bf16.h>
#include <cstring>
#include "workspace.h"
#include <cstdio>
#include <cstdlib>

namespace {

// ------------------------------------------------------------------------------------------------------------
// convert
// ------------------------------------------------------------------------------------------------------------

template <typename S, typename D>
__global__ void convert_kernel(const S* __restrict__ src, D* __restrict__ dst, size_t n)
{
    osb_pdl_prologue();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = from_float<D>(to_float(src[i]));
}

template <typename D>
__global__ void dequant_kernel(const uint8_t* __restrict__ src, D* __restrict__ dst, size_t n, float scale, int zp)
{
    osb_pdl_prologue();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = from_float<D>((float)((int)src[i] - zp) * scale);
}

template <typename S>
__global__ void quant_kernel(const S* __restrict__ src, uint8_t* __restrict__ dst, size_t n, float scale, int zp)
{
    osb_pdl_prologue();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        // XNNPACK f32-qu8-vcvt (xnn_run_convert_nc_f32_qu8): x * (1 / scale), clamp to [0 - zp, 255 - zp], round to nearest even, + zp
        float q = to_float(src[i]) * (1.0f / scale);
        q = fminf(fmaxf(q, (float)(0 - zp)), (float)(255 - zp));
        dst[i] = (uint8_t)((int)rintf(q) + zp);
    }
}

__global__ void i64_to_float_kernel(const int64_t* __restrict__ src, float* __restrict__ dst, size_t n)
{
    osb_pdl_prologue();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = (float)src[i];
}

// ------------------------------------------------------------------------------------------------------------
// unary
// ------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ float apply_unary(int op, float x, float alpha)
{
    switch (op) {
    case OSB_UN_SIGMOID: return 1.f / (1.f + expf(-x));
    case OSB_UN_SILU: return x / (1.f + expf(-x));
    case OSB_UN_ERF: return erff(x);
    case OSB_UN_SQRT: return sqrtf(x);
    case OSB_UN_SIN: return sinf(x);
    case OSB_UN_COS: return cosf(x);
    case OSB_UN_POW: return alpha == 2.f ? x * x : powf(x, alpha);
    case OSB_UN_NEG: return -x;
    case OSB_UN_GELU_ERF: return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
    case OSB_UN_MULC: return x * alpha;
    case OSB_UN_ADDC: return x + alpha;
    case OSB_UN_RECIP_SQRT: return rsqrtf(x);
    default: return x;
    }
}

template <typename T, int VEC>
__global__ void unary_kernel(int op, const T* __restrict__ x, T* __restrict__ y, size_t n, float alpha)
{
    osb_pdl_prologue();
    size_t nvec = n / VEC;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        Vec<T, VEC> v = load_vec<T, VEC>(x + i * VEC);
#pragma unroll
        for (int k = 0; k < VEC; k++) v.v[k] = from_float<T>(apply_unary(op, to_float(v.v[k]), alpha));
        store_vec<T, VEC>(y + i * VEC, v);
    }
    if (blockIdx.x == 0) {
        for (size_t i = nvec * VEC + threadIdx.x; i < n; i += blockDim.x)
            y[i] = from_float<T>(apply_unary(op, to_float(x[i]), alpha));
    }
}

// ------------------------------------------------------------------------------------------------------------
// binary with broadcasting
// ------------------------------------------------------------------------------------------------------------

struct BinParams {
    int64_t shape[OSB_MAX_DIMS];
    int64_t as[OSB_MAX_DIMS];
    int64_t bs[OSB_MAX_DIMS];
    int ndim;
};

// fast path: both operands contiguous & same shape, or one of them a scalar
template <typename T, int VEC>
__global__ void binary_flat_kernel(int op, const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out, size_t n, int a_scalar, int b_scalar)
{
    osb_pdl_prologue();
    float sa = a_scalar ? to_float(a[0]) : 0.f, sb = b_scalar ? to_float(b[0]) : 0.f;
    size_t nvec = n / VEC;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        Vec<T, VEC> va, vb, vo;
        if (!a_scalar) va = load_vec<T, VEC>(a + i * VEC);
        if (!b_scalar) vb = load_vec<T, VEC>(b + i * VEC);
#pragma unroll
        for (int k = 0; k < VEC; k++)
            vo.v[k] = from_float<T>(apply_binary(op, a_scalar ? sa : to_float(va.v[k]), b_scalar ? sb : to_float(vb.v[k])));
        store_vec<T, VEC>(out + i * VEC, vo);
    }
    if (blockIdx.x == 0)
        for (size_t i = nvec * VEC + threadIdx.x; i < n; i += blockDim.x)
            out[i] = from_float<T>(apply_binary(op, a_scalar ? sa : to_float(a[i]), b_scalar ? sb : to_float(b[i])));
}

// inner-broadcast path: out[r, c] = a[r, c] (op) b[c]  (or b[r]); covers bias adds and gamma/beta in channel-last tensors
template <typename T, int VEC>
__global__ void binary_rowcol_kernel(int op, const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out,
                                     int64_t rows, int64_t cols, int b_per_row, int swap)
{
    osb_pdl_prologue();
    int64_t cvec = cols / VEC;
    int64_t total = rows * cvec;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = i / cvec, c = (i % cvec) * VEC;
        Vec<T, VEC> va = load_vec<T, VEC>(a + r * cols + c), vb, vo;
        float sb = 0.f;
        if (b_per_row) sb = to_float(b[r]); else vb = load_vec<T, VEC>(b + c);
#pragma unroll
        for (int k = 0; k < VEC; k++) {
            float x = to_float(va.v[k]), y = b_per_row ? sb : to_float(vb.v[k]);
            vo.v[k] = from_float<T>(swap ? apply_binary(op, y, x) : apply_binary(op, x, y));
        }
        store_vec<T, VEC>(out + r * cols + c, vo);
    }
}

// GEGLU: x is [rows, 2*inner]; out[r, c] = x[r, c] * gelu_erf(x[r, inner + c]) -- the two Slices, the Erf chain and the Mul of
// the feed-forward gate in one pass (same arithmetic as OSB_BIN_MUL_GELU on materialised halves)
template <typename T, int VEC>
__global__ void geglu_kernel(const T* __restrict__ x, T* __restrict__ out, int64_t rows, int64_t inner)
{
    osb_pdl_prologue();
    int64_t cvec = inner / VEC;
    int64_t total = rows * cvec;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = i / cvec, c = (i % cvec) * VEC;
        Vec<T, VEC> va = load_vec<T, VEC>(x + r * 2 * inner + c), vb = load_vec<T, VEC>(x + r * 2 * inner + inner + c), vo;
#pragma unroll
        for (int k = 0; k < VEC; k++) vo.v[k] = from_float<T>(apply_binary(OSB_BIN_MUL_GELU, to_float(va.v[k]), to_float(vb.v[k])));
        store_vec<T, VEC>(out + r * inner + c, vo);
    }
}

template <typename T>
__global__ void binary_generic_kernel(int op, const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out, BinParams p, size_t n)
{
    osb_pdl_prologue();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        size_t rem = i;
        int64_t ao = 0, bo = 0;
#pragma unroll
        for (int d = OSB_MAX_DIMS - 1; d >= 0; d--) {
            if (d < p.ndim) {
                int64_t idx = rem % p.shape[d];
                rem /= p.shape[d];
                ao += idx * p.as[d];
                bo += idx * p.bs[d];
            }
        }
        out[i] = from_float<T>(apply_binary(op, to_float(a[ao]), to_float(b[bo])));
    }
}


// XNNPACK qu8 elementwise add / multiply (xnn_run_binary_elementwise_nd with xnn_datatype_quint8, called at src/onnxstream.cpp:846-927
// and 1666-1746), restated and pinned bit-exact against the reference run (tests/test_cpu.py):
//   add: fixed point.  shift = 20 - exponent(max(|sa/so|, |sb/so|)); multipliers = lrintf(|s/so| * 2^shift);
//        acc = 2^(shift-1) - ma*za - mb*zb + a*ma + b*mb;  y = clamp(acc >> shift, -zo, 255 - zo) + zo
//   mul: acc = (a - za)(b - zb);  y = lrintf(clamp(acc * (sa*sb/so), -zo, 255 - zo)) + zo
struct Qu8BinParams { int op; int za, zb, zo; int ma, mb, shift, bias; float mul_scale; };

__global__ void binary_qu8_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, uint8_t* __restrict__ out, BinParams p, size_t n, Qu8BinParams q)
{
    osb_pdl_prologue();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        size_t rem = i;
        int64_t ao = 0, bo = 0;
#pragma unroll
        for (int d = OSB_MAX_DIMS - 1; d >= 0; d--) {
            if (d < p.ndim) {
                int64_t idx = rem % p.shape[d];
                rem /= p.shape[d];
                ao += idx * p.as[d];
                bo += idx * p.bs[d];
            }
        }
        const int va = a[ao], vb = b[bo];
        int y;
        if (q.op == OSB_BIN_ADD) {
            int acc = q.bias + va * q.ma + vb * q.mb;
            y = acc >> q.shift;                                   // arithmetic shift (math_asr_s32)
            y = max(y, 0 - q.zo); y = min(y, 255 - q.zo);
        } else {
            float f = (float)((va - q.za) * (vb - q.zb)) * q.mul_scale;
            f = fminf(fmaxf(f, (float)(0 - q.zo)), (float)(255 - q.zo));
            y = (int)rintf(f);
        }
        out[i] = (uint8_t)(y + q.zo);
    }
}

// qu8 softmax restated as plain arithmetic (dequantise with zero point 0, float softmax, requantise; XNNPACK's LUT rounding is not reproduced): the
// reference calls xnn_*_softmax_nc_qu8 (src/onnxstream.cpp:1958-2051) with output scale 2^-8 and zero point 0 (5971-5972).
__global__ void softmax_qu8_kernel(const uint8_t* __restrict__ x, uint8_t* __restrict__ y, int64_t rows, int64_t cols, float in_scale, float out_scale, int out_zp)
{
    osb_pdl_prologue();
    __shared__ float red[32];
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const uint8_t* xr = x + r * cols; uint8_t* yr = y + r * cols;
        float m = -INFINITY;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) m = fmaxf(m, (float)xr[c] * in_scale);
        m = block_reduce_max(m, red);
        float s = 0.f;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) s += expf((float)xr[c] * in_scale - m);
        s = block_reduce_sum(s, red);
        const float inv = 1.0f / s;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) {
            float v = expf((float)xr[c] * in_scale - m) * inv;
            long q = lrintf(v / out_scale) + out_zp;
            yr[c] = (uint8_t)(q < 0 ? 0 : (q > 255 ? 255 : q));
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------------------
// strided copy
// ------------------------------------------------------------------------------------------------------------

struct CopyParams {
    int64_t shape[OSB_MAX_DIMS];
    int64_t is[OSB_MAX_DIMS];
    int64_t idiv[OSB_MAX_DIMS];
    int64_t os[OSB_MAX_DIMS];
    int64_t in_off, out_off;
    int ndim;
};

template <typename T>
__global__ void strided_copy_kernel(const T* __restrict__ in, T* __restrict__ out, CopyParams p, size_t n)
{
    osb_pdl_prologue();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        size_t rem = i;
        int64_t io = p.in_off, oo = p.out_off;
#pragma unroll
        for (int d = OSB_MAX_DIMS - 1; d >= 0; d--) {
            if (d < p.ndim) {
                int64_t idx = rem % p.shape[d];
                rem /= p.shape[d];
                io += (idx / p.idiv[d]) * p.is[d];
                oo += idx * p.os[d];
            }
        }
        out[oo] = in[io];
    }
}

// [B, R, C] -> [B, C, R] through a 32x33 shared tile (coalesced on both sides)
template <typename T>
__global__ void transpose2d_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t rows, int64_t cols)
{
    osb_pdl_prologue();
    __shared__ T tile[32][33];
    int64_t b = blockIdx.z;
    const T* src = in + b * rows * cols;
    T* dst = out + b * rows * cols;
    int64_t c0 = (int64_t)blockIdx.x * 32, r0 = (int64_t)blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        int64_t r = r0 + j, c = c0 + threadIdx.x;
        if (r < rows && c < cols) tile[j][threadIdx.x] = src[r * cols + c];
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        int64_t c = c0 + j, r = r0 + threadIdx.x;
        if (r < rows && c < cols) dst[c * rows + r] = tile[threadIdx.x][j];
    }
}

// ------------------------------------------------------------------------------------------------------------
// reductions: softmax / layernorm / reduce-mean (one CTA per row, row cached in registers when it fits)
// ------------------------------------------------------------------------------------------------------------

template <typename T>
__global__ void softmax_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t rows, int64_t cols)
{
    osb_pdl_prologue();
    __shared__ float red[32];
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const T* xr = x + r * cols;
        T* yr = y + r * cols;
        float mx = -INFINITY;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) mx = fmaxf(mx, to_float(xr[c]));
        mx = block_reduce_max(mx, red);
        float sum = 0.f;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) sum += expf(to_float(xr[c]) - mx);
        sum = block_reduce_sum(sum, red);
        float inv = 1.f / sum;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) yr[c] = from_float<T>(expf(to_float(xr[c]) - mx) * inv);
    }
}

template <typename T>
__global__ void layer_norm_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t rows, int64_t cols,
                                  const T* __restrict__ gamma, const T* __restrict__ beta, float eps)
{
    osb_pdl_prologue();
    __shared__ float red[32];
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const T* xr = x + r * cols;
        T* yr = y + r * cols;
        float s = 0.f;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) s += to_float(xr[c]);
        float mean = block_reduce_sum(s, red) / (float)cols;
        float v = 0.f;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) { float d = to_float(xr[c]) - mean; v += d * d; }
        float var = block_reduce_sum(v, red) / (float)cols;
        float rstd = 1.f / sqrtf(var + eps);
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) {
            float o = (to_float(xr[c]) - mean) * rstd;
            if (gamma) o *= to_float(gamma[c]);
            if (beta) o += to_float(beta[c]);
            yr[c] = from_float<T>(o);
        }
    }
}

// LayerNorm, one warp per row, the row held in registers (cols <= 64 * ITERS, cols even): one global read, shuffle reductions
// only, same two-pass mean / variance arithmetic as the block kernel above.  Every load of a phase is issued before the first
// use (a load inside an `if (c < cols) { ...accumulate... }` body serialises the row on memory latency -- measured 2x slower).
constexpr int LN_MAX_ITERS = 20;
template <typename T, int ITERS>
__global__ void __launch_bounds__(128)
layer_norm_warp_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t rows, int cols,
                       const T* __restrict__ gamma, const T* __restrict__ beta, float eps)
{
    osb_pdl_prologue();
    const int lane = threadIdx.x & 31;
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= rows) return;
    const T* xr = x + r * cols;
    T* yr = y + r * cols;
    Vec<T, 2> raw[ITERS], gr[ITERS], br[ITERS];
#pragma unroll
    for (int i = 0; i < ITERS; i++) {
        int c = lane * 2 + i * 64;
        raw[i].v[0] = from_float<T>(0.f); raw[i].v[1] = from_float<T>(0.f);
        if (c < cols) raw[i] = load_vec<T, 2>(xr + c);
    }
#pragma unroll
    for (int i = 0; i < ITERS; i++) {
        int c = lane * 2 + i * 64;
        gr[i].v[0] = from_float<T>(1.f); gr[i].v[1] = from_float<T>(1.f);
        br[i].v[0] = from_float<T>(0.f); br[i].v[1] = from_float<T>(0.f);
        if (gamma && c < cols) gr[i] = load_vec<T, 2>(gamma + c);
        if (beta && c < cols) br[i] = load_vec<T, 2>(beta + c);
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < ITERS; i++) s += to_float(raw[i].v[0]) + to_float(raw[i].v[1]);   // padding lanes hold zeros
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)cols;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < ITERS; i++) {
        int c = lane * 2 + i * 64;
        float d0 = to_float(raw[i].v[0]) - mean, d1 = to_float(raw[i].v[1]) - mean;
        q += c < cols ? d0 * d0 + d1 * d1 : 0.f;
    }
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = 1.f / sqrtf(q / (float)cols + eps);
#pragma unroll
    for (int i = 0; i < ITERS; i++) {
        int c = lane * 2 + i * 64;
        float o0 = (to_float(raw[i].v[0]) - mean) * rstd, o1 = (to_float(raw[i].v[1]) - mean) * rstd;
        if (gamma) { o0 *= to_float(gr[i].v[0]); o1 *= to_float(gr[i].v[1]); }
        if (beta) { o0 += to_float(br[i].v[0]); o1 += to_float(br[i].v[1]); }
        Vec<T, 2> w; w.v[0] = from_float<T>(o0); w.v[1] = from_float<T>(o1);
        if (c < cols) store_vec<T, 2>(yr + c, w);
    }
}

template <typename T>
__global__ void reduce_mean_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t rows, int64_t cols)
{
    osb_pdl_prologue();
    __shared__ float red[32];
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const T* xr = x + r * cols;
        float s = 0.f;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) s += to_float(xr[c]);
        s = block_reduce_sum(s, red);
        if (threadIdx.x == 0) y[r] = from_float<T>(s / (float)cols);
    }
}

// ------------------------------------------------------------------------------------------------------------
// InstanceNorm on [C, N]: one CTA cluster-free design -- grid (C, splits); stats via fp32 partials + double finish
// ------------------------------------------------------------------------------------------------------------

// pass 1: per (channel, split) partial sum and sum of squares, accumulated in double like the reference.
template <typename T>
__global__ void inorm_stats_kernel(const T* __restrict__ x, double* __restrict__ partial, int64_t n_per_c, int splits)
{
    osb_pdl_prologue();
    __shared__ double red[64];
    int64_t c = blockIdx.x;
    int s = blockIdx.y;
    int64_t chunk = (n_per_c + splits - 1) / splits;
    int64_t lo = s * chunk, hi = min(lo + chunk, n_per_c);
    const T* xc = x + c * n_per_c;
    double sum = 0.0, sq = 0.0;
    for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) { double v = (double)to_float(xc[i]); sum += v; sq += v * v; }
    // block reduce (double)
    for (int o = 16; o > 0; o >>= 1) { sum += __shfl_xor_sync(0xffffffffu, sum, o); sq += __shfl_xor_sync(0xffffffffu, sq, o); }
    int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (l == 0) { red[w] = sum; red[32 + w] = sq; }
    __syncthreads();
    if (w == 0) {
        sum = l < nw ? red[l] : 0.0; sq = l < nw ? red[32 + l] : 0.0;
        for (int o = 16; o > 0; o >>= 1) { sum += __shfl_xor_sync(0xffffffffu, sum, o); sq += __shfl_xor_sync(0xffffffffu, sq, o); }
        if (l == 0) { partial[(c * splits + s) * 2] = sum; partial[(c * splits + s) * 2 + 1] = sq; }
    }
}

template <typename T>
__global__ void inorm_apply_kernel(const T* __restrict__ x, T* __restrict__ y, const double* __restrict__ partial, int64_t n_per_c, int splits,
                                   const T* __restrict__ scale, const T* __restrict__ bias, float eps)
{
    osb_pdl_prologue();
    int64_t c = blockIdx.x;
    double sum = 0.0, sq = 0.0;
    for (int s = 0; s < splits; s++) { sum += partial[(c * splits + s) * 2]; sq += partial[(c * splits + s) * 2 + 1]; }
    double mean = sum / (double)n_per_c;
    double var = sq / (double)n_per_c - mean * mean;
    if (var < 0) var = 0;
    float rstd = (float)(1.0 / sqrt(var + (double)eps));
    float g = scale ? to_float(scale[c]) : 1.f, b = bias ? to_float(bias[c]) : 0.f;
    float m = (float)mean;
    int64_t chunk = (n_per_c + gridDim.y - 1) / gridDim.y;
    int64_t lo = blockIdx.y * chunk, hi = min(lo + chunk, n_per_c);
    const T* xc = x + c * n_per_c;
    T* yc = y + c * n_per_c;
    for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) yc[i] = from_float<T>((to_float(xc[i]) - m) * rstd * g + b);
}

// ------------------------------------------------------------------------------------------------------------
// GroupNorm (+SiLU) on [C, HW] (NCHW) or [HW, C] (NHWC)
// ------------------------------------------------------------------------------------------------------------

// osb_group_norm's statistics are taken around a per-group pivot p, the group's first element in memory (NHWC: its first channel at
// pixel 0; NCHW: the start of its slab), which every CTA reads alike: stats = fp64 sums of the fp32 partials of x - p and (x - p)^2, and
// the readers form mean = p + S/n, var = Q/n - (S/n)^2.  Plain sums of x and x^2 cancel in E[x^2] - mean^2 when the mean is large
// against the spread (x = 1024 + N(0,1) in fp16: rstd up to 9 % off).  The stats stay fp64 sums of fp32 partials; only what is
// summed moved, so the producers and the scratch layout are unchanged.
__device__ __forceinline__ void gn_mean_var(const double* stats, int g, double inv_n, float p, double& mean, double& var)
{
    const double s = stats[2 * g] * inv_n;
    mean = (double)p + s;
    var = stats[2 * g + 1] * inv_n - s * s;
}

// NCHW: group g = contiguous slab of (C/G)*HW elements -> same as instance norm stats with C := G.
// NHWC: each pixel row holds C channels; a CTA takes a strip of pixels, accumulates per-channel partials in registers
// (thread t owns channels t, t+blockDim, ...), folds them to groups through shared memory, then atomically adds to stats.
template <typename T>
__global__ void gn_stats_nhwc_kernel(const T* __restrict__ x, double* __restrict__ stats, int64_t C, int64_t HW, int groups, int64_t pix_per_cta)
{
    osb_pdl_prologue();
    extern __shared__ float sm[];  // 2 * groups
    for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    int64_t p0 = (int64_t)blockIdx.x * pix_per_cta, p1 = min(p0 + pix_per_cta, HW);
    int cpg = (int)(C / groups);
    for (int64_t c = threadIdx.x; c < C; c += blockDim.x) {
        int g = (int)(c / cpg);
        const float pv = to_float(x[(int64_t)g * cpg]);
        float s = 0.f, q = 0.f;
        for (int64_t p = p0; p < p1; p++) { float v = to_float(x[p * C + c]) - pv; s += v; q += v * v; }
        atomicAdd(&sm[2 * g], s);
        atomicAdd(&sm[2 * g + 1], q);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) atomicAdd(&stats[i], (double)sm[i]);
}

// y's value at pixel 0, channel c (y = x, x + addv[c] rounded to T, or channel c of the concatenation [x | xb] with ca channels from x):
// the pivot of the group that starts at channel c, which every CTA computes alike
template <typename T, bool CAT>
__device__ __forceinline__ float gn_first_y(const T* __restrict__ x, const T* __restrict__ addv, int c, const T* __restrict__ xb, int ca)
{
    if (CAT) return to_float(c < ca ? x[c] : xb[c - ca]);
    const float v = to_float(x[c]);
    return addv ? to_float(from_float<T>(v + to_float(addv[c]))) : v;
}

// NHWC statistics, vectorised: a thread owns 8 consecutive channels (one 16-byte load per pixel) and walks down the
// CTA's pixel strip; 256/(C/8) pixels are in flight per iteration.  Per-channel fp32 partials of y - p (p: the group's pivot,
// gn_first_y) go to shared memory, are folded per group in fp64, then one double atomic per bin and CTA.
template <typename T, int VEC, bool CAT = false>
__global__ void gn_stats_nhwc_vec_kernel(const T* __restrict__ x, double* __restrict__ stats, int C, int64_t HW, int groups, int64_t pix_per_cta,
                                         const T* __restrict__ addv, T* __restrict__ y, int pivot, const T* __restrict__ xb, int ca)
{
    // CAT: y = the channel concatenation of x [HW, ca] and xb [HW, C - ca] (ca % VEC == 0: a thread's channels come from one source),
    // copied on the way; the statistics are those of y as for the Add.
    // addv / y != null: y = x + addv[c] (the per-channel time-embedding add of a resnet) is written on the way and the statistics
    // are those of y -- the producer side of a GroupNorm whose apply pass is gn_apply_pre_kernel.  pivot != 0: the sums of y - p
    // go out as they are (osb_group_norm's layout, see gn_mean_var); else they are shifted back to plain sums of y and y^2, which
    // gn_apply_pre_kernel reads: S += s + n p, Q += q + 2 p s + n p^2 in fp64 with n the CTA's element count of the group.  Plain fp32
    // sums of y and y^2 would cancel in E[y^2] - mean^2 when the mean is large against the spread.
    osb_pdl_prologue();
    extern __shared__ float sm[];  // the group pivots (groups of the 2 * groups floats), then the per-row partials
    for (int g = threadIdx.x; g < groups; g += blockDim.x) sm[g] = gn_first_y<T, CAT>(x, addv, g * (C / groups), xb, ca);
    __syncthreads();
    const int tpp = C / VEC;                        // threads per pixel
    const int rows = blockDim.x / tpp;              // pixels in flight
    const int cv = threadIdx.x % tpp, pr = threadIdx.x / tpp;
    // where this thread's channels are read: x + pixel * C, or (CAT) its source's channel offset and pixel stride
    const T* src = x + cv * VEC;
    int64_t src_ld = C;
    if (CAT) { if (cv * VEC < ca) src_ld = ca; else { src = xb + (cv * VEC - ca); src_ld = C - ca; } }
    int64_t p0 = (int64_t)blockIdx.x * pix_per_cta, p1 = min(p0 + pix_per_cta, HW);
    const int cpg = C / groups;
    if (pr < rows) {
        float s[VEC], q[VEC], a[VEC], pv[VEC];
#pragma unroll
        for (int k = 0; k < VEC; k++) { s[k] = 0.f; q[k] = 0.f; a[k] = 0.f; pv[k] = sm[(cv * VEC + k) / cpg]; }
        if (addv) {
            Vec<T, VEC> av = load_vec<T, VEC>(addv + cv * VEC);
#pragma unroll
            for (int k = 0; k < VEC; k++) a[k] = to_float(av.v[k]);
        }
        // 4 pixels (independent 16-byte loads) in flight per thread
        for (int64_t pb = p0 + pr; pb < p1; pb += 4 * (int64_t)rows) {
            Vec<T, VEC> v[4];
#pragma unroll
            for (int u = 0; u < 4; u++) { const int64_t p = pb + u * (int64_t)rows; if (p < p1) v[u] = load_vec<T, VEC>(src + p * src_ld); }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int64_t p = pb + u * (int64_t)rows;
                if (p >= p1) break;
                if (y) {
                    if (!CAT) {
#pragma unroll
                        for (int k = 0; k < VEC; k++) v[u].v[k] = from_float<T>(to_float(v[u].v[k]) + a[k]);
                    }
                    store_vec<T, VEC>(y + p * C + cv * VEC, v[u]);
                }
#pragma unroll
                for (int k = 0; k < VEC; k++) { float f = to_float(v[u].v[k]) - pv[k]; s[k] += f; q[k] += f * f; }
            }
        }
        // per-thread partials -> shared [rows][2][C] (no atomics: 256 threads hammering 2 * groups shared addresses serialise)
        float* part = sm + 2 * groups;
#pragma unroll
        for (int k = 0; k < VEC; k++) { part[(pr * 2 + 0) * C + cv * VEC + k] = s[k]; part[(pr * 2 + 1) * C + cv * VEC + k] = q[k]; }
    }
    __syncthreads();
    {
        // bin b = 2 g + which (which: 0 = sum, 1 = sum of squares) is summed in fp64 by tpb adjacent threads, each taking every tpb-th
        // of its rows x cpg partials, then combined by shuffle; bins 2 g and 2 g + 1 sit in one warp for the shift back
        const float* part = sm + 2 * groups;
        int tpb = 16;
        while (tpb > 1 && tpb * 2 * groups > (int)blockDim.x) tpb >>= 1;
        const int b = threadIdx.x / tpb, sub = threadIdx.x % tpb, g = b >> 1, which = b & 1;
        double v = 0.0;
        if (b < 2 * groups)
            for (int r = 0; r < rows; r++)
                for (int c = sub; c < cpg; c += tpb) v += part[(r * 2 + which) * C + g * cpg + c];
#pragma unroll
        for (int off = 1; off < 16; off <<= 1)
            if (off < tpb) v += __shfl_xor_sync(0xffffffffu, v, off);
        const double s_of_group = __shfl_xor_sync(0xffffffffu, v, which ? tpb : 0);   // the group's sum, in both bins' threads
        if (b < 2 * groups && sub == 0) {
            if (!pivot) {
                const double pg = sm[g], n = (double)(p1 - p0) * cpg;
                v += which ? (2.0 * pg) * s_of_group + n * pg * pg : n * pg;
            }
            atomicAdd(&stats[b], v);
        }
    }
}

// GroupNorm(+SiLU) on NHWC in ONE launch: statistics -> grid rendezvous -> apply.  All CTAs are co-resident (grid <= 2 per
// SM), so after publishing its partial sums every CTA waits on an arrival counter and then normalises its own pixel strip,
// which is still L2-resident.  The scratch (2*G doubles + 2 counters) is zero on entry and the last CTA out re-zeroes it, so
// a CUDA graph needs a single node per GroupNorm instead of memset + 2 kernels.
template <typename T, int VEC>
__global__ void __launch_bounds__(512, 1)
gn_fused_nhwc_kernel(const T* __restrict__ x, T* __restrict__ y, double* __restrict__ stats, int* __restrict__ counters,
                     int C, int64_t HW, int groups, int64_t pix_per_cta, const T* __restrict__ gamma, const T* __restrict__ beta, float eps, int silu)
{
    osb_pdl_prologue();
    // 2 * groups fp64 partials, then (as floats) 2 * groups (mean, rstd).  The per-thread fp32 partials are combined in fp64, as the
    // producers of gn_apply_pre_kernel's statistics do, so that both GroupNorm paths derive the same mean and rstd from the same input.
    extern __shared__ double smd[];
    float* sm = reinterpret_cast<float*>(smd);
    for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) smd[i] = 0.0;
    __syncthreads();
    const int tpp = C / VEC;
    const int rows = blockDim.x / tpp;
    const int cv = threadIdx.x % tpp, pr = threadIdx.x / tpp;
    const int cpg = C / groups;
    int64_t p0 = (int64_t)blockIdx.x * pix_per_cta, p1 = min(p0 + pix_per_cta, HW);
    if (pr < rows) {
        float s[VEC], q[VEC], pv[VEC];
#pragma unroll
        for (int k = 0; k < VEC; k++) { s[k] = 0.f; q[k] = 0.f; pv[k] = to_float(x[(cv * VEC + k) / cpg * cpg]); }
        for (int64_t p = p0 + pr; p < p1; p += rows) {
            Vec<T, VEC> v = load_vec<T, VEC>(x + p * C + cv * VEC);
#pragma unroll
            for (int k = 0; k < VEC; k++) { float f = to_float(v.v[k]) - pv[k]; s[k] += f; q[k] += f * f; }
        }
        // combine the channels of this vector that fall into the same group in registers first: 2 (not 2 * VEC) shared atomics
        // per group touched -- the contended shared atomics were the longest phase of the kernel
        int g_cur = (cv * VEC) / cpg;
        double gs = 0.0, gq = 0.0;
#pragma unroll
        for (int k = 0; k < VEC; k++) {
            int g = (cv * VEC + k) / cpg;
            if (g != g_cur) { atomicAdd(&smd[2 * g_cur], gs); atomicAdd(&smd[2 * g_cur + 1], gq); g_cur = g; gs = 0.0; gq = 0.0; }
            gs += s[k]; gq += q[k];
        }
        atomicAdd(&smd[2 * g_cur], gs);
        atomicAdd(&smd[2 * g_cur + 1], gq);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) atomicAdd(&stats[i], smd[i]);
    __syncthreads();      // every partial is read before sm (the same memory) takes the (mean, rstd) floats
    // ---- grid rendezvous ----
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(&counters[0], 1);
        long long t0 = clock64();
        while (true) {
            int seen;
            asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(counters) : "memory");
            if (seen >= (int)gridDim.x) break;
            if (clock64() - t0 > 4000000000LL) { printf("gn_fused_nhwc_kernel: rendezvous timed out (block %d)\n", blockIdx.x); __trap(); }
        }
    }
    __syncthreads();
    __threadfence();
    // ---- per-group mean / rstd into shared memory ----
    const double inv_n = 1.0 / (double)((int64_t)cpg * HW);
    for (int g = threadIdx.x; g < groups; g += blockDim.x) {
        const double s = __ldcg(&stats[2 * g]) * inv_n;
        const double mean = (double)to_float(x[(int64_t)g * cpg]) + s;
        const double var = __ldcg(&stats[2 * g + 1]) * inv_n - s * s;
        sm[2 * g] = (float)mean;
        sm[2 * g + 1] = rsqrtf(fmaxf((float)var, 0.f) + eps);
    }
    __syncthreads();
    if (pr < rows) {
        float gm[VEC], bt[VEC], mu[VEC], rs[VEC];
#pragma unroll
        for (int k = 0; k < VEC; k++) {
            int c = cv * VEC + k, g = c / cpg;
            gm[k] = gamma ? to_float(gamma[c]) : 1.f; bt[k] = beta ? to_float(beta[c]) : 0.f; mu[k] = sm[2 * g]; rs[k] = sm[2 * g + 1] * gm[k];
        }
        for (int64_t p = p0 + pr; p < p1; p += rows) {
            Vec<T, VEC> v = load_vec<T, VEC>(x + p * C + cv * VEC);
#pragma unroll
            for (int k = 0; k < VEC; k++) {
                float o = fmaf(to_float(v.v[k]) - mu[k], rs[k], bt[k]);      // rs: rstd * gamma, as gn_apply_pre_kernel's scale
                if (silu) o = __fdividef(o, 1.f + __expf(-o));
                v.v[k] = from_float<T>(o);
            }
            store_vec<T, VEC>(y + p * C + cv * VEC, v);
        }
    }
    // ---- last CTA out re-zeroes the scratch for the next launch ----
    __syncthreads();
    if (threadIdx.x == 0) {
        int done = atomicAdd(&counters[1], 1);
        if (done == (int)gridDim.x - 1) {
            for (int i = 0; i < 2 * groups; i++) stats[i] = 0.0;
            counters[0] = 0; counters[1] = 0;
            __threadfence();
        }
    }
}

template <typename T>
__global__ void gn_stats_nchw_kernel(const T* __restrict__ x, double* __restrict__ stats, int64_t n_per_g, int splits)
{
    osb_pdl_prologue();
    __shared__ float red[32];
    int64_t g = blockIdx.x;
    int64_t chunk = (n_per_g + splits - 1) / splits;
    int64_t lo = blockIdx.y * chunk, hi = min(lo + chunk, n_per_g);
    const T* xg = x + g * n_per_g;
    const float pv = to_float(xg[0]);
    float s = 0.f, q = 0.f;
    for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) { float v = to_float(xg[i]) - pv; s += v; q += v * v; }
    s = block_reduce_sum(s, red);
    q = block_reduce_sum(q, red);
    if (threadIdx.x == 0) { atomicAdd(&stats[2 * g], (double)s); atomicAdd(&stats[2 * g + 1], (double)q); }
}

template <typename T, int VEC>
__global__ void gn_apply_kernel(const T* __restrict__ x, T* __restrict__ y, const double* __restrict__ stats, int nhwc, int64_t C, int64_t HW, int groups,
                                const T* __restrict__ gamma, const T* __restrict__ beta, float eps, int silu)
{
    // stats around the group pivots (gn_mean_var): group g's first element is x[g * cpg] (NHWC) or x[g * cpg * HW] (NCHW)
    osb_pdl_prologue();
    int cpg = (int)(C / groups);
    double inv_n = 1.0 / (double)((int64_t)cpg * HW);
    size_t n = (size_t)C * HW, nvec = n / VEC;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        size_t e = i * VEC;
        Vec<T, VEC> v = load_vec<T, VEC>(x + e);
#pragma unroll
        for (int k = 0; k < VEC; k++) {
            int64_t c = nhwc ? (int64_t)((e + k) % C) : (int64_t)((e + k) / HW);
            int g = (int)(c / cpg);
            double meand, vard;
            gn_mean_var(stats, g, inv_n, to_float(x[(int64_t)g * cpg * (nhwc ? 1 : HW)]), meand, vard);
            float mean = (float)meand;
            float rstd = rsqrtf(fmaxf((float)vard, 0.f) + eps);
            float o = (to_float(v.v[k]) - mean) * rstd;
            o = o * (gamma ? to_float(gamma[c]) : 1.f) + (beta ? to_float(beta[c]) : 0.f);
            if (silu) o = o / (1.f + expf(-o));
            v.v[k] = from_float<T>(o);
        }
        store_vec<T, VEC>(y + e, v);
    }
}


// GroupNorm(+SiLU) apply pass for statistics gathered by the producing conv's epilogue (osb_conv2d_ex): one streaming pass, no grid
// rendezvous.  Each CTA lays out per-channel mean, scale = rstd * gamma and beta tables in shared memory, then y = (x - mean) * scale +
// beta (+ SiLU) over its strip of NHWC pixels with 16-byte vectors, a thread's VEC channels read from each table as 16-byte words.  This
// is gn_fused_nhwc_kernel's arithmetic, so a GroupNorm computes the same from the same statistics on either path.  The subtraction comes
// first: x * scale + (beta - mean * scale) would round mean * scale at the scale of the mean, several ulps of the mean times rstd when the
// mean is large against the spread.  CTA 0 zeroes `clear_stats` -- the buffer the NEXT statistics producer in stream order accumulates
// into (its previous reader finished before this kernel started).
template <typename T, int VEC>
__global__ void gn_apply_pre_kernel(const T* __restrict__ x, T* __restrict__ y, const double* __restrict__ stats, double* __restrict__ clear_stats,
                                    int C, int64_t HW, int groups, const T* __restrict__ gamma, const T* __restrict__ beta, float eps, int silu)
{
    osb_pdl_prologue();
    extern __shared__ float4 tab4[];        // [3 * C] floats: mean, scale, beta
    float* mu = reinterpret_cast<float*>(tab4); float* scale = mu + C; float* shift = mu + 2 * C;
    const int cpg = C / groups;
    const double inv_n = 1.0 / ((double)cpg * (double)HW);
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int g = c / cpg;
        const double mean = stats[2 * g] * inv_n;
        const double var = stats[2 * g + 1] * inv_n - mean * mean;
        const float rstd = rsqrtf(fmaxf((float)var, 0.f) + eps);
        const float ga = gamma ? to_float(gamma[c]) : 1.f, be = beta ? to_float(beta[c]) : 0.f;
        mu[c] = (float)mean; scale[c] = rstd * ga; shift[c] = be;
    }
    if (blockIdx.x == 0 && clear_stats) for (int t = threadIdx.x; t < 2 * groups; t += blockDim.x) clear_stats[t] = 0.0;
    __syncthreads();
    const int vpp = C / VEC;                                  // vectors per pixel
    const int64_t nvec = HW * vpp;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    // 4 independent 16-byte loads in flight per thread: the pass is pure streaming, latency is hidden by memory-level parallelism
    for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i0 < nvec; i0 += 4 * stride) {
        Vec<T, VEC> v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) { const int64_t i = i0 + u * stride; if (i < nvec) v[u] = load_vec<T, VEC>(x + i * VEC); }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int64_t i = i0 + u * stride;
            if (i >= nvec) break;
            const int c0 = (int)(i % vpp) * VEC;
            float tm[VEC], ts[VEC], tb[VEC];
#pragma unroll
            for (int k = 0; k < VEC; k += 4) {
                *reinterpret_cast<float4*>(tm + k) = *reinterpret_cast<const float4*>(mu + c0 + k);
                *reinterpret_cast<float4*>(ts + k) = *reinterpret_cast<const float4*>(scale + c0 + k);
                *reinterpret_cast<float4*>(tb + k) = *reinterpret_cast<const float4*>(shift + c0 + k);
            }
#pragma unroll
            for (int k = 0; k < VEC; k++) {
                float o = fmaf(to_float(v[u].v[k]) - tm[k], ts[k], tb[k]);
                if (silu) o = __fdividef(o, 1.f + __expf(-o));
                v[u].v[k] = from_float<T>(o);
            }
            store_vec<T, VEC>(y + i * VEC, v[u]);
        }
    }
}


// ------------------------------------------------------------------------------------------------------------
// dynamic-quantisation range: Model::get_percentiles (src/onnxstream.cpp:3104-3232) + FloatAsUInt::get_percentiles (2302-2386)
// ------------------------------------------------------------------------------------------------------------
// The reference splits the tensor across its `threads` pool workers (get_start_and_end, 3091-3102), each worker walks its span in
// 64 KiB chunks, sorts a chunk's bit patterns and takes the k-th smallest / k-th largest FINITE value with k = (size_t)(n * 0.001f);
// the tensor's range is the min of the chunk lows and the max of the chunk highs.  Here: one CTA per chunk, the chunk's values as
// order-preserving integer keys in shared memory, two radix selects (8 bits per round) instead of a sort, atomicMin / atomicMax on
// the keys.  out[0] = min low key (init 0xFFFFFFFF), out[1] = max high key (init 0), out[2] = number of chunks that had a result.
constexpr unsigned PCT_SENTINEL = 0xFFFFFFFFu;

__device__ unsigned pct_select(const unsigned* keys, int n, unsigned rank, int bits, unsigned* hist, unsigned* bcast)
{
    unsigned prefix = 0, mask = 0;
    for (int shift = bits - 8; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            unsigned k = keys[i];
            if (k != PCT_SENTINEL && (k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned cum = 0, d = 0;
            for (; d < 256; d++) { if (cum + hist[d] > rank) break; cum += hist[d]; }
            bcast[0] = d; bcast[1] = rank - cum;
        }
        __syncthreads();
        prefix |= bcast[0] << shift; mask |= 255u << shift; rank = bcast[1];
        __syncthreads();
    }
    return prefix;
}

template <typename T>
__global__ void __launch_bounds__(1024, 1)
percentile_chunks_kernel(const T* __restrict__ x, size_t size, size_t threads, size_t chunk, float from_left, float from_right, unsigned* __restrict__ out)
{
    extern __shared__ unsigned pk[];            // [chunk] keys
    __shared__ unsigned hist[256], bcast[2], n_finite;
    // span of reference worker blockIdx.y (get_start_and_end), chunk blockIdx.x inside it
    size_t per = size / threads; if (!per) per = 1;
    const size_t i = blockIdx.y;
    const size_t start = i * per, end = i >= threads - 1 ? size : (i + 1) * per;
    if (start >= end || start >= size) return;
    const size_t c0 = start + (size_t)blockIdx.x * chunk;
    if (c0 >= end) return;
    const int n = (int)min(chunk, end - c0);
    constexpr bool half = sizeof(T) == 2;
    if (threadIdx.x == 0) n_finite = 0;
    __syncthreads();
    unsigned local = 0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        unsigned key;
        if (half) {
            unsigned h = reinterpret_cast<const unsigned short*>(x)[c0 + j];
            bool fin = (h & 0x7C00u) != 0x7C00u;
            key = fin ? ((h & 0x8000u) ? (~h & 0xFFFFu) : (h | 0x8000u)) : PCT_SENTINEL;
            local += fin;
        } else {
            unsigned u = reinterpret_cast<const unsigned*>(x)[c0 + j];
            bool fin = (u & 0x7F800000u) != 0x7F800000u;
            key = fin ? ((u & 0x80000000u) ? ~u : (u | 0x80000000u)) : PCT_SENTINEL;
            if (key == PCT_SENTINEL) key = 0xFFFFFFFEu;      // (cannot happen for a finite value; keeps the sentinel exclusive)
            local += fin;
        }
        pk[j] = key;
    }
    atomicAdd(&n_finite, local);
    __syncthreads();
    const unsigned m = n_finite;
    const size_t kl = (size_t)((float)n * from_left), kr = (size_t)((float)n * from_right);
    if (kl >= m || kr >= m) return;              // FloatAsUInt::get_percentiles returns nullopt: this chunk contributes nothing
    const int bits = half ? 16 : 32;
    const unsigned lo = pct_select(pk, n, (unsigned)kl, bits, hist, bcast);
    const unsigned hi = pct_select(pk, n, m - 1 - (unsigned)kr, bits, hist, bcast);
    if (threadIdx.x == 0) { atomicMin(&out[0], lo); atomicMax(&out[1], hi); atomicAdd(&out[2], 1u); }
}


// ------------------------------------------------------------------------------------------------------------
// LLM decode fusions: RMSNorm and rotary embedding (the op chains llm.cpp's graphs spell out, src/onnxstream.cpp: Pow 5478-5604,
// ReduceMean 5237-5393, Sqrt 4001-4139, Div / Mul / Add / Neg / Slice / Concat)
// ------------------------------------------------------------------------------------------------------------
// y = w * (x * (1 / sqrt(mean(x^2) + eps))): one warp per row, fp32 arithmetic whatever the storage types (the reference keeps these
// ops in fp32 through m_requires_upcast, src/llm.cpp:385-389)
template <typename TI, typename TW, typename TO>
__global__ void rms_norm_kernel(const TI* __restrict__ x, const TW* __restrict__ w, TO* __restrict__ y, int64_t rows, int cols, float eps)
{
    osb_pdl_prologue();
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    for (int64_t r = (int64_t)blockIdx.x * wpb + wib; r < rows; r += (int64_t)gridDim.x * wpb) {
        const TI* xr = x + r * cols;
        float ss = 0.f;
        for (int c = lane; c < cols; c += 32) { const float v = to_float(xr[c]); ss = fmaf(v, v, ss); }
        ss = warp_sum(ss);
        const float inv = 1.0f / sqrtf(ss / (float)cols + eps);
        TO* yr = y + r * cols;
        for (int c = lane; c < cols; c += 32) yr[c] = from_float<TO>(to_float(w[c]) * (to_float(xr[c]) * inv));
    }
}

// few rows (a decode step has one): a whole CTA per row -- 256 threads, 4 independent loads each per pass, block reduction -- instead of one
// warp walking the row with one load in flight
template <typename TI, typename TW, typename TO>
__global__ void __launch_bounds__(256) rms_norm_block_kernel(const TI* __restrict__ x, const TW* __restrict__ w, TO* __restrict__ y, int cols, float eps)
{
    osb_pdl_prologue();
    __shared__ float red[8];
    const TI* xr = x + (int64_t)blockIdx.x * cols;
    TO* yr = y + (int64_t)blockIdx.x * cols;
    float ss = 0.f;
#pragma unroll 4
    for (int c = threadIdx.x; c < cols; c += 256) { const float v = to_float(xr[c]); ss = fmaf(v, v, ss); }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int k = 0; k < 8; k++) tot += red[k];
    const float inv = 1.0f / sqrtf(tot / (float)cols + eps);
#pragma unroll 4
    for (int c = threadIdx.x; c < cols; c += 256) yr[c] = from_float<TO>(to_float(w[c]) * (to_float(xr[c]) * inv));
}

// rotary embedding, "rotate_half" form: y[j] = x[j] * cos[j] + (j < D/2 ? -x[j + D/2] : x[j - D/2]) * sin[j]; cos / sin are one row of D
// values shared by every row (table_rows == 1) or one row per x row
template <typename T>
__global__ void rope_kernel(const T* __restrict__ x, const T* __restrict__ cs, const T* __restrict__ sn, T* __restrict__ y, int64_t rows, int D, int64_t table_rows)
{
    osb_pdl_prologue();
    const int64_t n = rows * D;
    const int half = D >> 1;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / D; const int j = (int)(i % D);
        // one table row for every x row (decode), or x [.., T, D] cycling through T rows (prefill); no 64-bit division on the decode path
        const int64_t t = table_rows == 1 ? 0 : (table_rows == rows ? r : r % table_rows);
        const float xv = to_float(x[i]);
        const float rot = j < half ? -to_float(x[i + half]) : to_float(x[i - half]);
        // the reference rounds each product and the sum to the storage type (three separate ops): keep those roundings
        // (__fmul_rn / __fadd_rn: no fused multiply-add across the three ops in fp32 either)
        const T a = from_float<T>(__fmul_rn(xv, to_float(cs[t * D + j]))), b = from_float<T>(__fmul_rn(to_float(from_float<T>(rot)), to_float(sn[t * D + j])));
        y[i] = from_float<T>(__fadd_rn(to_float(a), to_float(b)));
    }
}

// ------------------------------------------------------------------------------------------------------------
// gather rows, fill
// ------------------------------------------------------------------------------------------------------------

// ScatterND with full-rank indices (src/onnxstream.cpp:7939-8074): out[pos[i]] = updates[i]; positions are linearised (and range
// checked) on the host because the index tensor is int64 host data.  Duplicate positions: last writer wins is not guaranteed by
// the reference either (it scatters from a thread pool).
__global__ void scatter_elems_kernel(uint8_t* __restrict__ out, const int64_t* __restrict__ pos, const uint8_t* __restrict__ upd, int64_t n, int elem)
{
    osb_pdl_prologue();
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t p = pos[i];
        if (elem == 2) reinterpret_cast<uint16_t*>(out)[p] = reinterpret_cast<const uint16_t*>(upd)[i];
        else reinterpret_cast<uint32_t*>(out)[p] = reinterpret_cast<const uint32_t*>(upd)[i];
    }
}

// MaxPool on NHWC (XnnPack::maxpool_nhwc, src/onnxstream.cpp:1537-1664): dilation 1, padded taps are ignored (-inf), one thread
// per (output pixel, channel).
template <typename T>
__global__ void maxpool_nhwc_kernel(const T* __restrict__ x, T* __restrict__ y, int H, int W, int C, int kh, int kw, int stride, int pad_top, int pad_left, int Ho, int Wo)
{
    osb_pdl_prologue();
    const int64_t total = (int64_t)Ho * Wo * C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(i % C);
        int64_t pix = i / C;
        int ox = (int)(pix % Wo), oy = (int)(pix / Wo);
        float m = -INFINITY;
        for (int ky = 0; ky < kh; ky++) {
            int iy = oy * stride + ky - pad_top;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < kw; kx++) {
                int ix = ox * stride + kx - pad_left;
                if (ix < 0 || ix >= W) continue;
                m = fmaxf(m, to_float(x[((int64_t)iy * W + ix) * C + c]));
            }
        }
        y[i] = from_float<T>(m);
    }
}

__global__ void gather_rows_kernel(const uint8_t* __restrict__ table, const int64_t* __restrict__ idx, uint8_t* __restrict__ out,
                                   int64_t n_idx, int64_t table_rows, int64_t row_bytes)
{
    osb_pdl_prologue();
    for (int64_t r = blockIdx.x; r < n_idx; r += gridDim.x) {
        int64_t src = idx[r];
        if (src < 0) src += table_rows;
        src = src < 0 ? 0 : (src >= table_rows ? table_rows - 1 : src);      // indices may come from a device mirror the host did not validate (graph replay)
        const uint8_t* s = table + src * row_bytes;
        uint8_t* d = out + r * row_bytes;
        if ((row_bytes & 15) == 0 && (((uintptr_t)s | (uintptr_t)d) & 15) == 0) {
            for (int64_t i = threadIdx.x; i < row_bytes / 16; i += blockDim.x) ((int4*)d)[i] = ((const int4*)s)[i];
        } else {
            for (int64_t i = threadIdx.x; i < row_bytes; i += blockDim.x) d[i] = s[i];
        }
    }
}

template <typename T>
__global__ void fill_kernel(T* dst, size_t n, float v)
{
    osb_pdl_prologue();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = from_float<T>(v);
}

bool contiguous_like(const int64_t* strides, const int64_t* shape, int ndim)
{
    int64_t s = 1;
    for (int d = ndim - 1; d >= 0; d--) {
        if (shape[d] != 1 && strides[d] != s) return false;
        s *= shape[d];
    }
    return true;
}

bool all_zero(const int64_t* strides, const int64_t* shape, int ndim)
{
    for (int d = 0; d < ndim; d++) if (shape[d] != 1 && strides[d] != 0) return false;
    return true;
}

} // namespace

template <typename T, int VEC>
static int binary_dispatch(int op, const T* a, const int64_t* as, const T* b, const int64_t* bs, T* out, const int64_t* shape, int ndim, cudaStream_t st)
{
    size_t n = 1;
    for (int d = 0; d < ndim; d++) n *= (size_t)shape[d];
    if (n == 0) return 0;
    bool al = aligned16(a) && aligned16(b) && aligned16(out);
    bool a_contig = contiguous_like(as, shape, ndim), b_contig = contiguous_like(bs, shape, ndim);
    bool a_scalar = all_zero(as, shape, ndim), b_scalar = all_zero(bs, shape, ndim);
    if ((a_contig || a_scalar) && (b_contig || b_scalar)) {
        if (al || (a_scalar && aligned16(b) && aligned16(out)) || (b_scalar && aligned16(a) && aligned16(out)))
            osb_launch((binary_flat_kernel<T, VEC>), grid_for(n / VEC + 1, 256), 256, 0, st, op, a, b, out, n, a_scalar && !a_contig, b_scalar && !b_contig);
        else
            osb_launch((binary_flat_kernel<T, 1>), grid_for(n, 256), 256, 0, st, op, a, b, out, n, a_scalar && !a_contig, b_scalar && !b_contig);
        return launched();
    }
    // one operand contiguous, the other varies only along the last dim (per-column) or is constant along it (per-row)
    for (int swap = 0; swap < 2; swap++) {
        const int64_t* fs = swap ? bs : as;      // full operand
        const int64_t* ps = swap ? as : bs;      // partial operand
        const T* full = swap ? b : a;
        const T* part = swap ? a : b;
        if (!contiguous_like(fs, shape, ndim)) continue;
        int64_t cols = shape[ndim - 1], rows = (int64_t)(n / (size_t)cols);
        // per-column: strides zero on all but the last dim, last dim stride 1
        bool percol = (cols == 1 || ps[ndim - 1] == 1);
        for (int d = 0; d < ndim - 1 && percol; d++) if (shape[d] != 1 && ps[d] != 0) percol = false;
        if (percol && cols % VEC == 0 && aligned16(full) && aligned16(part) && aligned16(out)) {
            osb_launch((binary_rowcol_kernel<T, VEC>), grid_for((size_t)rows * (cols / VEC), 256), 256, 0, st, op, full, part, out, rows, cols, 0, swap);
            return launched();
        }
        // per-row: [R, 1] against [R, cols] where the partial operand is contiguous over the leading dims
        if (ps[ndim - 1] == 0 || cols == 1) {
            bool perrow = true;
            int64_t s = 1;
            for (int d = ndim - 2; d >= 0; d--) { if (shape[d] != 1 && ps[d] != s) perrow = false; s *= shape[d]; }
            if (perrow && cols % VEC == 0 && aligned16(full) && aligned16(out)) {
                osb_launch((binary_rowcol_kernel<T, VEC>), grid_for((size_t)rows * (cols / VEC), 256), 256, 0, st, op, full, part, out, rows, cols, 1, swap);
                return launched();
            }
        }
    }
    BinParams p;
    p.ndim = ndim;
    for (int d = 0; d < OSB_MAX_DIMS; d++) { p.shape[d] = d < ndim ? shape[d] : 1; p.as[d] = d < ndim ? as[d] : 0; p.bs[d] = d < ndim ? bs[d] : 0; }
    osb_launch((binary_generic_kernel<T>), grid_for(n, 256), 256, 0, st, op, a, b, out, p, n);
    return launched();
}

// ================================================================================================================
// C ABI
// ================================================================================================================

extern "C" {

int osb_convert(const void* src, int sd, void* dst, int dd, size_t n, float scale, int zp, void* stream)
{
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    int grid = grid_for(n, 256);
    if (sd == OSB_F16 && dd == OSB_F32) osb_launch((convert_kernel<__half, float>), grid, 256, 0, st, (const __half*)src, (float*)dst, n);
    else if (sd == OSB_F32 && dd == OSB_F16) osb_launch((convert_kernel<float, __half>), grid, 256, 0, st, (const float*)src, (__half*)dst, n);
    else if (sd == OSB_U8 && dd == OSB_F32) osb_launch((dequant_kernel<float>), grid, 256, 0, st, (const uint8_t*)src, (float*)dst, n, scale, zp);
    else if (sd == OSB_U8 && dd == OSB_F16) osb_launch((dequant_kernel<__half>), grid, 256, 0, st, (const uint8_t*)src, (__half*)dst, n, scale, zp);
    else if (sd == OSB_F32 && dd == OSB_U8) osb_launch((quant_kernel<float>), grid, 256, 0, st, (const float*)src, (uint8_t*)dst, n, scale, zp);
    else if (sd == OSB_F16 && dd == OSB_U8) osb_launch((quant_kernel<__half>), grid, 256, 0, st, (const __half*)src, (uint8_t*)dst, n, scale, zp);
    else if (sd == OSB_I64 && dd == OSB_F32) osb_launch((i64_to_float_kernel), grid, 256, 0, st, (const int64_t*)src, (float*)dst, n);
    else return (int)cudaErrorInvalidValue;
    return launched();
}

int osb_unary(int op, const void* x, void* y, int dtype, size_t n, float alpha, void* stream)
{
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    bool al = aligned16(x) && aligned16(y);
    if (dtype == OSB_F16) {
        if (al) osb_launch((unary_kernel<__half, 8>), grid_for(n / 8 + 1, 256), 256, 0, st, op, (const __half*)x, (__half*)y, n, alpha);
        else osb_launch((unary_kernel<__half, 1>), grid_for(n, 256), 256, 0, st, op, (const __half*)x, (__half*)y, n, alpha);
    } else if (dtype == OSB_F32) {
        if (al) osb_launch((unary_kernel<float, 4>), grid_for(n / 4 + 1, 256), 256, 0, st, op, (const float*)x, (float*)y, n, alpha);
        else osb_launch((unary_kernel<float, 1>), grid_for(n, 256), 256, 0, st, op, (const float*)x, (float*)y, n, alpha);
    } else return (int)cudaErrorInvalidValue;
    return launched();
}

int osb_geglu(const void* x, void* y, int dtype, int64_t rows, int64_t inner, void* stream)
{
    if (rows * inner == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    bool al = aligned16(x) && aligned16(y);
    if (dtype == OSB_F16) {
        if (al && inner % 8 == 0) osb_launch((geglu_kernel<__half, 8>), grid_for((size_t)rows * (inner / 8), 256), 256, 0, st, (const __half*)x, (__half*)y, rows, inner);
        else osb_launch((geglu_kernel<__half, 1>), grid_for((size_t)rows * inner, 256), 256, 0, st, (const __half*)x, (__half*)y, rows, inner);
    } else if (dtype == OSB_F32) {
        if (al && inner % 4 == 0) osb_launch((geglu_kernel<float, 4>), grid_for((size_t)rows * (inner / 4), 256), 256, 0, st, (const float*)x, (float*)y, rows, inner);
        else osb_launch((geglu_kernel<float, 1>), grid_for((size_t)rows * inner, 256), 256, 0, st, (const float*)x, (float*)y, rows, inner);
    } else return (int)cudaErrorInvalidValue;
    return launched();
}

int osb_binary(int op, const void* a, const int64_t* as, const void* b, const int64_t* bs, void* out, const int64_t* shape, int ndim, int dtype, void* stream)
{
    if (ndim < 1 || ndim > OSB_MAX_DIMS) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == OSB_F16) return binary_dispatch<__half, 8>(op, (const __half*)a, as, (const __half*)b, bs, (__half*)out, shape, ndim, st);
    if (dtype == OSB_F32) return binary_dispatch<float, 4>(op, (const float*)a, as, (const float*)b, bs, (float*)out, shape, ndim, st);
    return (int)cudaErrorInvalidValue;
}

// ---- fp32 -> bf16 triple split, expanded along K for the tensor-core fp32 path (gemm_wgmma.cu: osb_tc_gemm_f32x) -----------------
// x = h + m + l (common.cuh: bf16x3_split).  A side: segments [h|h|m|h|l|m]; B side: [h|m|h|l|h|m], so that segment s of A times
// segment s of B runs over the six products hh, hm, mh, hl, lh, mm.
__device__ __forceinline__ void bf16x3_parts(float x, int b_side, __nv_bfloat16* six)
{
    __nv_bfloat16 h, m, l;
    bf16x3_split(x, h, m, l);
    if (b_side) { six[0] = h; six[1] = m; six[2] = h; six[3] = l; six[4] = h; six[5] = m; }
    else        { six[0] = h; six[1] = h; six[2] = m; six[3] = h; six[4] = l; six[5] = m; }
}
// out[r][s * L + j] = part_s(in[r * ld_in + j]): rows of length L become rows of length 6 L (GEMM A rows, K-major B rows, NHWC pixels, OHWI taps)
__global__ void bf16x3_expand_cols_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t rows, int L, int64_t ld_in, int b_side)
{
    osb_pdl_prologue();
    const int64_t n = rows * L;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / L; const int j = (int)(i - r * L);
        __nv_bfloat16 six[6];
        bf16x3_parts(in[r * ld_in + j], b_side, six);
        __nv_bfloat16* o = out + r * 6 * L + j;
#pragma unroll
        for (int s = 0; s < 6; s++) o[(int64_t)s * L] = six[s];
    }
}
// out[s * Kr + k][n] = part_s(in[k][n]): a [K][N] MatMul weight becomes [6 K][N] (MN-major B operand)
__global__ void bf16x3_expand_rows_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t Kr, int64_t N, int b_side)
{
    osb_pdl_prologue();
    const int64_t n = Kr * N;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        __nv_bfloat16 six[6];
        bf16x3_parts(in[i], b_side, six);
#pragma unroll
        for (int s = 0; s < 6; s++) out[(int64_t)s * n + i] = six[s];
    }
}

int osb_bf16x3_expand_cols(const void* in, void* out, int64_t rows, int64_t L, int64_t ld_in, int b_side, void* stream)
{
    if (rows * L == 0) return 0;
    if (L > (1 << 30)) return (int)cudaErrorInvalidValue;
    osb_launch((bf16x3_expand_cols_kernel), grid_for((size_t)(rows * L), 256), 256, 0, (cudaStream_t)stream, (const float*)in, (__nv_bfloat16*)out, rows, (int)L, ld_in, b_side);
    return launched();
}

int osb_bf16x3_expand_rows(const void* in, void* out, int64_t K, int64_t N, int b_side, void* stream)
{
    if (K * N == 0) return 0;
    osb_launch((bf16x3_expand_rows_kernel), grid_for((size_t)(K * N), 256), 256, 0, (cudaStream_t)stream, (const float*)in, (__nv_bfloat16*)out, K, N, b_side);
    return launched();
}

// Concat of two sources along one axis as ONE launch: out[o][0:la) = a[o][:], out[o][la:la+lb) = b[o][:], lengths in 16-byte units
// (KV-cache append of a decode step: la = cached rows, lb = one row)
__global__ void concat2_vec_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ out, int64_t outer, int64_t la, int64_t lb)
{
    osb_pdl_prologue();
    const int64_t lo = la + lb, n = outer * lo;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t o = i / lo, j = i - o * lo;
        out[i] = j < la ? a[o * la + j] : b[o * lb + (j - la)];
    }
}

int osb_concat2(const void* a, const void* b, void* out, int64_t outer, int64_t a_bytes, int64_t b_bytes, void* stream)
{
    if (outer * (a_bytes + b_bytes) == 0) return 0;
    if ((a_bytes | b_bytes) & 15 || !aligned16(a) || !aligned16(b) || !aligned16(out)) return (int)cudaErrorNotSupported;
    osb_launch((concat2_vec_kernel), grid_for((size_t)(outer * (a_bytes + b_bytes) / 16), 256), 256, 0, (cudaStream_t)stream,
               (const uint4*)a, (const uint4*)b, (uint4*)out, outer, a_bytes / 16, b_bytes / 16);
    return launched();
}

int osb_strided_copy(const void* in, void* out, int elem_size, int ndim, const int64_t* shape, const int64_t* in_stride, const int64_t* in_div,
                     int64_t in_offset, const int64_t* out_stride, int64_t out_offset, void* stream)
{
    if (ndim < 1 || ndim > OSB_MAX_DIMS) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    CopyParams p;
    p.ndim = ndim; p.in_off = in_offset; p.out_off = out_offset;
    size_t n = 1;
    for (int d = 0; d < OSB_MAX_DIMS; d++) {
        p.shape[d] = d < ndim ? shape[d] : 1;
        p.is[d] = d < ndim ? in_stride[d] : 0;
        p.idiv[d] = (d < ndim && in_div) ? in_div[d] : 1;
        p.os[d] = d < ndim ? out_stride[d] : 0;
        if (d < ndim) n *= (size_t)shape[d];
    }
    if (n == 0) return 0;
    // widen the element when the innermost dimension is contiguous on both sides and everything is aligned
    int es = elem_size;
    if (p.is[ndim - 1] == 1 && p.os[ndim - 1] == 1 && p.idiv[ndim - 1] == 1) {
        for (int wide = 16; wide > es; wide >>= 1) {
            int f = wide / es;
            bool ok = (p.shape[ndim - 1] % f == 0) && (p.in_off % f == 0) && (p.out_off % f == 0) &&
                      ((uintptr_t)in % wide == 0) && ((uintptr_t)out % wide == 0);
            for (int d = 0; d < ndim - 1 && ok; d++) ok = (p.is[d] % f == 0) && (p.os[d] % f == 0);
            if (ok) {
                p.shape[ndim - 1] /= f; p.in_off /= f; p.out_off /= f;
                for (int d = 0; d < ndim - 1; d++) { p.is[d] /= f; p.os[d] /= f; }
                n /= f; es = wide;
                break;
            }
        }
    }
    int grid = grid_for(n, 256);
    switch (es) {
    case 1: osb_launch((strided_copy_kernel<uint8_t>), grid, 256, 0, st, (const uint8_t*)in, (uint8_t*)out, p, n); break;
    case 2: osb_launch((strided_copy_kernel<uint16_t>), grid, 256, 0, st, (const uint16_t*)in, (uint16_t*)out, p, n); break;
    case 4: osb_launch((strided_copy_kernel<uint32_t>), grid, 256, 0, st, (const uint32_t*)in, (uint32_t*)out, p, n); break;
    case 8: osb_launch((strided_copy_kernel<uint2>), grid, 256, 0, st, (const uint2*)in, (uint2*)out, p, n); break;
    case 16: osb_launch((strided_copy_kernel<uint4>), grid, 256, 0, st, (const uint4*)in, (uint4*)out, p, n); break;
    default: return (int)cudaErrorInvalidValue;
    }
    return launched();
}

int osb_transpose2d(const void* in, void* out, int elem_size, int64_t batch, int64_t rows, int64_t cols, void* stream)
{
    if (batch * rows * cols == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32), (unsigned)batch), block(32, 8);
    if (grid.y > 65535 || grid.z > 65535) return (int)cudaErrorInvalidValue;
    switch (elem_size) {
    case 1: osb_launch((transpose2d_kernel<uint8_t>), grid, block, 0, st, (const uint8_t*)in, (uint8_t*)out, rows, cols); break;
    case 2: osb_launch((transpose2d_kernel<uint16_t>), grid, block, 0, st, (const uint16_t*)in, (uint16_t*)out, rows, cols); break;
    case 4: osb_launch((transpose2d_kernel<uint32_t>), grid, block, 0, st, (const uint32_t*)in, (uint32_t*)out, rows, cols); break;
    default: return (int)cudaErrorInvalidValue;
    }
    return launched();
}

int osb_softmax(const void* x, void* y, int dtype, int64_t rows, int64_t cols, void* stream)
{
    if (rows * cols == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    int threads = cols >= 1024 ? 256 : (cols >= 256 ? 128 : 32);
    int grid = (int)min<int64_t>(rows, OSB_SMS * 16);
    if (dtype == OSB_F16) osb_launch((softmax_kernel<__half>), grid, threads, 0, st, (const __half*)x, (__half*)y, rows, cols);
    else if (dtype == OSB_F32) osb_launch((softmax_kernel<float>), grid, threads, 0, st, (const float*)x, (float*)y, rows, cols);
    else return (int)cudaErrorInvalidValue;
    return launched();
}

int osb_layer_norm(const void* x, void* y, int dtype, int64_t rows, int64_t cols, const void* gamma, const void* beta, float eps, void* stream)
{
    if (rows * cols == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int esz = dtype == OSB_F16 ? 2 : 4;
    auto al = [&](const void* p) { return p == nullptr || ((uintptr_t)p % (2 * esz)) == 0; };
    if ((cols % 2) == 0 && cols <= 64 * LN_MAX_ITERS && rows >= 64 && al(x) && al(y) && al(gamma) && al(beta) && (dtype == OSB_F16 || dtype == OSB_F32)) {
        unsigned grid_w = (unsigned)((rows + 3) / 4);
#define OSB_LN_LAUNCH(T_, IT_) osb_launch((layer_norm_warp_kernel<T_, IT_>), grid_w, 128, 0, st, (const T_*)x, (T_*)y, rows, (int)cols, (const T_*)gamma, (const T_*)beta, eps)
        if (dtype == OSB_F16) { if (cols <= 320) OSB_LN_LAUNCH(__half, 5); else if (cols <= 640) OSB_LN_LAUNCH(__half, 10); else OSB_LN_LAUNCH(__half, LN_MAX_ITERS); }
        else { if (cols <= 320) OSB_LN_LAUNCH(float, 5); else if (cols <= 640) OSB_LN_LAUNCH(float, 10); else OSB_LN_LAUNCH(float, LN_MAX_ITERS); }
#undef OSB_LN_LAUNCH
        return launched();
    }
    int threads = cols >= 1024 ? 256 : (cols >= 256 ? 128 : 32);
    int grid = (int)min<int64_t>(rows, OSB_SMS * 16);
    if (dtype == OSB_F16) osb_launch((layer_norm_kernel<__half>), grid, threads, 0, st, (const __half*)x, (__half*)y, rows, cols, (const __half*)gamma, (const __half*)beta, eps);
    else if (dtype == OSB_F32) osb_launch((layer_norm_kernel<float>), grid, threads, 0, st, (const float*)x, (float*)y, rows, cols, (const float*)gamma, (const float*)beta, eps);
    else return (int)cudaErrorInvalidValue;
    return launched();
}

int osb_reduce_mean(const void* x, void* y, int dtype, int64_t rows, int64_t cols, void* stream)
{
    if (rows * cols == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    int threads = cols >= 1024 ? 256 : (cols >= 256 ? 128 : 32);
    int grid = (int)min<int64_t>(rows, OSB_SMS * 16);
    if (dtype == OSB_F16) osb_launch((reduce_mean_kernel<__half>), grid, threads, 0, st, (const __half*)x, (__half*)y, rows, cols);
    else if (dtype == OSB_F32) osb_launch((reduce_mean_kernel<float>), grid, threads, 0, st, (const float*)x, (float*)y, rows, cols);
    else return (int)cudaErrorInvalidValue;
    return launched();
}

int osb_instance_norm(const void* x, void* y, int dtype, int64_t channels, int64_t n_per_c, const void* scale, const void* bias, float eps, void* stream)
{
    if (channels * n_per_c == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    int splits = (int)max<int64_t>(1, min<int64_t>(64, (OSB_SMS * 4 + channels - 1) / channels));
    while (splits > 1 && n_per_c / splits < 1024) splits--;
    while (splits > 1 && (size_t)channels * splits * 2 > OSB_WS_INORM_DOUBLES) splits--;
    if ((size_t)channels * splits * 2 > OSB_WS_INORM_DOUBLES) return (int)cudaErrorInvalidValue;
    // per-stream fixed-capacity partial sums (workspace.h): never re-allocated, so a captured graph keeps a valid address
    OsbWorkspace* ws = osb_workspace(st, OSB_WS_INORM);
    if (!ws) return (int)cudaErrorStreamCaptureUnsupported;
    double* g_inorm_partial = ws->inorm;
    dim3 grid((unsigned)channels, (unsigned)splits);
    if (dtype == OSB_F16) {
        osb_launch((inorm_stats_kernel<__half>), grid, 256, 0, st, (const __half*)x, g_inorm_partial, n_per_c, splits);
        osb_launch((inorm_apply_kernel<__half>), grid, 256, 0, st, (const __half*)x, (__half*)y, g_inorm_partial, n_per_c, splits, (const __half*)scale, (const __half*)bias, eps);
    } else if (dtype == OSB_F32) {
        osb_launch((inorm_stats_kernel<float>), grid, 256, 0, st, (const float*)x, g_inorm_partial, n_per_c, splits);
        osb_launch((inorm_apply_kernel<float>), grid, 256, 0, st, (const float*)x, (float*)y, g_inorm_partial, n_per_c, splits, (const float*)scale, (const float*)bias, eps);
    } else return (int)cudaErrorInvalidValue;
    launched();
    return launched();
}

int osb_group_norm(const void* x, void* y, int dtype, int nhwc, int64_t C, int64_t HW, int groups, const void* gamma, const void* beta,
                   float eps, int fuse_silu, void* stats_, void* stream)
{
    double* stats = (double*)stats_;
    if (C * HW == 0) return 0;
    if (C % groups) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    {
        // single-launch path: NHWC, vectorisable channel count, scratch layout [0,1024) two-pass stats | [1024,1920) fused stats
        // (zero-initialised by the caller, self-cleaning) | [1920,1928) rendezvous counters
        int vec = dtype == OSB_F16 ? 8 : 4;
        static int fused_ok = -1;
        if (fused_ok < 0) { const char* e = getenv("OSB_GN_FUSED"); fused_ok = (e && e[0] == '0') ? 0 : 1; }
        if (fused_ok && nhwc && groups <= 48 && C % vec == 0 && C / vec <= 512 && aligned16(x) && aligned16(y) && (dtype == OSB_F16 || dtype == OSB_F32)) {
            double* fstats = (double*)((char*)stats_ + 1024);
            int* counters = (int*)((char*)stats_ + 1920);
            // one CTA per SM by default (every CTA must be co-resident for the rendezvous; fewer CTAs = fewer same-address atomics)
            static const int cta_cap = [] { const char* e = getenv("OSB_GN_CTAS"); int v = e ? atoi(e) : 0; return v > 0 ? v : OSB_SMS; }();
            int threads = C / vec <= 256 ? 256 : 512;
            size_t smem = sizeof(double) * 2 * groups;
            // co-residency bound from the device itself (SM count x resident CTAs of THIS kernel at this block size), and a cooperative
            // launch so the driver gang-schedules the grid: with SMs held by other work the launch waits (or fails) instead of spinning
            int dev = 0, sms = 0, occ = 0;
            cudaGetDevice(&dev);
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            if (dtype == OSB_F16) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gn_fused_nhwc_kernel<__half, 8>, threads, smem);
            else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gn_fused_nhwc_kernel<float, 4>, threads, smem);
            const int64_t resident = (int64_t)sms * std::min(occ, 2);
            if (resident >= 1) {
                int64_t c2 = std::min<int64_t>(HW, std::min<int64_t>(cta_cap, resident));
                int64_t ppc2 = (HW + c2 - 1) / c2;
                c2 = (HW + ppc2 - 1) / ppc2;
                if (dtype == OSB_F16) osb_launch_coop((gn_fused_nhwc_kernel<__half, 8>), (unsigned)c2, threads, smem, st, (const __half*)x, (__half*)y, fstats, counters, (int)C, HW, groups, ppc2, (const __half*)gamma, (const __half*)beta, eps, fuse_silu);
                else osb_launch_coop((gn_fused_nhwc_kernel<float, 4>), (unsigned)c2, threads, smem, st, (const float*)x, (float*)y, fstats, counters, (int)C, HW, groups, ppc2, (const float*)gamma, (const float*)beta, eps, fuse_silu);
                int rc = launched();
                if (rc != (int)cudaErrorCooperativeLaunchTooLarge && rc != (int)cudaErrorNotSupported) return rc;
                // not schedulable as one gang on this device / partition: the two-pass path below has no rendezvous
            }
        }
    }
    cudaError_t e = cudaMemsetAsync(stats, 0, sizeof(double) * 2 * groups, st);
    if (e != cudaSuccess) return (int)e;
    size_t n = (size_t)C * HW;
    if (nhwc) {
        int64_t ctas = min<int64_t>(HW, OSB_SMS * 4);
        int64_t ppc = (HW + ctas - 1) / ctas;
        ctas = (HW + ppc - 1) / ppc;
        size_t smem = sizeof(float) * 2 * groups;
        int vec = dtype == OSB_F16 ? 8 : 4;
        if (C % vec == 0 && C / vec <= 256 && aligned16(x)) {
            int64_t c2 = min<int64_t>(HW, OSB_SMS * 2);
            int64_t ppc2 = (HW + c2 - 1) / c2;
            c2 = (HW + ppc2 - 1) / ppc2;
            const size_t smem2 = sizeof(float) * (2 * groups + (size_t)(256 / (C / vec)) * 2 * C);    // + the per-row partials
            if (dtype == OSB_F16) osb_launch((gn_stats_nhwc_vec_kernel<__half, 8>), (unsigned)c2, 256, smem2, st, (const __half*)x, stats, (int)C, HW, groups, ppc2, (const __half*)nullptr, (__half*)nullptr, 1, (const __half*)nullptr, 0);
            else if (dtype == OSB_F32) osb_launch((gn_stats_nhwc_vec_kernel<float, 4>), (unsigned)c2, 256, smem2, st, (const float*)x, stats, (int)C, HW, groups, ppc2, (const float*)nullptr, (float*)nullptr, 1, (const float*)nullptr, 0);
            else return (int)cudaErrorInvalidValue;
            goto stats_done;
        }
        int threads = (int)min<int64_t>(1024, ((C + 31) / 32) * 32);
        if (dtype == OSB_F16) osb_launch((gn_stats_nhwc_kernel<__half>), (unsigned)ctas, threads, smem, st, (const __half*)x, stats, C, HW, groups, ppc);
        else if (dtype == OSB_F32) osb_launch((gn_stats_nhwc_kernel<float>), (unsigned)ctas, threads, smem, st, (const float*)x, stats, C, HW, groups, ppc);
        else return (int)cudaErrorInvalidValue;
    } else {
        int64_t n_per_g = (C / groups) * HW;
        int splits = (int)max<int64_t>(1, min<int64_t>(64, (OSB_SMS * 4 + groups - 1) / groups));
        while (splits > 1 && n_per_g / splits < 2048) splits--;
        dim3 grid((unsigned)groups, (unsigned)splits);
        if (dtype == OSB_F16) osb_launch((gn_stats_nchw_kernel<__half>), grid, 256, 0, st, (const __half*)x, stats, n_per_g, splits);
        else if (dtype == OSB_F32) osb_launch((gn_stats_nchw_kernel<float>), grid, 256, 0, st, (const float*)x, stats, n_per_g, splits);
        else return (int)cudaErrorInvalidValue;
    }
stats_done:
    launched();
    bool al = aligned16(x) && aligned16(y);
    if (dtype == OSB_F16) {
        if (al && n % 8 == 0 && (nhwc ? C % 8 == 0 : HW % 8 == 0))
            osb_launch((gn_apply_kernel<__half, 8>), grid_for(n / 8, 256), 256, 0, st, (const __half*)x, (__half*)y, stats, nhwc, C, HW, groups, (const __half*)gamma, (const __half*)beta, eps, fuse_silu);
        else
            osb_launch((gn_apply_kernel<__half, 1>), grid_for(n, 256), 256, 0, st, (const __half*)x, (__half*)y, stats, nhwc, C, HW, groups, (const __half*)gamma, (const __half*)beta, eps, fuse_silu);
    } else {
        if (al && n % 4 == 0 && (nhwc ? C % 4 == 0 : HW % 4 == 0))
            osb_launch((gn_apply_kernel<float, 4>), grid_for(n / 4, 256), 256, 0, st, (const float*)x, (float*)y, stats, nhwc, C, HW, groups, (const float*)gamma, (const float*)beta, eps, fuse_silu);
        else
            osb_launch((gn_apply_kernel<float, 1>), grid_for(n, 256), 256, 0, st, (const float*)x, (float*)y, stats, nhwc, C, HW, groups, (const float*)gamma, (const float*)beta, eps, fuse_silu);
    }
    return launched();
}

int osb_group_norm_apply(const void* x, void* y, int dtype, int64_t C, int64_t HW, int groups, const void* gamma, const void* beta, float eps, int fuse_silu,
                         const void* stats, void* clear_stats, void* stream)
{
    if (C * HW == 0) return 0;
    const int vec = dtype == OSB_F16 ? 8 : 4;
    if (groups < 1 || C % groups || C % vec || C > 4096 || !aligned16(x) || !aligned16(y)) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = sizeof(float) * 3 * (size_t)C;      // <= 48 KB (C <= 4096)
    const int64_t nvec = HW * (C / vec);
    // every CTA pays the table set-up (C channels, a few hundred cycles); 4 vectors per thread per pass, up to 4 CTAs per SM
    const int grid = (int)max<int64_t>(1, min<int64_t>((nvec + 256 * 4 - 1) / (256 * 4), OSB_SMS * 4));
    if (dtype == OSB_F16) osb_launch((gn_apply_pre_kernel<__half, 8>), grid, 256, smem, st, (const __half*)x, (__half*)y, (const double*)stats, (double*)clear_stats, (int)C, HW, groups, (const __half*)gamma, (const __half*)beta, eps, fuse_silu);
    else if (dtype == OSB_F32) osb_launch((gn_apply_pre_kernel<float, 4>), grid, 256, smem, st, (const float*)x, (float*)y, (const double*)stats, (double*)clear_stats, (int)C, HW, groups, (const float*)gamma, (const float*)beta, eps, fuse_silu);
    else return (int)cudaErrorInvalidValue;
    return launched();
}

// NHWC statistics producer for osb_group_norm_apply: stats[2 * groups] += per-group (sum, sum of squares) of y = x + addv[c] (addv / y may
// both be null: statistics of x).  Returns cudaErrorInvalidValue for shapes the vector kernel does not cover (callers then take osb_group_norm).
int osb_channel_add_stats(const void* x, const void* addv, void* y, int dtype, int64_t C, int64_t HW, int groups, void* stats, void* stream)
{
    if (C * HW == 0) return 0;
    const int vec = dtype == OSB_F16 ? 8 : 4;
    if ((dtype != OSB_F16 && dtype != OSB_F32) || groups < 1 || C % groups || C % vec || C / vec > 256 || !aligned16(x) || (y && !aligned16(y)) || (addv && !aligned16(addv)) || ((addv == nullptr) != (y == nullptr)))
        return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    // pixels per CTA: enough CTAs to fill the machine (4 per SM), but >= 4 pixel rows per thread-row so the unrolled loop is used;
    // each CTA ends with 2 * groups fp64 atomics, so more CTAs is not free
    const int rows_per_cta = (int)max<int64_t>(1, 256 / (C / vec));
    int64_t c2 = min<int64_t>((HW + 4 * rows_per_cta - 1) / (4 * rows_per_cta), OSB_SMS * 4);
    c2 = max<int64_t>(c2, 1);
    int64_t ppc2 = (HW + c2 - 1) / c2;
    c2 = (HW + ppc2 - 1) / ppc2;
    size_t smem = sizeof(float) * (2 * groups + (size_t)rows_per_cta * 2 * C);
    if (dtype == OSB_F16) osb_launch((gn_stats_nhwc_vec_kernel<__half, 8>), (unsigned)c2, 256, smem, st, (const __half*)x, (double*)stats, (int)C, HW, groups, ppc2, (const __half*)addv, (__half*)y, 0, (const __half*)nullptr, 0);
    else osb_launch((gn_stats_nhwc_vec_kernel<float, 4>), (unsigned)c2, 256, smem, st, (const float*)x, (double*)stats, (int)C, HW, groups, ppc2, (const float*)addv, (float*)y, 0, (const float*)nullptr, 0);
    return launched();
}

// Channel Concat of two NHWC images that a GroupNorm reads next: y [HW, ca + cb] = [a | b] in one pass that also adds the per-group (sum, sum
// of squares) of y to stats[2 * groups], as osb_channel_add_stats does for the Add.  cudaErrorInvalidValue: a layout the kernel does not cover
// (a source's channels not a multiple of the vector, more than 1024 vectors per pixel, unaligned pointers); nothing is launched then.
int osb_concat2_stats(const void* a, const void* b, void* y, int dtype, int64_t ca, int64_t cb, int64_t HW, int groups, void* stats, void* stream)
{
    const int vec = dtype == OSB_F16 ? 8 : 4;
    const int64_t C = ca + cb;
    if ((dtype != OSB_F16 && dtype != OSB_F32) || HW < 1 || groups < 1 || ca < 1 || cb < 1 || C % groups || ca % vec || cb % vec || C / vec > 1024 ||
        !aligned16(a) || !aligned16(b) || !aligned16(y))
        return (int)cudaErrorInvalidValue;
    // one pixel's vectors per thread row, as many rows as fit 256 threads (a wider pixel takes a block of its own width)
    const int tpp = (int)(C / vec), threads = tpp <= 256 ? 256 : (tpp + 31) / 32 * 32, rows_per_cta = threads / tpp;
    int64_t c2 = max<int64_t>(1, min<int64_t>((HW + 4 * rows_per_cta - 1) / (4 * rows_per_cta), OSB_SMS * 4));
    const int64_t ppc2 = (HW + c2 - 1) / c2;
    c2 = (HW + ppc2 - 1) / ppc2;
    const size_t smem = sizeof(float) * (2 * groups + (size_t)rows_per_cta * 2 * C);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == OSB_F16) osb_launch((gn_stats_nhwc_vec_kernel<__half, 8, true>), (unsigned)c2, threads, smem, st, (const __half*)a, (double*)stats, (int)C, HW, groups, ppc2,
                                     (const __half*)nullptr, (__half*)y, 0, (const __half*)b, (int)ca);
    else osb_launch((gn_stats_nhwc_vec_kernel<float, 4, true>), (unsigned)c2, threads, smem, st, (const float*)a, (double*)stats, (int)C, HW, groups, ppc2,
                    (const float*)nullptr, (float*)y, 0, (const float*)b, (int)ca);
    return launched();
}

// Range of a float tensor for dynamic quantisation (Model::get_percentiles): out3 is a DEVICE array of 3 uint32 (see the kernel); the
// caller initialises it to { 0xFFFFFFFF, 0, 0 } and decodes the order-preserving keys with osb_percentile_key_to_float.
int osb_percentiles(const void* x, int dtype, size_t n, int threads, float from_left, float from_right, void* out3, void* stream)
{
    if (n == 0) return 0;
    if (dtype != OSB_F16 && dtype != OSB_F32) return (int)cudaErrorInvalidValue;
    if (threads < 1) threads = 1;
    const size_t chunk = dtype == OSB_F16 ? 32768 : 16384;       // m_perthread_buffer_size (64 KiB) / sizeof(element)
    size_t per = n / (size_t)threads; if (!per) per = 1;
    const size_t longest = std::max(per, n - per * ((size_t)threads - 1 < n / per ? (size_t)threads - 1 : n / per));
    dim3 grid((unsigned)((longest + chunk - 1) / chunk), (unsigned)threads);
    const size_t smem = chunk * sizeof(unsigned);
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(percentile_chunks_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(32768 * 4));
        cudaFuncSetAttribute(percentile_chunks_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(16384 * 4));
        attr = true;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == OSB_F16) percentile_chunks_kernel<__half><<<grid, 1024, smem, st>>>((const __half*)x, n, (size_t)threads, chunk, from_left, from_right, (unsigned*)out3);
    else percentile_chunks_kernel<float><<<grid, 1024, smem, st>>>((const float*)x, n, (size_t)threads, chunk, from_left, from_right, (unsigned*)out3);
    return launched();
}

float osb_percentile_key_to_float(unsigned key, int dtype)
{
    if (dtype == OSB_F16) {
        unsigned short h = (key & 0x8000u) ? (unsigned short)(key & 0x7FFFu) : (unsigned short)(~key & 0xFFFFu);
        __half hv; memcpy(&hv, &h, 2);
        return __half2float(hv);
    }
    unsigned u = (key & 0x80000000u) ? (key & 0x7FFFFFFFu) : ~key;
    float f; memcpy(&f, &u, 4);
    return f;
}

int osb_binary_qu8(int op, const void* a, const int64_t* as, float sa, int za, const void* b, const int64_t* bs, float sb, int zb,
                   void* out, float so, int zo, const int64_t* shape, int ndim, void* stream)
{
    if (ndim < 1 || ndim > OSB_MAX_DIMS || (op != OSB_BIN_ADD && op != OSB_BIN_MUL)) return (int)cudaErrorInvalidValue;
    size_t n = 1;
    BinParams p; p.ndim = ndim;
    for (int d = 0; d < OSB_MAX_DIMS; d++) { p.shape[d] = d < ndim ? shape[d] : 1; p.as[d] = d < ndim ? as[d] : 0; p.bs[d] = d < ndim ? bs[d] : 0; if (d < ndim) n *= (size_t)shape[d]; }
    if (n == 0) return 0;
    Qu8BinParams q{};
    q.op = op; q.za = za; q.zb = zb; q.zo = zo;
    if (op == OSB_BIN_ADD) {
        // xnn_init_qu8_add_minmax_*_params
        const float ao = sa / so, bo = sb / so;
        const float mx = fmaxf(fabsf(ao), fabsf(bo));
        uint32_t mbits; memcpy(&mbits, &mx, 4);
        const int32_t expo = (int32_t)(mbits >> 23) - 127;
        const uint32_t shift = (uint32_t)(20 - expo);
        if (shift < 1 || shift > 31) return (int)cudaErrorInvalidValue;
        auto mult = [&](float v) { float av = fabsf(v); uint32_t bits; memcpy(&bits, &av, 4); bits += shift << 23; float f; memcpy(&f, &bits, 4); int32_t m = (int32_t)lrintf(f); return v < 0 ? -m : m; };
        q.ma = mult(ao); q.mb = mult(bo); q.shift = (int)shift;
        q.bias = (int)((1u << (shift - 1)) - (uint32_t)(q.ma * za) - (uint32_t)(q.mb * zb));
    } else {
        q.mul_scale = sa * sb / so;
    }
    osb_launch((binary_qu8_kernel), grid_for(n, 256), 256, 0, (cudaStream_t)stream, (const uint8_t*)a, (const uint8_t*)b, (uint8_t*)out, p, n, q);
    return launched();
}

int osb_softmax_qu8(const void* x, void* y, int64_t rows, int64_t cols, float in_scale, float out_scale, int out_zp, void* stream)
{
    if (rows * cols == 0) return 0;
    int threads = cols >= 1024 ? 256 : (cols >= 256 ? 128 : 32);
    osb_launch((softmax_qu8_kernel), (unsigned)min<int64_t>(rows, OSB_SMS * 16), threads, 0, (cudaStream_t)stream, (const uint8_t*)x, (uint8_t*)y, rows, cols, in_scale, out_scale, out_zp);
    return launched();
}

int osb_rms_norm(const void* x, int xd, const void* w, int wd, void* y, int yd, int64_t rows, int64_t cols, float eps, void* stream)
{
    if (rows * cols == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = (unsigned)min<int64_t>((rows + 3) / 4, OSB_SMS * 8);
    const bool per_block = rows <= 64 && cols >= 512;
#define OSB_RMS(TI_, TW_, TO_) do { if (per_block) osb_launch((rms_norm_block_kernel<TI_, TW_, TO_>), (unsigned)rows, 256, 0, st, (const TI_*)x, (const TW_*)w, (TO_*)y, (int)cols, eps); \
                                    else osb_launch((rms_norm_kernel<TI_, TW_, TO_>), grid, 128, 0, st, (const TI_*)x, (const TW_*)w, (TO_*)y, rows, (int)cols, eps); } while (0)
    if (xd == OSB_F16 && wd == OSB_F16 && yd == OSB_F16) OSB_RMS(__half, __half, __half);
    else if (xd == OSB_F16 && wd == OSB_F16 && yd == OSB_F32) OSB_RMS(__half, __half, float);
    else if (xd == OSB_F16 && wd == OSB_F32 && yd == OSB_F32) OSB_RMS(__half, float, float);
    else if (xd == OSB_F16 && wd == OSB_F32 && yd == OSB_F16) OSB_RMS(__half, float, __half);
    else if (xd == OSB_F32 && wd == OSB_F32 && yd == OSB_F32) OSB_RMS(float, float, float);
    else if (xd == OSB_F32 && wd == OSB_F16 && yd == OSB_F32) OSB_RMS(float, __half, float);
    else if (xd == OSB_F32 && wd == OSB_F32 && yd == OSB_F16) OSB_RMS(float, float, __half);
    else if (xd == OSB_F32 && wd == OSB_F16 && yd == OSB_F16) OSB_RMS(float, __half, __half);
    else return (int)cudaErrorInvalidValue;
#undef OSB_RMS
    return launched();
}

int osb_rope(const void* x, const void* cs, const void* sn, void* y, int dtype, int64_t rows, int64_t D, int64_t table_rows, void* stream)
{
    if (rows * D == 0) return 0;
    if (D % 2 || table_rows < 1 || rows % table_rows) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == OSB_F16) osb_launch((rope_kernel<__half>), grid_for((size_t)(rows * D), 256), 256, 0, st, (const __half*)x, (const __half*)cs, (const __half*)sn, (__half*)y, rows, (int)D, table_rows);
    else if (dtype == OSB_F32) osb_launch((rope_kernel<float>), grid_for((size_t)(rows * D), 256), 256, 0, st, (const float*)x, (const float*)cs, (const float*)sn, (float*)y, rows, (int)D, table_rows);
    else return (int)cudaErrorInvalidValue;
    return launched();
}

int osb_gather_rows(const void* table, const int64_t* idx, void* out, int64_t n_idx, int64_t table_rows, int64_t row_bytes, void* stream)
{
    if (n_idx * row_bytes == 0) return 0;
    int threads = row_bytes >= 4096 ? 256 : 64;
    osb_launch((gather_rows_kernel), (unsigned)min<int64_t>(n_idx, OSB_SMS * 8), threads, 0, (cudaStream_t)stream, (const uint8_t*)table, idx, (uint8_t*)out, n_idx, table_rows, row_bytes);
    return launched();
}

int osb_scatter_elems(void* out, const int64_t* pos, const void* updates, int64_t n, int elem_size, void* stream)
{
    if (n == 0) return 0;
    if (elem_size != 2 && elem_size != 4) return (int)cudaErrorInvalidValue;
    osb_launch((scatter_elems_kernel), grid_for((size_t)n, 256), 256, 0, (cudaStream_t)stream, (uint8_t*)out, pos, (const uint8_t*)updates, n, elem_size);
    return launched();
}

int osb_maxpool_nhwc(const void* x, void* y, int dtype, int64_t H, int64_t W, int64_t C, int kh, int kw, int stride, int pad_top, int pad_left,
                     int64_t Ho, int64_t Wo, void* stream)
{
    if (Ho * Wo * C == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    size_t n = (size_t)Ho * Wo * C;
    if (dtype == OSB_F16) osb_launch((maxpool_nhwc_kernel<__half>), grid_for(n, 256), 256, 0, st, (const __half*)x, (__half*)y, (int)H, (int)W, (int)C, kh, kw, stride, pad_top, pad_left, (int)Ho, (int)Wo);
    else if (dtype == OSB_F32) osb_launch((maxpool_nhwc_kernel<float>), grid_for(n, 256), 256, 0, st, (const float*)x, (float*)y, (int)H, (int)W, (int)C, kh, kw, stride, pad_top, pad_left, (int)Ho, (int)Wo);
    else return (int)cudaErrorInvalidValue;
    return launched();
}

int osb_fill(void* dst, int dtype, size_t n, float value, void* stream)
{
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == OSB_F16) osb_launch((fill_kernel<__half>), grid_for(n, 256), 256, 0, st, (__half*)dst, n, value);
    else if (dtype == OSB_F32) osb_launch((fill_kernel<float>), grid_for(n, 256), 256, 0, st, (float*)dst, n, value);
    else return (int)cudaErrorInvalidValue;
    return launched();
}

} // extern "C"
