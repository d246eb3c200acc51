// common.cuh -- shared device helpers for the sm_90a kernels.
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <algorithm>
#include <utility>
#include "../../include/onnxstream_b200_kernels.h"

using std::min;
using std::max;

extern "C" void osb_count_launch(int tensor_core);

// ---- launch bookkeeping --------------------------------------------------------------------------------------
static inline int launched(int tensor_core = 0)
{
    osb_count_launch(tensor_core);
    return (int)cudaGetLastError();
}

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------------------------
// Every kernel (a) signals at entry that the next kernel in the stream may be scheduled and (b) waits for its own
// predecessor to complete before touching global memory.  With ~1000 short kernels per UNet step this hides the launch
// latency and prologue of kernel i+1 behind the tail of kernel i (CUDA graphs keep the programmatic edges).
__device__ __forceinline__ void osb_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void osb_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// OSB_PDL_LATE (build variant): short kernels do not trigger at all (the implicit trigger at exit stands), the tensor-core kernels
// trigger once their producer has issued the last tile's loads -- so dependents never take SM slots from CTAs that still have work.
#ifdef OSB_PDL_LATE
__device__ __forceinline__ void osb_pdl_trigger_entry() {}
__device__ __forceinline__ void osb_pdl_trigger_late() { osb_pdl_trigger(); }
#else
__device__ __forceinline__ void osb_pdl_trigger_entry() { osb_pdl_trigger(); }
__device__ __forceinline__ void osb_pdl_trigger_late() {}
#endif
__device__ __forceinline__ void osb_pdl_prologue() { osb_pdl_trigger_entry(); osb_pdl_wait(); }

extern "C" int osb_pdl_enabled(void);

// cluster > 1: thread-block clusters of `cluster` consecutive CTAs along x (grid.x must be a multiple of it)
template <typename... KArgs, typename... Args>
static inline void osb_launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, unsigned cluster, Args&&... args)
{
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[2];
    int n = 0;
    if (osb_pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        n++;
    }
    if (cluster > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = cluster; attr[n].val.clusterDim.y = 1; attr[n].val.clusterDim.z = 1;
        n++;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);   // errors surface through launched() / cudaGetLastError
}

template <typename... KArgs, typename... Args>
static inline void osb_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args)
{
    osb_launch_cluster(kernel, grid, block, smem, st, 1u, std::forward<Args>(args)...);
}

// Cooperative launch: the driver gang-schedules the grid (every CTA resident at once, or the launch fails with
// cudaErrorCooperativeLaunchTooLarge) -- what a kernel with a grid-wide rendezvous needs when other work (NCCL kernels, a second
// stream) may hold SMs.
template <typename... KArgs, typename... Args>
static inline void osb_launch_coop(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args)
{
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// streaming multiprocessors of an H100 SXM: caps the grids of the grid-stride kernels (the tensor-core launchers query the device)
constexpr int OSB_SMS = 132;

static inline int grid_for(size_t work_items, int threads)
{
    size_t blocks = (work_items + threads - 1) / threads;
    size_t cap = (size_t)OSB_SMS * 16;  // persistent-ish: at most 16 CTAs per SM, grid-stride loops cover the rest
    if (blocks < 1) blocks = 1;
    return (int)(blocks < cap ? blocks : cap);
}

static inline bool aligned16(const void* p) { return (((uintptr_t)p) & 15) == 0; }

// ---- scalar conversions ----------------------------------------------------------------------------------------
__device__ __forceinline__ float to_float(float v) { return v; }
__device__ __forceinline__ float to_float(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_float(uint8_t v) { return (float)v; }
template <typename T> __device__ __forceinline__ T from_float(float v);
template <> __device__ __forceinline__ float from_float<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }

// ---- binary elementwise arithmetic (OSB_BIN_*), fp32: the node kernels and the tensor-core GEMM's GEGLU epilogue ---------------------
__device__ __forceinline__ float apply_binary(int op, float a, float b)
{
    switch (op) {
    case OSB_BIN_ADD: return a + b;
    case OSB_BIN_SUB: return a - b;
    case OSB_BIN_MUL: return a * b;
    case OSB_BIN_DIV: return a / b;
    case OSB_BIN_MUL_GELU: return a * (0.5f * b * (1.f + erff(b * 0.70710678118654752f)));
    case OSB_BIN_MUL_SIGMOID: return a / (1.f + expf(-b));
    case OSB_BIN_SILU_MUL: return (a / (1.f + expf(-a))) * b;
    default: return a;
    }
}

// ---- fp32 -> bf16 triple split of the tensor-core fp32 paths (osb_tc_gemm_f32x, osb_flash_attention_f32x) ----------------------------
// x = h + m + l, h = bf16(x), m = bf16(x - h), l = bf16(x - h - m): 24 mantissa bits in three bf16 planes
__device__ __forceinline__ void bf16x3_split(float x, __nv_bfloat16& h, __nv_bfloat16& m, __nv_bfloat16& l)
{
    h = __float2bfloat16_rn(x);
    const float r1 = x - __bfloat162float(h);
    m = __float2bfloat16_rn(r1);
    l = __float2bfloat16_rn(r1 - __bfloat162float(m));
}

// ---- 128-bit vectors -------------------------------------------------------------------------------------------
template <typename T, int N> struct alignas(sizeof(T) * N) Vec { T v[N]; };

template <typename T, int N>
__device__ __forceinline__ Vec<T, N> load_vec(const T* p)
{
    return *reinterpret_cast<const Vec<T, N>*>(p);
}
template <typename T, int N>
__device__ __forceinline__ void store_vec(T* p, const Vec<T, N>& v)
{
    *reinterpret_cast<Vec<T, N>*>(p) = v;
}

// ---- block reductions (blockDim.x multiple of 32, <= 1024) -------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float block_reduce_sum(float v, float* red)
{
    v = warp_sum(v);
    int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    v = l < nw ? red[l] : 0.f;
    v = warp_sum(v);
    return v;
}
__device__ __forceinline__ float block_reduce_max(float v, float* red)
{
    v = warp_max(v);
    int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    v = l < nw ? red[l] : -INFINITY;
    v = warp_max(v);
    return v;
}
