// tc_ptx.cuh -- inline-PTX wrappers shared by the sm_90a tensor-core kernels (gemm_wgmma.cu, attention_wgmma.cu): mbarrier, TMA,
// shared-memory matrix descriptors and warpgroup MMA (wgmma); on the host, the TMA tensor maps they read through.
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cstdio>
#include <mutex>

namespace tcptx {

// ---- TMA tensor maps (host) ---------------------------------------------------------------------------------------

// the driver's cuTensorMapEncodeTiled, or nullptr when the driver has none
inline PFN_cuTensorMapEncodeTiled_v12000 get_encode()
{
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (PFN_cuTensorMapEncodeTiled_v12000)p;
    });
    return fn;
}

// rank-3 fp16 tensor map with 128B swizzle (or `swizzle`); dims/strides innermost first
inline bool make_map(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1_bytes, uint64_t s2_bytes,
                     uint32_t b0, uint32_t b1, uint32_t b2, uint32_t traversal_stride = 1, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                     CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B)
{
    auto enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[3] = { d0, d1, d2 };
    cuuint64_t strides[2] = { s1_bytes, s2_bytes };
    cuuint32_t box[3] = { b0, b1, b2 };
    cuuint32_t estr[3] = { 1, traversal_stride, traversal_stride };   // strided conv: every s-th pixel of the box span
    CUresult r = enc(map, dtype, 3, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// rank-4 bf16 tensor map with 128B swizzle; dims/strides innermost first, traversal strides (1, 1, s, s) (the bf16 planes of an NHWC
// image as (C, plane, W, H): a strided conv takes every s-th pixel of the box span)
inline bool make_map_4d(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3, uint64_t s1_bytes, uint64_t s2_bytes,
                        uint64_t s3_bytes, uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3, uint32_t traversal_stride)
{
    auto enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[4] = { d0, d1, d2, d3 };
    cuuint64_t strides[3] = { s1_bytes, s2_bytes, s3_bytes };
    cuuint32_t box[4] = { b0, b1, b2, b3 };
    cuuint32_t estr[4] = { 1, 1, traversal_stride, traversal_stride };
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// ---- PTX wrappers ---------------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    long long t0 = 0;
    while (true) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}" : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) break;
        // watchdog: a protocol bug must surface as a launch failure, never as a hung GPU (~2 s at 2 GHz).  No printf here: a function
        // call inside the MMA loop makes ptxas serialise every wgmma.
        long long now = clock64();
        if (t0 == 0) t0 = now;
        else if (now - t0 > 4000000000LL) __trap();
    }
}

__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(smem)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// The producer warp runs WARP-UNIFORM control flow and issues from an elect.sync-guarded region, so ptxas keeps the TMA operands in
// uniform registers.
__device__ __forceinline__ void tma_load_3d_s(uint32_t smem_addr, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_addr), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_4d_s(uint32_t smem_addr, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3)
{
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(smem_addr), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
// TMA multicast: the box lands at the same shared-memory offset in every CTA of `cta_mask` and completes bytes on the mbarrier at the
// same offset in each of them
__device__ __forceinline__ void tma_load_3d_mc(uint32_t smem_addr, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, uint16_t cta_mask)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5}], [%2], %6;"
                 ::"r"(smem_addr), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "h"(cta_mask) : "memory");
}

// ---- thread-block clusters ----
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_id_x() { uint32_t r; asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_count_x() { uint32_t r; asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r)); return r; }
// every thread of every CTA of the cluster; orders shared-memory writes (barrier init) before the peers use them
__device__ __forceinline__ void cluster_sync()
{
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t cta)
{
    asm volatile("{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\tmbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}"
                 ::"r"(smem_u32(bar)), "r"(cta) : "memory");
}

// one lane of a converged warp, chosen by the hardware (elect.sync): ptxas knows the guarded region runs on exactly one lane
__device__ __forceinline__ bool elect_one()
{
    uint32_t pred = 0;
    asm volatile("{\n\t.reg .pred px;\n\telect.sync _|px, 0xffffffff;\n\tselp.u32 %0, 1, 0, px;\n\t}" : "=r"(pred));
    return pred != 0;
}

// named barrier over `count` threads (id 0 is __syncthreads): sync waits for the count, arrive adds this warp's threads and goes on
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// per-thread register budget of the executing warpgroup (every warp of it executes the instruction)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// pins registers that an asynchronous wgmma reads or writes: the compiler may not move their other uses across this point
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N])
{
#pragma unroll
    for (int i = 0; i < N; i++) asm volatile("" : "+f"(r[i])::"memory");
}
template <int N>
__device__ __forceinline__ void fence_regs(uint32_t (&r)[N][4])
{
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int e = 0; e < 4; e++) asm volatile("" : "+r"(r[i][e])::"memory");
}

// shared-memory matrix descriptor for wgmma (cute/arch/mma_sm90_desc.hpp GmmaDescriptor): 128B swizzle, start / LBO / SBO in 16-byte units.
//   K-major: 8-row groups SBO bytes apart (LBO unused).  MN-major: 64-element MN atoms LBO bytes apart, 8-row K groups SBO bytes apart.
// Every operand tile starts on a 1024-byte boundary, so the base-offset field stays 0; advancing K inside a swizzle row adds to the start address.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)1 << 62;   // layout type SWIZZLE_128B
    return d;
}

// wgmma ordering: fence before the first MMA that reads registers written by ordinary code, commit the issued MMAs as one group, and
// wait until at most N groups are still in flight
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Accumulator fragments of an m64nN wgmma: thread t of the warpgroup holds, for every 8-column block j, d[4j], d[4j+1] at row
// 16 (t / 32) + (t % 32) / 4, columns 8j + 2 (t % 4) + {0, 1}, and d[4j+2], d[4j+3] at the row 8 below.
// Shared-A wgmma (A and B from shared-memory descriptors), fp32 accumulators: m64nNk16 for the N the kernels use, in fp16 and bf16.
// TC_R<n> is the asm list of n accumulator operands, TC_D<n> the matching "+f" operand list; the four operands after them are the A and B
// descriptors, the scale-d flag and the B transpose immediate (their operand numbers are ODA, ODB, OSC, OTB).
#define TC_R8(a, b, c, d, e, f, g, h) "%" #a ", %" #b ", %" #c ", %" #d ", %" #e ", %" #f ", %" #g ", %" #h
#define TC_R16 TC_R8(0, 1, 2, 3, 4, 5, 6, 7) ", " TC_R8(8, 9, 10, 11, 12, 13, 14, 15)
#define TC_R32 TC_R16 ", " TC_R8(16, 17, 18, 19, 20, 21, 22, 23) ", " TC_R8(24, 25, 26, 27, 28, 29, 30, 31)
#define TC_R40 TC_R32 ", " TC_R8(32, 33, 34, 35, 36, 37, 38, 39)
#define TC_R64 TC_R40 ", " TC_R8(40, 41, 42, 43, 44, 45, 46, 47) ", " TC_R8(48, 49, 50, 51, 52, 53, 54, 55) ", " TC_R8(56, 57, 58, 59, 60, 61, 62, 63)
#define TC_R80 TC_R64 ", " TC_R8(64, 65, 66, 67, 68, 69, 70, 71) ", " TC_R8(72, 73, 74, 75, 76, 77, 78, 79)
#define TC_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define TC_D16 TC_D8(0), TC_D8(8)
#define TC_D32 TC_D16, TC_D8(16), TC_D8(24)
#define TC_D40 TC_D32, TC_D8(32)
#define TC_D64 TC_D40, TC_D8(40), TC_D8(48), TC_D8(56)
#define TC_D80 TC_D64, TC_D8(64), TC_D8(72)
#define TC_WGMMA_SS(N, TY, NAME, R, ODA, ODB, OSC, OTB, ...)                                                                                 \
    template <int TRANS_B>                                                                                                              \
    __device__ __forceinline__ void NAME(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d)                                 \
    {                                                                                                                                   \
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " OSC ", 0;\n\t"                                                              \
                     "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." TY "." TY " {" R "}, " ODA ", " ODB ", p, 1, 1, 0, " OTB ";\n\t}" \
                     : __VA_ARGS__ : "l"(da), "l"(db), "r"(scale_d), "n"(TRANS_B));                                                     \
    }
#define TC_WGMMA_SS2(N, R, ODA, ODB, OSC, OTB, ...)                                      \
    TC_WGMMA_SS(N, "f16", wgmma_m64n##N##k16_f16, R, ODA, ODB, OSC, OTB, __VA_ARGS__)   \
    TC_WGMMA_SS(N, "bf16", wgmma_m64n##N##k16_bf16, R, ODA, ODB, OSC, OTB, __VA_ARGS__)
TC_WGMMA_SS2(32, TC_R16, "%16", "%17", "%18", "%19", TC_D16)
TC_WGMMA_SS2(64, TC_R32, "%32", "%33", "%34", "%35", TC_D32)
TC_WGMMA_SS2(80, TC_R40, "%40", "%41", "%42", "%43", TC_D40)
TC_WGMMA_SS2(128, TC_R64, "%64", "%65", "%66", "%67", TC_D64)
TC_WGMMA_SS2(160, TC_R80, "%80", "%81", "%82", "%83", TC_D80)

// m64nNk16 by N (the columns of one warpgroup's accumulator tile) and operand type
template <int N, int TRANS_B, bool BF16>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d)
{
#define TC_CASE(n) if constexpr (N == n) { if constexpr (BF16) wgmma_m64n##n##k16_bf16<TRANS_B>(d, da, db, scale_d); else wgmma_m64n##n##k16_f16<TRANS_B>(d, da, db, scale_d); }
    TC_CASE(32) TC_CASE(64) TC_CASE(80) TC_CASE(128) TC_CASE(160)
#undef TC_CASE
    static_assert(N == 32 || N == 64 || N == 80 || N == 128 || N == 160, "no wgmma wrapper for this N");
}
__device__ __forceinline__ void wgmma_m64n128k32_u8(int32_t (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_m64n64k16_f16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
// A from registers (bf16 pairs in the A-fragment order of the f16 variant above), B MN-major from shared memory
__device__ __forceinline__ void wgmma_m64n64k16_bf16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}


// ---- GroupNorm statistics of a GEMM / conv output, gathered in the producing kernel's epilogue -----------------------------------
// The consumer GroupNorm needs sum(x) and sum(x^2) per group of `cpg` consecutive channels over ALL rows (pixels).  A thread holds two
// adjacent columns of two rows per 8-column block (the accumulator fragment above): the 8 lanes that share those columns sum their rows by
// shuffle, and lanes 0..3 add the column totals to the CTA's per-group shared accumulators.  After the tile the accumulators are flushed to
// the global fp64 statistics (the reference accumulates in double).  Plain fp32 sums of y and y^2 would cancel in E[y^2] - mean^2 when
// the mean is large against the spread, so a column's fp32 warp partial is of y - p, p = that column's value in the warp's first valid
// row, and is shifted back in fp64 (S += s + c p, Q += q + 2 p s + c p^2, c = the warp's valid rows) into fp64 CTA accumulators.
constexpr int GN_MAX_GROUPS = 64;

// fp64 add into shared memory (a CAS loop in SASS; the explicit state space keeps the compiler from adding a global-memory path)
__device__ __forceinline__ void shared_add_f64(double* p, double v)
{
    asm volatile("red.shared.add.f64 [%0], %1;" ::"r"(smem_u32(p)), "d"(v) : "memory");
}

// v0 / v1: this thread's two columns (n, n + 1), each summed over its valid rows as y - p0 / y - p1 with y rounded as it is stored
// (columns outside the problem passed as zeros); q0 / q1 the same for the squares; c: the warp's valid rows.  Lanes 0..3 (the 8 columns
// of the block) combine their fp64 sums by group before the shared adds: one per group the block touches, not one per lane.
__device__ __forceinline__ void gn_stats_pair(float v0, float v1, float q0, float q1, float p0, float p1, int c, int n, int n_end, int cpg,
                                              double* cta_stats, int lane)
{
#pragma unroll
    for (int off = 4; off < 32; off <<= 1) {
        v0 += __shfl_xor_sync(0xffffffffu, v0, off); v1 += __shfl_xor_sync(0xffffffffu, v1, off);
        q0 += __shfl_xor_sync(0xffffffffu, q0, off); q1 += __shfl_xor_sync(0xffffffffu, q1, off);
    }
    const double dc = (double)c, d0 = p0, d1 = p1;
    const bool ok0 = n < n_end && c > 0, ok1 = n + 1 < n_end && c > 0;
    const int g0 = n / cpg;
    double s = ok0 ? (double)v0 + dc * d0 : 0.0, r = ok0 ? (double)q0 + (2.0 * d0) * v0 + dc * d0 * d0 : 0.0;
    if (ok1) {
        const double s1 = (double)v1 + dc * d1, r1 = (double)q1 + (2.0 * d1) * v1 + dc * d1 * d1;
        if ((n + 1) / cpg == g0) { s += s1; r += r1; }
        else if (lane < 4) { shared_add_f64(&cta_stats[2 * (g0 + 1)], s1); shared_add_f64(&cta_stats[2 * (g0 + 1) + 1], r1); }
    }
    // segmented sum over lanes 0..3 by group (groups are contiguous, so lane l's group <= lane l + 1's): lane 2k takes lane 2k + 1,
    // then lane 0 takes lane 2; a lane whose sums were taken adds nothing itself
    const int g = ok0 ? g0 : -1;
    bool taken = false;
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {
        const double so = __shfl_down_sync(0xffffffffu, s, off), ro = __shfl_down_sync(0xffffffffu, r, off);
        const int go = __shfl_down_sync(0xffffffffu, g, off);
        const int gu = __shfl_up_sync(0xffffffffu, g, off);
        if ((lane & (2 * off - 1)) == 0 && go == g && g >= 0) { s += so; r += ro; }
        if ((lane & (2 * off - 1)) == off && gu == g) taken = true;
    }
    if (lane < 4 && g >= 0 && !taken) { shared_add_f64(&cta_stats[2 * g], s); shared_add_f64(&cta_stats[2 * g + 1], r); }
}

// after a tile: thread t of the epilogue group moves accumulator t to the global fp64 statistics and re-arms it
__device__ __forceinline__ void gn_stats_flush(double* cta_stats, double* gstats, int groups, int t)
{
    if (t < 2 * groups) {
        const double v = __longlong_as_double((long long)atomicExch(reinterpret_cast<unsigned long long*>(&cta_stats[t]), 0ull));
        if (v != 0.0) atomicAdd(&gstats[t], v);
    }
}

}  // namespace tcptx
