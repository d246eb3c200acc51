// attention_wgmma.cu -- fused flash-style attention for sm_90a: softmax(Q K^T * scale) V in ONE kernel, score tile in registers,
// never in HBM.  Replaces the reference's sliced AttentionFusedOps loop (src/onnxstream.cpp:6696-6929: per head and per Q-slice a MatMul,
// a Mul, a Softmax and a MatMul, each through XNNPACK with the [Tq/parts, Tk] score tile round-tripping through two aux buffers,
// src/onnxstream.cpp:6798-6799).
//
// One CTA per (head, 128-query tile), 384 threads:
//   warpgroup 0      TMA producer (one warp): Q tile once, then a (K tile, V tile) pair per 128 keys into a KV_STAGES-deep ring
//   warpgroups 1, 2  64 query rows each: S = Q K_j^T (wgmma m64n128k16 from shared memory, fp32 in registers), online softmax in
//                    registers (fp32, exp2 with the scale folded in), P rounded to fp16 in registers is the A operand of O += P V_j
//                    (wgmma m64n64k16, V from shared memory), finally O / sum -> fp16 -> global
// Q, K, V are read in place from the [T, heads*d] projection buffers through strided tensor maps and O is written in the
// merged [T, heads*d] layout, so the exported graph's head split / merge costs nothing.  d <= 64, d % 8 == 0.

#include "common.cuh"
#include "tc_ptx.cuh"
#include <cstdlib>
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cstdio>
#include <mutex>

namespace {

using namespace tcptx;

constexpr int BQ = 128;                 // queries per CTA
constexpr int BKV = 128;                // keys per tile
constexpr int BD = 64;                  // head dim padded to one 128-byte swizzle row
constexpr int KV_STAGES = 4;            // K/V ring: the producer runs up to three tiles ahead of the slower warpgroup
constexpr int Q_BYTES = BQ * BD * 2;    // 16 KiB
constexpr int K_BYTES = BKV * BD * 2;   // 16 KiB
constexpr int V_BYTES = BKV * BD * 2;   // 16 KiB (128 key rows x 64 columns)
constexpr int FA_SMEM = Q_BYTES + KV_STAGES * (K_BYTES + V_BYTES) + 1024 + 256;
constexpr int FA_THREADS = 384;
constexpr int FA_CONSUMERS = 256;

struct FaParams {
    int T, Tk, d, heads;
    int q_tiles, kv_tiles;
    float scale_log2;        // scale * log2(e)
    float tau;               // lazy-rescaling threshold in log2 units (0 = exact running maximum)
    __half* out;             // [T, ldo] merged layout, head h at column h*d
    long long ldo;
};

// 2^x on the SFU, flush-to-zero: one MUFU.EX2 (exp2f() adds a range check and two scaling multiplies for denormal results,
// which a probability that is about to be rounded to fp16 does not need).  ex2(-inf) = +0.
__device__ __forceinline__ float ex2_approx(float x)
{
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi)
{
    __half2 h2 = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h2);
}

__global__ void __launch_bounds__(FA_THREADS, 1)
flash_attention_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                       const FaParams p)
{
    osb_pdl_trigger_entry();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + Q_BYTES;
    uint8_t* sV = sK + KV_STAGES * K_BYTES;
    uint64_t* bars = (uint64_t*)(sV + KV_STAGES * V_BYTES);
    uint64_t* q_full = bars;                           // [1]
    uint64_t* kv_full = bars + 1;                      // [KV_STAGES]
    uint64_t* kv_empty = kv_full + KV_STAGES;          // [KV_STAGES]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, head = blockIdx.y;
    const int q0 = qt * BQ;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_q) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_k) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_v) : "memory");
    }
    if (warp == 1 && lane == 0) {
        mbar_init(q_full, 1);
        for (int i = 0; i < KV_STAGES; i++) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], FA_CONSUMERS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    osb_pdl_wait();

    const int n_kv = p.kv_tiles;

    if (warp == 0) {
        if (elect_one()) {
            mbar_expect_tx(q_full, Q_BYTES);
            tma_load_3d(sQ, &map_q, q_full, 0, head, q0);
        }
        __syncwarp();
        for (int j = 0; j < n_kv; j++) {
            const int st = j % KV_STAGES;
            mbar_wait(&kv_empty[st], ((j / KV_STAGES) & 1) ^ 1);
            if (elect_one()) {
                mbar_expect_tx(&kv_full[st], K_BYTES + V_BYTES);
                tma_load_3d(sK + st * K_BYTES, &map_k, &kv_full[st], 0, head, j * BKV);
                tma_load_3d(sV + st * V_BYTES, &map_v, &kv_full[st], 0, head, j * BKV);
                tma_load_3d(sV + st * V_BYTES + V_BYTES / 2, &map_v, &kv_full[st], 0, head, j * BKV + 64);
            }
            __syncwarp();
        }
    } else if (warp >= 4) {
        // ===================== warpgroups 1, 2: 64 query rows each =====================
        // Accumulator fragments (tc_ptx.cuh): this thread holds rows r and r + 8 of the warpgroup's 64 (h = 0, 1) and, per 8-column
        // block c, the columns 8c + cq, 8c + cq + 1 -- of the 128 keys in s[], of the 64 output columns in o[].  The four lanes of a row
        // share its maximum and sum by two shuffles.
        const int wg = (warp >> 2) - 1;
        const int r = (warp & 3) * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);
        // descriptors (start address in 16-byte units moves): Q / K K-major, 8-row groups 1024 B apart, 32 B per 16-element K step;
        // V MN-major (key rows of 64 columns = one atom), 8-key groups 1024 B apart, 16 keys = 2048 B per K step
        const uint64_t qdesc = make_smem_desc(smem_u32(sQ) + wg * (BQ / 2) * 128, 16, 1024);
        const uint64_t kdesc0 = make_smem_desc(smem_u32(sK), 16, 1024);
        const uint64_t vdesc0 = make_smem_desc(smem_u32(sV), V_BYTES, 1024);
        float o[32];
#pragma unroll
        for (int i = 0; i < 32; i++) o[i] = 0.f;
        float m_run[2] = { -INFINITY, -INFINITY }, l_run[2] = { 0.f, 0.f };
        mbar_wait(q_full, 0);
        for (int j = 0; j < n_kv; j++) {
            const int ks = j % KV_STAGES;
            mbar_wait(&kv_full[ks], (j / KV_STAGES) & 1);
            float s[64];
#pragma unroll
            for (int i = 0; i < 64; i++) s[i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BD / 16; k++) wgmma_m64n128k16_f16<0>(s, qdesc + (uint64_t)(k * 2), kdesc0 + (uint64_t)(ks * (K_BYTES >> 4) + k * 2), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            // only the last tile has padding keys (K rows zero-filled by TMA): they get probability 0
            if (j * BKV + BKV > p.Tk) {
#pragma unroll
                for (int c = 0; c < BKV / 8; c++)
#pragma unroll
                    for (int e = 0; e < 2; e++)
                        if (j * BKV + 8 * c + cq + e >= p.Tk) { s[4 * c + e] = -INFINITY; s[4 * c + 2 + e] = -INFINITY; }
            }
            float alpha[2], neg_m[2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                float mt = -INFINITY;
#pragma unroll
                for (int c = 0; c < BKV / 8; c++) mt = fmaxf(mt, fmaxf(s[4 * c + 2 * h], s[4 * c + 2 * h + 1]));
                mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
                mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
                // Lazy rescaling: the stale maximum is kept while the new one exceeds it by at most tau (log2 units) -- P <= 2^tau stays well
                // inside fp16, O and l accumulate in fp32.  tau = 0 is the exact running maximum (the default; OSB_FLASH_TAU sets it).
                const float m_cand = fmaxf(m_run[h], mt * p.scale_log2);     // scale_log2 > 0
                const float m_new = (m_cand - m_run[h] > p.tau) ? m_cand : m_run[h];
                alpha[h] = ex2_approx(m_run[h] - m_new);                     // 0 on the first tile (m_run = -inf)
                neg_m[h] = -m_new;
                m_run[h] = m_new;
            }
            // p = 2^(s*scale*log2e - m_new): one FFMA + one MUFU.EX2 per score, packed to fp16 in the A-fragment order of the PV MMA
            // (k-step kk covers keys 16kk..16kk+15 = blocks 2kk, 2kk+1: {block 2kk row r, row r+8, block 2kk+1 row r, row r+8})
            uint32_t a[BKV / 16][4];
            float lsum[2] = { 0.f, 0.f };
#pragma unroll
            for (int c = 0; c < BKV / 8; c++) {
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const float p0 = ex2_approx(fmaf(s[4 * c + 2 * h], p.scale_log2, neg_m[h]));
                    const float p1 = ex2_approx(fmaf(s[4 * c + 2 * h + 1], p.scale_log2, neg_m[h]));
                    lsum[h] += p0 + p1;
                    a[c >> 1][(c & 1) * 2 + h] = pack_half2(p0, p1);
                }
            }
#pragma unroll
            for (int h = 0; h < 2; h++) {
                l_run[h] = l_run[h] * alpha[h] + lsum[h];    // this thread's partial row sum (the quad shares alpha)
#pragma unroll
                for (int c = 0; c < BD / 8; c++) { o[4 * c + 2 * h] *= alpha[h]; o[4 * c + 2 * h + 1] *= alpha[h]; }
            }
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < BKV / 16; kk++)
                wgmma_m64n64k16_f16_rs(o, a[kk], vdesc0 + (uint64_t)(ks * (V_BYTES >> 4) + kk * (2048 >> 4)), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            mbar_arrive(&kv_empty[ks]);
        }
        // epilogue: O / l -> fp16 -> out[q, head*d + c]
#pragma unroll
        for (int h = 0; h < 2; h++) {
            float l = l_run[h];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv = 1.f / l;
            const int qrow = q0 + wg * (BQ / 2) + r + 8 * h;
            if (qrow >= p.T) continue;
            __half* orow = p.out + (long long)qrow * p.ldo + (long long)head * p.d;
#pragma unroll
            for (int c = 0; c < BD / 8; c++) {
                const int col = 8 * c + cq;
                if (col < p.d)     // d % 8 == 0: the pair is inside
                    *reinterpret_cast<uint32_t*>(orow + col) = pack_half2(o[4 * c + 2 * h] * inv, o[4 * c + 2 * h + 1] * inv);
            }
        }
    }
}

PFN_cuTensorMapEncodeTiled_v12000 fa_encode()
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

// [rows, heads*d] projection viewed as (d, heads, rows): strides (d*2, ld*2) bytes; box (64, 1, box_rows)
bool head_map(CUtensorMap* map, const void* base, int d, int heads, int64_t rows, int64_t ld, uint32_t box_rows)
{
    auto enc = fa_encode();
    if (!enc) return false;
    cuuint64_t dims[3] = { (cuuint64_t)d, (cuuint64_t)heads, (cuuint64_t)rows };
    cuuint64_t strides[2] = { (cuuint64_t)d * 2, (cuuint64_t)ld * 2 };
    cuuint32_t box[3] = { 64, 1, box_rows };
    cuuint32_t estr[3] = { 1, 1, 1 };
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

extern "C" int osb_flash_attention_ok(int64_t T, int64_t Tk, int64_t d, int dtype)
{
    return dtype == OSB_F16 && d >= 8 && d <= 64 && d % 8 == 0 && T >= 64 && Tk >= 1 && fa_encode() != nullptr;
}

// q [T, heads*d] (row stride ldq), k / v [Tk, heads*d] (row strides ldk / ldv), out [T, heads*d] (row stride ldo); fp16.
extern "C" int osb_flash_attention(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out, int64_t ldo,
                                   int64_t heads, int64_t T, int64_t Tk, int64_t d, float scale, void* stream)
{
    if (heads * T == 0) return 0;
    if (d > 64 || d % 8 || (ldq % 8) || (ldk % 8) || (ldv % 8) || (ldo % 8)) return (int)cudaErrorInvalidValue;
    if ((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) & 15) != 0) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    CUtensorMap mq, mk, mv;
    if (!head_map(&mq, q, (int)d, (int)heads, T, ldq, BQ)) return (int)cudaErrorInvalidValue;
    if (!head_map(&mk, k, (int)d, (int)heads, Tk, ldk, BKV)) return (int)cudaErrorInvalidValue;
    if (!head_map(&mv, v, (int)d, (int)heads, Tk, ldv, 64)) return (int)cudaErrorInvalidValue;
    static bool attr = false;
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(flash_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM);
        if (e != cudaSuccess) return (int)e;
        attr = true;
    }
    FaParams p{};
    p.T = (int)T; p.Tk = (int)Tk; p.d = (int)d; p.heads = (int)heads;
    p.q_tiles = (int)((T + BQ - 1) / BQ); p.kv_tiles = (int)((Tk + BKV - 1) / BKV);
    p.scale_log2 = scale * 1.4426950408889634f;
    static const float tau_env = [] { const char* e = getenv("OSB_FLASH_TAU"); float v = e ? (float)atof(e) : 0.f; return v < 0.f ? 0.f : (v > 12.f ? 12.f : v); }();
    p.tau = tau_env;
    p.out = (__half*)out; p.ldo = ldo;
    dim3 grid((unsigned)p.q_tiles, (unsigned)heads);
    osb_launch((flash_attention_kernel), grid, FA_THREADS, (size_t)FA_SMEM, st, mq, mk, mv, p);
    return launched(1);
}
