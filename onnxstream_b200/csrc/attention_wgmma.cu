// attention_wgmma.cu -- fused flash-style attention for sm_90a: softmax(Q K^T * scale) V in ONE kernel, score tile in registers,
// never in HBM.  Replaces the reference's sliced AttentionFusedOps loop (src/onnxstream.cpp:6696-6929: per head and per Q-slice a MatMul,
// a Mul, a Softmax and a MatMul, each through XNNPACK with the [Tq/parts, Tk] score tile round-tripping through two aux buffers,
// src/onnxstream.cpp:6798-6799).
//
// One CTA per (head, 128-query tile), 384 threads:
//   warpgroup 0      TMA producer (one warp, 40 registers): Q tile once, then a (K tile, V tile) pair per BK keys into a ring
//   warpgroups 1, 2  64 query rows each (232 registers): S = Q K_j^T (wgmma from shared memory, fp32 in registers), online softmax
//                    in registers (fp32, exp2 with the scale folded in), P rounded to fp16 in registers is the A operand of
//                    O += P V_j (wgmma m64n64k16 per 64 output columns, V from shared memory), finally O / sum -> fp16 -> global
// The consumer loop is software-pipelined: S_{j+1} = Q K_{j+1}^T and O += P_j V_j are issued together, and the softmax of S_{j+1} runs
// while O += P_j V_j is in flight.  The two warpgroups take turns to issue their MMAs (two named barriers), so one warpgroup's
// softmax overlaps the other's MMAs.
// Q, K, V are read in place from the [T, heads*d] projection buffers through strided tensor maps and O is written in the
// merged [T, heads*d] layout, so the exported graph's head split / merge costs nothing.  d <= 160, d % 8 == 0.
//
// sdpa_flash_kernel (below): the unpipelined structure for ScaledDotProductAttention with grouped KV heads and an additive mask --
// llm.cpp's prompt prefill -- for d <= 128.
// flash_attention_wide_kernel (below): 160 < d <= 512 -- the VAE decoder's single-head d = 512 attention -- with O split over its columns.
// flash_attention_f32x_kernel (below): fp32 q / k / v / out on bf16 wgmma through the triple split, d <= 160.
// flash_attention_wide_f32x_kernel (below): the wide kernel's slices with the f32x kernel's numerics, fp32 and 160 < d <= 512.
// sdpa_flash_f32x_kernel (below): sdpa_flash_kernel's grouped-KV masked attention with the f32x kernel's numerics, fp32 and d <= 128.

#include "common.cuh"
#include "tc_ptx.cuh"
#include <cuda.h>
#include <cstdio>

namespace {

using namespace tcptx;

constexpr int BQ = 128;                 // queries per CTA
constexpr int BKV = 128;                // largest key tile
constexpr int KV_STAGES = 4;            // K/V ring: the producer runs up to three tiles ahead of the slower warpgroup
constexpr int FA_THREADS = 384;
constexpr int FA_CONSUMERS = 256;
constexpr int FA_PRODUCER_REGS = 40, FA_CONSUMER_REGS = 232;     // 128 * 40 + 256 * 232 = 168 * 384: the whole register file

// Tiling of flash_attention_kernel by head dim.  NCH = 64-column chunks of the head dim (one 128-byte swizzle row each; columns past d are
// zero-filled by TMA), BK = keys per tile, QKS = k-steps of 16 in Q K^T (ceil(d / 16) rounded to an instantiation).  Registers per
// consumer thread: O 32 * NCH, S BK / 2, P BK / 4 -- d <= 64: 128-key tiles (32 + 64 + 32), d <= 128: 64-key tiles (64 + 32 + 16),
// d <= 160: 32-key tiles (96 + 16 + 8; with 64-key tiles ptxas spills and serialises the wgmmas).
// The same layout serves the other 128-query kernels: KS = stages of the K / V ring, PLANES = operand planes per tile (3: the bf16 triple
// split of flash_attention_f32x_kernel).  Shared memory: Q, the K ring, the V ring, then the mbarriers at BARS.
template <int NCH, int BK, int QKS, int KS = KV_STAGES, int PLANES = 1>
struct FaCfg {
    static_assert(QKS <= 4 * NCH && (BK == 32 || BK == 64 || BK == 128), "tile");
    static constexpr int Q_CHUNK = BQ * 128;            // 128 rows x 64 2-byte columns
    static constexpr int KV_CHUNK = BK * 128;
    static constexpr int Q_PLANE = NCH * Q_CHUNK;
    static constexpr int KV_PLANE = NCH * KV_CHUNK;
    static constexpr int Q_BYTES = PLANES * Q_PLANE;
    static constexpr int KV_BYTES = PLANES * KV_PLANE;  // one K (or V) tile
    static constexpr int BARS = Q_BYTES + KS * 2 * KV_BYTES;
    static constexpr int SMEM = BARS + 1024 + 256;
};

struct FaParams {
    int T, Tk, d;
    int kv_tiles;
    float scale_log2;        // scale * log2(e)
    __half* out;             // [T, ldo] merged layout, head h at column h*d
    long long ldo;
};

// Kernel entry of the flash kernels after the PDL trigger, up to the wait for the previous grid: the dynamic shared memory aligned to 1024 bytes (128B-swizzled
// TMA boxes and wgmma operands), the three tensor maps prefetched and the mbarriers at smem + bar_off initialised -- q_full, then the
// n0 full and n0 empty barriers of the first ring, then the n1 full and n1 empty barriers of the second.  Full barriers take the
// producer's arrival (and the TMA bytes), empty barriers `arrivals` consumer arrivals.  Returns the aligned shared memory.
__device__ __forceinline__ uint8_t* fa_prologue(const CUtensorMap* map_q, const CUtensorMap* map_k, const CUtensorMap* map_v, int bar_off,
                                                uint32_t arrivals, int n0, int n1 = 0)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(map_q) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(map_k) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(map_v) : "memory");
    }
    if (warp == 1 && lane == 0) {
        uint64_t* bars = (uint64_t*)(smem + bar_off);
        mbar_init(bars, 1);
        for (int i = 0; i < n0; i++) { mbar_init(&bars[1 + i], 1); mbar_init(&bars[1 + n0 + i], arrivals); }
        for (int i = 0; i < n1; i++) { mbar_init(&bars[1 + 2 * n0 + i], 1); mbar_init(&bars[1 + 2 * n0 + n1 + i], arrivals); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    osb_pdl_wait();
    return smem;
}

// Producer warp of a K / V ring of KS stages: for key tile j, wait until the consumers have released slot j % KS, expect its bytes and
// issue its loads on one lane (load(slot, j, &kv_full[slot])).
template <int KS, typename Load>
__device__ __forceinline__ void fa_produce_kv(uint64_t* kv_full, uint64_t* kv_empty, int n_kv, uint32_t tile_bytes, Load load)
{
    for (int j = 0; j < n_kv; j++) {
        const int st = j % KS;
        mbar_wait(&kv_empty[st], ((j / KS) & 1) ^ 1);
        if (elect_one()) {
            mbar_expect_tx(&kv_full[st], tile_bytes);
            load(st, j, &kv_full[st]);
        }
        __syncwarp();
    }
    osb_pdl_trigger_late();
}

// The maximum of score row r + 8h (s in the accumulator fragment, see fa_softmax): this thread's columns, then its quad's.
template <int BK>
__device__ __forceinline__ float fa_row_max(const float (&s)[BK / 2], int h)
{
    float mt = -INFINITY;
#pragma unroll
    for (int c = 0; c < BK / 8; c++) mt = fmaxf(mt, fmaxf(s[4 * c + 2 * h], s[4 * c + 2 * h + 1]));
    mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
    mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
    return mt;
}

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

__device__ __forceinline__ void store_pair(__half* p, float lo, float hi) { *reinterpret_cast<uint32_t*>(p) = pack_half2(lo, hi); }
__device__ __forceinline__ void store_pair(float* p, float lo, float hi) { *reinterpret_cast<float2*>(p) = make_float2(lo, hi); }

// Epilogue: O / l -> out.  The quad sums its partial row sums; rows[h] is this thread's output row r + 8h (nullptr past the last row),
// which takes the column pairs 64 ch + 8 c + cq, + 1 below ncols (d % 8 == 0: a pair is inside or outside as a whole).
template <typename OutT, int NCH>
__device__ __forceinline__ void fa_store(const float (&o)[NCH][32], const float (&l_run)[2], OutT* const (&rows)[2], int ncols, int cq)
{
#pragma unroll
    for (int h = 0; h < 2; h++) {
        float l = l_run[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = 1.f / l;
        if (!rows[h]) continue;
#pragma unroll
        for (int ch = 0; ch < NCH; ch++)
#pragma unroll
            for (int c = 0; c < 8; c++) {
                const int col = 64 * ch + 8 * c + cq;
                if (col < ncols) store_pair(rows[h] + col, o[ch][4 * c + 2 * h] * inv, o[ch][4 * c + 2 * h + 1] * inv);
            }
    }
}

template <int BK>
__device__ __forceinline__ void qk_mma(float (&s)[BK / 2], uint64_t da, uint64_t db, uint32_t scale_d = 1u)
{
    if constexpr (BK == 128) wgmma_m64n128k16_f16<0>(s, da, db, scale_d);
    else if constexpr (BK == 64) wgmma_m64n64k16_f16<0>(s, da, db, scale_d);
    else wgmma_m64n32k16_f16<0>(s, da, db, scale_d);
}

// S = Q K^T for one key tile (kdesc: the tile's first chunk), issued as one wgmma group.  Q / K K-major: 32 B per 16-element k-step inside
// a 64-column chunk; the first k-step overwrites S.
template <int NCH, int BK, int QKS>
__device__ __forceinline__ void fa_issue_qk(float (&s)[BK / 2], uint64_t qdesc, uint64_t kdesc)
{
    using C = FaCfg<NCH, BK, QKS>;
    fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < QKS; k++)
        qk_mma<BK>(s, qdesc + (uint64_t)(((k >> 2) * C::Q_CHUNK >> 4) + (k & 3) * 2), kdesc + (uint64_t)(((k >> 2) * C::KV_CHUNK >> 4) + (k & 3) * 2), k > 0);
    wgmma_commit();
}

// O += P V for one key tile (vdesc: the tile's first chunk), one wgmma group.  V MN-major: 16 keys = 2048 B per k-step.
template <int NCH, int BK, int QKS>
__device__ __forceinline__ void fa_issue_pv(float (&o)[NCH][32], uint32_t (&a)[BK / 16][4], uint64_t vdesc)
{
    using C = FaCfg<NCH, BK, QKS>;
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) fence_regs(o[ch]);
    fence_regs(a);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BK / 16; kk++)
#pragma unroll
        for (int ch = 0; ch < NCH; ch++)
            wgmma_m64n64k16_f16_rs(o[ch], a[kk], vdesc + (uint64_t)((ch * C::KV_CHUNK + kk * 2048) >> 4), 1u);
    wgmma_commit();
}

// Online softmax of one score tile in place: padding keys (the last tile only; K rows zero-filled by TMA) get -inf, the running maximum
// and this thread's partial row sums advance, s becomes p = 2^(s*scale*log2e - m_new) in fp32 and alpha the factor that rescales O.
// Accumulator fragments (tc_ptx.cuh): this thread holds rows r and r + 8 of the warpgroup's 64 (h = 0, 1) and, per 8-column block c,
// the columns 8c + cq, 8c + cq + 1.  The four lanes of a row share its maximum by two shuffles.
template <int BK>
__device__ __forceinline__ void fa_softmax(float (&s)[BK / 2], float (&m_run)[2], float (&l_run)[2], float (&alpha)[2], int key0, int cq, const FaParams& p)
{
    if (key0 + BK > p.Tk) {
#pragma unroll
        for (int c = 0; c < BK / 8; c++)
#pragma unroll
            for (int e = 0; e < 2; e++)
                if (key0 + 8 * c + cq + e >= p.Tk) { s[4 * c + e] = -INFINITY; s[4 * c + 2 + e] = -INFINITY; }
    }
    float neg_m[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
        // the maximum of the raw scores times scale_log2 is the maximum of the scaled logits only for scale > 0: the entries refuse
        // other scales
        const float m_new = fmaxf(m_run[h], fa_row_max<BK>(s, h) * p.scale_log2);
        alpha[h] = ex2_approx(m_run[h] - m_new);                     // 0 on the first tile (m_run = -inf)
        neg_m[h] = -m_new;
        m_run[h] = m_new;
    }
    // one FFMA + one MUFU.EX2 per score
    float lsum[2] = { 0.f, 0.f };
#pragma unroll
    for (int c = 0; c < BK / 8; c++)
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const float pe = ex2_approx(fmaf(s[4 * c + 2 * h + e], p.scale_log2, neg_m[h]));
                s[4 * c + 2 * h + e] = pe;
                lsum[h] += pe;
            }
#pragma unroll
    for (int h = 0; h < 2; h++) l_run[h] = l_run[h] * alpha[h] + lsum[h];    // this thread's partial row sum (the quad shares alpha)
}

// O *= alpha, then P (fp32 in s) rounded to fp16 in the A-fragment order of the PV MMA (k-step kk covers keys 16kk..16kk+15 = blocks
// 2kk, 2kk+1: {block 2kk row r, row r+8, block 2kk+1 row r, row r+8})
template <int NCH, int BK>
__device__ __forceinline__ void fa_rescale_pack(float (&o)[NCH][32], uint32_t (&a)[BK / 16][4], const float (&s)[BK / 2], const float (&alpha)[2])
{
#pragma unroll
    for (int ch = 0; ch < NCH; ch++)
#pragma unroll
        for (int c = 0; c < 8; c++)
#pragma unroll
            for (int h = 0; h < 2; h++) { o[ch][4 * c + 2 * h] *= alpha[h]; o[ch][4 * c + 2 * h + 1] *= alpha[h]; }
#pragma unroll
    for (int c = 0; c < BK / 8; c++)
#pragma unroll
        for (int h = 0; h < 2; h++) a[c >> 1][(c & 1) * 2 + h] = pack_half2(s[4 * c + 2 * h], s[4 * c + 2 * h + 1]);
}

template <int NCH, int BK, int QKS>
__global__ void __launch_bounds__(FA_THREADS, 1)
flash_attention_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                       const FaParams p)
{
    using C = FaCfg<NCH, BK, QKS>;
    constexpr int S = KV_STAGES;
    osb_pdl_trigger_entry();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int head = blockIdx.y;
    const int q0 = blockIdx.x * BQ;
    const int n_kv = p.kv_tiles;
    uint8_t* smem = fa_prologue(&map_q, &map_k, &map_v, C::BARS, FA_CONSUMERS / 32, S);   // kv_empty: one arrival per consumer warp
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + C::Q_BYTES;
    uint8_t* sV = sK + S * C::KV_BYTES;
    uint64_t* q_full = (uint64_t*)(smem + C::BARS);   // [1]
    uint64_t* kv_full = q_full + 1;                    // [S]
    uint64_t* kv_empty = kv_full + S;                  // [S]

    if (warp < 4) {
        setmaxnreg_dec<FA_PRODUCER_REGS>();
        if (warp == 0) {
            if (elect_one()) {
                mbar_expect_tx(q_full, C::Q_BYTES);
#pragma unroll
                for (int c = 0; c < NCH; c++) tma_load_3d(sQ + c * C::Q_CHUNK, &map_q, q_full, 64 * c, head, q0);
            }
            __syncwarp();
            fa_produce_kv<S>(kv_full, kv_empty, n_kv, 2 * C::KV_BYTES, [&](int st, int j, uint64_t* bar) {
#pragma unroll
                for (int c = 0; c < NCH; c++) {
                    tma_load_3d(sK + st * C::KV_BYTES + c * C::KV_CHUNK, &map_k, bar, 64 * c, head, j * BK);
                    tma_load_3d(sV + st * C::KV_BYTES + c * C::KV_CHUNK, &map_v, bar, 64 * c, head, j * BK);
                }
            });
        }
    } else {
        // ===================== warpgroups 1, 2: 64 query rows each =====================
        setmaxnreg_inc<FA_CONSUMER_REGS>();
        const int wg = (warp >> 2) - 1;
        const int r = (warp & 3) * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);
        // Turn-taking: warpgroup w waits on named barrier 1 + w (its own 128 threads + the other's 128 arrivals) before it issues MMAs
        // and arrives on the other's barrier after.  Warpgroup 0 pre-arrives on its own barrier to take the first turn, so warpgroup 1's
        // last arrival would have no matching wait and is left out.
        const uint32_t my_bar = 1 + wg, other_bar = 2 - wg;
        if (wg == 0) named_bar_arrive(my_bar, FA_CONSUMERS);
        // descriptors (start address in 16-byte units moves): Q / K K-major, 8-row groups 1024 B apart; V MN-major, 8-key groups 1024 B apart
        const uint64_t qdesc = make_smem_desc(smem_u32(sQ) + wg * (BQ / 2) * 128, 16, 1024);
        const uint64_t kdesc0 = make_smem_desc(smem_u32(sK), 16, 1024);
        const uint64_t vdesc0 = make_smem_desc(smem_u32(sV), C::KV_CHUNK, 1024);
        float o[NCH][32];
#pragma unroll
        for (int ch = 0; ch < NCH; ch++)
#pragma unroll
            for (int i = 0; i < 32; i++) o[ch][i] = 0.f;
        float s[BK / 2];
        uint32_t a[BK / 16][4];
        float m_run[2] = { -INFINITY, -INFINITY }, l_run[2] = { 0.f, 0.f }, alpha[2];
        mbar_wait(q_full, 0);

        // tile 0: S_0, its softmax, P_0
        mbar_wait(&kv_full[0], 0);
        named_bar_sync(my_bar, FA_CONSUMERS);
        fa_issue_qk<NCH, BK, QKS>(s, qdesc, kdesc0);
        named_bar_arrive(other_bar, FA_CONSUMERS);
        wgmma_wait<0>();
        fence_regs(s);
        fa_softmax<BK>(s, m_run, l_run, alpha, 0, cq, p);
        fa_rescale_pack<NCH, BK>(o, a, s, alpha);
        // tile j: S_j and O += P_{j-1} V_{j-1} in flight together; the softmax of S_j waits for S_j only
        for (int j = 1; j < n_kv; j++) {
            const int st = j % S, prev = (j - 1) % S;
            mbar_wait(&kv_full[st], (j / S) & 1);
            named_bar_sync(my_bar, FA_CONSUMERS);
            fa_issue_qk<NCH, BK, QKS>(s, qdesc, kdesc0 + (uint64_t)(st * C::KV_BYTES >> 4));
            fa_issue_pv<NCH, BK, QKS>(o, a, vdesc0 + (uint64_t)(prev * C::KV_BYTES >> 4));
            named_bar_arrive(other_bar, FA_CONSUMERS);
            wgmma_wait<1>();
            fence_regs(s);
            fa_softmax<BK>(s, m_run, l_run, alpha, j * BK, cq, p);
            wgmma_wait<0>();
#pragma unroll
            for (int ch = 0; ch < NCH; ch++) fence_regs(o[ch]);
            fence_regs(a);
            __syncwarp();
            if (lane == 0) mbar_arrive(&kv_empty[prev]);
            fa_rescale_pack<NCH, BK>(o, a, s, alpha);
        }
        named_bar_sync(my_bar, FA_CONSUMERS);
        fa_issue_pv<NCH, BK, QKS>(o, a, vdesc0 + (uint64_t)((n_kv - 1) % S * C::KV_BYTES >> 4));
        if (wg == 0) named_bar_arrive(other_bar, FA_CONSUMERS);
        wgmma_wait<0>();
#pragma unroll
        for (int ch = 0; ch < NCH; ch++) fence_regs(o[ch]);
        // out[q, head*d + c]
        __half* rows[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int qrow = q0 + wg * (BQ / 2) + r + 8 * h;
            rows[h] = qrow < p.T ? p.out + (long long)qrow * p.ldo + (long long)head * p.d : nullptr;
        }
        fa_store(o, l_run, rows, p.d, cq);
    }
}

// One launch of a flash kernel; the first launch of each kernel raises its dynamic shared-memory limit to smem.
template <auto Kernel, typename... Args>
int fa_launch_kernel(dim3 grid, int threads, int smem, cudaStream_t st, const Args&... args)
{
    static bool attr = false;
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return (int)e;
        attr = true;
    }
    osb_launch(Kernel, grid, threads, (size_t)smem, st, args...);
    return launched(1);
}

// ---- grouped-KV masked attention (ScaledDotProductAttention: prompt prefill) ----------------------------------------------------------
// softmax(Q K^T * scale + mask) V with Hq / Hkv = G query heads per KV head.  The G heads of one KV head are contiguous in q
// ([G*Tq, d] rows) and in out, so one CTA takes 128 of those packed rows: each K / V tile it loads serves all G heads.  Packed row R
// is query t = R % Tq of head hk*G + R / Tq and reads mask row t.
// Same roles as flash_attention_kernel (one TMA producer warp, two consumer warpgroups of 64 rows, K / V ring).  NCH = 64-column
// chunks of the head dim (1: d <= 64, 2: 64 < d <= 128), BK = keys per tile.  At d = 128 the O accumulator is 64 fp32 registers per
// thread, so that instantiation takes 64-key tiles (a 32-register score tile) to stay inside the 168 registers of a 384-thread CTA.
// Masked keys keep their finite logit s*scale + mask (a row whose keys are all masked gets the softmax of those logits, as the
// reference computes it); keys past Tk are padding (zero-filled by TMA) and get probability 0.  Q K^T runs over the whole of each
// 64-column chunk (QKS = 4 NCH).
struct SdpaParams {
    int rows;                // G * Tq: packed query rows per KV head
    int Tq, Tk, d;
    int kv_tiles;
    float scale_log2;        // scale * log2(e)
    const __half* mask;      // [Tq, Tk] additive, or nullptr
    __half* out;             // [Hkv][G*Tq][d] (= [Hq, Tq, d])
};

// mask[row][col], mask[row][col + 1] as a packed half2; keys past Tk read as 0 (they are set to -inf afterwards).  vec: the pair is
// 4-byte aligned (Tk even).
__device__ __forceinline__ uint32_t ld_mask_pair(const __half* row, int col, int Tk, bool vec)
{
    const unsigned short* m = reinterpret_cast<const unsigned short*>(row) + col;
    if (col + 1 < Tk) {
        if (vec) return __ldg(reinterpret_cast<const unsigned int*>(m));
        return (uint32_t)__ldg(m) | ((uint32_t)__ldg(m + 1) << 16);
    }
    return col < Tk ? (uint32_t)__ldg(m) : 0u;
}

template <int NCH, int BK>
__global__ void __launch_bounds__(FA_THREADS, 1)
sdpa_flash_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                  const SdpaParams p)
{
    using C = FaCfg<NCH, BK, 4 * NCH>;
    constexpr float LOG2E = 1.4426950408889634f;
    osb_pdl_trigger_entry();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r0 = blockIdx.x * BQ, hk = blockIdx.y;
    const int n_kv = p.kv_tiles;
    uint8_t* smem = fa_prologue(&map_q, &map_k, &map_v, C::BARS, FA_CONSUMERS, KV_STAGES);   // kv_empty: one arrival per consumer thread
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + C::Q_BYTES;
    uint8_t* sV = sK + KV_STAGES * C::KV_BYTES;
    uint64_t* q_full = (uint64_t*)(smem + C::BARS);   // [1]
    uint64_t* kv_full = q_full + 1;                    // [KV_STAGES]
    uint64_t* kv_empty = kv_full + KV_STAGES;          // [KV_STAGES]

    if (warp == 0) {
        if (elect_one()) {
            mbar_expect_tx(q_full, C::Q_BYTES);
#pragma unroll
            for (int c = 0; c < NCH; c++) tma_load_3d(sQ + c * C::Q_CHUNK, &map_q, q_full, 64 * c, r0, hk);
        }
        __syncwarp();
        fa_produce_kv<KV_STAGES>(kv_full, kv_empty, n_kv, 2 * C::KV_BYTES, [&](int st, int j, uint64_t* bar) {
#pragma unroll
            for (int c = 0; c < NCH; c++) {
                tma_load_3d(sK + st * C::KV_BYTES + c * C::KV_CHUNK, &map_k, bar, 64 * c, j * BK, hk);
                tma_load_3d(sV + st * C::KV_BYTES + c * C::KV_CHUNK, &map_v, bar, 64 * c, j * BK, hk);
            }
        });
    } else if (warp >= 4) {
        // Fragments as in flash_attention_kernel: rows r, r + 8 of the warpgroup's 64; per 8-column block c the columns 8c + cq, + 1.
        const int wg = (warp >> 2) - 1;
        const int r = (warp & 3) * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);
        // Q / K K-major (one descriptor per 64-column chunk, 32 B per 16-element K step); V MN-major, 16 keys = 2048 B per K step
        const uint64_t qdesc = make_smem_desc(smem_u32(sQ) + wg * (BQ / 2) * 128, 16, 1024);
        const uint64_t kdesc0 = make_smem_desc(smem_u32(sK), 16, 1024);
        const uint64_t vdesc0 = make_smem_desc(smem_u32(sV), C::KV_CHUNK, 1024);
        const bool has_mask = p.mask != nullptr, vec = (p.Tk & 1) == 0;
        const __half* mrow[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int R = r0 + wg * (BQ / 2) + r + 8 * h;                     // rows past G*Tq (zero-filled by TMA) are never stored
            mrow[h] = has_mask ? p.mask + (long long)(R % p.Tq) * p.Tk : nullptr;
        }
        float o[NCH][32];
#pragma unroll
        for (int ch = 0; ch < NCH; ch++)
#pragma unroll
            for (int i = 0; i < 32; i++) o[ch][i] = 0.f;
        float m_run[2] = { -INFINITY, -INFINITY }, l_run[2] = { 0.f, 0.f };
        mbar_wait(q_full, 0);
        for (int j = 0; j < n_kv; j++) {
            const int ks = j % KV_STAGES;
            const int key0 = j * BK;
            mbar_wait(&kv_full[ks], (j / KV_STAGES) & 1);
            float s[BK / 2];
            fa_issue_qk<NCH, BK, 4 * NCH>(s, qdesc, kdesc0 + (uint64_t)(ks * C::KV_BYTES >> 4));
            // the mask loads (L2-resident: every head reads the same [Tq, Tk] block) are in flight while the MMAs run
            uint32_t mk[2][BK / 8];
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int c = 0; c < BK / 8; c++) mk[h][c] = has_mask ? ld_mask_pair(mrow[h], key0 + 8 * c + cq, p.Tk, vec) : 0u;
            wgmma_wait<0>();
            // logits in log2 units: s * scale * log2e + mask * log2e; padding keys (last tile only) -inf
            const bool tail = key0 + BK > p.Tk;
#pragma unroll
            for (int c = 0; c < BK / 8; c++)
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    __half2 m2 = *reinterpret_cast<__half2*>(&mk[h][c]);
                    const float2 mf = __half22float2(m2);
                    float x0 = fmaf(s[4 * c + 2 * h], p.scale_log2, mf.x * LOG2E);
                    float x1 = fmaf(s[4 * c + 2 * h + 1], p.scale_log2, mf.y * LOG2E);
                    if (tail) {
                        if (key0 + 8 * c + cq >= p.Tk) x0 = -INFINITY;
                        if (key0 + 8 * c + cq + 1 >= p.Tk) x1 = -INFINITY;
                    }
                    s[4 * c + 2 * h] = x0; s[4 * c + 2 * h + 1] = x1;
                }
            float alpha[2], neg_m[2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const float m_new = fmaxf(m_run[h], fa_row_max<BK>(s, h));
                // m_new = -inf only when every logit so far is -inf (a -inf mask): keep the sums at 0 instead of producing NaN here
                const bool none = m_new == -INFINITY;
                alpha[h] = none ? 1.f : ex2_approx(m_run[h] - m_new);          // 0 on the first tile (m_run = -inf)
                neg_m[h] = none ? 0.f : -m_new;
                m_run[h] = m_new;
            }
            float lsum[2] = { 0.f, 0.f };
#pragma unroll
            for (int c = 0; c < BK / 8; c++) {
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const float p0 = ex2_approx(s[4 * c + 2 * h] + neg_m[h]);
                    const float p1 = ex2_approx(s[4 * c + 2 * h + 1] + neg_m[h]);
                    lsum[h] += p0 + p1;
                    s[4 * c + 2 * h] = p0; s[4 * c + 2 * h + 1] = p1;
                }
            }
#pragma unroll
            for (int h = 0; h < 2; h++) l_run[h] = l_run[h] * alpha[h] + lsum[h];
            uint32_t a[BK / 16][4];
            fa_rescale_pack<NCH, BK>(o, a, s, alpha);
            fa_issue_pv<NCH, BK, 4 * NCH>(o, a, vdesc0 + (uint64_t)(ks * C::KV_BYTES >> 4));
            wgmma_wait<0>();
            mbar_arrive(&kv_empty[ks]);
        }
        // out[hk][R][col]
        __half* rows[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int R = r0 + wg * (BQ / 2) + r + 8 * h;
            rows[h] = R < p.rows ? p.out + ((long long)hk * p.rows + R) * p.d : nullptr;
        }
        fa_store(o, l_run, rows, p.d, cq);
    }
}

// q / k / v [Hkv, rows, d] contiguous viewed as (d, rows, Hkv); boxes (64, BQ or BK, 1)
template <int NCH, int BK>
int sdpa_launch(const void* q, const void* k, const void* v, SdpaParams p, int64_t Hkv, cudaStream_t st)
{
    using C = FaCfg<NCH, BK, 4 * NCH>;
    const uint64_t d = p.d;
    CUtensorMap mq, mk, mv;
    if (!make_map(&mq, q, d, p.rows, Hkv, d * 2, p.rows * d * 2, 64, BQ, 1) || !make_map(&mk, k, d, p.Tk, Hkv, d * 2, p.Tk * d * 2, 64, BK, 1) ||
        !make_map(&mv, v, d, p.Tk, Hkv, d * 2, p.Tk * d * 2, 64, BK, 1))
        return (int)cudaErrorInvalidValue;
    p.kv_tiles = (p.Tk + BK - 1) / BK;
    dim3 grid((unsigned)((p.rows + BQ - 1) / BQ), (unsigned)Hkv);
    return fa_launch_kernel<sdpa_flash_kernel<NCH, BK>>(grid, FA_THREADS, C::SMEM, st, mq, mk, mv, p);
}

// q / k / v [rows, heads*d] (row strides ld*) viewed as (d, heads, rows); boxes (64, 1, BQ or BK)
template <int NCH, int BK, int QKS>
int fa_launch(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, FaParams p, int64_t heads, cudaStream_t st)
{
    using C = FaCfg<NCH, BK, QKS>;
    const uint64_t d = p.d;
    CUtensorMap mq, mk, mv;
    if (!make_map(&mq, q, d, heads, p.T, d * 2, ldq * 2, 64, 1, BQ) || !make_map(&mk, k, d, heads, p.Tk, d * 2, ldk * 2, 64, 1, BK) ||
        !make_map(&mv, v, d, heads, p.Tk, d * 2, ldv * 2, 64, 1, BK))
        return (int)cudaErrorInvalidValue;
    p.kv_tiles = (p.Tk + BK - 1) / BK;
    dim3 grid((unsigned)((p.T + BQ - 1) / BQ), (unsigned)heads);
    return fa_launch_kernel<flash_attention_kernel<NCH, BK, QKS>>(grid, FA_THREADS, C::SMEM, st, mq, mk, mv, p);
}

// ---- wide heads: 160 < d <= 512 (the VAE's single-head d = 512 attention) --------------------------------------------------------------
// softmax(Q K^T * scale) V for q [h, T, d], k [h, Tk, d] (KT = false) or [h, d, Tk] (KT = true), v [h, Tk, d], out [h, T, d].
// A 64-row x 512-column fp32 O would take 256 registers per consumer thread, so O is split over its columns: one CTA per (256-column slice
// of V and O, 64-query tile, head).  Each CTA computes the full S = Q K^T over d in 64-column chunks and then O_slice += P V_slice, so
// Q K^T runs once per slice: at d = 512 the two slices make 2 + 1 = 3 units of MMA work where the unsplit product has 2.  Slices of the
// same query tile are adjacent in the grid, so their K / V tiles are read from HBM once and from L2 by the sibling.
// 256 threads: warpgroup 0 is the TMA producer (one warp, 40 registers), warpgroup 1 takes the 64 query rows (240 registers: O 128 + S 32
// + P 16).  With two consumer warpgroups (384 threads) ptxas allocates at most 168 registers per thread: a 256-column O spills and
// 128-column slices would make Q K^T 4 + 1 = 5 units of MMA work at d = 512.  Q stays in shared memory (up to 8 chunks, 64 KB); K streams
// through a ring of 64-column chunks of one 64-key tile (a chunk is released as soon as the MMAs that read it retire), V through a ring of
// 64-key x 256-column tiles.  The consumer loop is not software-pipelined (Q K^T is 2/3 of the MMA work).  Numerics are those of
// flash_attention_kernel with the exact running maximum.
constexpr int WD_BQ = 64;                 // queries per CTA: one consumer warpgroup
constexpr int WD_BK = 64;                 // keys per tile
constexpr int WD_NV = 4;                  // 64-column chunks of V / O per CTA
constexpr int WD_DCH = 8;                 // largest number of 64-column chunks of d
constexpr int WD_K_STAGES = 8, WD_V_STAGES = 2;
constexpr int WD_THREADS = 256, WD_CONSUMERS = 128;
constexpr int WD_PRODUCER_REGS = 40, WD_CONSUMER_REGS = 240;
constexpr int WD_Q_CHUNK = WD_BQ * 128;   // 64 rows x 64 fp16 columns
constexpr int WD_K_CHUNK = WD_BK * 128;   // 64 keys x 64 columns of d (or 64 rows of d x 64 keys)
constexpr int WD_V_CHUNK = WD_BK * 128;
constexpr int WD_V_BYTES = WD_NV * WD_V_CHUNK;
constexpr int WD_BARS = WD_DCH * WD_Q_CHUNK + WD_K_STAGES * WD_K_CHUNK + WD_V_STAGES * WD_V_BYTES;
constexpr int WD_SMEM = WD_BARS + 1024 + 256;

// S (+)= Q_c K_c^T for one 64-column chunk c of d: 4 k-steps.  K-major K: 32 B per k-step inside the swizzle row; MN-major K^T (rows of
// d): 16 rows of d = 2048 B per k-step.
template <bool KT>
__device__ __forceinline__ void wd_issue_qk_chunk(float (&s)[WD_BK / 2], uint64_t qdesc, uint64_t kdesc, bool first)
{
#pragma unroll
    for (int k = 0; k < 4; k++)
        wgmma_m64n64k16_f16<KT ? 1 : 0>(s, qdesc + (uint64_t)(k * 2), kdesc + (uint64_t)(KT ? (k * 2048) >> 4 : k * 2), (first && k == 0) ? 0u : 1u);
    wgmma_commit();
}

// O_slice += P V_slice for one key tile, one wgmma group: 64-column chunks of V WD_V_CHUNK bytes apart, MN-major, 16 keys = 2048 B per
// k-step.  Chunks wholly past d (d <= 192, or the last slice) are not loaded: their MMAs read stale shared memory into output columns
// that are never stored.
__device__ __forceinline__ void wd_issue_pv(float (&o)[WD_NV][32], uint32_t (&a)[WD_BK / 16][4], uint64_t vdesc)
{
#pragma unroll
    for (int ch = 0; ch < WD_NV; ch++) fence_regs(o[ch]);
    fence_regs(a);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < WD_BK / 16; kk++)
#pragma unroll
        for (int ch = 0; ch < WD_NV; ch++)
            wgmma_m64n64k16_f16_rs(o[ch], a[kk], vdesc + (uint64_t)((ch * WD_V_CHUNK + kk * 2048) >> 4), 1u);
    wgmma_commit();
}

template <bool KT>
__global__ void __launch_bounds__(WD_THREADS, 1)
flash_attention_wide_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                            const __grid_constant__ CUtensorMap map_v, const FaParams p)
{
    constexpr int KS = WD_K_STAGES, VS = WD_V_STAGES;
    osb_pdl_trigger_entry();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // blockIdx.x = query tile * slices + slice: the slices of one query tile are adjacent, and x takes any T (y would stop at 65535 tiles)
    const int n_slices = (p.d + 64 * WD_NV - 1) / (64 * WD_NV);
    const int col0 = (blockIdx.x % n_slices) * (64 * WD_NV);
    const int q0 = (blockIdx.x / n_slices) * WD_BQ;
    const int head = blockIdx.y;
    const int n_dch = (p.d + 63) >> 6;
    uint8_t* smem = fa_prologue(&map_q, &map_k, &map_v, WD_BARS, WD_CONSUMERS / 32, KS, VS);
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + WD_DCH * WD_Q_CHUNK;
    uint8_t* sV = sK + KS * WD_K_CHUNK;
    uint64_t* q_full = (uint64_t*)(smem + WD_BARS);   // [1]
    uint64_t* k_full = q_full + 1;                     // [KS]
    uint64_t* k_empty = k_full + KS;                   // [KS]: one arrival per consumer warp
    uint64_t* v_full = k_empty + KS;                   // [VS]
    uint64_t* v_empty = v_full + VS;                   // [VS]
    const int n_kv = p.kv_tiles;

    if (warp < 4) {
        setmaxnreg_dec<WD_PRODUCER_REGS>();
        if (warp == 0) {
            if (elect_one()) {
                mbar_expect_tx(q_full, n_dch * WD_Q_CHUNK);
                for (int c = 0; c < n_dch; c++) tma_load_3d(sQ + c * WD_Q_CHUNK, &map_q, q_full, 64 * c, q0, head);
            }
            __syncwarp();
            // V chunks wholly past d are not loaded: they only feed output columns that are never stored
            const int n_vch = min(WD_NV, (p.d - col0 + 63) >> 6);
            int kc = 0;
            for (int j = 0; j < n_kv; j++) {
                for (int c = 0; c < n_dch; c++, kc++) {
                    const int st = kc % KS;
                    mbar_wait(&k_empty[st], ((kc / KS) & 1) ^ 1);
                    if (elect_one()) {
                        mbar_expect_tx(&k_full[st], WD_K_CHUNK);
                        if (KT) tma_load_3d(sK + st * WD_K_CHUNK, &map_k, &k_full[st], j * WD_BK, 64 * c, head);
                        else tma_load_3d(sK + st * WD_K_CHUNK, &map_k, &k_full[st], 64 * c, j * WD_BK, head);
                    }
                    __syncwarp();
                }
                const int sv = j % VS;
                mbar_wait(&v_empty[sv], ((j / VS) & 1) ^ 1);
                if (elect_one()) {
                    mbar_expect_tx(&v_full[sv], n_vch * WD_V_CHUNK);
                    for (int ch = 0; ch < n_vch; ch++)
                        tma_load_3d(sV + sv * WD_V_BYTES + ch * WD_V_CHUNK, &map_v, &v_full[sv], col0 + 64 * ch, j * WD_BK, head);
                }
                __syncwarp();
            }
            osb_pdl_trigger_late();
        }
    } else {
        // ===================== warpgroup 1: the CTA's 64 query rows =====================
        setmaxnreg_inc<WD_CONSUMER_REGS>();
        const int r = (warp & 3) * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);
        // Q K-major (8-row groups 1024 B apart); K K-major or K^T MN-major and V MN-major, 8-row groups 1024 B apart
        const uint64_t qdesc0 = make_smem_desc(smem_u32(sQ), 16, 1024);
        const uint64_t kdesc0 = make_smem_desc(smem_u32(sK), KT ? WD_K_CHUNK : 16, 1024);
        const uint64_t vdesc0 = make_smem_desc(smem_u32(sV), WD_V_CHUNK, 1024);
        float o[WD_NV][32];
#pragma unroll
        for (int ch = 0; ch < WD_NV; ch++)
#pragma unroll
            for (int i = 0; i < 32; i++) o[ch][i] = 0.f;
        float s[WD_BK / 2];
        uint32_t a[WD_BK / 16][4];
        float m_run[2] = { -INFINITY, -INFINITY }, l_run[2] = { 0.f, 0.f }, alpha[2];
        mbar_wait(q_full, 0);
        int kc = 0;
        for (int j = 0; j < n_kv; j++) {
            // S = Q K_j^T, one wgmma group per chunk of d; a chunk's slot is released once the next chunk's group is issued and it retired
            fence_regs(s);
            for (int c = 0; c < n_dch; c++, kc++) {
                const int st = kc % KS;
                mbar_wait(&k_full[st], (kc / KS) & 1);
                wgmma_fence();
                wd_issue_qk_chunk<KT>(s, qdesc0 + (uint64_t)((c * WD_Q_CHUNK) >> 4), kdesc0 + (uint64_t)((st * WD_K_CHUNK) >> 4), c == 0);
                if (c > 0) {
                    wgmma_wait<1>();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&k_empty[(kc - 1) % KS]);
                }
            }
            wgmma_wait<0>();
            fence_regs(s);
            __syncwarp();
            if (lane == 0) mbar_arrive(&k_empty[(kc - 1) % KS]);
            fa_softmax<WD_BK>(s, m_run, l_run, alpha, j * WD_BK, cq, p);
            fa_rescale_pack<WD_NV, WD_BK>(o, a, s, alpha);
            // O_slice += P V_slice
            const int sv = j % VS;
            mbar_wait(&v_full[sv], (j / VS) & 1);
            wd_issue_pv(o, a, vdesc0 + (uint64_t)((sv * WD_V_BYTES) >> 4));
            wgmma_wait<0>();
#pragma unroll
            for (int ch = 0; ch < WD_NV; ch++) fence_regs(o[ch]);
            fence_regs(a);
            __syncwarp();
            if (lane == 0) mbar_arrive(&v_empty[sv]);
        }
        // out[head][q][col0 + c]
        __half* rows[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int qrow = q0 + r + 8 * h;
            rows[h] = qrow < p.T ? p.out + ((long long)head * p.T + qrow) * p.ldo + col0 : nullptr;
        }
        fa_store(o, l_run, rows, p.d - col0, cq);
    }
}

template <bool KT>
int wd_launch(const void* q, const void* k, const void* v, FaParams p, int64_t heads, cudaStream_t st)
{
    // q / v / out [heads, rows, d] viewed as (d, rows, heads); K^T [heads, d, Tk] as (Tk, d, heads) with 64 x 64 boxes
    const uint64_t d = p.d, T = p.T, Tk = p.Tk;
    CUtensorMap mq, mk, mv;
    const bool ok_k = KT ? make_map(&mk, k, Tk, d, heads, Tk * 2, d * Tk * 2, 64, 64, 1) : make_map(&mk, k, d, Tk, heads, d * 2, Tk * d * 2, 64, WD_BK, 1);
    if (!make_map(&mq, q, d, T, heads, d * 2, T * d * 2, 64, WD_BQ, 1) || !ok_k || !make_map(&mv, v, d, Tk, heads, d * 2, Tk * d * 2, 64, WD_BK, 1))
        return (int)cudaErrorInvalidValue;
    p.kv_tiles = (p.Tk + WD_BK - 1) / WD_BK;
    const int64_t n_slices = (p.d + 64 * WD_NV - 1) / (64 * WD_NV);
    dim3 grid((unsigned)((p.T + WD_BQ - 1) / WD_BQ * n_slices), (unsigned)heads);
    return fa_launch_kernel<flash_attention_wide_kernel<KT>>(grid, WD_THREADS, WD_SMEM, st, mq, mk, mv, p);
}

// ---- fp32 multi-head attention on the tensor cores: bf16 triple split --------------------------------------------------------------
// softmax(Q K^T * scale) V of flash_attention_kernel for fp32 q / k / v / out, to fp32 accuracy on bf16 wgmma.  Every operand is split
// x = h + m + l into three bf16 planes (common.cuh: bf16x3_split) and every product into the six cross terms hh + hm + mh + hl + lh + mm
// (the dropped ml, lm, ll are below ~2^-26 relative), all accumulated in fp32:
//   f32x_split_kernel splits q, k and v (one launch for the three) into plane buffers [rows][3][heads*d], which the attention kernel reads
//   through the strided tensor maps of the fp16 kernel: row stride 3 C, plane p of head h is "head" p * heads + h;
//   S = Q K^T is 6 QKS wgmmas per key tile; the online softmax is f32x_softmax (fp32, expf, exact running maximum); P is split into
//   three bf16 planes in registers and P V is 6 BK / 16 wgmmas per 64-column chunk of O, A from registers, V MN-major, added to O in fp32.
// Roles as in sdpa_flash_kernel, unpipelined like it: one TMA producer warp (40 registers), two consumer warpgroups of 64 query rows
// (232 registers), a K / V ring of KS stages.  Three planes take 3x the shared memory of the fp16 tiles:
//   d <= 64:  64-key tiles, 2 stages: Q 48 KB + 2 x 48 KB;   registers O 32 + S 32 + P 3 x 16 + a P V chunk 32
//   d <= 128: 32-key tiles, 2 stages: Q 96 KB + 2 x 48 KB;   O 64 + S 16 + P 3 x 8 + 32
//   d <= 160: 32-key tiles, 1 stage:  Q 144 KB + 72 KB;      O 96 + S 16 + P 3 x 8 + 32
// (FaCfg<NCH, BK, QKS, KS, 3>).

// cross product x = 0..5 (hh, hm, mh, hl, lh, mm): plane of the A operand (Q, P) and of the B operand (K, V); 0 = h, 1 = m, 2 = l
__host__ __device__ constexpr int x3a(int x) { return x == 2 || x == 5 ? 1 : (x == 4 ? 2 : 0); }
__host__ __device__ constexpr int x3b(int x) { return x == 1 || x == 5 ? 1 : (x == 3 ? 2 : 0); }

__device__ __forceinline__ uint32_t pack_bf162(__nv_bfloat16 lo, __nv_bfloat16 hi)
{
    __nv_bfloat162 b2 = __halves2bfloat162(lo, hi);
    return *reinterpret_cast<uint32_t*>(&b2);
}

// q [T, ldq], k / v [Tk, ldk / ldv] fp32 -> bf16 planes pq [T][3][C], pk / pv [Tk][3][C]; 4 columns per thread
__global__ void f32x_split_kernel(const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, int64_t ldk, const float* __restrict__ v,
                                  int64_t ldv, __nv_bfloat16* __restrict__ pq, __nv_bfloat16* __restrict__ pk, __nv_bfloat16* __restrict__ pv,
                                  int64_t T, int64_t Tk, int C)
{
    osb_pdl_prologue();
    const int C4 = C / 4;
    const int64_t nq = T * C4, nk = Tk * C4, n = nq + 2 * nk;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float* src = q; int64_t ld = ldq; __nv_bfloat16* dst = pq; int64_t e = i;
        if (e >= nq) {
            e -= nq;
            if (e < nk) { src = k; ld = ldk; dst = pk; }
            else { e -= nk; src = v; ld = ldv; dst = pv; }
        }
        const int64_t r = e / C4;
        const int c = (int)(e - r * C4) * 4;
        const float4 x = *reinterpret_cast<const float4*>(src + r * ld + c);
        const float xs[4] = { x.x, x.y, x.z, x.w };
        Vec<__nv_bfloat16, 4> h, m, l;
#pragma unroll
        for (int t = 0; t < 4; t++) bf16x3_split(xs[t], h.v[t], m.v[t], l.v[t]);
        __nv_bfloat16* o = dst + r * 3 * C + c;
        store_vec(o, h);
        store_vec(o + C, m);
        store_vec(o + 2 * C, l);
    }
}

// Online softmax of one score tile for the fp32 kernels: fa_softmax with fp32 arithmetic -- the logit s * scale rounded once, as fp32
// attention rounds it, and expf instead of the one-MUFU ex2 (whose ~2^-22 relative error and the rounding of scale * log2e show at fp32
// accuracy); the exact running maximum.  Padding keys (last tile only) get -inf.
// MASK: the logit is s * scale + mask in natural units, rounded as fp32 attention rounds the two steps; mk[h][c] holds the mask of this
// thread's row r + 8h at the columns 8c + cq, + 1.  The running maximum is then taken over the masked, scaled logits (any finite scale),
// and a tile whose logits so far are all -inf (a -inf mask over a row's first keys) leaves m_run, l_run and O as they are.
template <int BK, bool MASK = false>
__device__ __forceinline__ void f32x_softmax(float (&s)[BK / 2], float (&m_run)[2], float (&l_run)[2], float (&alpha)[2], int key0, int cq, int Tk, float scale,
                                             const float2 (*mk)[BK / 8] = nullptr)
{
#pragma unroll
    for (int c = 0; c < BK / 8; c++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const bool pad = key0 + 8 * c + cq + e >= Tk;
            if constexpr (MASK) {
                s[4 * c + e] = pad ? -INFINITY : __fmul_rn(s[4 * c + e], scale) + (e ? mk[0][c].y : mk[0][c].x);
                s[4 * c + 2 + e] = pad ? -INFINITY : __fmul_rn(s[4 * c + 2 + e], scale) + (e ? mk[1][c].y : mk[1][c].x);
            } else {
                s[4 * c + e] = pad ? -INFINITY : s[4 * c + e] * scale;
                s[4 * c + 2 + e] = pad ? -INFINITY : s[4 * c + 2 + e] * scale;
            }
        }
    float m_new[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
        m_new[h] = fmaxf(m_run[h], fa_row_max<BK>(s, h));
        alpha[h] = expf(m_run[h] - m_new[h]);                        // 0 on the first tile (m_run = -inf)
        m_run[h] = m_new[h];
        if constexpr (MASK) {
            // every logit so far -inf: p = expf(-inf - 0) = 0 and alpha = 1 instead of the NaN of -inf - -inf
            if (m_new[h] == -INFINITY) { alpha[h] = 1.f; m_new[h] = 0.f; }
        }
    }
    float lsum[2] = { 0.f, 0.f };
#pragma unroll
    for (int c = 0; c < BK / 8; c++)
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const float pe = expf(s[4 * c + 2 * h + e] - m_new[h]);
                s[4 * c + 2 * h + e] = pe;
                lsum[h] += pe;
            }
#pragma unroll
    for (int h = 0; h < 2; h++) l_run[h] = l_run[h] * alpha[h] + lsum[h];
}

template <int BK>
__device__ __forceinline__ void qk_mma_bf16(float (&s)[BK / 2], uint64_t da, uint64_t db, uint32_t scale_d)
{
    if constexpr (BK == 64) wgmma_m64n64k16_bf16<0>(s, da, db, scale_d);
    else wgmma_m64n32k16_bf16<0>(s, da, db, scale_d);
}

template <int NCH, int BK, int QKS, int KS>
__global__ void __launch_bounds__(FA_THREADS, 1)
flash_attention_f32x_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                            const FaParams p, float scale, float* __restrict__ out)
{
    using C = FaCfg<NCH, BK, QKS, KS, 3>;
    osb_pdl_trigger_entry();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int head = blockIdx.y, heads = gridDim.y;
    const int q0 = blockIdx.x * BQ;
    const int n_kv = p.kv_tiles;
    uint8_t* smem = fa_prologue(&map_q, &map_k, &map_v, C::BARS, FA_CONSUMERS / 32, KS);   // kv_empty: one arrival per consumer warp
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + C::Q_BYTES;
    uint8_t* sV = sK + KS * C::KV_BYTES;
    uint64_t* q_full = (uint64_t*)(smem + C::BARS);   // [1]
    uint64_t* kv_full = q_full + 1;                    // [KS]
    uint64_t* kv_empty = kv_full + KS;                 // [KS]

    if (warp < 4) {
        setmaxnreg_dec<FA_PRODUCER_REGS>();
        if (warp == 0) {
            if (elect_one()) {
                mbar_expect_tx(q_full, C::Q_BYTES);
#pragma unroll
                for (int pl = 0; pl < 3; pl++)
#pragma unroll
                    for (int c = 0; c < NCH; c++) tma_load_3d(sQ + pl * C::Q_PLANE + c * C::Q_CHUNK, &map_q, q_full, 64 * c, pl * heads + head, q0);
            }
            __syncwarp();
            fa_produce_kv<KS>(kv_full, kv_empty, n_kv, 2 * C::KV_BYTES, [&](int st, int j, uint64_t* bar) {
#pragma unroll
                for (int pl = 0; pl < 3; pl++)
#pragma unroll
                    for (int c = 0; c < NCH; c++) {
                        const int off = st * C::KV_BYTES + pl * C::KV_PLANE + c * C::KV_CHUNK;
                        tma_load_3d(sK + off, &map_k, bar, 64 * c, pl * heads + head, j * BK);
                        tma_load_3d(sV + off, &map_v, bar, 64 * c, pl * heads + head, j * BK);
                    }
            });
        }
    } else {
        // ===================== warpgroups 1, 2: 64 query rows each =====================
        setmaxnreg_inc<FA_CONSUMER_REGS>();
        const int wg = (warp >> 2) - 1;
        const int r = (warp & 3) * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);
        // Q / K K-major (32 B per 16-element k-step inside a 64-column chunk), V MN-major (16 keys = 2048 B per k-step); 8-row groups 1024 B apart
        const uint64_t qdesc = make_smem_desc(smem_u32(sQ) + wg * (BQ / 2) * 128, 16, 1024);
        const uint64_t kdesc0 = make_smem_desc(smem_u32(sK), 16, 1024);
        const uint64_t vdesc0 = make_smem_desc(smem_u32(sV), C::KV_CHUNK, 1024);
        float o[NCH][32];
#pragma unroll
        for (int ch = 0; ch < NCH; ch++)
#pragma unroll
            for (int i = 0; i < 32; i++) o[ch][i] = 0.f;
        float m_run[2] = { -INFINITY, -INFINITY }, l_run[2] = { 0.f, 0.f }, alpha[2];
        mbar_wait(q_full, 0);
        for (int j = 0; j < n_kv; j++) {
            const int st = j % KS;
            mbar_wait(&kv_full[st], (j / KS) & 1);
            // S = sum of the six cross products over the k-steps.  The tensor cores' fp32 accumulation is not round-to-nearest: the five
            // small products go first, while S is still small, and hh last.  The first MMA overwrites S.
            const uint64_t kdesc = kdesc0 + (uint64_t)(st * C::KV_BYTES >> 4), vdesc = vdesc0 + (uint64_t)(st * C::KV_BYTES >> 4);
            float s[BK / 2];
            fence_regs(s);
            wgmma_fence();
#pragma unroll
            for (int xx = 0; xx < 6; xx++)
#pragma unroll
                for (int k = 0; k < QKS; k++) {
                    const int x = 5 - xx;
                    qk_mma_bf16<BK>(s, qdesc + (uint64_t)(((x3a(x) * C::Q_PLANE + (k >> 2) * C::Q_CHUNK) >> 4) + (k & 3) * 2),
                                    kdesc + (uint64_t)(((x3b(x) * C::KV_PLANE + (k >> 2) * C::KV_CHUNK) >> 4) + (k & 3) * 2), (k | xx) != 0);
                }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(s);
            f32x_softmax<BK>(s, m_run, l_run, alpha, j * BK, cq, p.Tk, scale);
            // O *= alpha; P (fp32 in s) -> three bf16 planes in the A-fragment order of the PV MMA (see fa_rescale_pack)
#pragma unroll
            for (int ch = 0; ch < NCH; ch++)
#pragma unroll
                for (int c = 0; c < 8; c++)
#pragma unroll
                    for (int h = 0; h < 2; h++) { o[ch][4 * c + 2 * h] *= alpha[h]; o[ch][4 * c + 2 * h + 1] *= alpha[h]; }
            uint32_t a[3][BK / 16][4];
#pragma unroll
            for (int c = 0; c < BK / 8; c++)
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    __nv_bfloat16 p0[3], p1[3];
                    bf16x3_split(s[4 * c + 2 * h], p0[0], p0[1], p0[2]);
                    bf16x3_split(s[4 * c + 2 * h + 1], p1[0], p1[1], p1[2]);
#pragma unroll
                    for (int pl = 0; pl < 3; pl++) a[pl][c >> 1][(c & 1) * 2 + h] = pack_bf162(p0[pl], p1[pl]);
                }
            // O += P V one 64-column chunk at a time: the tile's product accumulates on the tensor cores in a fresh register tile (small
            // products first, as for S) and is added to O in fp32 here, so O never takes a tensor-core accumulation over the whole sequence
#pragma unroll
            for (int pl = 0; pl < 3; pl++) fence_regs(a[pl]);
#pragma unroll
            for (int ch = 0; ch < NCH; ch++) {
                float t[32];
                fence_regs(t);
                wgmma_fence();
#pragma unroll
                for (int xx = 0; xx < 6; xx++)
#pragma unroll
                    for (int kk = 0; kk < BK / 16; kk++) {
                        const int x = 5 - xx;
                        wgmma_m64n64k16_bf16_rs(t, a[x3a(x)][kk], vdesc + (uint64_t)((x3b(x) * C::KV_PLANE + ch * C::KV_CHUNK + kk * 2048) >> 4), (kk | xx) != 0);
                    }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(t);
#pragma unroll
                for (int i = 0; i < 32; i++) o[ch][i] += t[i];
            }
#pragma unroll
            for (int pl = 0; pl < 3; pl++) fence_regs(a[pl]);
            __syncwarp();
            if (lane == 0) mbar_arrive(&kv_empty[st]);
        }
        // out[q, head*d + c]
        float* rows[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int qrow = q0 + wg * (BQ / 2) + r + 8 * h;
            rows[h] = qrow < p.T ? out + (long long)qrow * p.ldo + (long long)head * p.d : nullptr;
        }
        fa_store(o, l_run, rows, p.d, cq);
    }
}

// Every tensor map is made before anything is enqueued, so a refused launch enqueues nothing.  The plane buffers [rows][3][C] (plane p of
// head h is "head" p * heads + h) hold 2-byte elements that the tensor maps only move: the fp16 element type serves for bf16.
template <int NCH, int BK, int QKS, int KS>
int f32x_launch(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, float* out, FaParams p, float scale,
                int64_t heads, __nv_bfloat16* planes, cudaStream_t st)
{
    using Cf = FaCfg<NCH, BK, QKS, KS, 3>;
    const int64_t C = heads * p.d;
    const uint64_t d = p.d;
    __nv_bfloat16* pq = planes;
    __nv_bfloat16* pk = pq + 3 * p.T * C;
    __nv_bfloat16* pv = pk + 3 * p.Tk * C;
    CUtensorMap mq, mk, mv;
    if (!make_map(&mq, pq, d, 3 * heads, p.T, d * 2, 3 * C * 2, 64, 1, BQ) || !make_map(&mk, pk, d, 3 * heads, p.Tk, d * 2, 3 * C * 2, 64, 1, BK) ||
        !make_map(&mv, pv, d, 3 * heads, p.Tk, d * 2, 3 * C * 2, 64, 1, BK))
        return (int)cudaErrorInvalidValue;
    osb_launch((f32x_split_kernel), grid_for((size_t)((p.T + 2 * (int64_t)p.Tk) * C / 4), 256), 256, 0, st, q, ldq, k, ldk, v, ldv, pq, pk, pv,
               (int64_t)p.T, (int64_t)p.Tk, (int)C);
    const int e = launched();
    if (e) return e;
    p.kv_tiles = (p.Tk + BK - 1) / BK;
    dim3 grid((unsigned)((p.T + BQ - 1) / BQ), (unsigned)heads);
    return fa_launch_kernel<flash_attention_f32x_kernel<NCH, BK, QKS, KS>>(grid, FA_THREADS, Cf::SMEM, st, mq, mk, mv, p, scale, out);
}

// 8 <= d <= 160, d % 8 == 0 (the 128-query kernels' head dims) and sequence lengths whose last query and key tiles start inside int32
bool fa_dims_ok(int64_t T, int64_t Tk, int64_t d)
{
    return d >= 8 && d <= 160 && d % 8 == 0 && T >= 1 && Tk >= 1 && T <= (int64_t)INT32_MAX - BQ && Tk <= (int64_t)INT32_MAX - BKV;
}

// Launch rules of the flash entries whose softmax takes the running maximum over the raw scores: that is the maximum of the scaled
// logits only for scale > 0 (and finite); heads are grid.y.
bool fa_launch_ok(int64_t heads, float scale)
{
    return heads >= 1 && heads <= 65535 && scale > 0.f && scale < INFINITY;
}

bool aligned16(const void* a, const void* b, const void* c, const void* d, const void* e = nullptr)
{
    return (((uintptr_t)a | (uintptr_t)b | (uintptr_t)c | (uintptr_t)d | (uintptr_t)e) & 15) == 0;
}

// ---- fp32 wide heads on the tensor cores: 160 < d <= 512 (the fp32 VAE decoder's single-head d = 512 attention) ---------------------
// softmax(Q K^T * scale) V of flash_attention_wide_kernel for fp32 q [h, T, d], k [h, Tk, d] or [h, d, Tk], v [h, Tk, d], out [h, T, d],
// with the numerics of flash_attention_f32x_kernel: bf16 planes x = h + m + l, six cross products, small ones first, f32x_softmax, P
// split into three planes in registers, each tile's P V added to O in fp32.  Slices, grid and roles are those of the wide kernel (one CTA
// per 256-column slice of V / O, 64-query tile and head; a TMA producer warp and one consumer warpgroup at 240 registers).
// Planes: f32x_split_kernel writes q and v as [h * rows][3][d] (C = d); f32x_split_k_kernel writes K, either layout, K-major as
// [h][3][Tk][d], so the kernel has one K layout.  Q / V are read through (3 d, rows, h) maps -- plane p's chunk c at column p d + 64 c, rows
// past the head's last zero-filled; a chunk that ends past d reads the next plane's first columns, which meet K's zero-filled columns
// (Q K^T) or feed output columns that are never stored (P V) -- and K through (d, Tk, 3 h).
// Three planes of Q do not fit beside the rings (64 x 512 x 3 x 2 B = 192 KB), so Q streams with K: a stage of the Q K^T ring holds one
// 64-column chunk of Q and of a 32-key K tile (3 x 8 KB + 3 x 4 KB); 3 stages (108 KB) + 2 stages of 32-key x 256-column V tiles (2 x
// 48 KB) = 204 KB.  Registers: O 128 + S 16 + a chunk's product 16, then P 3 x 8 + a P V chunk 32.  Each chunk's six products go to a
// fresh register tile that is added to S in fp32, so S, like O, never takes a tensor-core accumulation over more than one chunk.
constexpr int WX_BK = 32;                               // keys per tile
constexpr int WX_QK_STAGES = 3, WX_V_STAGES = 2;
constexpr int WX_Q_PLANE = WD_BQ * 128;                 // one 64-column chunk of one plane: 64 rows x 128 B
constexpr int WX_K_PLANE = WX_BK * 128;                 // 32 keys x 128 B
constexpr int WX_QK_BYTES = 3 * WX_Q_PLANE + 3 * WX_K_PLANE;
constexpr int WX_V_CHUNK = WX_BK * 128;                 // 32 keys x 64 columns of one plane
constexpr int WX_V_PLANE = WD_NV * WX_V_CHUNK;
constexpr int WX_V_BYTES = 3 * WX_V_PLANE;
constexpr int WX_BARS = WX_QK_STAGES * WX_QK_BYTES + WX_V_STAGES * WX_V_BYTES;
constexpr int WX_SMEM = WX_BARS + 1024 + 256;
static_assert(WX_SMEM <= 227 * 1024, "shared memory");

// k [h, Tk, d] (KT = false) or [h, d, Tk] (KT = true) fp32 -> bf16 planes pk [h][3][Tk][d]: a 32-key x 32-column tile through shared
// memory, read along the input's contiguous axis and written along d
template <bool KT>
__global__ void __launch_bounds__(256) f32x_split_k_kernel(const float* __restrict__ k, __nv_bfloat16* __restrict__ pk, int Tk, int d)
{
    osb_pdl_prologue();
    __shared__ float tile[32][33];     // [column][key]
    const int key0 = blockIdx.x * 32, c0 = blockIdx.y * 32, head = blockIdx.z;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const float* src = k + (int64_t)head * Tk * d;
    for (int i = ty; i < 32; i += 8) {
        const int key = key0 + (KT ? tx : i), c = c0 + (KT ? i : tx);
        if (key < Tk && c < d) tile[c - c0][key - key0] = KT ? src[(int64_t)c * Tk + key] : src[(int64_t)key * d + c];
    }
    __syncthreads();
    __nv_bfloat16* dst = pk + (int64_t)head * 3 * Tk * d;
    for (int i = ty; i < 32; i += 8) {
        const int key = key0 + i, c = c0 + tx;
        if (key < Tk && c < d) {
            __nv_bfloat16 h, m, l;
            bf16x3_split(tile[tx][i], h, m, l);
            const int64_t o = (int64_t)key * d + c;
            dst[o] = h;
            dst[(int64_t)Tk * d + o] = m;
            dst[2 * (int64_t)Tk * d + o] = l;
        }
    }
}

__global__ void __launch_bounds__(WD_THREADS, 1)
flash_attention_wide_f32x_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                                 const __grid_constant__ CUtensorMap map_v, const FaParams p, float scale, float* __restrict__ out)
{
    constexpr int QS = WX_QK_STAGES, VS = WX_V_STAGES;
    osb_pdl_trigger_entry();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // blockIdx.x = query tile * slices + slice, as in flash_attention_wide_kernel
    const int n_slices = (p.d + 64 * WD_NV - 1) / (64 * WD_NV);
    const int col0 = (blockIdx.x % n_slices) * (64 * WD_NV);
    const int q0 = (blockIdx.x / n_slices) * WD_BQ;
    const int head = blockIdx.y;
    const int n_dch = (p.d + 63) >> 6;
    const int n_vch = min(WD_NV, (p.d - col0 + 63) >> 6);     // V / O chunks of this slice inside d
    uint8_t* smem = fa_prologue(&map_q, &map_k, &map_v, WX_BARS, WD_CONSUMERS / 32, QS, VS);
    uint8_t* sQK = smem;
    uint8_t* sV = sQK + QS * WX_QK_BYTES;
    uint64_t* qk_full = (uint64_t*)(smem + WX_BARS) + 1;    // [QS] (after fa_prologue's q_full, unused here)
    uint64_t* qk_empty = qk_full + QS;                       // [QS]: one arrival per consumer warp
    uint64_t* v_full = qk_empty + QS;                        // [VS]
    uint64_t* v_empty = v_full + VS;                         // [VS]
    const int n_kv = p.kv_tiles;

    if (warp < 4) {
        setmaxnreg_dec<WD_PRODUCER_REGS>();
        if (warp == 0) {
            int kc = 0;
            for (int j = 0; j < n_kv; j++) {
                for (int c = 0; c < n_dch; c++, kc++) {
                    const int st = kc % QS;
                    mbar_wait(&qk_empty[st], ((kc / QS) & 1) ^ 1);
                    if (elect_one()) {
                        uint8_t* s = sQK + st * WX_QK_BYTES;
                        mbar_expect_tx(&qk_full[st], WX_QK_BYTES);
                        for (int pl = 0; pl < 3; pl++) {
                            tma_load_3d(s + pl * WX_Q_PLANE, &map_q, &qk_full[st], pl * p.d + 64 * c, q0, head);
                            tma_load_3d(s + 3 * WX_Q_PLANE + pl * WX_K_PLANE, &map_k, &qk_full[st], 64 * c, j * WX_BK, 3 * head + pl);
                        }
                    }
                    __syncwarp();
                }
                const int sv = j % VS;
                mbar_wait(&v_empty[sv], ((j / VS) & 1) ^ 1);
                if (elect_one()) {
                    mbar_expect_tx(&v_full[sv], 3 * n_vch * WX_V_CHUNK);
                    for (int pl = 0; pl < 3; pl++)
                        for (int ch = 0; ch < n_vch; ch++)
                            tma_load_3d(sV + sv * WX_V_BYTES + pl * WX_V_PLANE + ch * WX_V_CHUNK, &map_v, &v_full[sv], pl * p.d + col0 + 64 * ch,
                                        j * WX_BK, head);
                }
                __syncwarp();
            }
            osb_pdl_trigger_late();
        }
    } else {
        // ===================== warpgroup 1: the CTA's 64 query rows =====================
        setmaxnreg_inc<WD_CONSUMER_REGS>();
        const int r = (warp & 3) * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);
        // Q / K K-major (32 B per k-step inside the swizzle row), V MN-major (16 keys = 2048 B per k-step); 8-row groups 1024 B apart
        const uint64_t qdesc0 = make_smem_desc(smem_u32(sQK), 16, 1024);
        const uint64_t vdesc0 = make_smem_desc(smem_u32(sV), WX_V_CHUNK, 1024);
        float o[WD_NV][32];
#pragma unroll
        for (int ch = 0; ch < WD_NV; ch++)
#pragma unroll
            for (int i = 0; i < 32; i++) o[ch][i] = 0.f;
        float m_run[2] = { -INFINITY, -INFINITY }, l_run[2] = { 0.f, 0.f }, alpha[2];
        int kc = 0;
        for (int j = 0; j < n_kv; j++) {
            // S = sum over the chunks of d of the chunk's six cross products (small ones first, hh last; the first MMA overwrites t)
            float s[WX_BK / 2];
            for (int c = 0; c < n_dch; c++, kc++) {
                const int st = kc % QS;
                const uint64_t qdesc = qdesc0 + (uint64_t)((st * WX_QK_BYTES) >> 4);
                const uint64_t kdesc = qdesc + (uint64_t)((3 * WX_Q_PLANE) >> 4);
                mbar_wait(&qk_full[st], (kc / QS) & 1);
                float t[WX_BK / 2];
                fence_regs(t);
                wgmma_fence();
#pragma unroll
                for (int xx = 0; xx < 6; xx++)
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const int x = 5 - xx;
                        wgmma_m64n32k16_bf16<0>(t, qdesc + (uint64_t)(((x3a(x) * WX_Q_PLANE) >> 4) + k * 2),
                                                kdesc + (uint64_t)(((x3b(x) * WX_K_PLANE) >> 4) + k * 2), (k | xx) != 0);
                    }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(t);
                __syncwarp();
                if (lane == 0) mbar_arrive(&qk_empty[st]);
#pragma unroll
                for (int i = 0; i < WX_BK / 2; i++) s[i] = c == 0 ? t[i] : s[i] + t[i];
            }
            f32x_softmax<WX_BK>(s, m_run, l_run, alpha, j * WX_BK, cq, p.Tk, scale);
            // O *= alpha; P -> three bf16 planes in the A-fragment order of the P V MMA (see flash_attention_f32x_kernel)
#pragma unroll
            for (int ch = 0; ch < WD_NV; ch++)
#pragma unroll
                for (int c = 0; c < 8; c++)
#pragma unroll
                    for (int h = 0; h < 2; h++) { o[ch][4 * c + 2 * h] *= alpha[h]; o[ch][4 * c + 2 * h + 1] *= alpha[h]; }
            uint32_t a[3][WX_BK / 16][4];
#pragma unroll
            for (int c = 0; c < WX_BK / 8; c++)
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    __nv_bfloat16 p0[3], p1[3];
                    bf16x3_split(s[4 * c + 2 * h], p0[0], p0[1], p0[2]);
                    bf16x3_split(s[4 * c + 2 * h + 1], p1[0], p1[1], p1[2]);
#pragma unroll
                    for (int pl = 0; pl < 3; pl++) a[pl][c >> 1][(c & 1) * 2 + h] = pack_bf162(p0[pl], p1[pl]);
                }
            // O_slice += P V_slice one 64-column chunk at a time, each through a fresh register tile added to O in fp32; chunks past d
            // are neither loaded nor multiplied
            const int sv = j % VS;
            const uint64_t vdesc = vdesc0 + (uint64_t)((sv * WX_V_BYTES) >> 4);
            mbar_wait(&v_full[sv], (j / VS) & 1);
#pragma unroll
            for (int pl = 0; pl < 3; pl++) fence_regs(a[pl]);
#pragma unroll
            for (int ch = 0; ch < WD_NV; ch++) {
                if (ch >= n_vch) break;
                float t[32];
                fence_regs(t);
                wgmma_fence();
#pragma unroll
                for (int xx = 0; xx < 6; xx++)
#pragma unroll
                    for (int kk = 0; kk < WX_BK / 16; kk++) {
                        const int x = 5 - xx;
                        wgmma_m64n64k16_bf16_rs(t, a[x3a(x)][kk], vdesc + (uint64_t)((x3b(x) * WX_V_PLANE + ch * WX_V_CHUNK + kk * 2048) >> 4),
                                                (kk | xx) != 0);
                    }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(t);
#pragma unroll
                for (int i = 0; i < 32; i++) o[ch][i] += t[i];
            }
#pragma unroll
            for (int pl = 0; pl < 3; pl++) fence_regs(a[pl]);
            __syncwarp();
            if (lane == 0) mbar_arrive(&v_empty[sv]);
        }
        // out[head][q][col0 + c]
        float* rows[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int qrow = q0 + r + 8 * h;
            rows[h] = qrow < p.T ? out + ((long long)head * p.T + qrow) * p.d + col0 : nullptr;
        }
        fa_store(o, l_run, rows, p.d - col0, cq);
    }
}

// Every tensor map is made before the splits are enqueued.  planes: pq [h * T][3][d], pk [h][3][Tk][d], pv [h * Tk][3][d].
int wx_launch(const float* q, const float* k, const float* v, float* out, FaParams p, float scale, int64_t heads, bool kt,
              __nv_bfloat16* planes, cudaStream_t st)
{
    const int64_t T = p.T, Tk = p.Tk, d = p.d;
    __nv_bfloat16* pq = planes;
    __nv_bfloat16* pk = pq + 3 * heads * T * d;
    __nv_bfloat16* pv = pk + 3 * heads * Tk * d;
    CUtensorMap mq, mk, mv;
    if (!make_map(&mq, pq, 3 * d, T, heads, 3 * d * 2, T * 3 * d * 2, 64, WD_BQ, 1) ||
        !make_map(&mk, pk, d, Tk, 3 * heads, d * 2, Tk * d * 2, 64, WX_BK, 1) ||
        !make_map(&mv, pv, 3 * d, Tk, heads, 3 * d * 2, Tk * 3 * d * 2, 64, WX_BK, 1))
        return (int)cudaErrorInvalidValue;
    // q and v as [h * rows, d] with no K part, then K
    osb_launch((f32x_split_kernel), grid_for((size_t)(heads * T * d / 4), 256), 256, 0, st, q, d, q, d, q, d, pq, pq, pq, heads * T,
               (int64_t)0, (int)d);
    int e = launched();
    if (e) return e;
    osb_launch((f32x_split_kernel), grid_for((size_t)(heads * Tk * d / 4), 256), 256, 0, st, v, d, v, d, v, d, pv, pv, pv, heads * Tk,
               (int64_t)0, (int)d);
    if ((e = launched())) return e;
    const dim3 kgrid((unsigned)((Tk + 31) / 32), (unsigned)((d + 31) / 32), (unsigned)heads), kblock(32, 8);
    if (kt) osb_launch((f32x_split_k_kernel<true>), kgrid, kblock, 0, st, k, pk, (int)Tk, (int)d);
    else osb_launch((f32x_split_k_kernel<false>), kgrid, kblock, 0, st, k, pk, (int)Tk, (int)d);
    if ((e = launched())) return e;
    p.kv_tiles = (int)((Tk + WX_BK - 1) / WX_BK);
    const int64_t n_slices = (d + 64 * WD_NV - 1) / (64 * WD_NV);
    dim3 grid((unsigned)((T + WD_BQ - 1) / WD_BQ * n_slices), (unsigned)heads);
    return fa_launch_kernel<flash_attention_wide_f32x_kernel>(grid, WD_THREADS, WX_SMEM, st, mq, mk, mv, p, scale, out);
}

// ---- fp32 grouped-KV masked attention on the tensor cores (ScaledDotProductAttention in fp32 arithmetic: prompt prefill) -------------
// softmax(Q K^T * scale + mask) V of sdpa_flash_kernel for fp32 q [Hq, Tq, d], k / v [Hkv, Tk, d], mask [Tq, Tk], out [Hq, Tq, d], with
// the numerics of flash_attention_f32x_kernel: bf16 planes x = h + m + l, six cross products, small ones first, the fp32
// softmax with the mask added in natural units (f32x_softmax<BK, true>).  Roles and packing are sdpa_flash_kernel's: one CTA per 128
// packed rows [G*Tq, d] of one KV head (grid.y), packed row R is query R % Tq of head hk*G + R / Tq and reads mask row R % Tq; a TMA
// producer warp and two consumer warpgroups at 232 registers, unpipelined.  Tiles as the f32x kernel's (FaCfg<NCH, BK, QKS, KS, 3>):
// d <= 64: 64-key tiles, 2 stages; d <= 128: 32-key tiles, 2 stages.
// Planes as the wide fp32 kernel lays them out: q and v [rows][3][d] read through (3 d, rows, Hkv) maps, K [Hkv][3][Tk][d] through a
// (d, Tk, 3 Hkv) map.  Rows past G*Tq and keys past Tk are zero-filled by TMA; a Q chunk that ends past d reads the next plane's first
// columns, which meet K's zero-filled columns, and a V chunk's columns past d feed output columns that are never stored.
// The mask is not folded into log2 units: llm.cpp's fp32 masks hold -3.4028235e38, which times log2e overflows to -inf.
struct SdpaF32xParams {
    int rows;                // G * Tq: packed query rows per KV head
    int Tq, Tk, d;
    int kv_tiles;
    float scale;
    const float* mask;       // [Tq, Tk] additive, or nullptr
    int mask_vec;            // 8-byte mask loads: Tk even and the mask 8-byte aligned
    float* out;              // [Hkv][G*Tq][d] (= [Hq, Tq, d])
};

// mask[row][col], mask[row][col + 1]; keys past Tk read as 0 (they get -inf afterwards).  vec: the pair is 8-byte aligned.
__device__ __forceinline__ float2 ld_mask_pair_f32(const float* row, int col, int Tk, bool vec)
{
    if (col + 1 < Tk) {
        if (vec) return __ldg(reinterpret_cast<const float2*>(row + col));
        return make_float2(__ldg(row + col), __ldg(row + col + 1));
    }
    return make_float2(col < Tk ? __ldg(row + col) : 0.f, 0.f);
}

template <int NCH, int BK, int QKS, int KS>
__global__ void __launch_bounds__(FA_THREADS, 1)
sdpa_flash_f32x_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                       const SdpaF32xParams p)
{
    using C = FaCfg<NCH, BK, QKS, KS, 3>;
    osb_pdl_trigger_entry();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r0 = blockIdx.x * BQ, hk = blockIdx.y;
    const int n_kv = p.kv_tiles;
    uint8_t* smem = fa_prologue(&map_q, &map_k, &map_v, C::BARS, FA_CONSUMERS / 32, KS);   // kv_empty: one arrival per consumer warp
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + C::Q_BYTES;
    uint8_t* sV = sK + KS * C::KV_BYTES;
    uint64_t* q_full = (uint64_t*)(smem + C::BARS);   // [1]
    uint64_t* kv_full = q_full + 1;                    // [KS]
    uint64_t* kv_empty = kv_full + KS;                 // [KS]

    if (warp < 4) {
        setmaxnreg_dec<FA_PRODUCER_REGS>();
        if (warp == 0) {
            if (elect_one()) {
                mbar_expect_tx(q_full, C::Q_BYTES);
#pragma unroll
                for (int pl = 0; pl < 3; pl++)
#pragma unroll
                    for (int c = 0; c < NCH; c++) tma_load_3d(sQ + pl * C::Q_PLANE + c * C::Q_CHUNK, &map_q, q_full, pl * p.d + 64 * c, r0, hk);
            }
            __syncwarp();
            fa_produce_kv<KS>(kv_full, kv_empty, n_kv, 2 * C::KV_BYTES, [&](int st, int j, uint64_t* bar) {
#pragma unroll
                for (int pl = 0; pl < 3; pl++)
#pragma unroll
                    for (int c = 0; c < NCH; c++) {
                        const int off = st * C::KV_BYTES + pl * C::KV_PLANE + c * C::KV_CHUNK;
                        tma_load_3d(sK + off, &map_k, bar, 64 * c, j * BK, 3 * hk + pl);
                        tma_load_3d(sV + off, &map_v, bar, pl * p.d + 64 * c, j * BK, hk);
                    }
            });
        }
    } else {
        // ===================== warpgroups 1, 2: 64 packed rows each =====================
        setmaxnreg_inc<FA_CONSUMER_REGS>();
        const int wg = (warp >> 2) - 1;
        const int r = (warp & 3) * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);
        const uint64_t qdesc = make_smem_desc(smem_u32(sQ) + wg * (BQ / 2) * 128, 16, 1024);
        const uint64_t kdesc0 = make_smem_desc(smem_u32(sK), 16, 1024);
        const uint64_t vdesc0 = make_smem_desc(smem_u32(sV), C::KV_CHUNK, 1024);
        const bool has_mask = p.mask != nullptr, vec = p.mask_vec != 0;
        const float* mrow[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int R = r0 + wg * (BQ / 2) + r + 8 * h;                     // rows past G*Tq (zero-filled by TMA) are never stored
            mrow[h] = has_mask ? p.mask + (long long)(R % p.Tq) * p.Tk : nullptr;
        }
        float o[NCH][32];
#pragma unroll
        for (int ch = 0; ch < NCH; ch++)
#pragma unroll
            for (int i = 0; i < 32; i++) o[ch][i] = 0.f;
        float m_run[2] = { -INFINITY, -INFINITY }, l_run[2] = { 0.f, 0.f }, alpha[2];
        mbar_wait(q_full, 0);
        for (int j = 0; j < n_kv; j++) {
            const int st = j % KS;
            const int key0 = j * BK;
            mbar_wait(&kv_full[st], (j / KS) & 1);
            // S = the six cross products, small ones first, as in flash_attention_f32x_kernel
            const uint64_t kdesc = kdesc0 + (uint64_t)(st * C::KV_BYTES >> 4), vdesc = vdesc0 + (uint64_t)(st * C::KV_BYTES >> 4);
            float s[BK / 2];
            fence_regs(s);
            wgmma_fence();
#pragma unroll
            for (int xx = 0; xx < 6; xx++)
#pragma unroll
                for (int k = 0; k < QKS; k++) {
                    const int x = 5 - xx;
                    qk_mma_bf16<BK>(s, qdesc + (uint64_t)(((x3a(x) * C::Q_PLANE + (k >> 2) * C::Q_CHUNK) >> 4) + (k & 3) * 2),
                                    kdesc + (uint64_t)(((x3b(x) * C::KV_PLANE + (k >> 2) * C::KV_CHUNK) >> 4) + (k & 3) * 2), (k | xx) != 0);
                }
            wgmma_commit();
            // the mask loads (L2-resident: every head reads the same [Tq, Tk] block) are in flight while the MMAs run
            float2 mk[2][BK / 8];
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int c = 0; c < BK / 8; c++) mk[h][c] = has_mask ? ld_mask_pair_f32(mrow[h], key0 + 8 * c + cq, p.Tk, vec) : make_float2(0.f, 0.f);
            wgmma_wait<0>();
            fence_regs(s);
            f32x_softmax<BK, true>(s, m_run, l_run, alpha, key0, cq, p.Tk, p.scale, mk);
            // O *= alpha; P -> three bf16 planes; O += P V one 64-column chunk at a time through a fresh register tile added in fp32
#pragma unroll
            for (int ch = 0; ch < NCH; ch++)
#pragma unroll
                for (int c = 0; c < 8; c++)
#pragma unroll
                    for (int h = 0; h < 2; h++) { o[ch][4 * c + 2 * h] *= alpha[h]; o[ch][4 * c + 2 * h + 1] *= alpha[h]; }
            uint32_t a[3][BK / 16][4];
#pragma unroll
            for (int c = 0; c < BK / 8; c++)
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    __nv_bfloat16 p0[3], p1[3];
                    bf16x3_split(s[4 * c + 2 * h], p0[0], p0[1], p0[2]);
                    bf16x3_split(s[4 * c + 2 * h + 1], p1[0], p1[1], p1[2]);
#pragma unroll
                    for (int pl = 0; pl < 3; pl++) a[pl][c >> 1][(c & 1) * 2 + h] = pack_bf162(p0[pl], p1[pl]);
                }
#pragma unroll
            for (int pl = 0; pl < 3; pl++) fence_regs(a[pl]);
#pragma unroll
            for (int ch = 0; ch < NCH; ch++) {
                float t[32];
                fence_regs(t);
                wgmma_fence();
#pragma unroll
                for (int xx = 0; xx < 6; xx++)
#pragma unroll
                    for (int kk = 0; kk < BK / 16; kk++) {
                        const int x = 5 - xx;
                        wgmma_m64n64k16_bf16_rs(t, a[x3a(x)][kk], vdesc + (uint64_t)((x3b(x) * C::KV_PLANE + ch * C::KV_CHUNK + kk * 2048) >> 4), (kk | xx) != 0);
                    }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(t);
#pragma unroll
                for (int i = 0; i < 32; i++) o[ch][i] += t[i];
            }
#pragma unroll
            for (int pl = 0; pl < 3; pl++) fence_regs(a[pl]);
            __syncwarp();
            if (lane == 0) mbar_arrive(&kv_empty[st]);
        }
        // out[hk][R][col]
        float* rows[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int R = r0 + wg * (BQ / 2) + r + 8 * h;
            rows[h] = R < p.rows ? p.out + ((long long)hk * p.rows + R) * p.d : nullptr;
        }
        fa_store(o, l_run, rows, p.d, cq);
    }
}

// Every tensor map is made before the splits are enqueued.  planes: pq [Hq * Tq][3][d], pk [Hkv][3][Tk][d], pv [Hkv * Tk][3][d].
template <int NCH, int BK, int QKS, int KS>
int sdpa_f32x_launch(const float* q, const float* k, const float* v, SdpaF32xParams p, int64_t Hkv, __nv_bfloat16* planes, cudaStream_t st)
{
    using Cf = FaCfg<NCH, BK, QKS, KS, 3>;
    const int64_t rows = p.rows, Tk = p.Tk, d = p.d;
    __nv_bfloat16* pq = planes;
    __nv_bfloat16* pk = pq + 3 * Hkv * rows * d;
    __nv_bfloat16* pv = pk + 3 * Hkv * Tk * d;
    CUtensorMap mq, mk, mv;
    if (!make_map(&mq, pq, 3 * d, rows, Hkv, 3 * d * 2, rows * 3 * d * 2, 64, BQ, 1) ||
        !make_map(&mk, pk, d, Tk, 3 * Hkv, d * 2, Tk * d * 2, 64, BK, 1) ||
        !make_map(&mv, pv, 3 * d, Tk, Hkv, 3 * d * 2, Tk * 3 * d * 2, 64, BK, 1))
        return (int)cudaErrorInvalidValue;
    // q and v as [rows, d] with no K part, then K
    osb_launch((f32x_split_kernel), grid_for((size_t)(Hkv * rows * d / 4), 256), 256, 0, st, q, d, q, d, q, d, pq, pq, pq, Hkv * rows,
               (int64_t)0, (int)d);
    int e = launched();
    if (e) return e;
    osb_launch((f32x_split_kernel), grid_for((size_t)(Hkv * Tk * d / 4), 256), 256, 0, st, v, d, v, d, v, d, pv, pv, pv, Hkv * Tk,
               (int64_t)0, (int)d);
    if ((e = launched())) return e;
    const dim3 kgrid((unsigned)((Tk + 31) / 32), (unsigned)((d + 31) / 32), (unsigned)Hkv), kblock(32, 8);
    osb_launch((f32x_split_k_kernel<false>), kgrid, kblock, 0, st, k, pk, (int)Tk, (int)d);
    if ((e = launched())) return e;
    p.kv_tiles = (int)((Tk + BK - 1) / BK);
    dim3 grid((unsigned)((rows + BQ - 1) / BQ), (unsigned)Hkv);
    return fa_launch_kernel<sdpa_flash_f32x_kernel<NCH, BK, QKS, KS>>(grid, FA_THREADS, Cf::SMEM, st, mq, mk, mv, p);
}

}  // namespace

// fp32 rows [rows][C] -> bf16 planes [rows][3][C] (h, m, l), C % 4 == 0, 16-byte aligned: the A operand of osb_tc_gemm_f32x_f16w
int osb_f32x_split_rows(const float* x, __nv_bfloat16* planes, int64_t rows, int64_t C, cudaStream_t st)
{
    osb_launch((f32x_split_kernel), grid_for((size_t)(rows * C / 4), 256), 256, 0, st, x, C, x, C, x, C, planes, planes, planes, rows, (int64_t)0, (int)C);
    return launched();
}

extern "C" int osb_flash_attention_ok(int64_t T, int64_t Tk, int64_t d, int dtype)
{
    return dtype == OSB_F16 && T >= 64 && fa_dims_ok(T, Tk, d) && get_encode() != nullptr;
}

// q [T, heads*d] (row stride ldq), k / v [Tk, heads*d] (row strides ldk / ldv), out [T, heads*d] (row stride ldo); fp16, 16-byte aligned.
// scale > 0: the running maximum is taken over the raw scores.
extern "C" int osb_flash_attention(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out, int64_t ldo,
                                   int64_t heads, int64_t T, int64_t Tk, int64_t d, float scale, void* stream)
{
    if (heads * T == 0) return 0;
    if (!fa_dims_ok(T, Tk, d) || !fa_launch_ok(heads, scale) || (ldq % 8) || (ldk % 8) || (ldv % 8) || (ldo % 8) || !aligned16(q, k, v, out))
        return (int)cudaErrorInvalidValue;
    FaParams p{};
    p.T = (int)T; p.Tk = (int)Tk; p.d = (int)d;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.out = (__half*)out; p.ldo = ldo;
    cudaStream_t st = (cudaStream_t)stream;
    if (d <= 48) return fa_launch<1, 128, 3>(q, ldq, k, ldk, v, ldv, p, heads, st);
    if (d <= 64) return fa_launch<1, 128, 4>(q, ldq, k, ldk, v, ldv, p, heads, st);
    if (d <= 80) return fa_launch<2, 64, 5>(q, ldq, k, ldk, v, ldv, p, heads, st);
    if (d <= 128) return fa_launch<2, 64, 8>(q, ldq, k, ldk, v, ldv, p, heads, st);
    return fa_launch<3, 32, 10>(q, ldq, k, ldk, v, ldv, p, heads, st);
}

extern "C" int osb_flash_attention_f32x_ok(int64_t T, int64_t Tk, int64_t d, int dtype)
{
    return dtype == OSB_F32 && fa_dims_ok(T, Tk, d) && get_encode() != nullptr;
}

// osb_flash_attention for fp32 q / k / v / out (row strides in floats, multiples of 4, >= heads * d; 16-byte aligned pointers), planes: scratch
// of 6 (T + 2 Tk) heads d bytes for the bf16 planes.  Two launches: the split, then the attention.
extern "C" int osb_flash_attention_f32x(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out, int64_t ldo,
                                        int64_t heads, int64_t T, int64_t Tk, int64_t d, float scale, void* planes, void* stream)
{
    if (!osb_flash_attention_f32x_ok(T, Tk, d, OSB_F32) || !fa_launch_ok(heads, scale)) return (int)cudaErrorInvalidValue;
    const int64_t C = heads * d;
    if (ldq < C || ldk < C || ldv < C || ldo < C || (ldq % 4) || (ldk % 4) || (ldv % 4) || (ldo % 4) || C > INT32_MAX) return (int)cudaErrorInvalidValue;
    if (!aligned16(q, k, v, out, planes)) return (int)cudaErrorInvalidValue;
    FaParams p{};
    p.T = (int)T; p.Tk = (int)Tk; p.d = (int)d;
    p.out = nullptr; p.ldo = ldo;
    const float* fq = (const float*)q; const float* fk = (const float*)k; const float* fv = (const float*)v;
    float* fo = (float*)out;
    __nv_bfloat16* pl = (__nv_bfloat16*)planes;
    cudaStream_t st = (cudaStream_t)stream;
    if (d <= 48) return f32x_launch<1, 64, 3, 2>(fq, ldq, fk, ldk, fv, ldv, fo, p, scale, heads, pl, st);
    if (d <= 64) return f32x_launch<1, 64, 4, 2>(fq, ldq, fk, ldk, fv, ldv, fo, p, scale, heads, pl, st);
    if (d <= 80) return f32x_launch<2, 32, 5, 2>(fq, ldq, fk, ldk, fv, ldv, fo, p, scale, heads, pl, st);
    if (d <= 128) return f32x_launch<2, 32, 8, 2>(fq, ldq, fk, ldk, fv, ldv, fo, p, scale, heads, pl, st);
    return f32x_launch<3, 32, 10, 1>(fq, ldq, fk, ldk, fv, ldv, fo, p, scale, heads, pl, st);
}

extern "C" int osb_flash_attention_wide_ok(int64_t T, int64_t Tk, int64_t d, int dtype)
{
    return dtype == OSB_F16 && d > 160 && d <= 64 * WD_DCH && d % 8 == 0 && T >= 1 && Tk >= 1 && T <= (int64_t)INT32_MAX - WD_BQ &&
           Tk <= (int64_t)INT32_MAX - WD_BK && get_encode() != nullptr;
}

// q [h, T, d], k [h, Tk, d] or (k_transposed) [h, d, Tk], v [h, Tk, d], out [h, T, d]; fp16, contiguous, 16-byte aligned.  K^T rows are
// Tk elements long, so k_transposed needs Tk % 8 == 0 (TMA row strides are multiples of 16 bytes).  scale > 0: the running maximum is
// taken over the raw scores.
extern "C" int osb_flash_attention_wide(const void* q, const void* k, const void* v, void* out, int64_t heads, int64_t T, int64_t Tk, int64_t d,
                                        float scale, int k_transposed, int dtype, void* stream)
{
    if (!osb_flash_attention_wide_ok(T, Tk, d, dtype) || !fa_launch_ok(heads, scale) || (k_transposed && Tk % 8) || !aligned16(q, k, v, out))
        return (int)cudaErrorInvalidValue;
    FaParams p{};
    p.T = (int)T; p.Tk = (int)Tk; p.d = (int)d;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.out = (__half*)out; p.ldo = d;
    cudaStream_t st = (cudaStream_t)stream;
    return k_transposed ? wd_launch<true>(q, k, v, p, heads, st) : wd_launch<false>(q, k, v, p, heads, st);
}

extern "C" int osb_flash_attention_wide_f32x_ok(int64_t T, int64_t Tk, int64_t d, int dtype)
{
    return dtype == OSB_F32 && d > 160 && d <= 64 * WD_DCH && d % 8 == 0 && T >= 1 && Tk >= 1 && T <= (int64_t)INT32_MAX - WD_BQ &&
           Tk <= (int64_t)INT32_MAX - WX_BK && get_encode() != nullptr;
}

// osb_flash_attention_wide for fp32 q / k / v / out (contiguous, 16-byte aligned) on the bf16 tensor cores at fp32 accuracy.  K^T is
// transposed by the split, so any Tk takes either layout.  planes: scratch of 6 (T + 2 Tk) heads d bytes.  Four launches: the splits of q,
// v and k, then the attention.
extern "C" int osb_flash_attention_wide_f32x(const void* q, const void* k, const void* v, void* out, int64_t heads, int64_t T, int64_t Tk,
                                             int64_t d, float scale, int k_transposed, void* planes, void* stream)
{
    if (!osb_flash_attention_wide_f32x_ok(T, Tk, d, OSB_F32) || !fa_launch_ok(heads, scale) || !aligned16(q, k, v, out, planes))
        return (int)cudaErrorInvalidValue;
    FaParams p{};
    p.T = (int)T; p.Tk = (int)Tk; p.d = (int)d;
    p.out = nullptr; p.ldo = d;
    return wx_launch((const float*)q, (const float*)k, (const float*)v, (float*)out, p, scale, heads, k_transposed != 0, (__nv_bfloat16*)planes,
                     (cudaStream_t)stream);
}

extern "C" int osb_sdpa_flash_ok(int64_t Hq, int64_t Hkv, int64_t Tq, int64_t Tk, int64_t d, int64_t dv, int dtype)
{
    return dtype == OSB_F16 && d == dv && d >= 8 && d <= 128 && d % 8 == 0 && Hkv >= 1 && Hkv <= 65535 && Hq >= Hkv && Hq % Hkv == 0 &&
           Tq >= 1 && Tk >= 1 && (Hq / Hkv) * Tq <= (int64_t)INT32_MAX - BQ && Tk <= (int64_t)INT32_MAX - BKV && get_encode() != nullptr;
}

// q [Hq,Tq,d], k / v [Hkv,Tk,d], mask [Tq,Tk] (additive, may be null), out [Hq,Tq,d]; fp16, contiguous.  Any scale: the running maximum
// is taken over the scaled logits.
extern "C" int osb_sdpa_flash(const void* q, const void* k, const void* v, const void* mask, void* out,
                              int64_t Hq, int64_t Hkv, int64_t Tq, int64_t Tk, int64_t d, float scale, void* stream)
{
    if (Hq * Tq * d == 0) return 0;
    if (!osb_sdpa_flash_ok(Hq, Hkv, Tq, Tk, d, d, OSB_F16)) return (int)cudaErrorInvalidValue;
    if (!aligned16(q, k, v, out) || ((uintptr_t)mask & 3) != 0) return (int)cudaErrorInvalidValue;
    SdpaParams p{};
    p.rows = (int)((Hq / Hkv) * Tq); p.Tq = (int)Tq; p.Tk = (int)Tk; p.d = (int)d;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.mask = (const __half*)mask; p.out = (__half*)out;
    cudaStream_t st = (cudaStream_t)stream;
    return d <= 64 ? sdpa_launch<1, 128>(q, k, v, p, Hkv, st) : sdpa_launch<2, 64>(q, k, v, p, Hkv, st);
}

extern "C" int osb_sdpa_flash_f32x_ok(int64_t Hq, int64_t Hkv, int64_t Tq, int64_t Tk, int64_t d, int64_t dv, int dtype)
{
    return dtype == OSB_F32 && d == dv && d >= 8 && d <= 128 && d % 8 == 0 && Hkv >= 1 && Hkv <= 65535 && Hq >= Hkv && Hq % Hkv == 0 &&
           Tq >= 1 && Tk >= 1 && (Hq / Hkv) * Tq <= (int64_t)INT32_MAX - BQ && Tk <= (int64_t)INT32_MAX - BKV && get_encode() != nullptr;
}

// osb_sdpa_flash for fp32 q / k / v / mask / out (contiguous; q, k, v, out and planes 16-byte aligned, the mask 4-byte aligned) on the
// bf16 tensor cores at fp32 accuracy.  Any finite scale.  planes: scratch of 6 (Hq Tq + 2 Hkv Tk) d bytes.  Four launches: the splits of
// q, v and k, then the attention.
extern "C" int osb_sdpa_flash_f32x(const void* q, const void* k, const void* v, const void* mask, void* out,
                                   int64_t Hq, int64_t Hkv, int64_t Tq, int64_t Tk, int64_t d, float scale, void* planes, void* stream)
{
    if (!osb_sdpa_flash_f32x_ok(Hq, Hkv, Tq, Tk, d, d, OSB_F32) || !(fabsf(scale) < INFINITY)) return (int)cudaErrorInvalidValue;
    if (!aligned16(q, k, v, out, planes) || ((uintptr_t)mask & 3) != 0) return (int)cudaErrorInvalidValue;
    SdpaF32xParams p{};
    p.rows = (int)((Hq / Hkv) * Tq); p.Tq = (int)Tq; p.Tk = (int)Tk; p.d = (int)d;
    p.scale = scale;
    p.mask = (const float*)mask;
    p.mask_vec = (Tk % 2 == 0) && ((uintptr_t)mask & 7) == 0;
    p.out = (float*)out;
    const float* fq = (const float*)q; const float* fk = (const float*)k; const float* fv = (const float*)v;
    __nv_bfloat16* pl = (__nv_bfloat16*)planes;
    cudaStream_t st = (cudaStream_t)stream;
    if (d <= 48) return sdpa_f32x_launch<1, 64, 3, 2>(fq, fk, fv, p, Hkv, pl, st);
    if (d <= 64) return sdpa_f32x_launch<1, 64, 4, 2>(fq, fk, fv, p, Hkv, pl, st);
    if (d <= 80) return sdpa_f32x_launch<2, 32, 5, 2>(fq, fk, fv, p, Hkv, pl, st);
    return sdpa_f32x_launch<2, 32, 8, 2>(fq, fk, fv, p, Hkv, pl, st);
}
