// gemm_wgmma.cu -- the tensor-core path for fp16 MatMul / Gemm / Conv / attention GEMMs on sm_90a.
//
// One persistent, warp-specialised kernel, 384 threads:
//   warpgroup 0      TMA producer: one warp issues cp.async.bulk.tensor tiles of A and B into 128B-swizzled shared memory, mbarrier-tracked
//   warpgroups 1, 2  consumers: each issues wgmma (m64n128k16, fp32 accumulators in registers) for 64 rows of the 128 x 128 tile, then
//                    runs the epilogue from its registers: add bias / residual, round to fp16, store
// Shared memory holds a STAGES-deep ring of (A,B) k-blocks, so the producer is already fetching the next tile while the consumers run
// the epilogue of this one.
//
// CTA pairs (PAIR): a cluster of two CTAs computes two vertically adjacent 128 x 128 tiles that share their B tile.  Each CTA fetches
// its own A and HALF of the B k-block, multicast by TMA into both CTAs' shared memory, so the L2 -> SM traffic for B halves; a slot
// of the ring is refilled once the consumers of BOTH CTAs have released it (they arrive on the local and on the peer's barrier).
//
// A is always K-major ([M,K] activations).  B is either MN-major ([K,N] row-major: ONNX MatMul weights, the
// pre-transposed K of the attention pattern, V) or K-major ([N,K] row-major: OHWI conv weights).  A convolution is the
// same kernel with the A tiles fetched as 3-D boxes of the NHWC input -- one box per filter tap and 64-channel block,
// out-of-bounds (padding) elements zero-filled by TMA -- i.e. an implicit GEMM with no im2col buffer.
//
// Replaces: XnnPack::matrix_multiply / matrix_multiply_dynamic / convolution for T = uint16_t
// (src/onnxstream.cpp:929-1215, 1292-1534) and the cuBLAS offload CublasOps::OpFullyConnected::run (src/onnxstream.cpp:308-352).

#include "common.cuh"
#include "workspace.h"
#include "tc_ptx.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <vector>

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 128;
constexpr int BLOCK_K = 64;            // 64 fp16 = 128 bytes = one swizzle row
constexpr int WG_K = 16;
constexpr int STAGES = 6;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KiB
constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;  // 16 KiB
constexpr int SMEM_BYTES = STAGES * (A_STAGE_BYTES + B_STAGE_BYTES) + 1024 /*align slack*/ + 256 /*barriers*/ + 2 * tcptx::GN_MAX_GROUPS * 4;
constexpr int NUM_THREADS = 384;        // producer warpgroup + two consumer warpgroups
constexpr int CONSUMER_THREADS = 256;

struct TcParams {
    int M, N, K;                 // GEMM view of the problem (conv: M = Ho*Wo, K = Cin per tap)
    int batch;
    int m_tiles, n_tiles;
    int b_kmajor;                // 1: B is [N,K] row-major
    int a_swap, b_swap;          // tensor map has (batch, row) order swapped because the batch stride is the smaller one (per-head views)
    // conv geometry (taps == 1 for a plain GEMM)
    int taps, kw, pad_top, pad_left, Wo, Ho, bw, bh, tiles_x;
    int k_blocks_per_tap;
    int stride;                  // conv stride (TMA traversal stride on W and H)
    int split_k;                 // > 1: each tile's k-blocks are divided among split_k CTAs, fp32 partials go to `ws`
    float* ws;                   // split-K workspace [split][batch][M][N] fp32
    // grouped launch (groups > 1): `batch` problems share A and the shape; problem g has its own B map (map_b, map_b1, map_b2) and output
    int groups;
    __half* C1;
    __half* C2;
    // output
    __half* C;
    const __half* bias;
    const __half* bias2;         // second per-column addend (the time-embedding row a resnet adds to conv1's output), or null
    const __half* residual;
    double* gn_stats;            // != null: per-group (sum, sum of squares) of the stored output, for the GroupNorm that consumes it
    int gn_cpg, gn_groups;       // channels per group, number of groups (N == gn_cpg * gn_groups)
    int gn_debug;                // bisecting aid (OSB_GN_DEBUG): 1 = skip the per-column gathering, 2 = skip the per-tile flush, 3 = both
    int bf16;                    // operands are bfloat16 (the fp32 path: bf16 triple-split operands, see osb_tc_gemm_f32x)
    int f32_out;                 // raw fp32 accumulators go to `ws` even when split_k == 1; the reduce kernel writes fp32 C (+ fp32 bias / residual)
    long long stride_c;          // elements between batches
    long long ldc;               // elements between output rows (== N for a dense C)
};

using namespace tcptx;

// one k-block (64 elements of K) of a consumer warpgroup: 4 x m64n128k16
template <int B_MN_MAJOR, bool BF16>
__device__ __forceinline__ void mma_kblock(float (&acc)[64], uint64_t adesc, uint64_t bdesc)
{
    constexpr uint32_t b_kstep = B_MN_MAJOR ? (WG_K * 128) >> 4 : (WG_K * 2) >> 4;   // descriptor address units (16 B)
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / WG_K; k++) {
        const uint64_t a = adesc + (uint64_t)(k * ((WG_K * 2) >> 4)), b = bdesc + (uint64_t)(k * b_kstep);
        if (BF16) wgmma_m64n128k16_bf16<B_MN_MAJOR>(acc, a, b, 1u);
        else wgmma_m64n128k16_f16<B_MN_MAJOR>(acc, a, b, 1u);
    }
    wgmma_commit();
}

// ---- the kernel -----------------------------------------------------------------------------------------------

// EXTRAS = the epilogue also adds `bias2` and gathers GroupNorm statistics.  A separate instantiation, so the common launches do not
// carry the extra registers and code.  B_MN_MAJOR (== !p.b_kmajor) and BF16 (== p.bf16) are compile-time: the MMA loop has no branches.
// PAIR = launched as clusters of two CTAs (see the top of the file); split_k == 1 and groups == 1 there.
template <bool EXTRAS, int B_MN_MAJOR, bool BF16, bool PAIR>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const __grid_constant__ CUtensorMap map_b1,
               const __grid_constant__ CUtensorMap map_b2, const TcParams p)
{
    osb_pdl_trigger_entry();   // let the next kernel's CTAs be scheduled as ours drain; it waits for our completion before touching memory
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the 128B swizzle atoms
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
    uint64_t* bars = (uint64_t*)(smem + STAGES * (A_STAGE_BYTES + B_STAGE_BYTES));
    uint64_t* full = bars;                       // [STAGES]
    uint64_t* empty = bars + STAGES;             // [STAGES]
    float* gn_acc = (float*)((uint8_t*)bars + 256);         // [2 * GN_MAX_GROUPS] per-CTA (sum, sum of squares) accumulators

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (EXTRAS && p.gn_stats && threadIdx.x < 2 * GN_MAX_GROUPS) gn_acc[threadIdx.x] = 0.f;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
    }
    // a stage is released by every consumer thread, or (PAIR) by one lane per consumer warp of both CTAs
    constexpr uint32_t EMPTY_ARRIVALS = PAIR ? 2 * (CONSUMER_THREADS / 32) : CONSUMER_THREADS;
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < STAGES; i++) { mbar_init(&full[i], 1); mbar_init(&empty[i], EMPTY_ARRIVALS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (PAIR) cluster_sync();    // the peer multicasts into our ring and arrives on our barriers: both must be initialised
    else __syncthreads();
    osb_pdl_wait();      // everything above (barrier init, descriptor prefetch) overlapped the previous kernel's tail

    // PAIR: the unit of work is a pair of m-tiles (rank r of the cluster takes m-tile 2 * unit + r), walked by cluster
    const uint32_t rank = PAIR ? cluster_ctarank() : 0;
    const int first = PAIR ? (int)cluster_id_x() : (int)blockIdx.x, step = PAIR ? (int)cluster_count_x() : (int)gridDim.x;
    const int m_units = PAIR ? (p.m_tiles + 1) / 2 : p.m_tiles;
    const int tiles_per_batch = m_units * p.n_tiles;
    const int total_tiles = tiles_per_batch * p.batch * p.split_k;
    const int k_blocks_all = p.taps * p.k_blocks_per_tap;
    const int kb_per_split = (k_blocks_all + p.split_k - 1) / p.split_k;   // host guarantees (split_k - 1) * kb_per_split < k_blocks_all

    if (warp == 0) {
        // ===================== TMA producer (warp-uniform control flow, leader-predicated issue) =====================
        const uint32_t sa0 = smem_u32(smem_a), sb0 = smem_u32(smem_b);
        int stage = 0; uint32_t phase = 0;
        for (int tile = first; tile < total_tiles; tile += step) {
            int sp = tile % p.split_k, t2 = tile / p.split_k;
            int b = t2 / tiles_per_batch, r = t2 % tiles_per_batch;
            int mt = r % m_units, nt = r / m_units;
            if (PAIR) mt = 2 * mt + (int)rank;
            int n0 = nt * BLOCK_N;
            int y0 = 0, x0 = 0, m0 = mt * BLOCK_M;
            if (p.taps > 1 || p.bh > 0) { y0 = (mt / p.tiles_x) * p.bh; x0 = (mt % p.tiles_x) * p.bw; }
            // grouped launch: the batch index selects the B map; every operand is addressed at batch coordinate 0
            const CUtensorMap* mbp = &map_b;
            if (p.groups > 1) { if (b == 1) mbp = &map_b1; else if (b == 2) mbp = &map_b2; b = 0; }
            int kb_lo = sp * kb_per_split, kb_hi = min(kb_lo + kb_per_split, k_blocks_all);
            // (tap, channel block) walk incrementally: no divisions inside the k loop
            int tap = kb_lo / p.k_blocks_per_tap, kcb = kb_lo % p.k_blocks_per_tap;
            int ky = tap / p.kw, kx = tap % p.kw;
            const int ax = x0 * p.stride - p.pad_left, ay = y0 * p.stride - p.pad_top;
            for (int kb = kb_lo; kb < kb_hi; kb++) {
                mbar_wait(&empty[stage], phase ^ 1);
                if (elect_one()) {
                    // every box is complete in shared memory (TMA zero-fills and counts out-of-bounds elements)
                    mbar_expect_tx(&full[stage], A_STAGE_BYTES + B_STAGE_BYTES);
                    const int kc = kcb * BLOCK_K;
                    const uint32_t sa = sa0 + stage * A_STAGE_BYTES;
                    const uint32_t sb = sb0 + stage * B_STAGE_BYTES;
                    if (p.bh > 0) tma_load_3d_s(sa, &map_a, &full[stage], kc, ax + kx, ay + ky);
                    else if (p.a_swap) tma_load_3d_s(sa, &map_a, &full[stage], kc, b, m0);
                    else tma_load_3d_s(sa, &map_a, &full[stage], kc, m0, b);
                    const int kglob = tap * p.K + kc;   // K index into B (conv: taps are concatenated along K)
                    if (PAIR) {
                        // this CTA's half of B (K-major: 64 of the 128 rows; MN-major: one of the two 64-column atoms), into both CTAs
                        const uint32_t sbh = sb + rank * (B_STAGE_BYTES / 2);
                        const int nh = n0 + 64 * (int)rank;
                        if (p.b_kmajor) {
                            if (p.b_swap) tma_load_3d_mc(sbh, mbp, &full[stage], kglob, b, nh, 0x3);
                            else tma_load_3d_mc(sbh, mbp, &full[stage], kglob, nh, b, 0x3);
                        } else {
                            if (p.b_swap) tma_load_3d_mc(sbh, mbp, &full[stage], nh, b, kglob, 0x3);
                            else tma_load_3d_mc(sbh, mbp, &full[stage], nh, kglob, b, 0x3);
                        }
                    } else if (p.b_kmajor) {
                        if (p.b_swap) tma_load_3d_s(sb, mbp, &full[stage], kglob, b, n0);
                        else tma_load_3d_s(sb, mbp, &full[stage], kglob, n0, b);
                    } else {
                        // two 64-column atoms of 64 k-rows each
                        if (p.b_swap) {
                            tma_load_3d_s(sb, mbp, &full[stage], n0, b, kglob);
                            tma_load_3d_s(sb + B_STAGE_BYTES / 2, mbp, &full[stage], n0 + 64, b, kglob);
                        } else {
                            tma_load_3d_s(sb, mbp, &full[stage], n0, kglob, b);
                            tma_load_3d_s(sb + B_STAGE_BYTES / 2, mbp, &full[stage], n0 + 64, kglob, b);
                        }
                    }
                }
                __syncwarp();
                if (++kcb == p.k_blocks_per_tap) { kcb = 0; tap++; if (++kx == p.kw) { kx = 0; ky++; } }
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
        osb_pdl_trigger_late();   // every load of this CTA is issued: the next kernel may start its prologue on SMs that drain
    } else if (warp >= 4) {
        // ===================== consumers: MMA + epilogue (warpgroups 1 and 2) =====================
        const int wg = (warp >> 2) - 1;          // rows [64 wg, 64 wg + 64) of the tile
        const int ct = (int)threadIdx.x - (NUM_THREADS - CONSUMER_THREADS);
        // Descriptor templates: everything but the 14-bit start address is loop-invariant.
        //   A, K-major SW128: 8-row groups 1024 B apart; K advances 32 B inside the swizzle row; warpgroup wg starts 64 rows (8 KiB) in.
        //   B, K-major: same.  B, MN-major SW128: two 64-column atoms 8192 B apart (LBO), 8-row k-groups 1024 B apart (SBO);
        //   K advances 16 rows = 2048 B.
        const uint64_t adesc0 = make_smem_desc(smem_u32(smem_a) + wg * (BLOCK_M / 2) * 128, 16, 1024);
        const uint64_t bdesc0 = p.b_kmajor ? make_smem_desc(smem_u32(smem_b), 16, 1024) : make_smem_desc(smem_u32(smem_b), B_STAGE_BYTES / 2, 1024);
        const bool partial = p.split_k > 1 || p.f32_out;
        const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows of the tile: r_lo and r_lo + 8
        const int cq = 2 * (lane & 3);                               // and its column pair inside every 8-column block
        auto release = [&](int s) {
            if (PAIR) {
                __syncwarp();
                if (lane == 0) { mbar_arrive(&empty[s]); mbar_arrive_remote(&empty[s], rank ^ 1u); }
            } else {
                mbar_arrive(&empty[s]);
            }
        };
        int stage = 0; uint32_t phase = 0;
        for (int tile = first; tile < total_tiles; tile += step) {
            int sp = tile % p.split_k, t2 = tile / p.split_k;
            int b = t2 / tiles_per_batch, r = t2 % tiles_per_batch;
            int mt = r % m_units, nt = r / m_units;
            if (PAIR) mt = 2 * mt + (int)rank;      // past the last m-tile (odd count): no row is stored, the CTA still feeds its peer
            const int n0 = nt * BLOCK_N;
            const int n_end = min(p.N, n0 + BLOCK_N);
            const int kb_lo = sp * kb_per_split, kb_hi = min(kb_lo + kb_per_split, k_blocks_all);

            float acc[64];
#pragma unroll
            for (int i = 0; i < 64; i++) acc[i] = 0.f;
            // one k-block of MMAs stays in flight: the stage of k-block kb-1 is released once the MMAs of kb are issued
            int prev = -1;
            for (int kb = kb_lo; kb < kb_hi; kb++) {
                mbar_wait(&full[stage], phase);
                mma_kblock<B_MN_MAJOR, BF16>(acc, adesc0 + (uint64_t)(stage * (A_STAGE_BYTES >> 4)), bdesc0 + (uint64_t)(stage * (B_STAGE_BYTES >> 4)));
                if (prev >= 0) { wgmma_wait<1>(); release(prev); }
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            release(prev);

            // ---- epilogue ----
            long long out_row[2];   // row index into C (conv: output pixel index)
            bool row_ok[2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int row_in_tile = r_lo + 8 * h;
                if (p.bh > 0) {
                    int y = (mt / p.tiles_x) * p.bh + row_in_tile / p.bw, x = (mt % p.tiles_x) * p.bw + row_in_tile % p.bw;
                    row_ok[h] = y < p.Ho && x < p.Wo;
                    out_row[h] = (long long)y * p.Wo + x;
                } else {
                    int m = mt * BLOCK_M + row_in_tile;
                    row_ok[h] = m < p.M;
                    out_row[h] = m;
                }
            }
            __half* cbase = p.C;
            if (p.groups > 1) cbase = b == 0 ? p.C : (b == 1 ? p.C1 : p.C2);    // stride_c == 0 in a grouped launch
            const bool pair_ok = (p.N & 1) == 0 && (p.ldc & 1) == 0;           // two adjacent columns move as one 4- / 8-byte vector
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; j++) {
                if (n0 + 8 * j >= n_end) break;     // warp-uniform
                const int n = n0 + 8 * j + cq;
                const bool ok0 = n < n_end, ok1 = n + 1 < n_end;
                float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;   // GroupNorm statistics of the two columns
                float add0 = 0.f, add1 = 0.f;                   // per-column addends: bias (+ bias2)
                if (!partial) {
                    if (p.bias) { if (ok0) add0 += __half2float(p.bias[n]); if (ok1) add1 += __half2float(p.bias[n + 1]); }
                }
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    if (!row_ok[h]) continue;
                    float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
                    if (partial) {
                        // split-K / fp32 output: raw fp32 partials, reduced (with bias / residual) by the reduce kernel
                        float* wrow = p.ws + (((long long)sp * p.batch + b) * p.M + out_row[h]) * p.N;
                        if (ok1 && pair_ok) *reinterpret_cast<float2*>(wrow + n) = make_float2(f0, f1);
                        else { if (ok0) wrow[n] = f0; if (ok1) wrow[n + 1] = f1; }
                        continue;
                    }
                    const long long off = (long long)b * p.stride_c + out_row[h] * p.ldc;
                    f0 += add0; f1 += add1;
                    if (p.residual) { if (ok0) f0 += __half2float(p.residual[off + n]); if (ok1) f1 += __half2float(p.residual[off + n + 1]); }
                    if (EXTRAS && p.bias2) { if (ok0) f0 += __half2float(p.bias2[n]); if (ok1) f1 += __half2float(p.bias2[n + 1]); }
                    const __half o0 = __float2half_rn(f0), o1 = __float2half_rn(f1);
                    __half* crow = cbase + off;
                    if (ok1 && pair_ok) *reinterpret_cast<__half2*>(crow + n) = __halves2half2(o0, o1);
                    else { if (ok0) crow[n] = o0; if (ok1) crow[n + 1] = o1; }
                    if (EXTRAS) {
                        // the statistics see the values as they are stored
                        const float g0 = ok0 ? __half2float(o0) : 0.f, g1 = ok1 ? __half2float(o1) : 0.f;
                        s0 += g0; q0 = fmaf(g0, g0, q0); s1 += g1; q1 = fmaf(g1, g1, q1);
                    }
                }
                if (EXTRAS && p.gn_stats && !partial && !(p.gn_debug & 1)) gn_stats_pair(s0, s1, q0, q1, n, n_end, p.gn_cpg, gn_acc, lane);
            }
            if (EXTRAS && p.gn_stats && !partial && !(p.gn_debug & 2)) {
                asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_THREADS) : "memory");
                gn_stats_flush(gn_acc, p.gn_stats, p.gn_groups, ct);
            }
        }
    }
    if (PAIR) cluster_sync();    // no CTA leaves while its peer may still multicast into it or arrive on its barriers
}

// split-K second pass: out[row][n] = fp16(sum_s ws[s][row][n] + bias[n] + bias2[n] + residual[row][n]); rows = batch * M.
// Optionally gathers the GroupNorm statistics of the result (per-block shared accumulators -> global fp64).
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, __half* __restrict__ out, const __half* __restrict__ bias, const __half* __restrict__ bias2,
                                     const __half* __restrict__ residual, long long rows, int N, int splits, double* __restrict__ gn_stats, int gn_cpg, int gn_groups)
{
    osb_pdl_prologue();
    __shared__ float acc[2 * GN_MAX_GROUPS];
    if (gn_stats) { if (threadIdx.x < 2 * GN_MAX_GROUPS) acc[threadIdx.x] = 0.f; __syncthreads(); }
    // N % 4 == 0: one float4 of every split plane per thread, fully coalesced
    const long long total4 = rows * N / 4;
    const long long plane4 = total4;
    const float4* w4 = reinterpret_cast<const float4*>(ws);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
        float4 a = w4[i];
        for (int s = 1; s < splits; s++) { float4 t = w4[(long long)s * plane4 + i]; a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w; }
        long long e = i * 4;
        int n = (int)(e % N);
        if (bias) { a.x += __half2float(bias[n]); a.y += __half2float(bias[n + 1]); a.z += __half2float(bias[n + 2]); a.w += __half2float(bias[n + 3]); }
        if (bias2) { a.x += __half2float(bias2[n]); a.y += __half2float(bias2[n + 1]); a.z += __half2float(bias2[n + 2]); a.w += __half2float(bias2[n + 3]); }
        if (residual) {
            Vec<__half, 4> r = load_vec<__half, 4>(residual + e);
            a.x += __half2float(r.v[0]); a.y += __half2float(r.v[1]); a.z += __half2float(r.v[2]); a.w += __half2float(r.v[3]);
        }
        Vec<__half, 4> o;
        o.v[0] = __float2half_rn(a.x); o.v[1] = __float2half_rn(a.y); o.v[2] = __float2half_rn(a.z); o.v[3] = __float2half_rn(a.w);
        store_vec<__half, 4>(out + e, o);
        if (gn_stats) {
            // the 4 columns of a thread lie in one group when cpg % 4 == 0 (host guarantees it)
            float x0 = __half2float(o.v[0]), x1 = __half2float(o.v[1]), x2 = __half2float(o.v[2]), x3 = __half2float(o.v[3]);
            const int g = n / gn_cpg;
            atomicAdd(&acc[2 * g], (x0 + x1) + (x2 + x3));
            atomicAdd(&acc[2 * g + 1], fmaf(x0, x0, x1 * x1) + fmaf(x2, x2, x3 * x3));
        }
    }
    if (gn_stats) {
        __syncthreads();
        if (threadIdx.x < 2 * gn_groups) { float v = acc[threadIdx.x]; if (v != 0.f) atomicAdd(&gn_stats[threadIdx.x], (double)v); }
    }
}

// fp32-output variant (the bf16 triple-split path): out[row][n] = sum_s ws[s][row][n] + bias[n] + residual[row][n], everything fp32, any N
__global__ void splitk_reduce_f32_kernel(const float* __restrict__ ws, float* __restrict__ out, const float* __restrict__ bias, const float* __restrict__ residual,
                                         long long rows, int N, int splits)
{
    osb_pdl_prologue();
    const long long total = rows * N;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        float a = ws[i];
        for (int s = 1; s < splits; s++) a += ws[(long long)s * total + i];
        if (bias) a += bias[(int)(i % N)];
        if (residual) a += residual[i];
        out[i] = a;
    }
}

#include "gemm_i8.cuh"

// ---- host side -------------------------------------------------------------------------------------------------
constexpr size_t WS_MAX = OSB_WS_SPLITK_BYTES;   // fixed-capacity per-stream workspace (workspace.h): never re-allocated, graph-safe

int num_sms();

// pick a split factor: fill the SMs when the tile count is small, keep >= 2 k-blocks per split, stay inside the workspace
int choose_split(int tiles, int k_blocks, size_t out_elems, cudaStream_t st, OsbWorkspace** ws_out)
{
    static const int forced = [] { const char* e = getenv("OSB_TC_SPLIT"); return e ? atoi(e) : 0; }();   // tuning experiments only
    // over the tensor-core shapes of the SD 1.5 UNet: below ~32 k-blocks the second launch (the reduce) costs more
    // than the idle SMs do
    *ws_out = nullptr;
    static const int min_kb = [] { const char* e = getenv("OSB_TC_SPLIT_MINKB"); int v = e ? atoi(e) : 0; return v > 0 ? v : 32; }();
    if ((tiles >= 100 && forced <= 0) || k_blocks < 4 || (k_blocks < min_kb && forced <= 0)) return 1;
    int split = forced > 0 ? forced : num_sms() / tiles;
    split = std::min(split, k_blocks / 2);
    while (split > 1 && (size_t)split * out_elems * 4 > WS_MAX) split--;
    if (split <= 1) return 1;
    int kb_per = (k_blocks + split - 1) / split;
    split = (k_blocks + kb_per - 1) / kb_per;          // no empty splits: every CTA must run at least one k-block
    if (split <= 1) return 1;
    OsbWorkspace* ws = osb_workspace(st, OSB_WS_SPLITK);
    if (!ws) return 1;                                  // capturing before any eager run, or out of memory: run unsplit
    *ws_out = ws;
    return split;
}

PFN_cuTensorMapEncodeTiled_v12000 get_encode()
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

// rank-3 fp16 tensor map with 128B swizzle; dims/strides innermost first
bool make_map(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1_bytes, uint64_t s2_bytes,
              uint32_t b0, uint32_t b1, uint32_t b2, uint32_t traversal_stride = 1, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16)
{
    auto enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[3] = { d0, d1, d2 };
    cuuint64_t strides[2] = { s1_bytes, s2_bytes };
    cuuint32_t box[3] = { b0, b1, b2 };
    cuuint32_t estr[3] = { 1, traversal_stride, traversal_stride };   // strided conv: every s-th pixel of the box span
    CUresult r = enc(map, dtype, 3, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// rank-3 map over (inner, row, batch) that keeps the global strides ascending: when the batch stride is the smaller one
// (per-head slices of a [T, heads*d] buffer) the two outer dimensions are swapped and *swapped is set.
bool make_map_rb(CUtensorMap* map, const void* base, uint64_t inner, uint64_t rows, uint64_t batch, uint64_t row_stride_bytes, uint64_t batch_stride_bytes,
                 uint32_t box_inner, uint32_t box_rows, int* swapped)
{
    if (batch > 1 && batch_stride_bytes < row_stride_bytes) {
        *swapped = 1;
        return make_map(map, base, inner, batch, rows, batch_stride_bytes, row_stride_bytes, box_inner, 1, box_rows);
    }
    *swapped = 0;
    return make_map(map, base, inner, rows, batch, row_stride_bytes, batch_stride_bytes, box_inner, box_rows, 1);
}

int num_sms()
{
    static int n = 0;
    if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); if (n <= 0) n = 132; }
    return n;
}

// optional per-launch timing (bench.py's roofline leg): CUDA events on the launching stream around every launch
struct ProfRec { cudaEvent_t a, b; double flops, bytes; int M, N, K, taps, batch, split, conv; };
bool g_prof = false;
std::vector<ProfRec> g_prof_list;

void prof_begin(ProfRec& rec, const TcParams& p, cudaStream_t st)
{
    cudaEventCreate(&rec.a); cudaEventCreate(&rec.b);
    // the fp32 path (bf16 triple split) runs a 6x longer K: ALGORITHMIC work is the fp32 problem's (K / 6, 4-byte elements)
    const double kdiv = p.bf16 ? 6.0 : 1.0, es = p.bf16 ? 4.0 : 2.0;
    double M = p.M, N = p.N, Kt = (double)p.K * p.taps / kdiv, B = p.batch;
    rec.flops = 2.0 * M * N * Kt * B;
    // algorithmic bytes: A once (conv: the input image once), B once, C once (+ residual / bias reads)
    double a_bytes = (p.bh > 0 ? M * (p.K / kdiv) : M * Kt) * es * B;
    rec.bytes = a_bytes + N * Kt * es * (p.bh > 0 ? 1.0 : B) + M * N * es * B * (p.residual ? 2.0 : 1.0) + (p.bias ? N * es : 0.0);
    rec.M = p.M; rec.N = p.N; rec.K = p.K; rec.taps = p.taps; rec.batch = p.batch; rec.split = p.split_k; rec.conv = p.bh > 0;
    cudaEventRecord(rec.a, st);
}

using TcKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, TcParams);

// pair: clusters of two CTAs sharing B (the B map's box covers half a tile: 64 rows K-major, one 64-column atom MN-major)
int launch(const CUtensorMap& ma, const CUtensorMap& mb, const TcParams& p, cudaStream_t st, const CUtensorMap* mb1p = nullptr, const CUtensorMap* mb2p = nullptr,
           bool pair = false)
{
    const CUtensorMap& mb1 = mb1p ? *mb1p : mb;
    const CUtensorMap& mb2 = mb2p ? *mb2p : mb;
    static bool attr_set = false;
    if (!attr_set) {
        TcKernel kernels[] = {
            tc_gemm_kernel<false, 0, false, false>, tc_gemm_kernel<false, 1, false, false>, tc_gemm_kernel<true, 0, false, false>, tc_gemm_kernel<true, 1, false, false>,
            tc_gemm_kernel<false, 0, true, false>, tc_gemm_kernel<false, 1, true, false>,
            tc_gemm_kernel<false, 0, false, true>, tc_gemm_kernel<false, 1, false, true>, tc_gemm_kernel<true, 0, false, true>, tc_gemm_kernel<true, 1, false, true> };
        for (auto k : kernels) {
            cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
            if (e != cudaSuccess) return (int)e;
        }
        attr_set = true;
    }
    const bool extras = p.bias2 != nullptr || p.gn_stats != nullptr;
    TcKernel k;
    if (pair) {
        if (p.bf16 || p.split_k != 1 || p.groups > 1) return (int)cudaErrorInvalidValue;
        k = extras ? (p.b_kmajor ? tc_gemm_kernel<true, 0, false, true> : tc_gemm_kernel<true, 1, false, true>)
                   : (p.b_kmajor ? tc_gemm_kernel<false, 0, false, true> : tc_gemm_kernel<false, 1, false, true>);
    } else if (p.bf16) {   // the fp32 path: no bias2 / statistics
        k = p.b_kmajor ? tc_gemm_kernel<false, 0, true, false> : tc_gemm_kernel<false, 1, true, false>;
    } else if (extras) {
        k = p.b_kmajor ? tc_gemm_kernel<true, 0, false, false> : tc_gemm_kernel<true, 1, false, false>;
    } else {
        k = p.b_kmajor ? tc_gemm_kernel<false, 0, false, false> : tc_gemm_kernel<false, 1, false, false>;
    }
    int grid;
    if (pair) {
        // a persistent grid must be co-resident: clusters need both SMs in one GPC, so fewer than num_sms / 2 of them may fit at once
        static int max_clusters = 0;
        if (!max_clusters) {
            cudaLaunchConfig_t cfg{};
            cfg.gridDim = dim3(2 * (num_sms() / 2)); cfg.blockDim = dim3(NUM_THREADS); cfg.dynamicSmemBytes = SMEM_BYTES;
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
            cfg.attrs = attr; cfg.numAttrs = 1;
            int n = 0;
            if (cudaOccupancyMaxActiveClusters(&n, k, &cfg) != cudaSuccess || n <= 0) { cudaGetLastError(); n = num_sms() / 2; }
            max_clusters = std::min(n, num_sms() / 2);
        }
        const int units = (p.m_tiles + 1) / 2 * p.n_tiles * p.batch;
        grid = 2 * std::min(units, max_clusters);
    } else {
        grid = std::min(p.m_tiles * p.n_tiles * p.batch * p.split_k, num_sms());
    }
    ProfRec rec{};
    if (g_prof) prof_begin(rec, p, st);
    osb_launch_cluster(k, grid, NUM_THREADS, (size_t)SMEM_BYTES, st, pair ? 2u : 1u, ma, mb, mb1, mb2, p);
    if (p.f32_out) {
        launched(1);
        const long long total = (long long)p.batch * p.M * p.N;
        int rgrid = (int)std::min<long long>((total + 255) / 256, num_sms() * 8);
        osb_launch((splitk_reduce_f32_kernel), rgrid, 256, 0, st, (const float*)p.ws, (float*)p.C, (const float*)p.bias, (const float*)p.residual, (long long)p.batch * p.M, p.N, p.split_k);
        if (g_prof) { cudaEventRecord(rec.b, st); g_prof_list.push_back(rec); }
        return launched(0);
    }
    if (p.split_k > 1) {
        launched(1);
        long long total4 = (long long)p.batch * p.M * p.N / 4;
        int rgrid = (int)std::min<long long>((total4 + 255) / 256, num_sms() * 8);
        osb_launch((splitk_reduce_kernel), rgrid, 256, 0, st, (const float*)p.ws, p.C, p.bias, p.bias2, p.residual, (long long)p.batch * p.M, p.N, p.split_k,
                   p.gn_stats, p.gn_cpg, p.gn_groups);
        if (g_prof) { cudaEventRecord(rec.b, st); g_prof_list.push_back(rec); }
        return launched(0);
    }
    if (g_prof) { cudaEventRecord(rec.b, st); g_prof_list.push_back(rec); }
    return launched(1);
}

int env_int(const char* name)
{
    const char* e = getenv(name);
    return e ? atoi(e) : 0;
}

inline uint32_t next_pow2(uint32_t v) { uint32_t r = 1; while (r < v) r <<= 1; return r; }

// ---- CTA pairs: when to use them ------------------------------------------------------------------------------------
// 0: single CTAs only, 1: the default rule below, 2: pairs wherever eligible (tests / A-B runs); OSB_TC_PAIR sets the start value
int g_pair_mode = -1;
int pair_mode()
{
    if (g_pair_mode < 0) { const char* e = getenv("OSB_TC_PAIR"); g_pair_mode = e ? atoi(e) : 1; }
    return g_pair_mode;
}

// Pairs halve the B bytes each CTA pulls through L2 per k-block.  On the H100 they measured slower than single tiles on every shape
// tried (GEMMs up to 8192^3, the SD 1.5 UNet and VAE convs: 1.6-2.2x the time), so the default rule takes single tiles; the pair
// path is kept, tested, for tuning (DESIGN.md section 7).
bool use_pair(int64_t m_tiles, int64_t N)
{
    return pair_mode() == 2 && m_tiles >= 2 && N % 8 == 0;
}

}  // namespace

extern "C" void osb_tc_set_pair_mode(int mode) { g_pair_mode = mode; }

extern "C" void osb_tc_profile(int enable)
{
    for (auto& r : g_prof_list) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    g_prof_list.clear();
    g_prof = enable != 0;
}

// Sums over the launches recorded since osb_tc_profile(1): out = { launches, total ms, total flops, total algorithmic bytes }
extern "C" int osb_tc_profile_read(double* out4)
{
    double ms = 0, fl = 0, by = 0;
    for (auto& r : g_prof_list) {
        if (cudaEventSynchronize(r.b) != cudaSuccess) return -1;
        float t = 0.f;
        if (cudaEventElapsedTime(&t, r.a, r.b) != cudaSuccess) return -1;
        ms += t; fl += r.flops; by += r.bytes;
    }
    out4[0] = (double)g_prof_list.size(); out4[1] = ms; out4[2] = fl; out4[3] = by;
    return 0;
}

// One text line per recorded launch: "M N K taps batch split conv ms gflop"
extern "C" int osb_tc_profile_dump(char* buf, int cap)
{
    int off = 0;
    for (auto& r : g_prof_list) {
        float t = 0.f;
        if (cudaEventSynchronize(r.b) != cudaSuccess || cudaEventElapsedTime(&t, r.a, r.b) != cudaSuccess) return -1;
        int n = snprintf(buf + off, cap - off, "%d %d %d %d %d %d %d %.4f %.3f\n", r.M, r.N, r.K, r.taps, r.batch, r.split, r.conv, t, r.flops * 1e-9);
        if (n < 0 || off + n >= cap) break;
        off += n;
    }
    return off;
}


// ---- W8A8 (kind::i8) entry points ------------------------------------------------------------------------------------
// TMA needs 16-byte global strides: K % 16 (K-major operands), N % 16 (MN-major weights and the 16-byte output vectors)
extern "C" int osb_qu8_tc_gemm_ok(int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C)
{
    if (M < 32 || N < 16 || K < 16 || (N % 16) || (K % 16)) return 0;
    if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)C) & 15) return 0;
    static const int off = env_int("OSB_QU8_TC_OFF");
    return get_encode() != nullptr && !off;
}

extern "C" int osb_qu8_tc_conv_ok(int64_t Cin, int64_t Cout, int64_t Ho, int64_t Wo, int kh, int kw, int stride, const void* x, const void* w, const void* y)
{
    if ((Cin % 16) || (Cout % 16) || Ho * Wo < 64 || kh > 7 || kw > 7 || stride < 1 || stride > 2) return 0;
    if (((uintptr_t)x | (uintptr_t)w | (uintptr_t)y) & 15) return 0;
    static const int off = env_int("OSB_QU8_TC_OFF");
    return get_encode() != nullptr && !off;
}

extern "C" int osb_rowsum_u8(const void* x, void* out, int64_t rows, int64_t cols, void* stream)
{
    if (rows * cols == 0) return 0;
    osb_launch((i8k::rowsum_u8_kernel), (unsigned)std::min<int64_t>((rows + 7) / 8, num_sms() * 8), 256, 0, (cudaStream_t)stream, (const uint8_t*)x, (int32_t*)out, (long long)rows, (long long)cols);
    return launched();
}

extern "C" int osb_colsum_u8(const void* w, void* out, int64_t K, int64_t N, void* stream)
{
    if (K * N == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(out, 0, (size_t)N * 4, st);
    if (e != cudaSuccess) return (int)e;
    const int64_t gx = (N + 255) / 256;
    const int64_t gy = std::max<int64_t>(1, std::min<int64_t>((K + 63) / 64, (num_sms() * 4 + gx - 1) / gx));
    const int64_t k_per = (K + gy - 1) / gy;
    osb_launch((i8k::colsum_u8_kernel), dim3((unsigned)gx, (unsigned)((K + k_per - 1) / k_per)), 256, 0, st, (const uint8_t*)w, (int32_t*)out, (long long)K, (long long)N, (long long)k_per);
    return launched();
}

extern "C" int osb_pad_sum_u8(const void* x, void* xp, void* psum, int64_t H, int64_t W, int64_t C, int64_t Hp, int64_t Wp, int pad_top, int pad_left, int zx, void* stream)
{
    if (Hp * Wp * C == 0) return 0;
    if (C % 16) return (int)cudaErrorInvalidValue;
    osb_launch((i8k::pad_sum_u8_kernel), (unsigned)std::min<int64_t>((Hp * Wp + 7) / 8, num_sms() * 16), 256, 0, (cudaStream_t)stream, (const uint8_t*)x, (uint8_t*)xp, (int32_t*)psum,
               (int)H, (int)W, (int)C, (int)Hp, (int)Wp, pad_top, pad_left, zx);
    return launched();
}

static int launch_i8(const CUtensorMap& ma, const CUtensorMap& mb, const i8k::I8Params& p, cudaStream_t st)
{
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(i8k::tc_i8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, i8k::I8_SMEM);
        if (e != cudaSuccess) return (int)e;
        attr_set = true;
    }
    const int total = p.m_tiles * p.n_tiles;
    osb_launch((i8k::tc_i8_kernel), std::min(total, num_sms()), NUM_THREADS, (size_t)i8k::I8_SMEM, st, ma, mb, p);
    return launched(1);
}

// C[M,N] (uint8) = requant((A - zx) (B - zw) + bias): A [M,K] uint8, B [K,N] (bt = 0, ONNX MatMul) or [N,K] (bt = 1); rsum = rowsum_x[M],
// csum = colsum_w[N] (osb_rowsum_u8 / osb_colsum_u8)
extern "C" int osb_qu8_tc_gemm(const void* A, const void* B, void* C, const void* bias, const void* rsum, const void* csum, int64_t M, int64_t N, int64_t K, int bt,
                               int zx, float sx, int zw, float sw, int zy, float sy, void* stream)
{
    CUtensorMap ma, mb;
    if (!make_map(&ma, A, (uint64_t)K, (uint64_t)M, 1, (uint64_t)K, (uint64_t)M * K, i8k::I8_BLOCK_K, BLOCK_M, 1, 1, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return (int)cudaErrorInvalidValue;
    bool ok = bt ? make_map(&mb, B, (uint64_t)K, (uint64_t)N, 1, (uint64_t)K, (uint64_t)N * K, i8k::I8_BLOCK_K, BLOCK_N, 1, 1, CU_TENSOR_MAP_DATA_TYPE_UINT8)
                 : make_map(&mb, B, (uint64_t)N, (uint64_t)K, 1, (uint64_t)N, (uint64_t)N * K, BLOCK_N, i8k::I8_BLOCK_K, 1, 1, CU_TENSOR_MAP_DATA_TYPE_UINT8);
    if (!ok) return (int)cudaErrorInvalidValue;
    i8k::I8Params p{};
    p.M = (int)M; p.N = (int)N; p.K = (int)K;
    p.m_tiles = (int)((M + BLOCK_M - 1) / BLOCK_M); p.n_tiles = (int)((N + BLOCK_N - 1) / BLOCK_N);
    p.b_kmajor = bt ? 1 : 0;
    p.taps = 1; p.kw = 1; p.bh = 0; p.bw = 0; p.tiles_x = 1; p.stride = 1;
    p.k_blocks_per_tap = (int)((K + i8k::I8_BLOCK_K - 1) / i8k::I8_BLOCK_K);
    p.rsum = (const int32_t*)rsum; p.csum = (const int32_t*)csum; p.bias = (const int32_t*)bias;
    p.zx = zx; p.zw = zw; p.zy = zy; p.kzz = (int)(K * zx * zw); p.requant = sx * sw / sy;
    p.C = (uint8_t*)C; p.ldc = N;
    return launch_i8(ma, mb, p, (cudaStream_t)stream);
}

// y[Ho,Wo,Cout] (uint8): xp = the zero-point-padded NHWC image [Hp,Wp,Cin] with its per-pixel channel sums psum (osb_pad_sum_u8), w = OHWI
extern "C" int osb_qu8_tc_conv(const void* xp, const void* psum, const void* w, const void* bias, const void* csum, void* y, int64_t Hp, int64_t Wp, int64_t Cin, int64_t Cout,
                               int kh, int kw, int stride, int64_t Ho, int64_t Wo, int zx, float sx, int zw, float sw, int zy, float sy, void* stream)
{
    const uint32_t bw = std::min<uint32_t>(128, next_pow2((uint32_t)Wo)), bh = 128 / bw;
    CUtensorMap ma, mb;
    const int64_t Ktot = (int64_t)kh * kw * Cin;
    if (!make_map(&ma, xp, (uint64_t)Cin, (uint64_t)Wp, (uint64_t)Hp, (uint64_t)Cin, (uint64_t)Wp * Cin, i8k::I8_BLOCK_K, bw * stride, bh * stride, (uint32_t)stride, CU_TENSOR_MAP_DATA_TYPE_UINT8))
        return (int)cudaErrorInvalidValue;
    if (!make_map(&mb, w, (uint64_t)Ktot, (uint64_t)Cout, 1, (uint64_t)Ktot, (uint64_t)Ktot * Cout, i8k::I8_BLOCK_K, BLOCK_N, 1, 1, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return (int)cudaErrorInvalidValue;
    i8k::I8Params p{};
    p.M = (int)(Ho * Wo); p.N = (int)Cout; p.K = (int)Cin;
    p.tiles_x = (int)((Wo + bw - 1) / bw);
    p.m_tiles = p.tiles_x * (int)((Ho + bh - 1) / bh);
    p.n_tiles = (int)((Cout + BLOCK_N - 1) / BLOCK_N);
    p.b_kmajor = 1;
    p.taps = kh * kw; p.kw = kw; p.Wo = (int)Wo; p.Ho = (int)Ho; p.bw = (int)bw; p.bh = (int)bh; p.stride = stride; p.Wp = (int)Wp;
    p.k_blocks_per_tap = (int)((Cin + i8k::I8_BLOCK_K - 1) / i8k::I8_BLOCK_K);
    p.rsum = (const int32_t*)psum; p.csum = (const int32_t*)csum; p.bias = (const int32_t*)bias;
    p.zx = zx; p.zw = zw; p.zy = zy; p.kzz = (int)(Ktot * zx * zw); p.requant = sx * sw / sy;
    p.C = (uint8_t*)y; p.ldc = Cout;
    return launch_i8(ma, mb, p, (cudaStream_t)stream);
}

bool osb_tc_gemm_ok(int64_t M, int64_t N, int64_t K, int bt, const void* A, const void* B, const void* C, int64_t sa, int64_t sb, int64_t sc,
                    int64_t lda, int64_t ldb, int64_t ldc)
{
    if ((lda % 8) || (ldb % 8) || (ldc % 8)) return false;
    if (M < 32 || N < 1 || K < 8) return false;
    if (K % 8) return false;
    if (N % 8) return false;   // ragged N only through the conv entry (K-major B, scalar epilogue)
    if (M > (1 << 30) || N > (1 << 30) || K > (1 << 30)) return false;
    if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)C) & 15) return false;
    if ((sa % 8) || (sb % 8) || (sc % 8)) return false;
    (void)bt;
    return get_encode() != nullptr || A == nullptr;
}

// fp32 problems on the tensor cores (osb_tc_gemm_f32x / osb_tc_conv_f32x below): the launch builders run with this flag set -- operands are
// bf16 triple-split expansions, C / bias / residual are fp32, accumulators leave through the fp32 workspace
static thread_local int g_f32x = 0;

// finish a TcParams for the fp32 path; false = the fp32 partial planes do not fit the fixed workspace
static bool f32x_params(TcParams& p, OsbWorkspace* wsp, cudaStream_t st)
{
    p.bf16 = 1; p.f32_out = 1;
    p.bias2 = nullptr; p.gn_stats = nullptr;
    if ((size_t)p.split_k * p.batch * p.M * p.N * 4 > WS_MAX) p.split_k = 1;
    if ((size_t)p.batch * p.M * p.N * 4 > WS_MAX) return false;
    if (!wsp) wsp = osb_workspace(st, OSB_WS_SPLITK);
    if (!wsp) return false;
    p.ws = wsp->splitk;
    return true;
}

int osb_tc_gemm_launch(const void* A, const void* B, void* C, const void* bias, const void* residual, int64_t batch, int64_t M, int64_t N, int64_t K,
                       int64_t sa, int64_t sb, int64_t sc, int bt, cudaStream_t st, int64_t lda, int64_t ldb, int64_t ldc)
{
    if (g_f32x && batch != 1) return (int)cudaErrorNotSupported;
    if (lda <= 0) lda = K;
    if (ldb <= 0) ldb = bt ? K : N;
    if (ldc <= 0) ldc = N;
    CUtensorMap ma, mb;
    // A: [batch][M][K]; a shared operand (stride 0) is presented as batch extent 1 and the batch coordinate ignored
    uint64_t abatch = sa ? (uint64_t)batch : 1, bbatch = sb ? (uint64_t)batch : 1;
    if (batch > 1 && (!sa || !sb)) {
        // shared operands across the batch: fold the batch into per-batch launches (rare: 2-D weights with n > 1)
        for (int64_t i = 0; i < batch; i++) {
            int r = osb_tc_gemm_launch((const __half*)A + i * sa, (const __half*)B + i * sb, (__half*)C + i * sc, bias,
                                       residual ? (const __half*)residual + i * sc : nullptr, 1, M, N, K, M * lda, bt ? N * ldb : K * ldb, sc, bt, st, lda, ldb, ldc);
            if (r) return r;
        }
        return 0;
    }
    int a_swap = 0, b_swap = 0;
    if (!make_map_rb(&ma, A, (uint64_t)K, (uint64_t)M, abatch, (uint64_t)lda * 2, (uint64_t)(sa ? sa : M * lda) * 2, BLOCK_K, BLOCK_M, &a_swap)) return (int)cudaErrorInvalidValue;
    int64_t m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
    const bool pair = !g_f32x && use_pair(m_tiles, N);
    bool okb = bt ? make_map_rb(&mb, B, (uint64_t)K, (uint64_t)N, bbatch, (uint64_t)ldb * 2, (uint64_t)(sb ? sb : N * ldb) * 2, BLOCK_K, pair ? BLOCK_N / 2 : BLOCK_N, &b_swap)
                  : make_map_rb(&mb, B, (uint64_t)N, (uint64_t)K, bbatch, (uint64_t)ldb * 2, (uint64_t)(sb ? sb : K * ldb) * 2, 64, BLOCK_K, &b_swap);
    if (!okb) return (int)cudaErrorInvalidValue;
    TcParams p{};
    p.M = (int)M; p.N = (int)N; p.K = (int)K; p.batch = (int)batch;
    p.m_tiles = (int)m_tiles; p.n_tiles = (int)((N + BLOCK_N - 1) / BLOCK_N);
    p.b_kmajor = bt ? 1 : 0;
    p.a_swap = a_swap; p.b_swap = b_swap;
    p.taps = 1; p.kw = 1; p.bh = 0; p.bw = 0; p.tiles_x = 1;
    p.k_blocks_per_tap = (int)((K + BLOCK_K - 1) / BLOCK_K);
    p.stride = 1;
    p.C = (__half*)C; p.bias = (const __half*)bias; p.residual = (const __half*)residual; p.stride_c = sc; p.ldc = ldc;
    if (pair) { p.split_k = 1; return launch(ma, mb, p, st, nullptr, nullptr, true); }
    OsbWorkspace* wsp = nullptr;
    p.split_k = (ldc == N && (sc == M * N || batch == 1)) ? choose_split(p.m_tiles * p.n_tiles * p.batch, p.k_blocks_per_tap, (size_t)batch * M * N, st, &wsp) : 1;
    p.ws = wsp ? wsp->splitk : nullptr;
    if (g_f32x && !f32x_params(p, wsp, st)) return (int)cudaErrorNotSupported;
    return launch(ma, mb, p, st);
}

// `groups` (2 or 3) GEMMs C_g = A * B_g that share A and the shape, in ONE launch (the q/k/v projections of an attention block):
// three times the tiles per launch, one dependency instead of three.  No bias / residual / split-K.
int osb_tc_gemm_grouped_launch(const void* A, const void* const* B, void* const* C, int groups, int64_t M, int64_t N, int64_t K, int bt, cudaStream_t st,
                               int64_t lda, int64_t ldb, int64_t ldc)
{
    if (groups < 2 || groups > 3) return (int)cudaErrorInvalidValue;
    CUtensorMap ma, mb[3];
    int a_swap = 0, b_swap = 0;
    if (!make_map_rb(&ma, A, (uint64_t)K, (uint64_t)M, 1, (uint64_t)lda * 2, (uint64_t)(M * lda) * 2, BLOCK_K, BLOCK_M, &a_swap)) return (int)cudaErrorInvalidValue;
    int64_t m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
    for (int g = 0; g < groups; g++) {
        int sw = 0;
        bool ok = bt ? make_map_rb(&mb[g], B[g], (uint64_t)K, (uint64_t)N, 1, (uint64_t)ldb * 2, (uint64_t)(N * ldb) * 2, BLOCK_K, BLOCK_N, &sw)
                     : make_map_rb(&mb[g], B[g], (uint64_t)N, (uint64_t)K, 1, (uint64_t)ldb * 2, (uint64_t)(K * ldb) * 2, 64, BLOCK_K, &sw);
        if (!ok || (g > 0 && sw != b_swap)) return (int)cudaErrorInvalidValue;
        b_swap = sw;
    }
    TcParams p{};
    p.M = (int)M; p.N = (int)N; p.K = (int)K; p.batch = groups; p.groups = groups;
    p.m_tiles = (int)m_tiles; p.n_tiles = (int)((N + BLOCK_N - 1) / BLOCK_N);
    p.b_kmajor = bt ? 1 : 0;
    p.a_swap = a_swap; p.b_swap = b_swap;
    p.taps = 1; p.kw = 1; p.bh = 0; p.bw = 0; p.tiles_x = 1;
    p.k_blocks_per_tap = (int)((K + BLOCK_K - 1) / BLOCK_K);
    p.stride = 1;
    p.C = (__half*)C[0]; p.C1 = (__half*)C[1]; p.C2 = (__half*)(groups > 2 ? C[2] : C[1]);
    p.bias = nullptr; p.residual = nullptr; p.stride_c = 0; p.ldc = ldc;
    p.split_k = 1; p.ws = nullptr;
    return launch(ma, mb[0], p, st, &mb[1], groups > 2 ? &mb[2] : &mb[1]);
}

bool osb_tc_conv_ok(int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, const void* x, const void* w, const void* y)
{
    if (stride < 1 || stride > 2) return false;
    if (Cin % 8 || Cin < 16) return false;     // TMA needs 16-byte pixel strides; tiny-Cin stems stay on the CUDA-core kernel
    if (H * W < 64) return false;
    if (kh > 7 || kw > 7) return false;
    if (((uintptr_t)x | (uintptr_t)w | (uintptr_t)y) & 15) return false;
    return get_encode() != nullptr;
}

// bias2: second per-channel addend or null.  gn_stats != null (and Cout % gn_groups == 0): the kernel adds the per-group (sum, sum of
// squares) of the stored output to gn_stats[2 * groups] (fp64) and sets *gn_done = 1 -- when the chosen decomposition cannot (ragged
// Cout, split-K with a group width that is not a multiple of 4, in-kernel reduce) *gn_done stays 0 and the caller computes them itself.
int osb_tc_conv_launch(const void* x, const void* w, const void* bias, const void* residual, void* y, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                       int kh, int kw, int stride, int pad_top, int pad_left, int64_t Ho, int64_t Wo, cudaStream_t st,
                       const void* bias2, double* gn_stats, int gn_groups, int* gn_done)
{
    if (gn_done) *gn_done = 0;
    if (gn_stats && (gn_groups < 1 || gn_groups > tcptx::GN_MAX_GROUPS || Cout % gn_groups || Cout % 8)) gn_stats = nullptr;
    const int gn_cpg = gn_stats ? (int)(Cout / gn_groups) : 0;
    uint32_t bw = std::min<uint32_t>(128, next_pow2((uint32_t)Wo)), bh = 128 / bw;
    CUtensorMap ma, mb;
    // A: NHWC input as (C, W, H); one box = bh rows x bw pixels x 64 channels, zero-filled outside the image.  With a
    // traversal stride s the box spans bw*s x bh*s input pixels and TMA delivers every s-th one.
    if (!make_map(&ma, x, (uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)Cin * 2, (uint64_t)W * Cin * 2, BLOCK_K, bw * stride, bh * stride, (uint32_t)stride))
        return (int)cudaErrorInvalidValue;
    // B: OHWI weights = [Cout][kh*kw*Cin], K-major
    int64_t Ktot = (int64_t)kh * kw * Cin;
    const int64_t m_tiles_ = ((Wo + bw - 1) / bw) * ((Ho + bh - 1) / bh);
    const bool pair = !g_f32x && Cout % 8 == 0 && use_pair(m_tiles_, Cout);
    if (!make_map(&mb, w, (uint64_t)Ktot, (uint64_t)Cout, 1, (uint64_t)Ktot * 2, (uint64_t)Ktot * Cout * 2, BLOCK_K, pair ? BLOCK_N / 2 : BLOCK_N, 1))
        return (int)cudaErrorInvalidValue;
    TcParams p{};
    p.M = (int)(Ho * Wo); p.N = (int)Cout; p.K = (int)Cin; p.batch = 1;
    p.tiles_x = (int)((Wo + bw - 1) / bw);
    p.m_tiles = p.tiles_x * (int)((Ho + bh - 1) / bh);
    p.n_tiles = (int)((Cout + BLOCK_N - 1) / BLOCK_N);
    p.b_kmajor = 1;
    p.taps = kh * kw; p.kw = kw; p.pad_top = pad_top; p.pad_left = pad_left; p.Wo = (int)Wo; p.Ho = (int)Ho; p.bw = (int)bw; p.bh = (int)bh;
    p.k_blocks_per_tap = (int)((Cin + BLOCK_K - 1) / BLOCK_K);
    p.stride = stride;
    p.C = (__half*)y; p.bias = (const __half*)bias; p.residual = (const __half*)residual; p.stride_c = 0; p.ldc = Cout;
    if (pair) {
        p.split_k = 1;
        p.bias2 = (const __half*)bias2;
        if (gn_stats) { p.gn_stats = gn_stats; p.gn_cpg = gn_cpg; p.gn_groups = gn_groups; if (gn_done) *gn_done = 1; }
        { static const int dbg = env_int("OSB_GN_DEBUG"); p.gn_debug = dbg; }
        return launch(ma, mb, p, st, nullptr, nullptr, true);
    }
    // the split-K reduce paths move float4 / half4 vectors: ragged Cout (conv_out, 3 or 4 channels) runs unsplit
    OsbWorkspace* wsp = nullptr;
    p.split_k = (Cout % 4 == 0) ? choose_split(p.m_tiles * p.n_tiles, p.taps * p.k_blocks_per_tap, (size_t)Ho * Wo * Cout, st, &wsp) : 1;
    p.ws = wsp ? wsp->splitk : nullptr;
    p.bias2 = (const __half*)bias2;
    // statistics: the tile epilogue (unsplit) or the reduce kernel (split-K; needs 4 consecutive columns inside one group)
    const bool stats_ok = gn_stats && (p.split_k == 1 || gn_cpg % 4 == 0);     // tile epilogue (unsplit) or the reduce kernel
    if (stats_ok) { p.gn_stats = gn_stats; p.gn_cpg = gn_cpg; p.gn_groups = gn_groups; if (gn_done) *gn_done = 1; }
    { static const int dbg = env_int("OSB_GN_DEBUG"); p.gn_debug = dbg; }
    if (g_f32x) {
        if (!f32x_params(p, wsp, st)) return (int)cudaErrorNotSupported;
    }
    return launch(ma, mb, p, st);
}

// ---- fp32 GEMM / conv on the tensor cores: bf16 triple split ------------------------------------------------------------------------
// x = h + m + l with h = bf16(x), m = bf16(x - h), l = bf16(x - h - m) carries 24 mantissa bits; a.b ~= ah.bh + ah.bm + am.bh + ah.bl + al.bh + am.bm
// (the dropped terms are below 2^-24 relative).  The six products are ONE tensor-core contraction over a 6x longer K: the caller expands
// A to [h|h|m|h|l|m] and B to [h|m|h|l|h|m] along K (osb_bf16x3_expand_*), products are exact in fp32 and accumulate in the fp32 register
// accumulator.  A, B: bf16 expansions (K6 = 6 K); C, bias, residual: fp32; C dense [M][N].  cudaErrorNotSupported: run the CUDA-core kernel.
// shape predicates of the fp32 tensor-core path (before the caller spends time expanding operands)
extern "C" int osb_tc_gemm_f32x_ok(int64_t M, int64_t N, int64_t K)
{
    static const bool on = [] { const char* e = getenv("OSB_F32_TC"); return !(e && e[0] == '0'); }();
    return on && M >= 32 && N >= 8 && N % 8 == 0 && K >= 8 && (6 * K) % 8 == 0 && (size_t)M * N * 4 <= WS_MAX && get_encode() != nullptr ? 1 : 0;
}
extern "C" int osb_tc_conv_f32x_ok(int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, int64_t Ho, int64_t Wo)
{
    static const bool on = [] { const char* e = getenv("OSB_F32_TC"); return !(e && e[0] == '0'); }();
    return on && (6 * Cin) % 8 == 0 && 6 * Cin >= 16 && stride >= 1 && stride <= 2 && H * W >= 64 && kh <= 7 && kw <= 7 && (size_t)Ho * Wo * Cout * 4 <= WS_MAX &&
           get_encode() != nullptr ? 1 : 0;
}

extern "C" int osb_tc_gemm_f32x(const void* A6, const void* B6, void* C, const void* bias, const void* residual, int64_t M, int64_t N, int64_t K6, int bt, void* stream)
{
    const int64_t ldb = bt ? K6 : N;
    // (ldc is a float pitch here: only 16-byte pointer alignment of C matters to the workspace reduce)
    if (!osb_tc_gemm_ok(M, N, K6, bt, A6, B6, nullptr, 0, 0, 0, K6, ldb, 8) || (N % 8)) return (int)cudaErrorNotSupported;
    g_f32x = 1;
    int r = osb_tc_gemm_launch(A6, B6, C, bias, residual, 1, M, N, K6, 0, 0, M * N, bt, (cudaStream_t)stream, K6, ldb, N);
    g_f32x = 0;
    return r;
}

extern "C" int osb_tc_conv_f32x(const void* x6, const void* w6, const void* bias, const void* residual, void* y, int64_t H, int64_t W, int64_t Cin6, int64_t Cout,
                     int kh, int kw, int stride, int pad_top, int pad_left, int64_t Ho, int64_t Wo, void* stream)
{
    if (!osb_tc_conv_ok(H, W, Cin6, Cout, kh, kw, stride, x6, w6, nullptr)) return (int)cudaErrorNotSupported;
    g_f32x = 1;
    int r = osb_tc_conv_launch(x6, w6, bias, residual, y, H, W, Cin6, Cout, kh, kw, stride, pad_top, pad_left, Ho, Wo, (cudaStream_t)stream, nullptr, nullptr, 0, nullptr);
    g_f32x = 0;
    return r;
}
