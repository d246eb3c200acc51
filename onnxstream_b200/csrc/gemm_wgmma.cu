// gemm_wgmma.cu -- the tensor-core path for fp16 MatMul / Gemm / Conv / attention GEMMs on sm_90a.
//
// One persistent, warp-specialised kernel, 384 threads:
//   warpgroup 0      TMA producer: one warp issues cp.async.bulk.tensor tiles of A and B into 128B-swizzled shared memory, mbarrier-tracked
//   warpgroups 1, 2  consumers: each issues wgmma (fp32 accumulators in registers) for its part of the BM x BN tile -- 64 rows at
//                    BM = 128, half the columns at BM = 64 (TileCfg) -- then runs the epilogue from its registers: add bias /
//                    residual, round to fp16, store
// The tile shape and the split-K factor are chosen per launch (choose_tile: a cost model fit to measured times).
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
#include <cstdio>
#include <cstdlib>
#include <vector>

namespace {

constexpr int BLOCK_M = 128;           // the default tile, the uint8 kernel's and the CTA pairs' tile
constexpr int BLOCK_N = 128;
constexpr int BLOCK_K = 64;            // 64 fp16 = 128 bytes = one swizzle row
constexpr int WG_K = 16;
constexpr int RING_BYTES = 6 * 32768;  // the (A, B) ring of every tile shape: 6 stages of the 128 x 128 tile
constexpr int NUM_THREADS = 384;        // producer warpgroup + two consumer warpgroups
constexpr int CONSUMER_THREADS = 256;

// One tile shape, BM x BN.  BM = 128: consumer warpgroup wg owns rows [64 wg, 64 wg + 64) and all BN columns (m64nBN).  BM = 64: both
// warpgroups share the 64 rows and split the columns, wg owns [wg BN/2, (wg + 1) BN/2) (m64n(BN/2)).  An MN-major B stage is BN/64 atoms of
// 64 columns x 64 k-rows, so there BN (BM = 128) or BN/2 (BM = 64) is a multiple of 64.  The ring takes as many stages as fit RING_BYTES.
template <int BM, int BN>
struct TileCfg {
    static constexpr int A_STAGE_BYTES = BM * BLOCK_K * 2;
    static constexpr int B_STAGE_BYTES = BN * BLOCK_K * 2;
    static constexpr int STAGES_FIT = RING_BYTES / (A_STAGE_BYTES + B_STAGE_BYTES);
    static constexpr int STAGES = STAGES_FIT < 16 ? STAGES_FIT : 16;      // 2 * STAGES mbarriers in the 256-byte barrier area
    static constexpr int WN = BM == 128 ? BN : BN / 2;                    // accumulator columns of one consumer warpgroup
    static constexpr int SMEM_BYTES = STAGES * (A_STAGE_BYTES + B_STAGE_BYTES) + 1024 /*align slack*/ + 256 /*barriers*/ + 2 * tcptx::GN_MAX_GROUPS * 8;
    static_assert(BM == 64 || BM == 128, "BM");
    static_assert(BN % 16 == 0 && B_STAGE_BYTES % 1024 == 0, "every stage and every warpgroup's B rows start on a 1024-byte swizzle boundary");
};
constexpr int A_STAGE_BYTES = TileCfg<BLOCK_M, BLOCK_N>::A_STAGE_BYTES;   // the uint8 kernel's stages (gemm_i8.cuh)
constexpr int B_STAGE_BYTES = TileCfg<BLOCK_M, BLOCK_N>::B_STAGE_BYTES;

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
    int bm, bn;                  // the tile shape the launch runs (the kernel's template arguments; kept for the launch profile)
    int geglu;                   // GEGLU epilogue (osb_tc_gemm_geglu): B is [K, 2 N], C [M, N] = value * gelu(gate)
    float wscale;                // uint8 weight (tc_gemm_u8w_kernel): per-tensor scale and zero point
    int wzero;
};

using namespace tcptx;

// one k-block (64 elements of K) of a consumer warpgroup: 4 x m64nWNk16
template <int WN, int B_MN_MAJOR, bool BF16>
__device__ __forceinline__ void mma_kblock(float (&acc)[WN / 2], uint64_t adesc, uint64_t bdesc)
{
    constexpr uint32_t b_kstep = B_MN_MAJOR ? (WG_K * 128) >> 4 : (WG_K * 2) >> 4;   // descriptor address units (16 B)
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / WG_K; k++) {
        const uint64_t a = adesc + (uint64_t)(k * ((WG_K * 2) >> 4)), b = bdesc + (uint64_t)(k * b_kstep);
        wgmma_ss<WN, B_MN_MAJOR, BF16>(acc, a, b, 1u);
    }
    wgmma_commit();
}

// x[0], x[1] as a packed half2, columns outside the problem (ok0 / ok1 false) read as 0.  vec: the pair is 4-byte aligned, one load.
// NC: through the read-only path (bias, bias2: never written by a launch; the residual may be C itself, so it takes plain loads).
template <bool NC>
__device__ __forceinline__ __half2 ld_pair(const __half* x, bool ok0, bool ok1, bool vec)
{
    const unsigned short* s = reinterpret_cast<const unsigned short*>(x);
    uint32_t v;
    if (ok1 && vec) v = NC ? __ldg(reinterpret_cast<const unsigned int*>(s)) : *reinterpret_cast<const unsigned int*>(s);
    else v = (ok0 ? (uint32_t)(NC ? __ldg(s) : s[0]) : 0u) | (ok1 ? (uint32_t)(NC ? __ldg(s + 1) : s[1]) << 16 : 0u);
    return *reinterpret_cast<__half2*>(&v);
}

// ---- the kernel -----------------------------------------------------------------------------------------------

// BM x BN = the tile (TileCfg).  EXTRAS = the epilogue also adds `bias2` and gathers GroupNorm statistics.  A separate instantiation, so
// the common launches do not carry the extra registers and code.  B_MN_MAJOR (== !p.b_kmajor) and BF16 (== p.bf16) are compile-time: the
// MMA loop has no branches.  PAIR = launched as clusters of two CTAs (see the top of the file); 128 x 128 tiles, split_k == 1 and
// groups == 1 there.  GEGLU (== p.geglu; 128 x 128 tiles, MN-major B, split_k == 1): the feed-forward gate of a [K, 2 N] weight in the
// epilogue.  The tile's B atom 0 holds value columns [64 nt, 64 nt + 64), atom 1 the gate columns N + [64 nt, 64 nt + 64), so every thread
// holds value block j and its gate block j + 8 in the same rows and column pair; the tile stores 64 columns of C [M, N].
template <int BM, int BN, bool EXTRAS, int B_MN_MAJOR, bool BF16, bool PAIR, bool GEGLU = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const __grid_constant__ CUtensorMap map_b1,
               const __grid_constant__ CUtensorMap map_b2, const TcParams p)
{
    using Cfg = TileCfg<BM, BN>;
    constexpr int STAGES = Cfg::STAGES, A_STAGE_BYTES = Cfg::A_STAGE_BYTES, B_STAGE_BYTES = Cfg::B_STAGE_BYTES, WN = Cfg::WN;
    static_assert(!PAIR || (BM == 128 && BN == 128), "CTA pairs run 128 x 128 tiles");
    static_assert(!B_MN_MAJOR || WN % 64 == 0, "an MN-major B is read in 64-column atoms");
    static_assert(!GEGLU || (BM == 128 && BN == 128 && B_MN_MAJOR && !EXTRAS && !BF16 && !PAIR), "GEGLU: 128 x 128 tiles of an fp16 [K, 2 N] weight");
    osb_pdl_trigger_entry();   // let the next kernel's CTAs be scheduled as ours drain; it waits for our completion before touching memory
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the 128B swizzle atoms
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
    uint64_t* bars = (uint64_t*)(smem + STAGES * (A_STAGE_BYTES + B_STAGE_BYTES));
    uint64_t* full = bars;                       // [STAGES]
    uint64_t* empty = bars + STAGES;             // [STAGES]
    double* gn_acc = (double*)((uint8_t*)bars + 256);       // [2 * GN_MAX_GROUPS] per-CTA (sum, sum of squares) accumulators

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (EXTRAS && p.gn_stats && threadIdx.x < 2 * GN_MAX_GROUPS) gn_acc[threadIdx.x] = 0.0;

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
            int n0 = nt * BN;
            int y0 = 0, x0 = 0, m0 = mt * BM;
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
                        // BN/64 atoms of 64 columns x 64 k-rows
#pragma unroll
                        for (int at = 0; at < BN / 64; at++) {
                            const int col = GEGLU ? 64 * nt + at * p.N : n0 + 64 * at;     // GEGLU: the value atom, then the gate atom
                            if (p.b_swap) tma_load_3d_s(sb + at * 8192, mbp, &full[stage], col, b, kglob);
                            else tma_load_3d_s(sb + at * 8192, mbp, &full[stage], col, kglob, b);
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
        const int wg = (warp >> 2) - 1;          // BM = 128: rows [64 wg, 64 wg + 64) of the tile; BM = 64: columns [WN wg, WN wg + WN)
        const int ct = (int)threadIdx.x - (NUM_THREADS - CONSUMER_THREADS);
        const int wrow = BM == 128 ? 64 * wg : 0, wcol = BM == 128 ? 0 : WN * wg;
        // Descriptor templates: everything but the 14-bit start address is loop-invariant.
        //   A, K-major SW128: 8-row groups 1024 B apart; K advances 32 B inside the swizzle row; warpgroup wg starts wrow rows in.
        //   B, K-major: same, starting wcol rows in.  B, MN-major SW128: 64-column atoms 8192 B apart (LBO), 8-row k-groups 1024 B apart
        //   (SBO); K advances 16 rows = 2048 B; warpgroup wg starts wcol / 64 atoms in.
        const uint64_t adesc0 = make_smem_desc(smem_u32(smem_a) + wrow * 128, 16, 1024);
        const uint64_t bdesc0 = B_MN_MAJOR ? make_smem_desc(smem_u32(smem_b) + (wcol / 64) * 8192, 8192, 1024) : make_smem_desc(smem_u32(smem_b) + wcol * 128, 16, 1024);
        const bool partial = p.split_k > 1 || p.f32_out;
        const int r_lo = wrow + (warp & 3) * 16 + (lane >> 2);      // this thread's rows of the tile: r_lo and r_lo + 8
        const int cq = 2 * (lane & 3);                               // and its column pair inside every 8-column block
        // the epilogue's column pairs load as one 4-byte word where the operand is aligned to it
        const bool vec_bias = ((uintptr_t)p.bias & 3) == 0, vec_bias2 = ((uintptr_t)p.bias2 & 3) == 0;
        const bool vec_res = ((uintptr_t)p.residual & 3) == 0 && ((p.ldc | p.stride_c) & 1) == 0;
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
            const int n0 = nt * BN, c0 = n0 + wcol;      // tile and warpgroup column origins
            const int n_end = min(p.N, n0 + BN);
            const int kb_lo = sp * kb_per_split, kb_hi = min(kb_lo + kb_per_split, k_blocks_all);
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
                    int m = mt * BM + row_in_tile;
                    row_ok[h] = m < p.M;
                    out_row[h] = m;
                }
            }
            const long long off[2] = { (long long)b * p.stride_c + out_row[0] * p.ldc, (long long)b * p.stride_c + out_row[1] * p.ldc };
            // GroupNorm statistics: the warp's valid rows (lanes 4r..4r+3 hold rows r (h = 0) and r + 8 (h = 1) of its 16), and the lane
            // group + row half that holds the first of them -- each column's pivot is read from there (gn_stats_pair)
            int gn_rows = 0, gn_src = 0, gn_h = 0;
            if (EXTRAS && p.gn_stats) {
                const unsigned b0 = __ballot_sync(0xffffffffu, row_ok[0]), b1 = __ballot_sync(0xffffffffu, row_ok[1]);
                gn_rows = (__popc(b0) + __popc(b1)) >> 2;
                gn_h = b0 ? 0 : 1;
                gn_src = b0 ? __ffs(b0) - 1 : (b1 ? __ffs(b1) - 1 : 0);
                gn_src = (gn_src & ~3) | (lane & 3);
            }
            // The tile's residual rows are fetched into L2 while the main loop runs (a residual written several launches ago may have been
            // evicted by the weights streaming through since), so the epilogue's loads do not wait on HBM.  The 4 lanes that share a row
            // take one 128-byte line each of the warpgroup's (at most 320-byte) column span.
            if (p.residual && !partial) {
                const int span = (min(p.N, c0 + WN) - c0) * 2;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const uintptr_t a0 = (uintptr_t)(p.residual + off[h] + c0), line = (a0 & ~(uintptr_t)127) + 128 * (lane & 3);
                    if (row_ok[h] && span > 0 && line < a0 + span) {
                        asm volatile("prefetch.global.L2 [%0];" ::"l"(line));
                    }
                }
            }

            float acc[WN / 2];
#pragma unroll
            for (int i = 0; i < WN / 2; i++) acc[i] = 0.f;
            // one k-block of MMAs stays in flight: the stage of k-block kb-1 is released once the MMAs of kb are issued
            int prev = -1;
            for (int kb = kb_lo; kb < kb_hi; kb++) {
                mbar_wait(&full[stage], phase);
                mma_kblock<WN, B_MN_MAJOR, BF16>(acc, adesc0 + (uint64_t)(stage * (A_STAGE_BYTES >> 4)), bdesc0 + (uint64_t)(stage * (B_STAGE_BYTES >> 4)));
                if (prev >= 0) { wgmma_wait<1>(); release(prev); }
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            release(prev);

            // ---- epilogue ----
            if constexpr (GEGLU) {
                // each half rounded to fp16 as the plain bias epilogue stores it, then value * gelu(gate) in fp32 (the node kernel's
                // arithmetic), rounded once: bit-identical to the unsplit GEMM followed by osb_geglu
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const int n = 64 * nt + 8 * j + cq;      // value column; the gate is column p.N + n
                    float av0 = 0.f, av1 = 0.f, ag0 = 0.f, ag1 = 0.f;
                    if (p.bias) {
                        const __half2 bv = ld_pair<true>(p.bias + n, true, true, vec_bias), bg = ld_pair<true>(p.bias + p.N + n, true, true, vec_bias);
                        av0 += __low2float(bv); av1 += __high2float(bv); ag0 += __low2float(bg); ag1 += __high2float(bg);
                    }
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        if (!row_ok[h]) continue;
                        const float a0 = __half2float(__float2half_rn(acc[4 * j + 2 * h] + av0)), a1 = __half2float(__float2half_rn(acc[4 * j + 2 * h + 1] + av1));
                        const float g0 = __half2float(__float2half_rn(acc[4 * (j + 8) + 2 * h] + ag0)), g1 = __half2float(__float2half_rn(acc[4 * (j + 8) + 2 * h + 1] + ag1));
                        *reinterpret_cast<__half2*>(p.C + off[h] + n) =
                            __halves2half2(__float2half_rn(apply_binary(OSB_BIN_MUL_GELU, a0, g0)), __float2half_rn(apply_binary(OSB_BIN_MUL_GELU, a1, g1)));
                    }
                }
                continue;
            }
            __half* cbase = p.C;
            if (p.groups > 1) cbase = b == 0 ? p.C : (b == 1 ? p.C1 : p.C2);    // stride_c == 0 in a grouped launch
            const bool pair_ok = (p.N & 1) == 0 && (p.ldc & 1) == 0;           // two adjacent columns move as one 4- / 8-byte vector
            // The addends of EG 8-column blocks are loaded before any of their stores: bias and residual may alias C for all the compiler
            // knows, so it cannot move a block's loads above an earlier block's stores, and loads interleaved with the stores wait one by one.
            constexpr int EG = 4;   // 2 and 8 measured no faster (DESIGN.md section 5)
#pragma unroll
            for (int j0 = 0; j0 < WN / 8; j0 += EG) {
                if (c0 + 8 * j0 >= n_end) break;    // warp-uniform
                __half2 bias_v[EG], bias2_v[EG], res_v[EG][2];
#pragma unroll
                for (int jj = 0; jj < EG && j0 + jj < WN / 8; jj++) {
                    const int n = c0 + 8 * (j0 + jj) + cq;
                    const bool ok0 = n < n_end, ok1 = n + 1 < n_end;
                    if (partial) continue;
                    if (p.bias) bias_v[jj] = ld_pair<true>(p.bias + n, ok0, ok1, vec_bias);
                    if (EXTRAS && p.bias2) bias2_v[jj] = ld_pair<true>(p.bias2 + n, ok0, ok1, vec_bias2);
                    if (p.residual) {
#pragma unroll
                        for (int h = 0; h < 2; h++) res_v[jj][h] = ld_pair<false>(p.residual + off[h] + n, ok0 && row_ok[h], ok1 && row_ok[h], vec_res);
                    }
                }
#pragma unroll
                for (int jj = 0; jj < EG && j0 + jj < WN / 8; jj++) {
                    const int j = j0 + jj;
                    if (c0 + 8 * j >= n_end) break;     // warp-uniform
                    const int n = c0 + 8 * j + cq;
                    const bool ok0 = n < n_end, ok1 = n + 1 < n_end;
                    float y0[2] = { 0.f, 0.f }, y1[2] = { 0.f, 0.f };   // the two columns as stored, for the GroupNorm statistics
                    float add0 = 0.f, add1 = 0.f;                   // per-column addend: bias
                    if (!partial && p.bias) { add0 += __low2float(bias_v[jj]); add1 += __high2float(bias_v[jj]); }
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
                        f0 += add0; f1 += add1;
                        if (p.residual) { f0 += __low2float(res_v[jj][h]); f1 += __high2float(res_v[jj][h]); }
                        if (EXTRAS && p.bias2) { f0 += __low2float(bias2_v[jj]); f1 += __high2float(bias2_v[jj]); }
                        const __half o0 = __float2half_rn(f0), o1 = __float2half_rn(f1);
                        __half* crow = cbase + off[h];
                        if (ok1 && pair_ok) *reinterpret_cast<__half2*>(crow + n) = __halves2half2(o0, o1);
                        else { if (ok0) crow[n] = o0; if (ok1) crow[n + 1] = o1; }
                        if (EXTRAS) {
                            // the statistics see the values as they are stored
                            y0[h] = ok0 ? __half2float(o0) : 0.f; y1[h] = ok1 ? __half2float(o1) : 0.f;
                        }
                    }
                    if (EXTRAS && p.gn_stats && !partial && !(p.gn_debug & 1)) {
                        const float p0 = __shfl_sync(0xffffffffu, gn_h ? y0[1] : y0[0], gn_src), p1 = __shfl_sync(0xffffffffu, gn_h ? y1[1] : y1[0], gn_src);
                        float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            if (!row_ok[h]) continue;
                            const float d0 = y0[h] - p0, d1 = y1[h] - p1;
                            s0 += d0; q0 = fmaf(d0, d0, q0); s1 += d1; q1 = fmaf(d1, d1, q1);
                        }
                        gn_stats_pair(s0, s1, q0, q1, p0, p1, gn_rows, n, n_end, p.gn_cpg, gn_acc, lane);
                    }
                }
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
// Optionally gathers the GroupNorm statistics of the result as plain fp64 sums of y and y^2: per-block fp32 shared accumulators of
// y - p around the group's pivot p (its first output, row 0, which every block computes alike), shifted back in fp64: each block adds s and
// q + 2 p s, block 0 also n p and n p^2 for the n = rows * cpg elements of the group.
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, __half* __restrict__ out, const __half* __restrict__ bias, const __half* __restrict__ bias2,
                                     const __half* __restrict__ residual, long long rows, int N, int splits, double* __restrict__ gn_stats, int gn_cpg, int gn_groups)
{
    osb_pdl_prologue();
    __shared__ float acc[2 * GN_MAX_GROUPS];
    __shared__ float piv[GN_MAX_GROUPS];
    // N % 4 == 0: one float4 of every split plane per thread, fully coalesced
    const long long total4 = rows * N / 4;
    const long long plane4 = total4;
    const float4* w4 = reinterpret_cast<const float4*>(ws);
    if (gn_stats) {
        if (threadIdx.x < 2 * GN_MAX_GROUPS) acc[threadIdx.x] = 0.f;
        if (threadIdx.x < gn_groups) {
            // group g's pivot: the output at row 0, column g * cpg, as the loop below computes and rounds it
            const int n = threadIdx.x * gn_cpg;
            float v = ws[n];
#pragma unroll 8
            for (int s = 1; s < splits; s++) v += __ldg(ws + (long long)s * rows * N + n);    // independent loads: few round trips
            if (bias) v += __half2float(bias[n]);
            if (bias2) v += __half2float(bias2[n]);
            if (residual) v += __half2float(residual[n]);
            piv[threadIdx.x] = __half2float(__float2half_rn(v));
        }
        __syncthreads();
    }
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
            const int g = n / gn_cpg;
            const float pg = piv[g];
            float x0 = __half2float(o.v[0]) - pg, x1 = __half2float(o.v[1]) - pg, x2 = __half2float(o.v[2]) - pg, x3 = __half2float(o.v[3]) - pg;
            atomicAdd(&acc[2 * g], (x0 + x1) + (x2 + x3));
            atomicAdd(&acc[2 * g + 1], fmaf(x0, x0, x1 * x1) + fmaf(x2, x2, x3 * x3));
        }
    }
    if (gn_stats) {
        __syncthreads();
        if (threadIdx.x < gn_groups) {
            const int g = threadIdx.x;
            const double s = acc[2 * g], q = acc[2 * g + 1], pg = piv[g], n = blockIdx.x == 0 ? (double)rows * gn_cpg : 0.0;
            atomicAdd(&gn_stats[2 * g], s + n * pg);
            atomicAdd(&gn_stats[2 * g + 1], q + (2.0 * pg) * s + n * pg * pg);
        }
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


// ---- fp32 activations x an fp16 weight read in place (osb_tc_gemm_f32x_f16w) --------------------------------------------------------
// An fp16 value w is exactly hi + lo with hi = bf16(w) and lo = bf16(w - hi) (the remainder has at most 3 significant bits, and fp16
// subnormals are bf16 normals), so the bf16 triple split of the widened weight is (hi, lo, 0): of the six products of the fp32 path (hh,
// hm, mh, hl, lh, mm; osb_tc_gemm_f32x) hl is zero, and five remain.  One 128 x 128 tile per CTA, 384 threads, persistent:
//   warp 0            TMA producer: per raw k-block (64 of K) the three bf16 planes of A ([M][3][K], one map over [M, 3 K]: plane p's
//                     k-block kc at column p K + kc; a chunk past K reads the next plane against B rows that TMA zero-fills) and the fp16
//                     B block as stored (two 64-column atoms, MN-major), which completes `landed`
//   warps 1-3         B splitters: every fp16 element of the block once -> hi in place and lo into the stage's second B buffer (elementwise
//                     at the same offset, so the 128B swizzle carries over), fence.proxy.async, arrive on `full` (one per warp)
//   warpgroups 1, 2   consumers: per stage the five products (h, hi), (h, lo), (m, hi), (l, hi), (m, lo) as 5 x 4 wgmma m64n128k16 into
//                     the fp32 accumulators, one stage in flight; the tile's raw fp32 sums go to the split-K workspace [split][M][N] and
//                     splitk_reduce_f32_kernel adds the splits, fp32 bias and residual.
// Each raw B block is converted once and its 16 KB read from L2 once; a stage is 48 KB of A planes + 32 KB of B parts, 2 stages.
//
// CONV (osb_tc_conv_f32x_f16w): the same pipeline as an implicit-GEMM convolution.  A is the NHWC image split into planes [H W][3][Cin],
// read through a 4-D map (Cin, plane, W, H): plane p of k-block (tap, channel block) is one box of bh x bw pixels at the tap's offset,
// zero-filled outside the image and past Cin (a 3-D map over 3 Cin channels would read the next plane there, against the next tap's
// weights in B).  B is the OHWI fp16 blob [Cout][kh kw Cin] as stored, K-major, as the fp16 conv reads it.  An unsplit launch stores fp32
// from the registers (acc + bias[n] + residual, the reduce kernel's order), so the output is not bounded by the workspace; a split
// launch writes its partials to the workspace for splitk_reduce_f32_kernel.  Ragged Cout stores are guarded by column.
//
// U8 (tc_gemm_u8w_kernel: osb_tc_gemm_f32x_u8w, osb_tc_conv_f32x_u8w): the weight is a uint8 blob with a per-tensor scale s and zero
// point z.  q - z is an integer of at most 255 in magnitude, exact as one bf16, and each product of a bf16 part of x with it has at most 16
// significant bits, so x (q - z) = h (q - z) + m (q - z) + l (q - z) exactly: three products per stage, (l, q), (m, q), (h, q), small ones
// first.  Warp 0 lands the uint8 block as stored (GEMM: [64 k][128 n] of the [K][N] blob; CONV: [128 n][64 k] of the OHWI blob, both
// unswizzled) in a buffer of its own; warps 1-3 write bf16(q - z) into the 128B-swizzled layout the consumers read (MN-major 64-column atoms
// for the GEMM, K-major rows for the conv) -- GEMM rows past K as 0, since A reads the next plane there.  s is applied once, in fp32, in the
// epilogue: unsplit, acc s + bias + residual is stored from the registers (GEMM and conv alike, so no output bound from the workspace);
// split, acc s goes to the workspace for the unchanged splitk_reduce_f32_kernel.  A stage is 48 KB of A planes + 16 KB of bf16 B + 8 KB
// landing, 3 stages.
namespace f16w {
constexpr int A_PLANE_BYTES = BLOCK_M * BLOCK_K * 2;            // 16 KB
constexpr int A_BYTES = 3 * A_PLANE_BYTES;
constexpr int B_PART_BYTES = BLOCK_N * BLOCK_K * 2;             // 16 KB
constexpr int B_BYTES = 2 * B_PART_BYTES;
constexpr int STAGES = 2;
constexpr int SMEM_BYTES = STAGES * (A_BYTES + B_BYTES) + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int SPLIT_THREADS = 96;
// U8: the bf16 (q - z) block, then the uint8 block as it lands
constexpr int U8_LAND_BYTES = BLOCK_N * BLOCK_K;                // 8 KB
constexpr int U8_B_BYTES = B_PART_BYTES + U8_LAND_BYTES;
constexpr int U8_STAGES = 3;
constexpr int U8_SMEM_BYTES = U8_STAGES * (A_BYTES + U8_B_BYTES) + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(U8_SMEM_BYTES <= 227 * 1024 && U8_B_BYTES % 1024 == 0, "three uint8 stages fit, every bf16 B block on a swizzle boundary");
}

// 8 uint8 weights (two words) -> 8 bf16 (q - z), exact: 2^23 + q is a float whose low byte is q, and subtracting 2^23 + z (fz) leaves q - z
__device__ __forceinline__ uint4 u8x8_bf16_minus_zero(uint2 v, float fz)
{
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint32_t w = i < 2 ? v.x : v.y, b = 2 * (i & 1);
        const float f0 = __uint_as_float(__byte_perm(w, 0x4Bu, 0x4550u + b)) - fz, f1 = __uint_as_float(__byte_perm(w, 0x4Bu, 0x4551u + b)) - fz;
        const __nv_bfloat162 h = __floats2bfloat162_rn(f0, f1);
        o[i] = *reinterpret_cast<const uint32_t*>(&h);
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
}

// two fp16 values (one 32-bit word) -> their bf16 hi and lo parts
__device__ __forceinline__ void f16x2_bf16_parts(uint32_t v, uint32_t& hi, uint32_t& lo)
{
    const float2 x = __half22float2(*reinterpret_cast<const __half2*>(&v));
    const __nv_bfloat162 h = __float22bfloat162_rn(x);
    const float2 hf = __bfloat1622float2(h);
    const __nv_bfloat162 l = __float22bfloat162_rn(make_float2(x.x - hf.x, x.y - hf.y));
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

// p: M, N, K, m_tiles, n_tiles, k_blocks_per_tap (= ceil(K / 64)), split_k, ws; CONV also the conv geometry (K = Cin, M = Ho Wo, taps,
// kw, pads, stride, bw x bh boxes, tiles_x) and, unsplit, C / bias / residual as fp32; U8 also wscale, wzero and, unsplit, C / bias /
// residual as fp32 in the GEMM mode too.  The body of tc_gemm_f16w_kernel (U8 = false) and tc_gemm_u8w_kernel (U8 = true); map_a, map_b and
// p are the kernel's own parameters.
template <bool CONV, bool U8>
__device__ __forceinline__ void f16w_u8w_body(const CUtensorMap& map_a, const CUtensorMap& map_b, const TcParams& p)
{
    using namespace f16w;
    constexpr int STAGES = U8 ? U8_STAGES : f16w::STAGES, B_BYTES = U8 ? U8_B_BYTES : f16w::B_BYTES;
    osb_pdl_trigger_entry();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* smem_a = smem;                             // [STAGES][3 planes][128 rows][64]
    uint8_t* smem_b = smem + STAGES * A_BYTES;          // [STAGES][hi, lo][2 atoms][64 k][64]; U8: [STAGES][q - z, landed uint8]
    uint64_t* bars = (uint64_t*)(smem + STAGES * (A_BYTES + B_BYTES));
    uint64_t* full = bars;
    uint64_t* empty = bars + STAGES;
    uint64_t* landed = bars + 2 * STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < STAGES; i++) { mbar_init(&full[i], 3); mbar_init(&empty[i], CONSUMER_THREADS); mbar_init(&landed[i], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    osb_pdl_wait();     // the planes of A are written by the split launched just before

    const int tiles = p.m_tiles * p.n_tiles;
    const int total = tiles * p.split_k;
    const int kbk = CONV ? p.taps * p.k_blocks_per_tap : p.k_blocks_per_tap;
    const int kb_per_split = (kbk + p.split_k - 1) / p.split_k;   // host guarantees every split runs >= 1 k-block

    if (warp == 0) {
        // ===================== TMA producer =====================
        const uint32_t sa0 = smem_u32(smem_a), sb0 = smem_u32(smem_b);
        int stage = 0; uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
            const int sp = tile % p.split_k, r = tile / p.split_k;
            const int m0 = (r % p.m_tiles) * BLOCK_M, n0 = (r / p.m_tiles) * BLOCK_N;
            const int kb_lo = sp * kb_per_split, kb_hi = min(kb_lo + kb_per_split, kbk);
            // CONV: the box origin of the tile's pixels and the (tap, channel block) walk, incremental inside the k loop
            int tap = 0, kcb = 0, ky = 0, kx = 0, ax = 0, ay = 0;
            if constexpr (CONV) {
                const int mt = r % p.m_tiles;
                ax = (mt % p.tiles_x) * p.bw * p.stride - p.pad_left; ay = (mt / p.tiles_x) * p.bh * p.stride - p.pad_top;
                tap = kb_lo / p.k_blocks_per_tap; kcb = kb_lo % p.k_blocks_per_tap; ky = tap / p.kw; kx = tap % p.kw;
            }
            for (int kb = kb_lo; kb < kb_hi; kb++) {
                mbar_wait(&empty[stage], phase ^ 1);
                if (elect_one()) {
                    mbar_expect_tx(&landed[stage], A_BYTES + (U8 ? U8_LAND_BYTES : B_PART_BYTES));
                    const uint32_t sa = sa0 + stage * A_BYTES, sb = sb0 + stage * B_BYTES;
                    if constexpr (CONV) {
                        const int kc = kcb * BLOCK_K;
#pragma unroll
                        for (int pl = 0; pl < 3; pl++) tma_load_4d_s(sa + pl * A_PLANE_BYTES, &map_a, &landed[stage], kc, pl, ax + kx, ay + ky);
                        tma_load_3d_s(U8 ? sb + B_PART_BYTES : sb, &map_b, &landed[stage], tap * p.K + kc, n0, 0);
                    } else {
                        const int kc = kb * BLOCK_K;
#pragma unroll
                        for (int pl = 0; pl < 3; pl++) tma_load_3d_s(sa + pl * A_PLANE_BYTES, &map_a, &landed[stage], pl * p.K + kc, m0, 0);
                        if constexpr (U8) {
                            tma_load_3d_s(sb + B_PART_BYTES, &map_b, &landed[stage], n0, kc, 0);     // one [64 k][128 n] uint8 box
                        } else {
#pragma unroll
                            for (int at = 0; at < 2; at++) tma_load_3d_s(sb + at * 8192, &map_b, &landed[stage], n0 + 64 * at, kc, 0);
                        }
                    }
                }
                __syncwarp();
                if constexpr (CONV) {
                    if (++kcb == p.k_blocks_per_tap) { kcb = 0; tap++; if (++kx == p.kw) { kx = 0; ky++; } }
                }
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
        osb_pdl_trigger_late();
    } else if (U8 && warp < 4) {
        // ===================== B converters: uint8 q -> bf16 (q - z) in the swizzled layout, once per raw block =====================
        // 8 landed bytes per thread -> one 16-byte chunk of a 128-byte swizzle row: chunk c of row r sits at chunk c ^ (r & 7)
        const int t = (int)threadIdx.x - 32;
        const float fz = 8388608.f + (float)p.wzero;
        int stage = 0; uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
            const int sp = tile % p.split_k;
            const int kb_lo = sp * kb_per_split, kb_hi = min(kb_lo + kb_per_split, kbk);
            for (int kb = kb_lo; kb < kb_hi; kb++) {
                mbar_wait(&landed[stage], phase);
                uint8_t* bq = smem_b + stage * B_BYTES;
                const uint2* land = reinterpret_cast<const uint2*>(bq + B_PART_BYTES);
                const int k_valid = CONV ? BLOCK_K : p.K - kb * BLOCK_K;     // GEMM: the block's rows inside K
#pragma unroll 4
                for (int g = t; g < U8_LAND_BYTES / 8; g += SPLIT_THREADS) {
                    uint4 o = u8x8_bf16_minus_zero(land[g], fz);
                    int off;
                    if constexpr (CONV) {
                        const int n = g >> 3, c = g & 7;            // landed row n: 64 k = 8 chunks
                        off = n * 128 + ((c ^ (n & 7)) << 4);
                    } else {
                        const int k = g >> 4, c = g & 15;           // landed row k: 128 n = 16 chunks, two 64-column atoms
                        off = (c >> 3) * 8192 + k * 128 + (((c & 7) ^ (k & 7)) << 4);
                        if (k >= k_valid) o = make_uint4(0u, 0u, 0u, 0u);
                    }
                    *reinterpret_cast<uint4*>(bq + off) = o;
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor cores
                __syncwarp();
                if (lane == 0) mbar_arrive(&full[stage]);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else if (warp < 4) {
        // ===================== B splitters: fp16 -> hi (in place) and lo, once per raw block =====================
        const int t = (int)threadIdx.x - 32;
        constexpr int PER = (B_PART_BYTES / 16 + SPLIT_THREADS - 1) / SPLIT_THREADS;
        int stage = 0; uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
            const int sp = tile % p.split_k;
            const int kb_lo = sp * kb_per_split, kb_hi = min(kb_lo + kb_per_split, kbk);
            for (int kb = kb_lo; kb < kb_hi; kb++) {
                mbar_wait(&landed[stage], phase);
                uint4* bh = reinterpret_cast<uint4*>(smem_b + stage * B_BYTES);
                uint4* bl = reinterpret_cast<uint4*>(smem_b + stage * B_BYTES + B_PART_BYTES);
                uint4 v[PER];
#pragma unroll
                for (int j = 0; j < PER; j++) if (t + j * SPLIT_THREADS < B_PART_BYTES / 16) v[j] = bh[t + j * SPLIT_THREADS];
#pragma unroll
                for (int j = 0; j < PER; j++) {
                    const int i = t + j * SPLIT_THREADS;
                    if (i >= B_PART_BYTES / 16) continue;
                    uint4 h, l;
                    f16x2_bf16_parts(v[j].x, h.x, l.x); f16x2_bf16_parts(v[j].y, h.y, l.y);
                    f16x2_bf16_parts(v[j].z, h.z, l.z); f16x2_bf16_parts(v[j].w, h.w, l.w);
                    bh[i] = h; bl[i] = l;
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor cores
                __syncwarp();
                if (lane == 0) mbar_arrive(&full[stage]);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // ===================== consumers: 5 products per stage (U8: 3), fp32 partials out =====================
        const int wg = (warp >> 2) - 1;
        const uint64_t adesc0 = make_smem_desc(smem_u32(smem_a) + 64 * wg * 128, 16, 1024);
        // B: MN-major (GEMM: [K][N] weight, two 64-column atoms) or K-major (CONV: 128 OHWI rows of 64 k)
        const uint64_t bdesc0 = CONV ? make_smem_desc(smem_u32(smem_b), 16, 1024) : make_smem_desc(smem_u32(smem_b), 8192, 1024);
        constexpr uint32_t b_kstep = CONV ? (WG_K * 2) >> 4 : (WG_K * 128) >> 4;
        constexpr uint64_t AP = A_PLANE_BYTES >> 4, BP = B_PART_BYTES >> 4;   // descriptor units (16 B)
        const int r_lo = 64 * wg + (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
        const bool pair_ok = (p.N & 1) == 0;
        int stage = 0; uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
            const int sp = tile % p.split_k, r = tile / p.split_k;
            const int m0 = (r % p.m_tiles) * BLOCK_M, n0 = (r / p.m_tiles) * BLOCK_N;
            const int kb_lo = sp * kb_per_split, kb_hi = min(kb_lo + kb_per_split, kbk);
            float acc[64];
#pragma unroll
            for (int i = 0; i < 64; i++) acc[i] = 0.f;
            int prev = -1;
            for (int kb = kb_lo; kb < kb_hi; kb++) {
                mbar_wait(&full[stage], phase);
                const uint64_t a = adesc0 + (uint64_t)(stage * (A_BYTES >> 4)), b = bdesc0 + (uint64_t)(stage * (B_BYTES >> 4));
                // (A plane, B part): (h, hi), (h, lo), (m, hi), (l, hi), (m, lo); U8: (l, q), (m, q), (h, q)
                const uint64_t ad[5] = { U8 ? a + 2 * AP : a, U8 ? a + AP : a, U8 ? a : a + AP, a + 2 * AP, a + AP }, bd[5] = { b, U8 ? b : b + BP, b, b, b + BP };
                wgmma_fence();
#pragma unroll
                for (int x = 0; x < (U8 ? 3 : 5); x++) {
#pragma unroll
                    for (int k = 0; k < BLOCK_K / WG_K; k++)
                        wgmma_ss<128, CONV ? 0 : 1, true>(acc, ad[x] + (uint64_t)(k * ((WG_K * 2) >> 4)), bd[x] + (uint64_t)(k * b_kstep), 1u);
                }
                wgmma_commit();
                if (prev >= 0) { wgmma_wait<1>(); mbar_arrive(&empty[prev]); }
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            mbar_arrive(&empty[prev]);
            if constexpr (CONV || U8) {
                // CONV: the tile's rows are a bw x bh box of output pixels
                const int mt = r % p.m_tiles, ty = CONV ? (mt / p.tiles_x) * p.bh : 0, tx = CONV ? (mt % p.tiles_x) * p.bw : 0;
                const float* bias = reinterpret_cast<const float*>(p.bias);
                const float* res = reinterpret_cast<const float*>(p.residual);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int rt = r_lo + 8 * h;
                    long long row;
                    if constexpr (CONV) {
                        const int y = ty + rt / p.bw, x = tx + rt % p.bw;
                        if (y >= p.Ho || x >= p.Wo) continue;
                        row = (long long)y * p.Wo + x;
                    } else {
                        if (m0 + rt >= p.M) continue;
                        row = m0 + rt;
                    }
                    // split: raw partials (U8: times s) -> ws[sp][M][N]; unsplit: acc (U8: times s) + bias + residual -> C, fp32
                    float* out = p.split_k > 1 ? p.ws + ((long long)sp * p.M + row) * p.N : reinterpret_cast<float*>(p.C) + row * p.N;
                    const float* rrow = p.split_k > 1 || !res ? nullptr : res + row * p.N;
                    const float* b = p.split_k > 1 ? nullptr : bias;
#pragma unroll
                    for (int j = 0; j < 16; j++) {
                        const int n = n0 + 8 * j + cq;
                        const bool ok0 = n < p.N, ok1 = n + 1 < p.N;
                        float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
                        if constexpr (U8) { f0 = __fmul_rn(f0, p.wscale); f1 = __fmul_rn(f1, p.wscale); }   // rounded before the bias, as a split launch does
                        if (b) { if (ok0) f0 += b[n]; if (ok1) f1 += b[n + 1]; }
                        if (rrow) {
                            if (ok1 && pair_ok) { const float2 rv = *reinterpret_cast<const float2*>(rrow + n); f0 += rv.x; f1 += rv.y; }
                            else { if (ok0) f0 += rrow[n]; if (ok1) f1 += rrow[n + 1]; }
                        }
                        if (ok1 && pair_ok) *reinterpret_cast<float2*>(out + n) = make_float2(f0, f1);
                        else { if (ok0) out[n] = f0; if (ok1) out[n + 1] = f1; }
                    }
                }
            } else {
                // raw fp32 sums of this split -> ws[sp][M][N]
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int m = m0 + r_lo + 8 * h;
                    if (m >= p.M) continue;
                    float* wrow = p.ws + ((long long)sp * p.M + m) * p.N;
#pragma unroll
                    for (int j = 0; j < 16; j++) {
                        const int n = n0 + 8 * j + cq;
                        const float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
                        if (n + 1 < p.N && pair_ok) *reinterpret_cast<float2*>(wrow + n) = make_float2(f0, f1);
                        else { if (n < p.N) wrow[n] = f0; if (n + 1 < p.N) wrow[n + 1] = f1; }
                    }
                }
            }
        }
    }
}

template <bool CONV>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tc_gemm_f16w_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const TcParams p)
{
    f16w_u8w_body<CONV, false>(map_a, map_b, p);
}

template <bool CONV>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tc_gemm_u8w_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const TcParams p)
{
    f16w_u8w_body<CONV, true>(map_a, map_b, p);
}

#include "gemm_i8.cuh"

// ---- host side -------------------------------------------------------------------------------------------------
constexpr size_t WS_MAX = OSB_WS_SPLITK_BYTES;   // fixed-capacity per-stream workspace (workspace.h): never re-allocated, graph-safe

int num_sms();

// The previous rule, kept selectable (osb_tc_set_tile(-1, 0, 0)) for A/B runs: 128 x 128 tiles, split K when there are fewer than 100 tiles
// and at least 32 (min_k_blocks) k-blocks, fill the SMs, keep >= 2 k-blocks per split, stay inside the workspace
int old_split(int tiles, int k_blocks, size_t out_elems, int min_k_blocks = 32)
{
    if (tiles >= 100 || k_blocks < min_k_blocks) return 1;
    int split = std::min(num_sms() / tiles, k_blocks / 2);
    while (split > 1 && (size_t)split * out_elems * 4 > WS_MAX) split--;
    if (split <= 1) return 1;
    int kb_per = (k_blocks + split - 1) / split;
    return (k_blocks + kb_per - 1) / kb_per;          // no empty splits: every CTA must run at least one k-block
}

// ---- tile shapes and the rule that picks one per launch ------------------------------------------------------------------------------
// The instantiated (BM, BN), each with the time one CTA takes for one k-block of it (ns; the cost model below).  K-major B (conv
// weights, transposed GEMM weights) with and without EXTRAS; MN-major B ([K, N] MatMul weights) without.  The fp32 path (BF16) and CTA
// pairs run 128 x 128 only.
#define TC_TILES_KMAJOR(X) X(128, 128, 468.0) X(128, 64, 327.0) X(128, 80, 365.0) X(128, 160, 606.0) X(64, 64, 266.0) X(64, 128, 329.0) X(64, 160, 358.0)
#define TC_TILES_MNMAJOR(X) X(128, 128, 499.0) X(128, 64, 284.0) X(64, 128, 300.0)
struct TileShape { int bm, bn; double kb_ns; };
#define TC_SHAPE(bm, bn, kb_ns) { bm, bn, kb_ns },
const TileShape kTilesK[] = { TC_TILES_KMAJOR(TC_SHAPE) };
const TileShape kTilesMN[] = { TC_TILES_MNMAJOR(TC_SHAPE) };
#undef TC_SHAPE

// forced by osb_tc_set_tile: 0 = the rule; g_tile_bm = -1: the previous rule (old_split) for every launch
int g_tile_bm = 0, g_tile_bn = 0, g_tile_split = 0;

// What the rule needs to know about a launch
struct TileProblem {
    int M, N;            // GEMM rows (per batch) and columns
    int Ho, Wo;          // conv output (conv != 0): the tile's rows are a bw x bh box of pixels
    int conv, batch, k_blocks, kmajor;
    bool may_split;      // the epilogue and the workspace allow a split-K launch
    bool only_128;       // the fp32 path: 128 x 128 tiles under the previous rule
};
struct TilePick { int bm, bn, split; };

int conv_box_w(int bm, int Wo) { uint32_t r = 1; while ((int)r < Wo) r <<= 1; return std::min<int>(bm, (int)r); }
int problem_m_tiles(const TileProblem& q, int bm)
{
    if (!q.conv) return (q.M + bm - 1) / bm;
    const int bw = conv_box_w(bm, q.Wo), bh = bm / bw;
    return ((q.Wo + bw - 1) / bw) * ((q.Ho + bh - 1) / bh);
}

// Cost model (ns), fit by least squares to the device times of the SD 1.5 UNet's tensor-core shapes under every tile on an H100 SXM
// (scripts/tile_bench.py; DESIGN.md section 5):
//   waves * (k-blocks per CTA * k-block time of the tile + WAVE_NS) + the reduce pass when split > 1.
// Median error of the fit 7 %, 90th percentile 20 %.
constexpr double WAVE_NS = 4500.0;         // per wave of CTAs: prologue, the first TMA round trip, the epilogue, the launch tail
constexpr double REDUCE_NS = 4050.0;       // the reduce launch and its dependency
constexpr double REDUCE_NS_PER_BYTE = 2.6e-5;   // the reduce's traffic: split fp32 planes read, fp16 output written

double tile_cost(const TileProblem& q, const TileShape& t, int split)
{
    const long long ctas = (long long)problem_m_tiles(q, t.bm) * ((q.N + t.bn - 1) / t.bn) * q.batch * split;
    const long long waves = (ctas + num_sms() - 1) / num_sms();
    const int kb_cta = (q.k_blocks + split - 1) / split;
    const double reduce_bytes = (double)q.batch * q.M * q.N * (4.0 * split + 2.0);
    return (double)waves * (kb_cta * t.kb_ns + WAVE_NS) + (split > 1 ? REDUCE_NS + REDUCE_NS_PER_BYTE * reduce_bytes : 0.0);
}

// the split factors worth trying for one tile: none, or enough CTAs for one or two waves, each with >= 2 k-blocks and no empty split
int split_for(const TileProblem& q, int tiles, int waves)
{
    if (!q.may_split || q.k_blocks < 4) return 1;
    int split = std::min(waves * num_sms() / std::max(tiles, 1), q.k_blocks / 2);
    while (split > 1 && (size_t)split * q.batch * q.M * q.N * 4 > WS_MAX) split--;
    if (split <= 1) return 1;
    int kb_per = (q.k_blocks + split - 1) / split;
    return (q.k_blocks + kb_per - 1) / kb_per;
}

TilePick choose_tile(const TileProblem& q)
{
    if (g_tile_bm < 0 || q.only_128) {
        const int tiles = problem_m_tiles(q, BLOCK_M) * ((q.N + BLOCK_N - 1) / BLOCK_N) * q.batch;
        return { BLOCK_M, BLOCK_N, q.may_split && q.k_blocks >= 4 ? old_split(tiles, q.k_blocks, (size_t)q.batch * q.M * q.N) : 1 };
    }
    const TileShape* shapes = q.kmajor ? kTilesK : kTilesMN;
    const int n_shapes = q.kmajor ? (int)(sizeof(kTilesK) / sizeof(kTilesK[0])) : (int)(sizeof(kTilesMN) / sizeof(kTilesMN[0]));
    // a forced shape without an instantiation for this B layout leaves the launch to the rule
    bool forced_shape = false;
    for (int i = 0; i < n_shapes; i++)
        forced_shape |= (g_tile_bm > 0 || g_tile_bn > 0) && (g_tile_bm <= 0 || shapes[i].bm == g_tile_bm) && (g_tile_bn <= 0 || shapes[i].bn == g_tile_bn);
    const bool forced_split = g_tile_split > 0 && (forced_shape || (g_tile_bm <= 0 && g_tile_bn <= 0));
    TilePick best{ BLOCK_M, BLOCK_N, 1 };
    double best_t = 1e300;
    for (int i = 0; i < n_shapes; i++) {
        const int bm = shapes[i].bm, bn = shapes[i].bn;
        if (forced_shape && ((g_tile_bm > 0 && bm != g_tile_bm) || (g_tile_bn > 0 && bn != g_tile_bn))) continue;
        const int tiles = problem_m_tiles(q, bm) * ((q.N + bn - 1) / bn) * q.batch;
        int cand[3] = { 1, split_for(q, tiles, 1), split_for(q, tiles, 2) };
        if (forced_split) {      // clamped to what the launch allows
            int sp = q.may_split && q.k_blocks >= 2 ? std::min(g_tile_split, q.k_blocks) : 1;
            while (sp > 1 && (size_t)sp * q.batch * q.M * q.N * 4 > WS_MAX) sp--;
            if (sp > 1) { int kb_per = (q.k_blocks + sp - 1) / sp; sp = (q.k_blocks + kb_per - 1) / kb_per; }
            cand[0] = cand[1] = cand[2] = std::max(sp, 1);
        }
        for (int sp : cand) {
            const double t = tile_cost(q, shapes[i], sp);
            if (t < best_t) { best_t = t; best = { bm, bn, sp }; }
        }
    }
    return best;
}

// the pick, with the split-K workspace attached; no workspace (capturing before any eager run, or out of memory): the best unsplit pick
TilePick choose_tile_ws(TileProblem q, cudaStream_t st, OsbWorkspace** ws_out)
{
    *ws_out = nullptr;
    TilePick t = choose_tile(q);
    if (t.split > 1) {
        *ws_out = osb_workspace(st, OSB_WS_SPLITK);
        if (!*ws_out) { q.may_split = false; t = choose_tile(q); }
    }
    return t;
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
struct ProfRec { cudaEvent_t a, b; double flops, bytes; int M, N, K, taps, batch, split, conv, bm, bn, kmajor; };
bool g_prof = false;
std::vector<ProfRec> g_prof_list;

void prof_begin(ProfRec& rec, const TcParams& p, cudaStream_t st)
{
    cudaEventCreate(&rec.a); cudaEventCreate(&rec.b);
    // the fp32 path (bf16 triple split) runs a 6x longer K: ALGORITHMIC work is the fp32 problem's (K / 6, 4-byte elements)
    const double kdiv = p.bf16 ? 6.0 : 1.0, es = p.bf16 ? 4.0 : 2.0;
    double M = p.M, N = p.geglu ? 2.0 * p.N : p.N, Kt = (double)p.K * p.taps / kdiv, B = p.batch;
    rec.flops = 2.0 * M * N * Kt * B;
    // algorithmic bytes: A once (conv: the input image once), B once, C once (+ residual / bias reads)
    double a_bytes = (p.bh > 0 ? M * (p.K / kdiv) : M * Kt) * es * B;
    rec.bytes = a_bytes + N * Kt * es * (p.bh > 0 ? 1.0 : B) + M * p.N * es * B * (p.residual ? 2.0 : 1.0) + (p.bias ? N * es : 0.0);
    rec.M = p.M; rec.N = (int)N; rec.K = p.K; rec.taps = p.taps; rec.batch = p.batch; rec.split = p.split_k; rec.conv = p.bh > 0;
    rec.bm = p.bm; rec.bn = p.bn; rec.kmajor = p.b_kmajor;
    cudaEventRecord(rec.a, st);
}

using TcKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, TcParams);

// the instantiation, with its shared-memory limit raised once
template <int BM, int BN, bool EXTRAS, int B_MN_MAJOR, bool BF16, bool PAIR, bool GEGLU = false>
TcKernel ready_kernel(int* err)
{
    static const cudaError_t e = cudaFuncSetAttribute(tc_gemm_kernel<BM, BN, EXTRAS, B_MN_MAJOR, BF16, PAIR, GEGLU>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                      TileCfg<BM, BN>::SMEM_BYTES);
    *err = (int)e;
    return tc_gemm_kernel<BM, BN, EXTRAS, B_MN_MAJOR, BF16, PAIR, GEGLU>;
}

// the kernel for a launch; nullptr when (bm, bn) is not instantiated for its B layout / epilogue / type
TcKernel pick_kernel(const TcParams& p, bool extras, bool pair, int* smem, int* err)
{
    *err = 0;
    *smem = TileCfg<BLOCK_M, BLOCK_N>::SMEM_BYTES;
    if (pair) {
        if (p.bf16 || p.split_k != 1 || p.groups > 1 || p.bm != 128 || p.bn != 128) return nullptr;
        return extras ? (p.b_kmajor ? ready_kernel<128, 128, true, 0, false, true>(err) : ready_kernel<128, 128, true, 1, false, true>(err))
                      : (p.b_kmajor ? ready_kernel<128, 128, false, 0, false, true>(err) : ready_kernel<128, 128, false, 1, false, true>(err));
    }
    if (p.geglu) {
        if (extras || p.bf16 || p.b_kmajor || p.split_k != 1 || p.groups > 1 || p.bm != 128 || p.bn != 128) return nullptr;
        return ready_kernel<128, 128, false, 1, false, false, true>(err);
    }
    if (p.bf16) {   // the fp32 path: no bias2 / statistics
        if (p.bm != 128 || p.bn != 128) return nullptr;
        return p.b_kmajor ? ready_kernel<128, 128, false, 0, true, false>(err) : ready_kernel<128, 128, false, 1, true, false>(err);
    }
#define TC_PICK_K(M_, N_, COST_) \
    if (p.bm == M_ && p.bn == N_) { *smem = TileCfg<M_, N_>::SMEM_BYTES; return extras ? ready_kernel<M_, N_, true, 0, false, false>(err) : ready_kernel<M_, N_, false, 0, false, false>(err); }
#define TC_PICK_MN(M_, N_, COST_) \
    if (p.bm == M_ && p.bn == N_) { *smem = TileCfg<M_, N_>::SMEM_BYTES; return ready_kernel<M_, N_, false, 1, false, false>(err); }
    if (p.b_kmajor) { TC_TILES_KMAJOR(TC_PICK_K) }
    else if (!extras) { TC_TILES_MNMAJOR(TC_PICK_MN) }
#undef TC_PICK_K
#undef TC_PICK_MN
    return nullptr;
}

// pair: clusters of two CTAs sharing B (the B map's box covers half a tile: 64 rows K-major, one 64-column atom MN-major)
int launch(const CUtensorMap& ma, const CUtensorMap& mb, const TcParams& p, cudaStream_t st, const CUtensorMap* mb1p = nullptr, const CUtensorMap* mb2p = nullptr,
           bool pair = false)
{
    const CUtensorMap& mb1 = mb1p ? *mb1p : mb;
    const CUtensorMap& mb2 = mb2p ? *mb2p : mb;
    const bool extras = p.bias2 != nullptr || p.gn_stats != nullptr;
    int smem = 0, err = 0;
    TcKernel k = pick_kernel(p, extras, pair, &smem, &err);
    if (err) return err;
    if (!k) return (int)cudaErrorInvalidValue;
    int grid;
    if (pair) {
        // a persistent grid must be co-resident: clusters need both SMs in one GPC, so fewer than num_sms / 2 of them may fit at once
        static int max_clusters = 0;
        if (!max_clusters) {
            cudaLaunchConfig_t cfg{};
            cfg.gridDim = dim3(2 * (num_sms() / 2)); cfg.blockDim = dim3(NUM_THREADS); cfg.dynamicSmemBytes = smem;
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
    osb_launch_cluster(k, grid, NUM_THREADS, (size_t)smem, st, pair ? 2u : 1u, ma, mb, mb1, mb2, p);
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

extern "C" void osb_tc_set_tile(int bm, int bn, int split)
{
    g_tile_bm = bm; g_tile_bn = bm < 0 ? 0 : bn; g_tile_split = bm < 0 ? 0 : split;
}

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

// One text line per recorded launch: "M N K taps batch split conv ms gflop bm bn kmajor"
extern "C" int osb_tc_profile_dump(char* buf, int cap)
{
    int off = 0;
    for (auto& r : g_prof_list) {
        float t = 0.f;
        if (cudaEventSynchronize(r.b) != cudaSuccess || cudaEventElapsedTime(&t, r.a, r.b) != cudaSuccess) return -1;
        int n = snprintf(buf + off, cap - off, "%d %d %d %d %d %d %d %.4f %.3f %d %d %d\n", r.M, r.N, r.K, r.taps, r.batch, r.split, r.conv, t, r.flops * 1e-9,
                         r.bm, r.bn, r.kmajor);
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
    const int64_t k_blocks = (K + BLOCK_K - 1) / BLOCK_K;
    const bool pair = !g_f32x && use_pair((M + BLOCK_M - 1) / BLOCK_M, N);
    // the split-K reduce reads the residual as 8-byte vectors: a residual that is not 8-byte aligned runs unsplit (scalar epilogue reads)
    const bool split_ok = ldc == N && (sc == M * N || batch == 1) && ((uintptr_t)residual & 7) == 0;
    TileProblem q{ (int)M, (int)N, 0, 0, 0, (int)batch, (int)k_blocks, bt ? 1 : 0, split_ok && !pair, g_f32x != 0 };
    OsbWorkspace* wsp = nullptr;
    const TilePick t = pair ? TilePick{ BLOCK_M, BLOCK_N, 1 } : choose_tile_ws(q, st, &wsp);
    int a_swap = 0, b_swap = 0;
    if (!make_map_rb(&ma, A, (uint64_t)K, (uint64_t)M, abatch, (uint64_t)lda * 2, (uint64_t)(sa ? sa : M * lda) * 2, BLOCK_K, t.bm, &a_swap)) return (int)cudaErrorInvalidValue;
    bool okb = bt ? make_map_rb(&mb, B, (uint64_t)K, (uint64_t)N, bbatch, (uint64_t)ldb * 2, (uint64_t)(sb ? sb : N * ldb) * 2, BLOCK_K, pair ? BLOCK_N / 2 : t.bn, &b_swap)
                  : make_map_rb(&mb, B, (uint64_t)N, (uint64_t)K, bbatch, (uint64_t)ldb * 2, (uint64_t)(sb ? sb : K * ldb) * 2, 64, BLOCK_K, &b_swap);
    if (!okb) return (int)cudaErrorInvalidValue;
    TcParams p{};
    p.M = (int)M; p.N = (int)N; p.K = (int)K; p.batch = (int)batch;
    p.bm = t.bm; p.bn = t.bn;
    p.m_tiles = (int)((M + t.bm - 1) / t.bm); p.n_tiles = (int)((N + t.bn - 1) / t.bn);
    p.b_kmajor = bt ? 1 : 0;
    p.a_swap = a_swap; p.b_swap = b_swap;
    p.taps = 1; p.kw = 1; p.bh = 0; p.bw = 0; p.tiles_x = 1;
    p.k_blocks_per_tap = (int)k_blocks;
    p.stride = 1;
    p.C = (__half*)C; p.bias = (const __half*)bias; p.residual = (const __half*)residual; p.stride_c = sc; p.ldc = ldc;
    p.split_k = t.split;
    if (pair) return launch(ma, mb, p, st, nullptr, nullptr, true);
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
    // one launch whatever the tile: the rule picks the shape, never a split
    const TilePick t = choose_tile(TileProblem{ (int)M, (int)N, 0, 0, 0, groups, (int)((K + BLOCK_K - 1) / BLOCK_K), bt ? 1 : 0, false, false });
    CUtensorMap ma, mb[3];
    int a_swap = 0, b_swap = 0;
    if (!make_map_rb(&ma, A, (uint64_t)K, (uint64_t)M, 1, (uint64_t)lda * 2, (uint64_t)(M * lda) * 2, BLOCK_K, t.bm, &a_swap)) return (int)cudaErrorInvalidValue;
    for (int g = 0; g < groups; g++) {
        int sw = 0;
        bool ok = bt ? make_map_rb(&mb[g], B[g], (uint64_t)K, (uint64_t)N, 1, (uint64_t)ldb * 2, (uint64_t)(N * ldb) * 2, BLOCK_K, t.bn, &sw)
                     : make_map_rb(&mb[g], B[g], (uint64_t)N, (uint64_t)K, 1, (uint64_t)ldb * 2, (uint64_t)(K * ldb) * 2, 64, BLOCK_K, &sw);
        if (!ok || (g > 0 && sw != b_swap)) return (int)cudaErrorInvalidValue;
        b_swap = sw;
    }
    TcParams p{};
    p.M = (int)M; p.N = (int)N; p.K = (int)K; p.batch = groups; p.groups = groups;
    p.bm = t.bm; p.bn = t.bn;
    p.m_tiles = (int)((M + t.bm - 1) / t.bm); p.n_tiles = (int)((N + t.bn - 1) / t.bn);
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

// The GEGLU feed-forward gate in the GEMM epilogue: C [M, inner] = value * gelu_erf(gate) of (A [M, K] . B [K, 2 inner] + bias [2 inner]),
// one unsplit launch of 128 x 128 tiles (64 value + 64 gate columns each), fp16, dense operands.  Measured faster than the rule's GEMM plus
// the GEGLU pass at every SD 1.5 feed-forward shape, the 8x8 level's (M = 64, where the rule's pick is a 64 x 128 tile) included (DESIGN.md
// section 5), so it has no rule of its own.
extern "C" int osb_tc_gemm_geglu(const void* A, const void* B, void* C, const void* bias, int64_t M, int64_t inner, int64_t K, void* stream)
{
    if (inner < 64 || inner % 64 || !osb_tc_gemm_ok(M, 2 * inner, K, 0, A, B, C, 0, 0, 0, K, 2 * inner, inner) || ((uintptr_t)bias & 3)) return (int)cudaErrorNotSupported;
    CUtensorMap ma, mb;
    int a_swap = 0, b_swap = 0;
    if (!make_map_rb(&ma, A, (uint64_t)K, (uint64_t)M, 1, (uint64_t)K * 2, (uint64_t)(M * K) * 2, BLOCK_K, BLOCK_M, &a_swap)) return (int)cudaErrorInvalidValue;
    if (!make_map_rb(&mb, B, (uint64_t)(2 * inner), (uint64_t)K, 1, (uint64_t)(2 * inner) * 2, (uint64_t)(2 * inner * K) * 2, 64, BLOCK_K, &b_swap))
        return (int)cudaErrorInvalidValue;
    TcParams p{};
    p.M = (int)M; p.N = (int)inner; p.K = (int)K; p.batch = 1;
    p.bm = BLOCK_M; p.bn = BLOCK_N; p.geglu = 1;
    p.m_tiles = (int)((M + BLOCK_M - 1) / BLOCK_M); p.n_tiles = (int)(inner / 64);
    p.taps = 1; p.kw = 1; p.tiles_x = 1; p.stride = 1;
    p.k_blocks_per_tap = (int)((K + BLOCK_K - 1) / BLOCK_K);
    p.C = (__half*)C; p.bias = (const __half*)bias; p.ldc = inner;
    p.split_k = 1;
    return launch(ma, mb, p, (cudaStream_t)stream);
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
    const int k_blocks = kh * kw * (int)((Cin + BLOCK_K - 1) / BLOCK_K);
    TileProblem q{ (int)(Ho * Wo), (int)Cout, (int)Ho, (int)Wo, 1, 1, k_blocks, 1, false, g_f32x != 0 };
    const bool pair = !g_f32x && Cout % 8 == 0 && use_pair(problem_m_tiles(q, BLOCK_M), Cout);
    // the split-K reduce paths move float4 / half4 vectors: ragged Cout (conv_out, 3 or 4 channels) and a residual that is not 8-byte
    // aligned run unsplit
    q.may_split = !pair && Cout % 4 == 0 && ((uintptr_t)residual & 7) == 0;
    OsbWorkspace* wsp = nullptr;
    const TilePick t = pair ? TilePick{ BLOCK_M, BLOCK_N, 1 } : choose_tile_ws(q, st, &wsp);
    const uint32_t bw = (uint32_t)conv_box_w(t.bm, (int)Wo), bh = (uint32_t)t.bm / bw;
    CUtensorMap ma, mb;
    // A: NHWC input as (C, W, H); one box = bh rows x bw pixels x 64 channels, zero-filled outside the image.  With a
    // traversal stride s the box spans bw*s x bh*s input pixels and TMA delivers every s-th one.
    if (!make_map(&ma, x, (uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)Cin * 2, (uint64_t)W * Cin * 2, BLOCK_K, bw * stride, bh * stride, (uint32_t)stride))
        return (int)cudaErrorInvalidValue;
    // B: OHWI weights = [Cout][kh*kw*Cin], K-major
    int64_t Ktot = (int64_t)kh * kw * Cin;
    if (!make_map(&mb, w, (uint64_t)Ktot, (uint64_t)Cout, 1, (uint64_t)Ktot * 2, (uint64_t)Ktot * Cout * 2, BLOCK_K, pair ? BLOCK_N / 2 : t.bn, 1))
        return (int)cudaErrorInvalidValue;
    TcParams p{};
    p.M = (int)(Ho * Wo); p.N = (int)Cout; p.K = (int)Cin; p.batch = 1;
    p.bm = t.bm; p.bn = t.bn;
    p.tiles_x = (int)((Wo + bw - 1) / bw);
    p.m_tiles = p.tiles_x * (int)((Ho + bh - 1) / bh);
    p.n_tiles = (int)((Cout + t.bn - 1) / t.bn);
    p.b_kmajor = 1;
    p.taps = kh * kw; p.kw = kw; p.pad_top = pad_top; p.pad_left = pad_left; p.Wo = (int)Wo; p.Ho = (int)Ho; p.bw = (int)bw; p.bh = (int)bh;
    p.k_blocks_per_tap = (int)((Cin + BLOCK_K - 1) / BLOCK_K);
    p.stride = stride;
    p.C = (__half*)y; p.bias = (const __half*)bias; p.residual = (const __half*)residual; p.stride_c = 0; p.ldc = Cout;
    p.split_k = t.split;
    p.ws = wsp ? wsp->splitk : nullptr;
    p.bias2 = (const __half*)bias2;
    // statistics: the tile epilogue (unsplit) or the reduce kernel (split-K; needs 4 consecutive columns inside one group)
    const bool stats_ok = gn_stats && (p.split_k == 1 || gn_cpg % 4 == 0);
    if (stats_ok) { p.gn_stats = gn_stats; p.gn_cpg = gn_cpg; p.gn_groups = gn_groups; if (gn_done) *gn_done = 1; }
    { static const int dbg = env_int("OSB_GN_DEBUG"); p.gn_debug = dbg; }
    if (pair) return launch(ma, mb, p, st, nullptr, nullptr, true);
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
static bool f32_tc_on()
{
    static const bool on = [] { const char* e = getenv("OSB_F32_TC"); return !(e && e[0] == '0'); }();
    return on;
}
extern "C" int osb_tc_gemm_f32x_ok(int64_t M, int64_t N, int64_t K)
{
    return f32_tc_on() && M >= 32 && N >= 8 && N % 8 == 0 && K >= 8 && (6 * K) % 8 == 0 && (size_t)M * N * 4 <= WS_MAX && get_encode() != nullptr ? 1 : 0;
}
extern "C" int osb_tc_conv_f32x_ok(int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, int64_t Ho, int64_t Wo)
{
    return f32_tc_on() && (6 * Cin) % 8 == 0 && 6 * Cin >= 16 && stride >= 1 && stride <= 2 && H * W >= 64 && kh <= 7 && kw <= 7 && (size_t)Ho * Wo * Cout * 4 <= WS_MAX &&
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

// ---- fp32 GEMM on an fp16 weight read in place ------------------------------------------------------------------------------------------
int osb_f32x_split_rows(const float* x, __nv_bfloat16* planes, int64_t rows, int64_t C, cudaStream_t st);   // attention_wgmma.cu

extern "C" int osb_tc_gemm_f32x_f16w_ok(int64_t M, int64_t N, int64_t K, int64_t ldb)
{
    return f32_tc_on() && M >= 1 && N >= 1 && K >= 8 && K % 8 == 0 && ldb % 8 == 0 && ldb >= N && M <= (1 << 30) && ldb <= (1 << 30) &&
           3 * K <= (1 << 30) && (size_t)N * 4 * BLOCK_M <= WS_MAX && get_encode() != nullptr ? 1 : 0;
}

// C [M, N] fp32 = A [M, K] fp32 . B [K, N] fp16 (rows ldb apart) + bias [N] + residual [M, N] (fp32, either may be null): the split of A into
// `planes`, then tc_gemm_f16w_kernel and the fp32 reduce, once per block of rows whose fp32 partials fit the workspace.
extern "C" int osb_tc_gemm_f32x_f16w(const void* A, const void* B, int64_t ldb, void* C, const void* bias, const void* residual, int64_t M, int64_t N,
                                     int64_t K, void* planes, void* stream)
{
    if (!osb_tc_gemm_f32x_f16w_ok(M, N, K, ldb) || !aligned16(A) || !aligned16(B) || !aligned16(planes) || ((uintptr_t)C & 3) || ((uintptr_t)bias & 3) ||
        ((uintptr_t)residual & 3))
        return (int)cudaErrorNotSupported;
    cudaStream_t st = (cudaStream_t)stream;
    OsbWorkspace* wsp = osb_workspace(st, OSB_WS_SPLITK);
    if (!wsp) return (int)cudaErrorNotSupported;
    const int64_t rows_max = std::min<int64_t>(M, (int64_t)(WS_MAX / ((size_t)N * 4)) / BLOCK_M * BLOCK_M);
    const int64_t K3 = 3 * K, kbk = (K + BLOCK_K - 1) / BLOCK_K;
    const __nv_bfloat16* pl = (const __nv_bfloat16*)planes;
    CUtensorMap mb;
    int sw = 0;
    if (!make_map_rb(&mb, B, (uint64_t)N, (uint64_t)K, 1, (uint64_t)ldb * 2, (uint64_t)(K * ldb) * 2, 64, BLOCK_K, &sw)) return (int)cudaErrorNotSupported;
    std::vector<CUtensorMap> ma((size_t)((M + rows_max - 1) / rows_max));
    for (size_t i = 0; i < ma.size(); i++) {
        const int64_t m0 = (int64_t)i * rows_max, rows = std::min(rows_max, M - m0);
        if (!make_map_rb(&ma[i], pl + m0 * K3, (uint64_t)K3, (uint64_t)rows, 1, (uint64_t)K3 * 2, (uint64_t)(rows * K3) * 2, BLOCK_K, BLOCK_M, &sw))
            return (int)cudaErrorNotSupported;
    }
    static const cudaError_t attr = cudaFuncSetAttribute(tc_gemm_f16w_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, f16w::SMEM_BYTES);
    if (attr != cudaSuccess) return (int)attr;
    int e = osb_f32x_split_rows((const float*)A, (__nv_bfloat16*)planes, M, K, st);
    if (e) return e;
    for (size_t i = 0; i < ma.size(); i++) {
        const int64_t m0 = (int64_t)i * rows_max, rows = std::min(rows_max, M - m0);
        TcParams p{};
        p.M = (int)rows; p.N = (int)N; p.K = (int)K; p.batch = 1;
        p.m_tiles = (int)((rows + BLOCK_M - 1) / BLOCK_M); p.n_tiles = (int)((N + BLOCK_N - 1) / BLOCK_N);
        p.k_blocks_per_tap = (int)kbk;
        // the fp32 path's split rule (old_split) over the raw k-blocks, each five products deep
        p.split_k = choose_tile(TileProblem{ (int)rows, (int)N, 0, 0, 0, 1, (int)kbk, 0, true, true }).split;
        if ((size_t)p.split_k * rows * N * 4 > WS_MAX) p.split_k = 1;
        p.ws = wsp->splitk;
        const int grid = (int)std::min<int64_t>((int64_t)p.m_tiles * p.n_tiles * p.split_k, num_sms());
        osb_launch((tc_gemm_f16w_kernel<false>), grid, NUM_THREADS, (size_t)f16w::SMEM_BYTES, st, ma[i], mb, p);
        if ((e = launched(1))) return e;
        const long long total = rows * N;
        osb_launch((splitk_reduce_f32_kernel), (int)std::min<long long>((total + 255) / 256, num_sms() * 8), 256, 0, st, (const float*)p.ws,
                   (float*)C + m0 * N, (const float*)bias, residual ? (const float*)residual + m0 * N : nullptr, (long long)rows, (int)N, p.split_k);
        if ((e = launched())) return e;
    }
    return 0;
}

// ---- fp32 conv on an fp16 weight read in place ------------------------------------------------------------------------------------------
// The shapes of osb_tc_conv_ok; the output is stored from the registers, so its size is not bounded by the workspace.
extern "C" int osb_tc_conv_f32x_f16w_ok(int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, int64_t Ho, int64_t Wo)
{
    return f32_tc_on() && Cout >= 1 && kh >= 1 && kw >= 1 && Ho >= 1 && Wo >= 1 && Ho * Wo <= (1 << 30) && Cout <= (1 << 30) &&
           (int64_t)kh * kw * Cin <= (1 << 30) && osb_tc_conv_ok(H, W, Cin, Cout, kh, kw, stride, nullptr, nullptr, nullptr) ? 1 : 0;
}

// y [Ho, Wo, Cout] fp32 = conv(x [H, W, Cin] fp32, float(w) [Cout][kh][kw][Cin] fp16) + bias [Cout] + residual [Ho, Wo, Cout] (fp32, either may
// be null): the split of x into `planes`, tc_gemm_f16w_kernel<true>, and the fp32 reduce when the launch splits K.
extern "C" int osb_tc_conv_f32x_f16w(const void* x, const void* w, const void* bias, const void* residual, void* y, int64_t H, int64_t W, int64_t Cin,
                                     int64_t Cout, int kh, int kw, int stride, int pad_top, int pad_left, int64_t Ho, int64_t Wo, void* planes, void* stream)
{
    if (!osb_tc_conv_f32x_f16w_ok(H, W, Cin, Cout, kh, kw, stride, Ho, Wo) || !aligned16(x) || !aligned16(w) || !aligned16(planes) || ((uintptr_t)y & 7) ||
        ((uintptr_t)bias & 3) || ((uintptr_t)residual & 7))
        return (int)cudaErrorNotSupported;
    cudaStream_t st = (cudaStream_t)stream;
    const int kbpt = (int)((Cin + BLOCK_K - 1) / BLOCK_K), k_blocks = kh * kw * kbpt;
    const int64_t M = Ho * Wo;
    // the fp32 path's split rule (old_split) over the raw k-blocks, each five products deep; osb_tc_set_tile's forced split, clamped so
    // that no split is empty.  A split runs only where its partials fit the workspace; unsplit, the kernel stores the output itself.
    int split = choose_tile(TileProblem{ (int)M, (int)Cout, (int)Ho, (int)Wo, 1, 1, k_blocks, 1, true, true }).split;
    if (g_tile_split > 0) {
        split = std::min(g_tile_split, k_blocks);
        if (split > 1) { const int kb_per = (k_blocks + split - 1) / split; split = (k_blocks + kb_per - 1) / kb_per; }
    }
    if ((size_t)split * M * Cout * 4 > WS_MAX) split = 1;
    OsbWorkspace* wsp = split > 1 ? osb_workspace(st, OSB_WS_SPLITK) : nullptr;
    if (!wsp) split = 1;
    const uint32_t bw = (uint32_t)conv_box_w(BLOCK_M, (int)Wo), bh = BLOCK_M / bw;
    CUtensorMap ma, mb;
    // A: the planes [H][W][3][Cin] as (Cin, plane, W, H); one box = one plane of bh rows x bw pixels x 64 channels
    if (!make_map_4d(&ma, planes, (uint64_t)Cin, 3, (uint64_t)W, (uint64_t)H, (uint64_t)Cin * 2, (uint64_t)Cin * 6, (uint64_t)W * Cin * 6, BLOCK_K, 1,
                     bw * stride, bh * stride, (uint32_t)stride))
        return (int)cudaErrorNotSupported;
    // B: OHWI weights = [Cout][kh*kw*Cin], K-major
    const int64_t Ktot = (int64_t)kh * kw * Cin;
    if (!make_map(&mb, w, (uint64_t)Ktot, (uint64_t)Cout, 1, (uint64_t)Ktot * 2, (uint64_t)Ktot * Cout * 2, BLOCK_K, BLOCK_N, 1)) return (int)cudaErrorNotSupported;
    static const cudaError_t attr = cudaFuncSetAttribute(tc_gemm_f16w_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, f16w::SMEM_BYTES);
    if (attr != cudaSuccess) return (int)attr;
    TcParams p{};
    p.M = (int)M; p.N = (int)Cout; p.K = (int)Cin; p.batch = 1;
    p.bm = BLOCK_M; p.bn = BLOCK_N;
    p.tiles_x = (int)((Wo + bw - 1) / bw);
    p.m_tiles = p.tiles_x * (int)((Ho + bh - 1) / bh);
    p.n_tiles = (int)((Cout + BLOCK_N - 1) / BLOCK_N);
    p.b_kmajor = 1;
    p.taps = kh * kw; p.kw = kw; p.pad_top = pad_top; p.pad_left = pad_left; p.Wo = (int)Wo; p.Ho = (int)Ho; p.bw = (int)bw; p.bh = (int)bh;
    p.k_blocks_per_tap = kbpt;
    p.stride = stride;
    p.C = (__half*)y; p.bias = (const __half*)bias; p.residual = (const __half*)residual; p.ldc = Cout;   // fp32 (see the kernel)
    p.split_k = split;
    p.ws = wsp ? wsp->splitk : nullptr;
    int e = osb_f32x_split_rows((const float*)x, (__nv_bfloat16*)planes, H * W, Cin, st);
    if (e) return e;
    const int grid = (int)std::min<int64_t>((int64_t)p.m_tiles * p.n_tiles * split, num_sms());
    osb_launch((tc_gemm_f16w_kernel<true>), grid, NUM_THREADS, (size_t)f16w::SMEM_BYTES, st, ma, mb, p);
    if ((e = launched(1))) return e;
    if (split == 1) return 0;
    const long long total = M * Cout;
    osb_launch((splitk_reduce_f32_kernel), (int)std::min<long long>((total + 255) / 256, num_sms() * 8), 256, 0, st, (const float*)p.ws, (float*)y,
               (const float*)bias, (const float*)residual, (long long)M, (int)Cout, split);
    return launched();
}

// ---- fp32 GEMM and conv on a uint8 weight read in place ---------------------------------------------------------------------------------
// The split rule of the fp16-weight launches (old_split: fewer than 100 tiles fill the SMs, >= 2 k-blocks per split) over the raw k-blocks,
// from 10 of them instead of 32: a k-block here is three products deep.  SDXL's few-tile launches of 10-31 k-blocks (the 1x1 skip convs at
// 16 x 16 and 32 x 32, its 256-row GEMMs) ran up to 1.6x slower than the expanded route unsplit and 1.1-1.5x faster split (H100, DESIGN.md
// section 5).  osb_tc_set_tile's forced split, clamped so that no split is empty; a split runs only where its partials fit the workspace
// (unsplit, the kernel stores the output).
static int u8w_split(const TileProblem& q, int k_blocks, size_t out_elems)
{
    int split = old_split(problem_m_tiles(q, BLOCK_M) * ((q.N + BLOCK_N - 1) / BLOCK_N), k_blocks, out_elems, 10);
    if (g_tile_split > 0) {
        split = std::min(g_tile_split, k_blocks);
        if (split > 1) { const int kb_per = (k_blocks + split - 1) / split; split = (k_blocks + kb_per - 1) / kb_per; }
    }
    if ((size_t)split * out_elems * 4 > WS_MAX) split = 1;
    return split;
}

// the uint8 launch: the split of the activation into `planes` (done by the caller), tc_gemm_u8w_kernel, and the fp32 reduce
// when the launch splits K
template <bool CONV>
static int u8w_launch(const CUtensorMap& ma, const CUtensorMap& mb, TcParams& p, int split, const void* y, const void* bias, const void* residual, cudaStream_t st)
{
    static const cudaError_t attr = cudaFuncSetAttribute(tc_gemm_u8w_kernel<CONV>, cudaFuncAttributeMaxDynamicSharedMemorySize, f16w::U8_SMEM_BYTES);
    if (attr != cudaSuccess) return (int)attr;
    OsbWorkspace* wsp = split > 1 ? osb_workspace(st, OSB_WS_SPLITK) : nullptr;
    if (!wsp) split = 1;
    p.split_k = split;
    p.ws = wsp ? wsp->splitk : nullptr;
    p.C = (__half*)y; p.bias = (const __half*)bias; p.residual = (const __half*)residual; p.ldc = p.N;   // fp32 (see the kernel)
    const int grid = (int)std::min<int64_t>((int64_t)p.m_tiles * p.n_tiles * split, num_sms());
    osb_launch((tc_gemm_u8w_kernel<CONV>), grid, NUM_THREADS, (size_t)f16w::U8_SMEM_BYTES, st, ma, mb, p);
    int e = launched(1);
    if (e || split == 1) return e;
    const long long total = (long long)p.M * p.N;
    osb_launch((splitk_reduce_f32_kernel), (int)std::min<long long>((total + 255) / 256, num_sms() * 8), 256, 0, st, (const float*)p.ws, (float*)y,
               (const float*)bias, (const float*)residual, (long long)p.M, p.N, split);
    return launched();
}

extern "C" int osb_tc_gemm_f32x_u8w_ok(int64_t M, int64_t N, int64_t K, int64_t ldb, int zero_point)
{
    return f32_tc_on() && M >= 1 && N >= 1 && K >= 8 && K % 8 == 0 && ldb % 16 == 0 && ldb >= N && M <= (1 << 30) && ldb <= (1 << 30) &&
           3 * K <= (1 << 30) && zero_point >= 0 && zero_point <= 255 && get_encode() != nullptr ? 1 : 0;
}

// C [M, N] fp32 = A [M, K] fp32 . ((B [K, N] uint8, rows ldb apart) - zero_point) scale + bias [N] + residual [M, N] (fp32, either may be null)
extern "C" int osb_tc_gemm_f32x_u8w(const void* A, const void* B, int64_t ldb, void* C, const void* bias, const void* residual, int64_t M, int64_t N,
                                    int64_t K, float scale, int zero_point, void* planes, void* stream)
{
    if (!osb_tc_gemm_f32x_u8w_ok(M, N, K, ldb, zero_point) || !aligned16(A) || !aligned16(B) || !aligned16(planes) || ((uintptr_t)C & 7) ||
        ((uintptr_t)bias & 3) || ((uintptr_t)residual & 7))
        return (int)cudaErrorNotSupported;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t K3 = 3 * K;
    const int kbk = (int)((K + BLOCK_K - 1) / BLOCK_K);
    CUtensorMap ma, mb;
    int sw = 0;
    // A: the planes [M][3][K] as one [M, 3 K] map (a chunk past K reads the next plane, against B rows the converters zero)
    if (!make_map_rb(&ma, planes, (uint64_t)K3, (uint64_t)M, 1, (uint64_t)K3 * 2, (uint64_t)(M * K3) * 2, BLOCK_K, BLOCK_M, &sw)) return (int)cudaErrorNotSupported;
    // B: the [K][N] uint8 blob, one unswizzled [64 k][128 n] box per k-block
    if (!make_map(&mb, B, (uint64_t)N, (uint64_t)K, 1, (uint64_t)ldb, (uint64_t)(K * ldb), BLOCK_N, BLOCK_K, 1, 1, CU_TENSOR_MAP_DATA_TYPE_UINT8,
                  CU_TENSOR_MAP_SWIZZLE_NONE))
        return (int)cudaErrorNotSupported;
    TcParams p{};
    p.M = (int)M; p.N = (int)N; p.K = (int)K; p.batch = 1;
    p.bm = BLOCK_M; p.bn = BLOCK_N;
    p.m_tiles = (int)((M + BLOCK_M - 1) / BLOCK_M); p.n_tiles = (int)((N + BLOCK_N - 1) / BLOCK_N);
    p.k_blocks_per_tap = kbk;
    p.wscale = scale; p.wzero = zero_point;
    const int split = u8w_split(TileProblem{ (int)M, (int)N, 0, 0, 0, 1, kbk, 0, true, true }, kbk, (size_t)M * N);
    int e = osb_f32x_split_rows((const float*)A, (__nv_bfloat16*)planes, M, K, st);
    if (e) return e;
    return u8w_launch<false>(ma, mb, p, split, C, bias, residual, st);
}

extern "C" int osb_tc_conv_f32x_u8w_ok(int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, int64_t Ho, int64_t Wo, int zero_point)
{
    return osb_tc_conv_f32x_f16w_ok(H, W, Cin, Cout, kh, kw, stride, Ho, Wo) && ((int64_t)kh * kw * Cin) % 16 == 0 && zero_point >= 0 && zero_point <= 255 ? 1 : 0;
}

// y [Ho, Wo, Cout] fp32 = conv(x [H, W, Cin] fp32, (w [Cout][kh][kw][Cin] uint8 - zero_point) scale) + bias [Cout] + residual [Ho, Wo, Cout]
extern "C" int osb_tc_conv_f32x_u8w(const void* x, const void* w, const void* bias, const void* residual, void* y, int64_t H, int64_t W, int64_t Cin,
                                    int64_t Cout, int kh, int kw, int stride, int pad_top, int pad_left, int64_t Ho, int64_t Wo, float scale, int zero_point,
                                    void* planes, void* stream)
{
    if (!osb_tc_conv_f32x_u8w_ok(H, W, Cin, Cout, kh, kw, stride, Ho, Wo, zero_point) || !aligned16(x) || !aligned16(w) || !aligned16(planes) ||
        ((uintptr_t)y & 7) || ((uintptr_t)bias & 3) || ((uintptr_t)residual & 7))
        return (int)cudaErrorNotSupported;
    cudaStream_t st = (cudaStream_t)stream;
    const int kbpt = (int)((Cin + BLOCK_K - 1) / BLOCK_K), k_blocks = kh * kw * kbpt;
    const int64_t M = Ho * Wo, Ktot = (int64_t)kh * kw * Cin;
    const uint32_t bw = (uint32_t)conv_box_w(BLOCK_M, (int)Wo), bh = BLOCK_M / bw;
    CUtensorMap ma, mb;
    // A: the planes [H][W][3][Cin] as (Cin, plane, W, H), as in osb_tc_conv_f32x_f16w
    if (!make_map_4d(&ma, planes, (uint64_t)Cin, 3, (uint64_t)W, (uint64_t)H, (uint64_t)Cin * 2, (uint64_t)Cin * 6, (uint64_t)W * Cin * 6, BLOCK_K, 1,
                     bw * stride, bh * stride, (uint32_t)stride))
        return (int)cudaErrorNotSupported;
    // B: the OHWI uint8 blob [Cout][kh kw Cin], one unswizzled [128 n][64 k] box per k-block
    if (!make_map(&mb, w, (uint64_t)Ktot, (uint64_t)Cout, 1, (uint64_t)Ktot, (uint64_t)(Ktot * Cout), BLOCK_K, BLOCK_N, 1, 1, CU_TENSOR_MAP_DATA_TYPE_UINT8,
                  CU_TENSOR_MAP_SWIZZLE_NONE))
        return (int)cudaErrorNotSupported;
    TcParams p{};
    p.M = (int)M; p.N = (int)Cout; p.K = (int)Cin; p.batch = 1;
    p.bm = BLOCK_M; p.bn = BLOCK_N;
    p.tiles_x = (int)((Wo + bw - 1) / bw);
    p.m_tiles = p.tiles_x * (int)((Ho + bh - 1) / bh);
    p.n_tiles = (int)((Cout + BLOCK_N - 1) / BLOCK_N);
    p.b_kmajor = 1;
    p.taps = kh * kw; p.kw = kw; p.pad_top = pad_top; p.pad_left = pad_left; p.Wo = (int)Wo; p.Ho = (int)Ho; p.bw = (int)bw; p.bh = (int)bh;
    p.k_blocks_per_tap = kbpt;
    p.stride = stride;
    p.wscale = scale; p.wzero = zero_point;
    const int split = u8w_split(TileProblem{ (int)M, (int)Cout, (int)Ho, (int)Wo, 1, 1, k_blocks, 1, true, true }, k_blocks, (size_t)M * Cout);
    int e = osb_f32x_split_rows((const float*)x, (__nv_bfloat16*)planes, H * W, Cin, st);
    if (e) return e;
    return u8w_launch<true>(ma, mb, p, split, y, bias, residual, st);
}
