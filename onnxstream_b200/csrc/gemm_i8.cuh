// gemm_i8.cuh -- W8A8 on the tensor cores: `wgmma ... .s32.u8.u8`, uint8 x uint8 -> int32 in registers (included by gemm_wgmma.cu).
//
// Replaces XnnPack::matrix_multiply<uint8_t,int32_t> / convolution for T = uint8_t (src/onnxstream.cpp:1035-1215, 1292-1534; the reference
// drives XNNPACK's qu8 GEMM / conv with the parameters of Qu8MatMulData / Qu8ConvData, 1025-1033) for the shapes TMA can address
// (16-byte strides); other shapes stay on the CUDA-core igemm_kernel (kernels_gemm.cu), same arithmetic.
//
// Arithmetic (bit-exact with XNNPACK's "fp32" requantisation, pinned in tests against the reference run):
//     acc[m,n] = sum_k (x[m,k] - zx) * (w[k,n] - zw) + bias[n]                    (int32)
//     y[m,n]   = clamp(lrintf(acc * (sx * sw / sy)), 0 - zy, 255 - zy) + zy       (uint8)
// The tensor core multiplies the RAW unsigned bytes: raw[m,n] = sum_k x*w, and the epilogue applies
//     acc = raw - zw * rowsum_x[m] - zx * colsum_w[n] + K * zx * zw + bias[n]
// with rowsum_x / colsum_w from small byte-sum kernels.  A convolution pads with the INPUT ZERO POINT in XNNPACK, while TMA fills
// out-of-bounds elements with 0: the host therefore pads the NHWC image once (value zx, kernel in this file) and the conv runs
// un-padded on it, so every tap of every output pixel is a real byte and rowsum_x[m] is the sum of kh*kw per-pixel channel sums.
//
// Structure = tc_gemm_kernel (warp 0 TMA producer, warpgroups 1 and 2 MMA + epilogue on 64 rows each), with 128-byte k-blocks = 128
// elements, m64n128k32 MMAs.  A is K-major; B is K-major (OHWI conv weights) or MN-major ([K,N] MatMul weights).  wgmma reads 8-bit
// operands K-major only, so an MN-major B k-block lands in a staging buffer and warps 1..3 of the producer warpgroup transpose it
// into the K-major swizzled stage the MMAs read.

namespace i8k {

constexpr int I8_BLOCK_K = 128;        // elements = bytes: one 128B swizzle row
constexpr int I8_WG_K = 32;
constexpr int I8_STAGES = 4;
constexpr int I8_STAGE_BYTES = A_STAGE_BYTES + 2 * B_STAGE_BYTES;   // A, B, the MN-major staging buffer
constexpr int I8_SMEM = I8_STAGES * I8_STAGE_BYTES + 1024 + 256;
constexpr int TRANSPOSE_THREADS = 96;

struct I8Params {
    int M, N, K;                 // GEMM view (conv: M = Ho*Wo, K = Cin per tap)
    int m_tiles, n_tiles;
    int b_kmajor;
    int taps, kw, Wo, Ho, bw, bh, tiles_x, k_blocks_per_tap, stride;
    int Wp;                      // conv: width of the zero-point-padded image (rows of `psum`)
    const int32_t* rsum;         // GEMM: rowsum_x[M];  conv: per-pixel channel sums of the padded image [Hp * Wp]
    const int32_t* csum;         // colsum_w[N]
    const int32_t* bias;         // int32 bias[N] or null
    int zx, zw, zy;
    int kzz;                     // K_total * zx * zw
    float requant;               // sx * sw / sy
    uint8_t* C;
    long long ldc;
};

__global__ void __launch_bounds__(NUM_THREADS, 1)
tc_i8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const I8Params p)
{
    osb_pdl_trigger_entry();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + I8_STAGES * A_STAGE_BYTES;
    uint8_t* smem_stg = smem_b + I8_STAGES * B_STAGE_BYTES;
    uint64_t* bars = (uint64_t*)(smem + I8_STAGES * I8_STAGE_BYTES);
    uint64_t* full = bars;                    // [I8_STAGES] A and (K-major) B landed / (MN-major) B transposed
    uint64_t* empty = bars + I8_STAGES;       // [I8_STAGES] consumers are done with the stage
    uint64_t* stg_full = empty + I8_STAGES;   // [I8_STAGES] MN-major B landed in the staging buffer

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < I8_STAGES; i++) {
            mbar_init(&full[i], p.b_kmajor ? 1 : 2);   // MN-major: the TMA of A and the transposers' arrival
            mbar_init(&empty[i], CONSUMER_THREADS);
            mbar_init(&stg_full[i], 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    osb_pdl_wait();

    const int total_tiles = p.m_tiles * p.n_tiles;
    const int k_blocks = p.taps * p.k_blocks_per_tap;

    if (warp == 0) {
        // ===================== TMA producer =====================
        const uint32_t sa0 = smem_u32(smem_a), sb0 = smem_u32(smem_b), sg0 = smem_u32(smem_stg);
        int stage = 0; uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int mt = tile % p.m_tiles, nt = tile / p.m_tiles;
            const int n0 = nt * BLOCK_N, m0 = mt * BLOCK_M;
            int y0 = 0, x0 = 0;
            if (p.bh > 0) { y0 = (mt / p.tiles_x) * p.bh; x0 = (mt % p.tiles_x) * p.bw; }
            int tap = 0, kcb = 0, ky = 0, kx = 0;
            const int ax = x0 * p.stride, ay = y0 * p.stride;       // the image is already padded: no negative coordinates
            for (int kb = 0; kb < k_blocks; kb++) {
                mbar_wait(&empty[stage], phase ^ 1);
                if (elect_one()) {
                    const int kc = kcb * I8_BLOCK_K;
                    const uint32_t sa = sa0 + stage * A_STAGE_BYTES;
                    const int kglob = tap * p.K + kc;
                    if (p.b_kmajor) {
                        mbar_expect_tx(&full[stage], A_STAGE_BYTES + B_STAGE_BYTES);
                        tma_load_3d_s(sb0 + stage * B_STAGE_BYTES, &map_b, &full[stage], kglob, n0, 0);
                    } else {
                        mbar_expect_tx(&full[stage], A_STAGE_BYTES);
                        mbar_expect_tx(&stg_full[stage], B_STAGE_BYTES);
                        tma_load_3d_s(sg0 + stage * B_STAGE_BYTES, &map_b, &stg_full[stage], n0, kglob, 0);   // 128 columns x 128 k-rows
                    }
                    if (p.bh > 0) tma_load_3d_s(sa, &map_a, &full[stage], kc, ax + kx, ay + ky);
                    else tma_load_3d_s(sa, &map_a, &full[stage], kc, m0, 0);
                }
                __syncwarp();
                if (++kcb == p.k_blocks_per_tap) { kcb = 0; tap++; if (++kx == p.kw) { kx = 0; ky++; } }
                if (++stage == I8_STAGES) { stage = 0; phase ^= 1; }
            }
        }
        osb_pdl_trigger_late();
    } else if (warp < 4) {
        // ===================== transposers (MN-major B only): staging [k][n] -> B stage [n][k], both 128B-swizzled =====================
        if (p.b_kmajor) return;
        const int t = (int)threadIdx.x - 32;
        int stage = 0; uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            for (int kb = 0; kb < k_blocks; kb++) {
                mbar_wait(&stg_full[stage], phase);
                const uint8_t* stg = smem_stg + stage * B_STAGE_BYTES;
                uint8_t* dst = smem_b + stage * B_STAGE_BYTES;
                for (int n = t; n < BLOCK_N; n += TRANSPOSE_THREADS) {
#pragma unroll
                    for (int c = 0; c < I8_BLOCK_K / 16; c++) {
                        uint32_t w[4];
#pragma unroll
                        for (int q = 0; q < 4; q++) {
                            uint32_t v = 0;
#pragma unroll
                            for (int e = 0; e < 4; e++) {
                                const int k = 16 * c + 4 * q + e;   // row k of the staging tile: 16-byte unit (n / 16) sits at unit (n / 16) ^ (k % 8)
                                v |= (uint32_t)stg[k * 128 + ((((n >> 4) ^ (k & 7))) << 4) + (n & 15)] << (8 * e);
                            }
                            w[q] = v;
                        }
                        *reinterpret_cast<uint4*>(dst + n * 128 + ((c ^ (n & 7)) << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor cores
                asm volatile("bar.sync 2, %0;" ::"n"(TRANSPOSE_THREADS) : "memory");
                if (t == 0) mbar_arrive(&full[stage]);
                if (++stage == I8_STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // ===================== consumers: MMA + zero-point corrections + fp32 requantisation =====================
        const int wg = (warp >> 2) - 1;
        const uint64_t adesc0 = make_smem_desc(smem_u32(smem_a) + wg * (BLOCK_M / 2) * 128, 16, 1024);
        const uint64_t bdesc0 = make_smem_desc(smem_u32(smem_b), 16, 1024);
        const uint32_t kstep = I8_WG_K >> 4;                                      // 32 bytes along K, both operands
        const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);
        int stage = 0; uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int mt = tile % p.m_tiles, nt = tile / p.m_tiles;
            const int n0 = nt * BLOCK_N;
            const int n_end = min(p.N, n0 + BLOCK_N);
            int32_t acc[64];
#pragma unroll
            for (int i = 0; i < 64; i++) acc[i] = 0;
            int prev = -1;
            for (int kb = 0; kb < k_blocks; kb++) {
                mbar_wait(&full[stage], phase);
                const uint64_t adesc = adesc0 + (uint64_t)(stage * (A_STAGE_BYTES >> 4));
                const uint64_t bdesc = bdesc0 + (uint64_t)(stage * (B_STAGE_BYTES >> 4));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < I8_BLOCK_K / I8_WG_K; k++) wgmma_m64n128k32_u8(acc, adesc + (uint64_t)(k * kstep), bdesc + (uint64_t)(k * kstep), 1u);
                wgmma_commit();
                if (prev >= 0) { wgmma_wait<1>(); mbar_arrive(&empty[prev]); }
                prev = stage;
                if (++stage == I8_STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            mbar_arrive(&empty[prev]);
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int row_in_tile = r_lo + 8 * h;
                long long out_row; bool row_ok; int rs = 0;
                if (p.bh > 0) {
                    const int y = (mt / p.tiles_x) * p.bh + row_in_tile / p.bw, x = (mt % p.tiles_x) * p.bw + row_in_tile % p.bw;
                    row_ok = y < p.Ho && x < p.Wo;
                    out_row = (long long)y * p.Wo + x;
                    if (row_ok) {
                        const int kh = p.taps / p.kw;
                        for (int ky = 0; ky < kh; ky++)
                            for (int kx = 0; kx < p.kw; kx++) rs += p.rsum[(long long)(y * p.stride + ky) * p.Wp + (x * p.stride + kx)];
                    }
                } else {
                    const int m = mt * BLOCK_M + row_in_tile;
                    row_ok = m < p.M;
                    out_row = m;
                    if (row_ok) rs = p.rsum[m];
                }
                if (!row_ok) continue;
                const int row_term = p.kzz - p.zw * rs;
                uint8_t* crow = p.C + out_row * p.ldc;
#pragma unroll
                for (int j = 0; j < BLOCK_N / 8; j++) {
                    const int n = n0 + 8 * j + cq;
                    if (n >= n_end) break;            // N % 16 == 0: both columns of the pair are inside
                    uint32_t o2 = 0;
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        int a = acc[4 * j + 2 * h + e] + row_term - p.zx * __ldg(p.csum + n + e);
                        if (p.bias) a += __ldg(p.bias + n + e);
                        float f = (float)a * p.requant;
                        f = fminf(fmaxf(f, (float)(0 - p.zy)), (float)(255 - p.zy));
                        o2 |= ((uint32_t)((int)rintf(f) + p.zy) & 0xFFu) << (8 * e);
                    }
                    *reinterpret_cast<uint16_t*>(crow + n) = (uint16_t)o2;
                }
            }
        }
    }
}

// ---- byte-sum helpers -----------------------------------------------------------------------------------------------

// out[r] = sum of the `cols` bytes of row r (row sums of A, column sums of K-major weights [N][K]); one warp per row
__global__ void rowsum_u8_kernel(const uint8_t* __restrict__ x, int32_t* __restrict__ out, long long rows, long long cols)
{
    osb_pdl_prologue();
    const int lane = threadIdx.x & 31;
    for (long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows; r += (long long)gridDim.x * (blockDim.x >> 5)) {
        const uint8_t* row = x + r * cols;
        int s = 0;
        long long c = 0;
        if (((uintptr_t)row & 15) == 0)
            for (c = (long long)lane * 16; c + 16 <= cols; c += 512) {
                const uint4 v = *reinterpret_cast<const uint4*>(row + c);
                s = (int)__dp4a((unsigned)v.x, 0x01010101u, (unsigned)s); s = (int)__dp4a((unsigned)v.y, 0x01010101u, (unsigned)s); s = (int)__dp4a((unsigned)v.z, 0x01010101u, (unsigned)s); s = (int)__dp4a((unsigned)v.w, 0x01010101u, (unsigned)s);
            }
        // tail (and the unaligned case): bytes not covered by the vector loop
        const long long done = ((uintptr_t)row & 15) == 0 ? (cols / 16) * 16 : 0;
        for (long long t = done + lane; t < cols; t += 32) s += row[t];
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) out[r] = s;
    }
}

// out[n] = sum over k of w[k][n] for an MN-major weight matrix [K][N] (ONNX MatMul layout): thread per column, K split over blockIdx.y
__global__ void colsum_u8_kernel(const uint8_t* __restrict__ w, int32_t* __restrict__ out, long long K, long long N, long long k_per)
{
    osb_pdl_prologue();
    const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const long long k0 = (long long)blockIdx.y * k_per, k1 = min(K, k0 + k_per);
    int s = 0;
    for (long long k = k0; k < k1; k++) s += w[k * N + n];
    atomicAdd(&out[n], s);
}

// Pads an NHWC uint8 image with the input zero point (what XNNPACK's qu8 convolution does, and TMA's zero fill cannot) and writes the
// per-pixel channel sums of the padded image: xp[Hp][Wp][C], psum[Hp * Wp].  One warp per padded pixel.
__global__ void pad_sum_u8_kernel(const uint8_t* __restrict__ x, uint8_t* __restrict__ xp, int32_t* __restrict__ psum, int H, int W, int C, int Hp, int Wp,
                                  int pad_top, int pad_left, int zx)
{
    osb_pdl_prologue();
    const int lane = threadIdx.x & 31;
    const long long pixels = (long long)Hp * Wp;
    for (long long pix = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pix < pixels; pix += (long long)gridDim.x * (blockDim.x >> 5)) {
        const int yp = (int)(pix / Wp), xq = (int)(pix % Wp);
        const int y = yp - pad_top, xx = xq - pad_left;
        uint8_t* dst = xp + pix * C;
        int s = 0;
        if (y >= 0 && y < H && xx >= 0 && xx < W) {
            const uint8_t* src = x + ((long long)y * W + xx) * C;
            for (int c = lane * 16; c < C; c += 512) {          // C % 16 == 0
                const uint4 v = *reinterpret_cast<const uint4*>(src + c);
                *reinterpret_cast<uint4*>(dst + c) = v;
                s = (int)__dp4a((unsigned)v.x, 0x01010101u, (unsigned)s); s = (int)__dp4a((unsigned)v.y, 0x01010101u, (unsigned)s); s = (int)__dp4a((unsigned)v.z, 0x01010101u, (unsigned)s); s = (int)__dp4a((unsigned)v.w, 0x01010101u, (unsigned)s);
            }
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        } else {
            const uint32_t z4 = (uint32_t)zx * 0x01010101u;
            for (int c = lane * 16; c < C; c += 512) *reinterpret_cast<uint4*>(dst + c) = make_uint4(z4, z4, z4, z4);
            s = zx * C;
        }
        if (lane == 0) psum[pix] = s;
    }
}

}  // namespace i8k
