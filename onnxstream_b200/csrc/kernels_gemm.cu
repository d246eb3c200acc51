// kernels_gemm.cu -- dispatch for MatMul/Gemm/Conv plus the CUDA-core implicit-GEMM kernels that serve as
//   (a) the fp32 path (bit-faithful fp32 FMA accumulation, needed for parity with the reference's f32 XNNPACK path),
//   (b) the fallback for fp16 problems the tensor-core kernel (gemm_wgmma.cu) does not take (ragged K, tiny M/N),
//   (c) the qu8 (W8A8) path with XNNPACK's exact requantisation.
// The tensor-core path for fp16 lives in gemm_wgmma.cu; osb_gemm/osb_conv2d choose between them.
//
// One kernel template covers GEMM and convolution: a convolution is a GEMM whose A operand is gathered on the fly
// from the NHWC input (M = Ho*Wo, K = kh*kw*Cin in OHWI order, N = Cout, B = the OHWI weights read as [N, K]).

#include "common.cuh"
#include "workspace.h"
#include <cstdlib>

// implemented in gemm_wgmma.cu
int osb_tc_gemm_launch(const void* A, const void* B, void* C, const void* bias, const void* residual,
                       int64_t batch, int64_t M, int64_t N, int64_t K, int64_t sa, int64_t sb, int64_t sc,
                       int b_transposed, cudaStream_t st, int64_t lda, int64_t ldb, int64_t ldc);
int osb_tc_conv_launch(const void* x, const void* w, const void* bias, const void* residual, void* y,
                       int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, int pad_top, int pad_left,
                       int64_t Ho, int64_t Wo, cudaStream_t st, const void* bias2, double* gn_stats, int gn_groups, int* gn_done);
int osb_tc_gemm_grouped_launch(const void* A, const void* const* B, void* const* C, int groups, int64_t M, int64_t N, int64_t K, int bt, cudaStream_t st,
                               int64_t lda, int64_t ldb, int64_t ldc);
bool osb_tc_gemm_ok(int64_t M, int64_t N, int64_t K, int b_transposed, const void* A, const void* B, const void* C, int64_t sa, int64_t sb, int64_t sc,
                    int64_t lda, int64_t ldb, int64_t ldc);
bool osb_tc_conv_ok(int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, const void* x, const void* w, const void* y);

namespace {

struct ConvGeom {
    int H, W, Cin, kh, kw, stride, pad_top, pad_left, Ho, Wo;
};

constexpr int BM = 64, BN = 64, BK = 16;

// acc type: float for f32/f16, int for u8
template <typename T, bool CONV, bool QU8>
__global__ void __launch_bounds__(256)
igemm_kernel(const T* __restrict__ A, const T* __restrict__ B, T* __restrict__ C,
             const void* __restrict__ bias, const T* __restrict__ residual,
             int M, int N, int K, int64_t sa, int64_t sb, int64_t sc, int b_transposed, ConvGeom g,
             int zx, int zw, int zy, float requant, int lda, int ldb, int ldc)
{
    if (lda <= 0) lda = K;
    if (ldb <= 0) ldb = b_transposed ? K : N;
    if (ldc <= 0) ldc = N;
    osb_pdl_prologue();
    using Acc = typename std::conditional<QU8, int, float>::type;
    __shared__ Acc As[BK][BM + 4];
    __shared__ Acc Bs[BK][BN + 4];

    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;  // 16 x 16 threads, each 4x4 outputs
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int64_t bz = blockIdx.z;
    A += bz * sa; B += bz * sb; C += bz * sc;
    if (residual) residual += bz * sc;

    Acc acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0;

    // loader mapping: A tile 64x16 -> 1024 elements, 4 per thread; B tile 16x64 likewise
    for (int k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
        for (int e = 0; e < 4; e++) {
            int idx = tid + e * 256;
            // A: idx -> (m, k) with k fastest (contiguous in memory for GEMM rows / conv channels)
            int am = idx / BK, ak = idx % BK;
            int m = m0 + am, k = k0 + ak;
            Acc v = 0;
            if (m < M && k < K) {
                if (CONV) {
                    int oy = m / g.Wo, ox = m % g.Wo;
                    int ci = k % g.Cin, t = k / g.Cin;
                    int kx = t % g.kw, ky = t / g.kw;
                    int iy = oy * g.stride - g.pad_top + ky, ix = ox * g.stride - g.pad_left + kx;
                    if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) {
                        T raw = A[((int64_t)iy * g.W + ix) * g.Cin + ci];
                        if (QU8) v = (Acc)((int)raw - zx); else v = (Acc)to_float(raw);
                    }
                } else {
                    T raw = A[(int64_t)m * lda + k];
                    if (QU8) v = (Acc)((int)raw - zx); else v = (Acc)to_float(raw);
                }
            }
            As[ak][am] = v;
            // B
            int bk, bn;
            if (b_transposed) { bn = idx / BK; bk = idx % BK; } else { bk = idx / BN; bn = idx % BN; }
            int kk = k0 + bk, n = n0 + bn;
            Acc w = 0;
            if (kk < K && n < N) {
                T raw = b_transposed ? B[(int64_t)n * ldb + kk] : B[(int64_t)kk * ldb + n];
                if (QU8) w = (Acc)((int)raw - zw); else w = (Acc)to_float(raw);
            }
            Bs[bk][bn] = w;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; k++) {
            Acc a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; i++) a[i] = As[k][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; j++) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] += a[i] * b[j];
        }
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < 4; i++) {
        int m = m0 + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            if constexpr (QU8) {
                int a = acc[i][j];
                if (bias) a += ((const int32_t*)bias)[n];
                float scaled = (float)a * requant;
                scaled = fmaxf(scaled, (float)(0 - zy));
                scaled = fminf(scaled, (float)(255 - zy));
                int q = (int)lrintf(scaled) + zy;
                C[(int64_t)m * ldc + n] = (uint8_t)q;
            } else {
                float v = acc[i][j];
                if (bias) v += to_float(((const T*)bias)[n]);
                if (residual) v += to_float(residual[(int64_t)m * ldc + n]);
                C[(int64_t)m * ldc + n] = from_float<T>(v);
            }
        }
    }
}

// Skinny GEMM (M <= 8): weight-bandwidth bound (time-embedding Gemms, llm decode).  One warp per output column
// block; each lane strides K; B is read exactly once, coalesced along N.
template <typename T, int MAXM>
__global__ void __launch_bounds__(256)
skinny_gemm_kernel(const T* __restrict__ A, const T* __restrict__ B, T* __restrict__ C, const T* __restrict__ bias, const T* __restrict__ residual,
                   int M, int N, int K, int b_transposed)
{
    osb_pdl_prologue();
    // block handles 64 columns x all M rows; 256 threads = 4 k-slices x 64 columns (non-transposed B, coalesced over n)
    __shared__ float red[4][MAXM][64];
    if (!b_transposed) {
        int nl = threadIdx.x & 63, ks = threadIdx.x >> 6;
        int n = blockIdx.x * 64 + nl;
        float acc[MAXM];
#pragma unroll
        for (int m = 0; m < MAXM; m++) acc[m] = 0.f;
        if (n < N) {
            for (int k = ks; k < K; k += 4) {
                float b = to_float(B[(int64_t)k * N + n]);
#pragma unroll
                for (int m = 0; m < MAXM; m++) if (m < M) acc[m] += to_float(A[(int64_t)m * K + k]) * b;
            }
        }
#pragma unroll
        for (int m = 0; m < MAXM; m++) red[ks][m][nl] = acc[m];
        __syncthreads();
        if (ks == 0 && n < N) {
            for (int m = 0; m < M; m++) {
                float v = red[0][m][nl] + red[1][m][nl] + red[2][m][nl] + red[3][m][nl];
                if (bias) v += to_float(bias[n]);
                if (residual) v += to_float(residual[(int64_t)m * N + n]);
                C[(int64_t)m * N + n] = from_float<T>(v);
            }
        }
    } else {
        // B is [N, K]: one warp per column, lanes stride K (coalesced along K)
        int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        for (int n = blockIdx.x * 8 + warp; n < N; n += gridDim.x * 8) {
            float acc[MAXM];
#pragma unroll
            for (int m = 0; m < MAXM; m++) acc[m] = 0.f;
            for (int k = lane; k < K; k += 32) {
                float b = to_float(B[(int64_t)n * K + k]);
#pragma unroll
                for (int m = 0; m < MAXM; m++) if (m < M) acc[m] += to_float(A[(int64_t)m * K + k]) * b;
            }
#pragma unroll
            for (int m = 0; m < MAXM; m++) {
                float v = warp_sum(acc[m]);
                if (lane == 0 && m < M) {
                    if (bias) v += to_float(bias[n]);
                    if (residual) v += to_float(residual[(int64_t)m * N + n]);
                    C[(int64_t)m * N + n] = from_float<T>(v);
                }
            }
        }
    }
}

// Skinny GEMM, B stored [K, N] (ONNX MatMul / Gemm weights), M <= 8: pure weight bandwidth.  The weight matrix is cut
// into (256-column x k-slice) panels so that ~2 waves of CTAs stream it with 16-byte loads; partial sums are reduced in
// shared memory, then added with fp32 atomics into a zeroed scratch row; a second tiny kernel applies bias / residual and
// rounds to the storage type.  Reads every weight exactly once.
constexpr int GEMV_U = 8;
// CTAs a GEMV launch aims for (4 per SM); OSB_GEMV_CTAS overrides for tuning runs
static inline int gemv_ctas() { static const int v = [] { const char* e = getenv("OSB_GEMV_CTAS"); int x = e ? atoi(e) : 0; return x > 0 ? x : 592; }(); return v; }
template <typename T, int MAXM>
__device__ __forceinline__ void gemv_panel_body(const T* __restrict__ A, const T* __restrict__ B, float* __restrict__ acc_out, int M, int N, int K, int k_per_cta,
                                                int* __restrict__ counter, T* __restrict__ C, const T* __restrict__ bias, const T* __restrict__ residual, int panel, int ldb)
{
    constexpr int VEC = 16 / sizeof(T);           // columns per thread
    constexpr int COLS = 32 * VEC;                // columns per CTA
    __shared__ float red[4][MAXM][COLS];
    const int cg = threadIdx.x & 31, kl = threadIdx.x >> 5;       // 32 column groups x 4 k-lanes
    const int n0 = panel * COLS + cg * VEC;
    const int k_lo = blockIdx.y * k_per_cta, k_hi = min(k_lo + k_per_cta, K);
    float acc[MAXM][VEC];
#pragma unroll
    for (int m = 0; m < MAXM; m++)
#pragma unroll
        for (int v = 0; v < VEC; v++) acc[m][v] = 0.f;
    if (n0 < N) {
        // GEMV_U independent 16-byte loads per thread before the first FMA: a decode GEMV is pure weight streaming and one load in
        // flight per thread leaves HBM bandwidth unused; 8 x 16 B x 128 threads x 4 CTAs = 64 KB in flight per SM
        for (int k = k_lo + kl; k < k_hi; k += 4 * GEMV_U) {
            Vec<T, VEC> b[GEMV_U];
#pragma unroll
            for (int u = 0; u < GEMV_U; u++) {
                const int kk = k + 4 * u;
                if (kk < k_hi) b[u] = load_vec<T, VEC>(B + (int64_t)kk * ldb + n0);
            }
#pragma unroll
            for (int u = 0; u < GEMV_U; u++) {
                const int kk = k + 4 * u;
                if (kk < k_hi) {
#pragma unroll
                    for (int m = 0; m < MAXM; m++) {
                        if (m < M) {
                            float a = to_float(A[(int64_t)m * K + kk]);
#pragma unroll
                            for (int v = 0; v < VEC; v++) acc[m][v] += a * to_float(b[u].v[v]);
                        }
                    }
                }
            }
        }
    }
#pragma unroll
    for (int m = 0; m < MAXM; m++)
#pragma unroll
        for (int v = 0; v < VEC; v++) red[kl][m][cg * VEC + v] = acc[m][v];
    __syncthreads();
    for (int i = threadIdx.x; i < M * COLS; i += 128) {
        int m = i / COLS, c = i % COLS;
        int n = panel * COLS + c;
        if (n >= N) continue;
        float v = 0.f;
#pragma unroll
        for (int j = 0; j < 4; j++) v += red[j][m][c];
        atomicAdd(&acc_out[(int64_t)m * N + n], v);
    }
    // The last K-slice CTA of this column panel to arrive finishes the panel: fp32 sums (+ bias, + residual) -> one rounding ->
    // C, and re-arms the scratch (zero sums, zero counter) for the next launch.  One graph node per GEMV instead of
    // memset + panel + finalize.
    __shared__ int is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(counter, 1) == (int)gridDim.y - 1;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    for (int i = threadIdx.x; i < M * COLS; i += 128) {
        int m = i / COLS, c = i % COLS;
        int n = panel * COLS + c;
        if (n >= N) continue;
        float v = __ldcg(&acc_out[(int64_t)m * N + n]);
        acc_out[(int64_t)m * N + n] = 0.f;
        if (bias) v += to_float(bias[n]);
        if (residual) v += to_float(residual[(int64_t)m * N + n]);
        C[(int64_t)m * N + n] = from_float<T>(v);
    }
    if (threadIdx.x == 0) *counter = 0;
}

template <typename T, int MAXM>
__global__ void __launch_bounds__(128)
gemv_panel_kernel(const T* __restrict__ A, const T* __restrict__ B, float* __restrict__ acc_out, int M, int N, int K, int k_per_cta,
                  int* __restrict__ counters, T* __restrict__ C, const T* __restrict__ bias, const T* __restrict__ residual, int ldb)
{
    osb_pdl_prologue();
    gemv_panel_body<T, MAXM>(A, B, acc_out, M, N, K, k_per_cta, counters + blockIdx.x, C, bias, residual, (int)blockIdx.x, ldb);
}

// Up to three GEMVs that share their input row(s) and K (q / k / v projections, gate / up of a gated MLP) as ONE launch: blockIdx.x walks
// the column panels of all groups, each group with its own weight, output, scratch slice and arrival counters.
struct GemvGroups {
    const void* B[3]; void* C[3];
    int N[3], panel0[4], acc0[3];      // first panel / first scratch float of each group; panel0[groups] = total panels
    float wscale[3]; int wzp[3];
    int groups;
};
template <typename T, int MAXM>
__global__ void __launch_bounds__(128)
gemv_panel_grouped_kernel(const T* __restrict__ A, GemvGroups g, float* __restrict__ acc_out, int M, int K, int k_per_cta, int* __restrict__ counters)
{
    osb_pdl_prologue();
    const int bx = (int)blockIdx.x;
    const int gi = bx >= g.panel0[2] && g.groups > 2 ? 2 : (bx >= g.panel0[1] ? 1 : 0);
    gemv_panel_body<T, MAXM>(A, (const T*)g.B[gi], acc_out + g.acc0[gi], M, g.N[gi], K, k_per_cta, counters + bx, (T*)g.C[gi], nullptr, nullptr, bx - g.panel0[gi], g.N[gi]);
}

// The same panel GEMV with uint8 weights [K, N] (per-tensor scale / zero point), M <= 2: 16 columns per thread per 16-byte load, the
// weight dequantised in registers to the activation type T -- (q - zp) * scale ROUNDED TO T, i.e. exactly the operand the reference
// builds when it converts a uint8 blob at load time (src/onnxstream.cpp:2885-2890) -- then fp32 FMA.  Half (fp16) / a quarter (fp32) of
// the HBM bytes of the float GEMV: LLM decode is weight-bandwidth bound.
template <typename T>
__device__ __forceinline__ void gemv_w8_panel_body(const T* __restrict__ A, const uint8_t* __restrict__ B, float* __restrict__ acc_out, int M, int N, int K, int k_per_cta,
                                                   int* __restrict__ counter, T* __restrict__ C, const T* __restrict__ bias, const T* __restrict__ residual, float wscale, int wzp, int panel)
{
    constexpr int VEC = 16, COLS = 32 * VEC, MAXM = 2;
    __shared__ float red[4][MAXM][COLS];
    const int cg = threadIdx.x & 31, kl = threadIdx.x >> 5;
    const int n0 = panel * COLS + cg * VEC;
    const int k_lo = blockIdx.y * k_per_cta, k_hi = min(k_lo + k_per_cta, K);
    float acc[MAXM][VEC];
#pragma unroll
    for (int m = 0; m < MAXM; m++)
#pragma unroll
        for (int v = 0; v < VEC; v++) acc[m][v] = 0.f;
    if (n0 < N) {
        for (int k = k_lo + kl; k < k_hi; k += 4 * GEMV_U) {
            uint4 raws[GEMV_U];
#pragma unroll
            for (int u = 0; u < GEMV_U; u++) {
                const int kk = k + 4 * u;
                if (kk < k_hi) raws[u] = *reinterpret_cast<const uint4*>(B + (int64_t)kk * N + n0);
            }
#pragma unroll
            for (int u = 0; u < GEMV_U; u++) {
                const int kk = k + 4 * u;
                if (kk < k_hi) {
                    const uint32_t words[4] = { raws[u].x, raws[u].y, raws[u].z, raws[u].w };
                    float w[VEC];
#pragma unroll
                    for (int v = 0; v < VEC; v++) w[v] = to_float(from_float<T>((float)((int)((words[v >> 2] >> (8 * (v & 3))) & 0xFFu) - wzp) * wscale));
#pragma unroll
                    for (int m = 0; m < MAXM; m++) {
                        if (m < M) {
                            const float a = to_float(A[(int64_t)m * K + kk]);
#pragma unroll
                            for (int v = 0; v < VEC; v++) acc[m][v] += a * w[v];
                        }
                    }
                }
            }
        }
    }
#pragma unroll
    for (int m = 0; m < MAXM; m++)
#pragma unroll
        for (int v = 0; v < VEC; v++) red[kl][m][cg * VEC + v] = acc[m][v];
    __syncthreads();
    for (int i = threadIdx.x; i < M * COLS; i += 128) {
        int m = i / COLS, c = i % COLS;
        int n = panel * COLS + c;
        if (n >= N) continue;
        float v = 0.f;
#pragma unroll
        for (int j = 0; j < 4; j++) v += red[j][m][c];
        atomicAdd(&acc_out[(int64_t)m * N + n], v);
    }
    __shared__ int is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(counter, 1) == (int)gridDim.y - 1;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    for (int i = threadIdx.x; i < M * COLS; i += 128) {
        int m = i / COLS, c = i % COLS;
        int n = panel * COLS + c;
        if (n >= N) continue;
        float v = __ldcg(&acc_out[(int64_t)m * N + n]);
        acc_out[(int64_t)m * N + n] = 0.f;
        if (bias) v += to_float(bias[n]);
        if (residual) v += to_float(residual[(int64_t)m * N + n]);
        C[(int64_t)m * N + n] = from_float<T>(v);
    }
    if (threadIdx.x == 0) *counter = 0;
}

template <typename T>
__global__ void __launch_bounds__(128)
gemv_w8_panel_kernel(const T* __restrict__ A, const uint8_t* __restrict__ B, float* __restrict__ acc_out, int M, int N, int K, int k_per_cta,
                     int* __restrict__ counters, T* __restrict__ C, const T* __restrict__ bias, const T* __restrict__ residual, float wscale, int wzp)
{
    osb_pdl_prologue();
    gemv_w8_panel_body<T>(A, B, acc_out, M, N, K, k_per_cta, counters + blockIdx.x, C, bias, residual, wscale, wzp, (int)blockIdx.x);
}

template <typename T>
__global__ void __launch_bounds__(128)
gemv_w8_panel_grouped_kernel(const T* __restrict__ A, GemvGroups g, float* __restrict__ acc_out, int M, int K, int k_per_cta, int* __restrict__ counters)
{
    osb_pdl_prologue();
    const int bx = (int)blockIdx.x;
    const int gi = bx >= g.panel0[2] && g.groups > 2 ? 2 : (bx >= g.panel0[1] ? 1 : 0);
    gemv_w8_panel_body<T>(A, (const uint8_t*)g.B[gi], acc_out + g.acc0[gi], M, g.N[gi], K, k_per_cta, counters + bx, (T*)g.C[gi], nullptr, nullptr, g.wscale[gi], g.wzp[gi], bx - g.panel0[gi]);
}

// ---- softmax with scale + additive mask (score tile of the attention decomposition) ---------------------------
template <typename T>
__global__ void softmax_scaled_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t rows, int64_t cols, float scale,
                                      const T* __restrict__ mask, int64_t mask_rows)
{
    osb_pdl_prologue();
    __shared__ float red[32];
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const T* xr = x + r * cols;
        const T* mr = mask ? mask + (r % mask_rows) * cols : nullptr;
        T* yr = y + r * cols;
        float mx = -INFINITY;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) mx = fmaxf(mx, to_float(xr[c]) * scale + (mr ? to_float(mr[c]) : 0.f));
        mx = block_reduce_max(mx, red);
        float sum = 0.f;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x) sum += expf(to_float(xr[c]) * scale + (mr ? to_float(mr[c]) : 0.f) - mx);
        sum = block_reduce_sum(sum, red);
        float inv = 1.f / sum;
        for (int64_t c = threadIdx.x; c < cols; c += blockDim.x)
            yr[c] = from_float<T>(expf(to_float(xr[c]) * scale + (mr ? to_float(mr[c]) : 0.f) - mx) * inv);
    }
}

// Short rows (cross-attention: 77 keys): one warp per row, values kept in registers (cols <= 256), row stride `ld`,
// pad columns [cols, ld) zero-filled so the tile can feed a GEMM whose K is padded to a multiple of 8.
template <typename T>
__global__ void softmax_scaled_warp_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t rows, int cols, int ld, float scale,
                                           const T* __restrict__ mask, int64_t mask_rows)
{
    osb_pdl_prologue();
    const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    for (int64_t r = (int64_t)blockIdx.x * wpb + (threadIdx.x >> 5); r < rows; r += (int64_t)gridDim.x * wpb) {
        const T* xr = x + r * ld;
        const T* mr = mask ? mask + (r % mask_rows) * cols : nullptr;
        T* yr = y + r * ld;
        float v[8];
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            int c = lane + 32 * j;
            v[j] = c < cols ? to_float(xr[c]) * scale + (mr ? to_float(mr[c]) : 0.f) : -INFINITY;
            mx = fmaxf(mx, v[j]);
        }
        mx = warp_max(mx);
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 8; j++) { v[j] = (lane + 32 * j) < cols ? __expf(v[j] - mx) : 0.f; sum += v[j]; }
        sum = warp_sum(sum);
        float inv = 1.f / sum;
#pragma unroll
        for (int j = 0; j < 8; j++) { int c = lane + 32 * j; if (c < ld) yr[c] = from_float<T>(v[j] * inv); }
    }
}

// Same, one global read per element: the row is staged in shared memory as fp32 (cols <= 12288)
template <typename T>
__global__ void softmax_scaled_smem_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t rows, int cols, float scale,
                                           const T* __restrict__ mask, int64_t mask_rows)
{
    osb_pdl_prologue();
    extern __shared__ float row[];
    __shared__ float red[32];
    constexpr int VEC = 16 / sizeof(T);
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const T* xr = x + r * cols;
        const T* mr = mask ? mask + (r % mask_rows) * cols : nullptr;
        T* yr = y + r * cols;
        float mx = -INFINITY;
        for (int c = threadIdx.x * VEC; c < cols; c += blockDim.x * VEC) {
            Vec<T, VEC> v = load_vec<T, VEC>(xr + c);
#pragma unroll
            for (int k = 0; k < VEC; k++) {
                float f = to_float(v.v[k]) * scale + (mr ? to_float(mr[c + k]) : 0.f);
                row[c + k] = f;
                mx = fmaxf(mx, f);
            }
        }
        mx = block_reduce_max(mx, red);
        float sum = 0.f;
        for (int c = threadIdx.x; c < cols; c += blockDim.x) { float e = __expf(row[c] - mx); row[c] = e; sum += e; }
        sum = block_reduce_sum(sum, red);
        float inv = 1.f / sum;
        for (int c = threadIdx.x * VEC; c < cols; c += blockDim.x * VEC) {
            Vec<T, VEC> o;
#pragma unroll
            for (int k = 0; k < VEC; k++) o.v[k] = from_float<T>(row[c + k] * inv);
            store_vec<T, VEC>(yr + c, o);
        }
        __syncthreads();
    }
}

// ---- direct attention for short query lengths (decode): one warp per (head, query row), online softmax -------
// ---- split-KV decode attention: grid (key splits, heads * Tq); each warp scores 32 keys (one per lane), the block folds its 128 keys
// into one partial (max, sum, acc[dv]) and the last block of a row to arrive (self-resetting ticket) merges the partials.  A decode
// step at 2048 cached positions becomes 16 x 32 blocks instead of 32 warps walking 2048 keys each.
constexpr int DEC_KEYS = 128;
template <typename T>
__device__ __forceinline__ float dec_dot(const float* qs, const T* kr, int d)
{
    float dot = 0.f;
    for (int c = 0; c < d; c++) dot += qs[c] * to_float(kr[c]);
    return dot;
}
template <>
__device__ __forceinline__ float dec_dot<__half>(const float* qs, const __half* kr, int d)
{
    float dot = 0.f;
    if ((d & 7) == 0 && ((uintptr_t)kr & 15) == 0) {
        const uint4* k4 = reinterpret_cast<const uint4*>(kr);
        for (int c = 0; c < d; c += 8) {
            uint4 u = k4[c >> 3];
            const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
            for (int j = 0; j < 4; j++) { float2 f = __half22float2(h2[j]); dot += qs[c + 2 * j] * f.x + qs[c + 2 * j + 1] * f.y; }
        }
    } else {
        for (int c = 0; c < d; c++) dot += qs[c] * __half2float(kr[c]);
    }
    return dot;
}

template <typename T>
__global__ void __launch_bounds__(128) attention_decode_kernel(const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v,
                                                               const T* __restrict__ mask, T* __restrict__ out, float* part, int* tickets,
                                                               int64_t Tq, int64_t Tk, int d, int dv, float scale, int64_t kv_group, int nsplit)
{
    osb_pdl_prologue();
    extern __shared__ float smem[];   // q [d] | acc of each warp [4][dv] | (max, sum) of each warp [4][2] | p [4][32]
    float* qs = smem;
    float* wacc = qs + d;
    float* wml = wacc + 4 * dv;
    float* ps = wml + 8;
    __shared__ int s_last;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t row = blockIdx.y, sp = blockIdx.x;
    const int64_t h = row / Tq, t = row % Tq, hk = h / kv_group;
    for (int c = tid; c < d; c += 128) qs[c] = to_float(q[row * d + c]) * scale;
    __syncthreads();
    const int64_t s0 = sp * DEC_KEYS + warp * 32, s = s0 + lane;
    float logit = -INFINITY;
    if (s < Tk) {
        logit = dec_dot<T>(qs, k + (hk * Tk + s) * d, d);
        if (mask) logit += to_float(mask[t * Tk + s]);
    }
    const float m = warp_max(logit);
    const float p = (s < Tk && m > -INFINITY) ? expf(logit - m) : 0.f;
    const float l = warp_sum(p);
    ps[warp * 32 + lane] = p;
    __syncwarp();
    const int jn = (Tk - s0) < 32 ? (int)max((int64_t)0, Tk - s0) : 32;
    const T* vb = v + (hk * Tk + s0) * dv;
    bool pv_done = false;
    if constexpr (std::is_same<T, __half>::value) {
        if ((dv & 7) == 0 && ((uintptr_t)vb & 15) == 0) {
            // 16-byte V loads: lane = (key group kg of 4, column group cg of 8 halves); every lane has its 8 loads in flight at once, then two
            // shuffles fold the 4 key groups (the scalar loop below issues 2-byte loads, 64 per lane)
            const int kg = lane >> 3, cg = lane & 7;
            for (int c0 = 0; c0 < dv; c0 += 64) {
                const int c = c0 + cg * 8;
                float a8[8];
#pragma unroll
                for (int t = 0; t < 8; t++) a8[t] = 0.f;
                if (c < dv) {
                    uint4 u[8];
#pragma unroll
                    for (int jj = 0; jj < 8; jj++) { const int j = jj * 4 + kg; if (j < jn) u[jj] = *reinterpret_cast<const uint4*>(vb + (int64_t)j * dv + c); }
#pragma unroll
                    for (int jj = 0; jj < 8; jj++) {
                        const int j = jj * 4 + kg;
                        if (j < jn) {
                            const float pj = ps[warp * 32 + j];
                            const __half2* h2 = reinterpret_cast<const __half2*>(&u[jj]);
#pragma unroll
                            for (int t = 0; t < 4; t++) { const float2 f = __half22float2(h2[t]); a8[2 * t] += pj * f.x; a8[2 * t + 1] += pj * f.y; }
                        }
                    }
                }
#pragma unroll
                for (int t = 0; t < 8; t++) {       // all 32 lanes shuffle (inactive column groups carry zeros)
                    a8[t] += __shfl_xor_sync(0xffffffffu, a8[t], 8);
                    a8[t] += __shfl_xor_sync(0xffffffffu, a8[t], 16);
                }
                if (kg == 0 && c < dv) {
#pragma unroll
                    for (int t = 0; t < 8; t++) wacc[warp * dv + c + t] = a8[t];
                }
            }
            pv_done = true;
        }
    }
    if (!pv_done)
    for (int c = lane; c < dv; c += 32) {
        float a = 0.f;
#pragma unroll 8
        for (int j = 0; j < jn; j++) a += ps[warp * 32 + j] * to_float(vb[(int64_t)j * dv + c]);
        wacc[warp * dv + c] = a;
    }
    if (lane == 0) { wml[warp * 2] = m; wml[warp * 2 + 1] = l; }
    __syncthreads();
    float* mine = part + (row * nsplit + sp) * (dv + 2);
    {
        float M = fmaxf(fmaxf(wml[0], wml[2]), fmaxf(wml[4], wml[6]));
        float w[4];
#pragma unroll
        for (int x = 0; x < 4; x++) w[x] = wml[2 * x] > -INFINITY ? expf(wml[2 * x] - M) : 0.f;
        for (int c = tid; c < dv; c += 128) __stcg(mine + c, wacc[c] * w[0] + wacc[dv + c] * w[1] + wacc[2 * dv + c] * w[2] + wacc[3 * dv + c] * w[3]);
        if (tid == 0) { __stcg(mine + dv, M); __stcg(mine + dv + 1, wml[1] * w[0] + wml[3] * w[1] + wml[5] * w[2] + wml[7] * w[3]); }
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        int ticket = atomicAdd(&tickets[row], 1);
        s_last = ticket == nsplit - 1;
        if (s_last) tickets[row] = 0;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    // merge: the per-split (max, sum) pairs are fetched by one thread each (parallel L2 round trips, not a dependent chain), the
    // weights land in shared memory (ps / wacc are free again), then every output column is a sum of independent loads
    const float* pr = part + row * nsplit * (dv + 2);
    float* sw = wacc;                       // [nsplit] weights; nsplit <= 4 * dv is checked by the launcher
    float Mx = -INFINITY;
    for (int x0 = 0; x0 < nsplit; x0 += 128) {
        const int x = x0 + tid;
        const float mx = x < nsplit ? __ldcg(pr + x * (dv + 2) + dv) : -INFINITY;
        if (x < nsplit) sw[x] = mx;
        Mx = fmaxf(Mx, mx);
    }
    Mx = warp_max(Mx);
    if (lane == 0) wml[warp] = Mx;
    __syncthreads();
    const float M = fmaxf(fmaxf(wml[0], wml[1]), fmaxf(wml[2], wml[3]));
    float Lp = 0.f;
    for (int x0 = 0; x0 < nsplit; x0 += 128) {
        const int x = x0 + tid;
        if (x < nsplit) {
            const float wgt = sw[x] > -INFINITY ? expf(sw[x] - M) : 0.f;
            Lp += __ldcg(pr + x * (dv + 2) + dv + 1) * wgt;
            sw[x] = wgt;
        }
    }
    Lp = warp_sum(Lp);
    __syncthreads();                        // wml[0..3] read by everyone before it is overwritten; sw complete
    if (lane == 0) wml[4 + warp] = Lp;
    __syncthreads();
    const float inv = 1.f / (wml[4] + wml[5] + wml[6] + wml[7]);
    for (int c = tid; c < dv; c += 128) {
        float a = 0.f;
#pragma unroll 8
        for (int x = 0; x < nsplit; x++) a += __ldcg(pr + x * (dv + 2) + c) * sw[x];
        out[row * dv + c] = from_float<T>(a * inv);
    }
}

template <typename T>
__global__ void attention_rows_kernel(const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, const T* __restrict__ mask,
                                      T* __restrict__ out, int64_t heads, int64_t Tq, int64_t Tk, int d, int dv, float scale,
                                      int k_transposed, int64_t kv_group)
{
    osb_pdl_prologue();
    extern __shared__ float smem[];  // per warp: q row [d] + acc [dv] + p [32]
    int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    float* qs = smem + warp * (d + dv + 32);
    float* acc = qs + d;
    float* ps = acc + dv;
    int64_t total = heads * Tq;
    for (int64_t row = (int64_t)blockIdx.x * nwarps + warp; row < total; row += (int64_t)gridDim.x * nwarps) {
        int64_t h = row / Tq, t = row % Tq, hk = h / kv_group;
        const T* qr = q + row * d;
        for (int c = lane; c < d; c += 32) qs[c] = to_float(qr[c]) * scale;
        for (int c = lane; c < dv; c += 32) acc[c] = 0.f;
        __syncwarp();
        float m = -INFINITY, l = 0.f;
        const T* kb = k + hk * Tk * d;
        const T* vb = v + hk * Tk * dv;
        for (int64_t s0 = 0; s0 < Tk; s0 += 32) {
            int64_t s = s0 + lane;
            float logit = -INFINITY;
            if (s < Tk) {
                float dot = 0.f;
                if (k_transposed) for (int c = 0; c < d; c++) dot += qs[c] * to_float(kb[(int64_t)c * Tk + s]);
                else for (int c = 0; c < d; c++) dot += qs[c] * to_float(kb[s * d + c]);
                if (mask) dot += to_float(mask[t * Tk + s]);
                logit = dot;
            }
            float mnew = fmaxf(m, warp_max(logit));
            float corr = expf(m - mnew);
            float p = s < Tk ? expf(logit - mnew) : 0.f;
            l = l * corr + warp_sum(p);
            // acc = acc * corr + sum_s p_s * v[s]   (p staged through shared memory: trip counts differ per lane)
            ps[lane] = p;
            __syncwarp();
            int jn = (Tk - s0) < 32 ? (int)(Tk - s0) : 32;
            for (int c = lane; c < dv; c += 32) {
                float a = acc[c] * corr;
                for (int j = 0; j < jn; j++) a += ps[j] * to_float(vb[(s0 + j) * dv + c]);
                acc[c] = a;
            }
            m = mnew;
            __syncwarp();
        }
        float inv = 1.f / l;
        T* orow = out + row * dv;
        for (int c = lane; c < dv; c += 32) orow[c] = from_float<T>(acc[c] * inv);
        __syncwarp();
    }
}

template <typename T>
int launch_igemm(const T* A, const T* B, T* C, const void* bias, const T* residual, int64_t batch, int64_t M, int64_t N, int64_t K,
                 int64_t sa, int64_t sb, int64_t sc, int bt, bool conv, ConvGeom g, cudaStream_t st, int64_t lda = 0, int64_t ldb = 0, int64_t ldc = 0)
{
    dim3 grid((unsigned)((N + BN - 1) / BN), (unsigned)((M + BM - 1) / BM), (unsigned)batch);
    if (grid.y > 65535 || grid.z > 65535) return (int)cudaErrorInvalidValue;
    if (conv) osb_launch((igemm_kernel<T, true, false>), grid, 256, 0, st, A, B, C, bias, residual, (int)M, (int)N, (int)K, sa, sb, sc, bt, g, 0, 0, 0, 0.f, 0, 0, 0);
    else osb_launch((igemm_kernel<T, false, false>), grid, 256, 0, st, A, B, C, bias, residual, (int)M, (int)N, (int)K, sa, sb, sc, bt, g, 0, 0, 0, 0.f, (int)lda, (int)ldb, (int)ldc);
    return launched();
}

} // namespace

extern "C" {

int osb_gemm_tc_eligible(int64_t M, int64_t N, int64_t K, int dtype)
{
    return dtype == OSB_F16 && osb_tc_gemm_ok(M, N, K, 0, nullptr, nullptr, nullptr, 0, 0, 0, K, N, N) ? 1 : 0;
}

int osb_gemm_grouped(const void* A, const void* const* B, void* const* C, int groups, int64_t M, int64_t N, int64_t K, int bt, int dtype, int impl, void* stream)
{
    if (groups < 1 || groups > 3) return (int)cudaErrorInvalidValue;
    if (M * N == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t lda = K, ldb = bt ? K : N, ldc = N;
    bool tc_ok = groups >= 2 && dtype == OSB_F16 && impl != 1;
    for (int g = 0; g < groups && tc_ok; g++) tc_ok = osb_tc_gemm_ok(M, N, K, bt, A, B[g], C[g], 0, 0, 0, lda, ldb, ldc);
    if (tc_ok) return osb_tc_gemm_grouped_launch(A, B, C, groups, M, N, K, bt, st, lda, ldb, ldc);
    for (int g = 0; g < groups; g++) {
        int r = osb_gemm(A, B[g], C[g], nullptr, nullptr, 1, M, N, K, 0, 0, 0, bt, dtype, impl, stream);
        if (r) return r;
    }
    return 0;
}

int osb_gemm(const void* A, const void* B, void* C, const void* bias, const void* residual, int64_t batch, int64_t M, int64_t N, int64_t K,
             int64_t sa, int64_t sb, int64_t sc, int bt, int dtype, int impl, void* stream)
{
    return osb_gemm_ld(A, K, B, bt ? K : N, C, N, bias, residual, batch, M, N, K, sa, sb, sc, bt, dtype, impl, stream);
}

int osb_gemm_ld(const void* A, int64_t lda, const void* B, int64_t ldb, void* C, int64_t ldc, const void* bias, const void* residual,
                int64_t batch, int64_t M, int64_t N, int64_t K, int64_t sa, int64_t sb, int64_t sc, int bt, int dtype, int impl, void* stream)
{
    const bool dense = lda == K && ldb == (bt ? K : N) && ldc == N;
    if (batch * M * N == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype != OSB_F16 && dtype != OSB_F32) return (int)cudaErrorInvalidValue;
    if (K == 0) return (int)cudaErrorInvalidValue;
    bool tc_ok = dtype == OSB_F16 && osb_tc_gemm_ok(M, N, K, bt, A, B, C, sa, sb, sc, lda, ldb, ldc);
    if (impl == 2 && !tc_ok) return (int)cudaErrorInvalidValue;
    if (tc_ok && impl != 1) return osb_tc_gemm_launch(A, B, C, bias, residual, batch, M, N, K, sa, sb, sc, bt, st, lda, ldb, ldc);
    ConvGeom g{};
    // (ldb > N: a row-padded copy of a weight whose N is not a multiple of the 16-byte vector, e.g. a 32003-entry vocabulary)
    if (lda == K && ldc == N && M <= 8 && batch == 1 && !bt && ldb >= N && ldb % (dtype == OSB_F16 ? 8 : 4) == 0 && aligned16(B) && N >= 256 && K >= 64) {
        // weight-bandwidth path
        // scratch (per-stream, fixed capacity, workspace.h): fp32 sums [M][N] + one arrival counter per column panel; zeroed when
        // allocated, re-armed by the kernel.  Shapes beyond the fixed capacity take the skinny kernel below.
        int vec = dtype == OSB_F16 ? 8 : 4, cols = 32 * vec;
        int gx = (int)((N + cols - 1) / cols);
        OsbWorkspace* ws = (gx <= 4096 && (size_t)M * N <= OSB_WS_GEMV_FLOATS) ? osb_workspace(st, OSB_WS_GEMV) : nullptr;
        if (ws) {
        float* scratch = ws->gemv;
        int* counters = ws->gemv_counters;
        int gy = (int)max<int64_t>(1, min<int64_t>((K + 15) / 16, (gemv_ctas() + gx - 1) / gx));
        int k_per = (int)((K + gy - 1) / gy);
        gy = (int)((K + k_per - 1) / k_per);
        dim3 grid(gx, gy);
#define OSB_GEMV(T_, MM_) osb_launch((gemv_panel_kernel<T_, MM_>), grid, 128, 0, st, (const T_*)A, (const T_*)B, scratch, (int)M, (int)N, (int)K, k_per, \
                                    counters, (T_*)C, (const T_*)bias, (const T_*)residual, (int)ldb)
        // row-count instantiations: the M = 1 decode GEMV keeps 8 accumulators instead of 64
        if (dtype == OSB_F16) { if (M == 1) OSB_GEMV(__half, 1); else if (M == 2) OSB_GEMV(__half, 2); else if (M <= 4) OSB_GEMV(__half, 4); else OSB_GEMV(__half, 8); }
        else { if (M == 1) OSB_GEMV(float, 1); else if (M == 2) OSB_GEMV(float, 2); else if (M <= 4) OSB_GEMV(float, 4); else OSB_GEMV(float, 8); }
#undef OSB_GEMV
        return launched();
        }
    }
    if (dense && M <= 8 && batch == 1) {
        int grid = bt ? (int)min<int64_t>((N + 7) / 8, OSB_SMS * 8) : (int)((N + 63) / 64);
        if (dtype == OSB_F16) osb_launch((skinny_gemm_kernel<__half, 8>), grid, 256, 0, st, (const __half*)A, (const __half*)B, (__half*)C, (const __half*)bias, (const __half*)residual, (int)M, (int)N, (int)K, bt);
        else osb_launch((skinny_gemm_kernel<float, 8>), grid, 256, 0, st, (const float*)A, (const float*)B, (float*)C, (const float*)bias, (const float*)residual, (int)M, (int)N, (int)K, bt);
        return launched();
    }
    if (dtype == OSB_F16) return launch_igemm<__half>((const __half*)A, (const __half*)B, (__half*)C, bias, (const __half*)residual, batch, M, N, K, sa, sb, sc, bt, false, g, st, lda, ldb, ldc);
    return launch_igemm<float>((const float*)A, (const float*)B, (float*)C, bias, (const float*)residual, batch, M, N, K, sa, sb, sc, bt, false, g, st, lda, ldb, ldc);
}

// y[M,N] = x[M,K] . dequant(Wq[K,N]) (+ bias, + residual), M <= 2, uint8 weights dequantised in registers (see gemv_w8_panel_kernel)
int osb_gemv_w8(const void* A, const void* Wq, void* C, const void* bias, const void* residual, int64_t M, int64_t N, int64_t K, float wscale, int wzp, int dtype, void* stream)
{
    if (M < 1 || M > 2 || (N % 16) || N < 16 || K < 1 || (dtype != OSB_F16 && dtype != OSB_F32) || !aligned16(Wq)) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    const int cols = 512;
    const int gx = (int)((N + cols - 1) / cols);
    OsbWorkspace* ws = (gx <= 4096 && (size_t)M * N <= OSB_WS_GEMV_FLOATS) ? osb_workspace(st, OSB_WS_GEMV) : nullptr;
    if (!ws) return (int)cudaErrorNotReady;
    int gy = (int)max<int64_t>(1, min<int64_t>((K + 15) / 16, (gemv_ctas() + gx - 1) / gx));
    int k_per = (int)((K + gy - 1) / gy);
    gy = (int)((K + k_per - 1) / k_per);
    dim3 grid(gx, gy);
    if (dtype == OSB_F16) osb_launch((gemv_w8_panel_kernel<__half>), grid, 128, 0, st, (const __half*)A, (const uint8_t*)Wq, ws->gemv, (int)M, (int)N, (int)K, k_per, ws->gemv_counters,
                                     (__half*)C, (const __half*)bias, (const __half*)residual, wscale, wzp);
    else osb_launch((gemv_w8_panel_kernel<float>), grid, 128, 0, st, (const float*)A, (const uint8_t*)Wq, ws->gemv, (int)M, (int)N, (int)K, k_per, ws->gemv_counters,
                    (float*)C, (const float*)bias, (const float*)residual, wscale, wzp);
    return launched();
}

// groups (2 or 3) GEMVs y_g[M,N_g] = x[M,K] . W_g[K,N_g] sharing x, as one launch.  wdtype == OSB_U8: uint8 weights dequantised in
// registers (M <= 2); otherwise weights of the activation type.  cudaErrorNotSupported = shape outside what the grouped kernels cover
// (the caller launches the GEMVs one by one).
int osb_gemv_grouped(const void* A, const void* const* B, void* const* C, const int64_t* N, const float* wscale, const int* wzp, int groups,
                     int64_t M, int64_t K, int wdtype, int dtype, void* stream)
{
    if (groups < 2 || groups > 3 || (dtype != OSB_F16 && dtype != OSB_F32) || M < 1 || K < 64) return (int)cudaErrorNotSupported;
    const bool w8 = wdtype == OSB_U8;
    if (!w8 && wdtype != dtype) return (int)cudaErrorNotSupported;
    if (M > (w8 ? 2 : 8)) return (int)cudaErrorNotSupported;
    const int cols = w8 ? 512 : (dtype == OSB_F16 ? 256 : 128);
    GemvGroups g{};
    g.groups = groups;
    int panels = 0; int64_t acc = 0;
    for (int i = 0; i < groups; i++) {
        if (N[i] < 256 || N[i] % (w8 ? 16 : 8) || !aligned16(B[i])) return (int)cudaErrorNotSupported;
        g.B[i] = B[i]; g.C[i] = C[i]; g.N[i] = (int)N[i]; g.panel0[i] = panels; g.acc0[i] = (int)acc;
        g.wscale[i] = w8 ? wscale[i] : 0.f; g.wzp[i] = w8 ? wzp[i] : 0;
        panels += (int)((N[i] + cols - 1) / cols);
        acc += M * N[i];
    }
    for (int i = groups; i < 4; i++) g.panel0[i] = panels;
    if (panels > 4096 || (size_t)acc > OSB_WS_GEMV_FLOATS) return (int)cudaErrorNotSupported;
    cudaStream_t st = (cudaStream_t)stream;
    OsbWorkspace* ws = osb_workspace(st, OSB_WS_GEMV);
    if (!ws) return (int)cudaErrorNotSupported;
    int gy = (int)max<int64_t>(1, min<int64_t>((K + 15) / 16, (gemv_ctas() + panels - 1) / panels));
    int k_per = (int)((K + gy - 1) / gy);
    gy = (int)((K + k_per - 1) / k_per);
    dim3 grid(panels, gy);
    if (w8) {
        if (dtype == OSB_F16) osb_launch((gemv_w8_panel_grouped_kernel<__half>), grid, 128, 0, st, (const __half*)A, g, ws->gemv, (int)M, (int)K, k_per, ws->gemv_counters);
        else osb_launch((gemv_w8_panel_grouped_kernel<float>), grid, 128, 0, st, (const float*)A, g, ws->gemv, (int)M, (int)K, k_per, ws->gemv_counters);
    } else {
#define OSB_GEMVG(T_, MM_) osb_launch((gemv_panel_grouped_kernel<T_, MM_>), grid, 128, 0, st, (const T_*)A, g, ws->gemv, (int)M, (int)K, k_per, ws->gemv_counters)
        if (dtype == OSB_F16) { if (M == 1) OSB_GEMVG(__half, 1); else if (M == 2) OSB_GEMVG(__half, 2); else if (M <= 4) OSB_GEMVG(__half, 4); else OSB_GEMVG(__half, 8); }
        else { if (M == 1) OSB_GEMVG(float, 1); else if (M == 2) OSB_GEMVG(float, 2); else if (M <= 4) OSB_GEMVG(float, 4); else OSB_GEMVG(float, 8); }
#undef OSB_GEMVG
    }
    return launched();
}

int osb_conv2d(const void* x, const void* w, const void* bias, const void* residual, void* y, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
               int kh, int kw, int stride, int pad_top, int pad_left, int64_t Ho, int64_t Wo, int dtype, int impl, void* stream)
{
    return osb_conv2d_ex(x, w, bias, nullptr, residual, y, H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left, Ho, Wo, dtype, impl, stream, nullptr, 0, nullptr);
}

// 1 when osb_conv2d_ex will take the tensor-core path for this problem, i.e. when `bias2` and `gn_stats` are honoured
int osb_conv2d_fusable(const void* x, const void* w, const void* y, int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, int dtype, int impl)
{
    return dtype == OSB_F16 && impl != 1 && Cout % 8 == 0 && osb_tc_conv_ok(H, W, Cin, Cout, kh, kw, stride, x, w, y) ? 1 : 0;
}

int osb_conv2d_ex(const void* x, const void* w, const void* bias, const void* bias2, const void* residual, void* y, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                  int kh, int kw, int stride, int pad_top, int pad_left, int64_t Ho, int64_t Wo, int dtype, int impl, void* stream,
                  void* gn_stats, int gn_groups, int* gn_done)
{
    if (gn_done) *gn_done = 0;
    if (Ho * Wo * Cout == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype != OSB_F16 && dtype != OSB_F32) return (int)cudaErrorInvalidValue;
    bool tc_ok = dtype == OSB_F16 && osb_tc_conv_ok(H, W, Cin, Cout, kh, kw, stride, x, w, y);
    if (impl == 2 && !tc_ok) return (int)cudaErrorInvalidValue;
    if (tc_ok && impl != 1) return osb_tc_conv_launch(x, w, bias, residual, y, H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left, Ho, Wo, st, bias2, (double*)gn_stats, gn_groups, gn_done);
    if (bias2) return (int)cudaErrorInvalidValue;     // callers ask osb_conv2d_fusable first
    ConvGeom g{ (int)H, (int)W, (int)Cin, kh, kw, stride, pad_top, pad_left, (int)Ho, (int)Wo };
    int64_t M = Ho * Wo, N = Cout, K = (int64_t)kh * kw * Cin;
    if (dtype == OSB_F16) return launch_igemm<__half>((const __half*)x, (const __half*)w, (__half*)y, bias, (const __half*)residual, 1, M, N, K, 0, 0, 0, 1, true, g, st);
    return launch_igemm<float>((const float*)x, (const float*)w, (float*)y, bias, (const float*)residual, 1, M, N, K, 0, 0, 0, 1, true, g, st);
}

int osb_gemm_qu8(const uint8_t* A, const uint8_t* B, uint8_t* C, const int32_t* bias, int64_t M, int64_t N, int64_t K,
                 int zx, float sx, int zw, float sw, int zy, float sy, void* stream)
{
    if (M * N == 0) return 0;
    ConvGeom g{};
    float requant = sx * sw / sy;
    dim3 grid((unsigned)((N + BN - 1) / BN), (unsigned)((M + BM - 1) / BM), 1);
    osb_launch((igemm_kernel<uint8_t, false, true>), grid, 256, 0, (cudaStream_t)stream, A, B, C, bias, nullptr, (int)M, (int)N, (int)K, 0, 0, 0, 0, g, zx, zw, zy, requant, 0, 0, 0);
    return launched();
}

int osb_conv2d_qu8(const uint8_t* x, const uint8_t* w, const int32_t* bias, uint8_t* y, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                   int kh, int kw, int stride, int pad_top, int pad_left, int64_t Ho, int64_t Wo,
                   int zx, float sx, int zw, float sw, int zy, float sy, void* stream)
{
    if (Ho * Wo * Cout == 0) return 0;
    ConvGeom g{ (int)H, (int)W, (int)Cin, kh, kw, stride, pad_top, pad_left, (int)Ho, (int)Wo };
    int64_t M = Ho * Wo, N = Cout, K = (int64_t)kh * kw * Cin;
    float requant = sx * sw / sy;
    dim3 grid((unsigned)((N + BN - 1) / BN), (unsigned)((M + BM - 1) / BM), 1);
    osb_launch((igemm_kernel<uint8_t, true, true>), grid, 256, 0, (cudaStream_t)stream, x, w, y, bias, nullptr, (int)M, (int)N, (int)K, 0, 0, 0, 1, g, zx, zw, zy, requant, 0, 0, 0);
    return launched();
}

int osb_softmax_scaled(const void* x, void* y, int dtype, int64_t rows, int64_t cols, float scale, const void* mask, int64_t mask_rows, void* stream)
{
    return osb_softmax_scaled_ld(x, y, dtype, rows, cols, cols, scale, mask, mask_rows, stream);
}

// rows of `cols` valid elements stored `ld` apart; the pad columns [cols, ld) of y are zero-filled (they feed a padded GEMM K)
int osb_softmax_scaled_ld(const void* x, void* y, int dtype, int64_t rows, int64_t cols, int64_t ld, float scale, const void* mask, int64_t mask_rows, void* stream)
{
    if (rows * cols == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    int threads = cols >= 1024 ? 256 : (cols >= 256 ? 128 : 32);
    int grid = (int)min<int64_t>(rows, OSB_SMS * 16);
    if (mask_rows <= 0) mask_rows = 1;
    int vecw = dtype == OSB_F16 ? 8 : 4;
    if (ld <= 256 && cols <= ld) {
        grid = (int)min<int64_t>((rows + 7) / 8, OSB_SMS * 8);
        if (dtype == OSB_F16) osb_launch((softmax_scaled_warp_kernel<__half>), grid, 256, 0, st, (const __half*)x, (__half*)y, rows, (int)cols, (int)ld, scale, (const __half*)mask, mask_rows);
        else if (dtype == OSB_F32) osb_launch((softmax_scaled_warp_kernel<float>), grid, 256, 0, st, (const float*)x, (float*)y, rows, (int)cols, (int)ld, scale, (const float*)mask, mask_rows);
        else return (int)cudaErrorInvalidValue;
        return launched();
    }
    if (ld != cols) return (int)cudaErrorInvalidValue;   // padded rows are only needed (and supported) for short rows
    if (cols >= 512 && cols <= 12288 && cols % vecw == 0 && aligned16(x) && aligned16(y)) {
        size_t smem = (size_t)cols * sizeof(float);
        grid = (int)min<int64_t>(rows, OSB_SMS * 4);
        if (dtype == OSB_F16) {
            static bool attr16 = false;
            if (!attr16) { cudaFuncSetAttribute(softmax_scaled_smem_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, 12288 * 4); attr16 = true; }
            osb_launch((softmax_scaled_smem_kernel<__half>), grid, 256, smem, st, (const __half*)x, (__half*)y, rows, (int)cols, scale, (const __half*)mask, mask_rows);
        } else if (dtype == OSB_F32) {
            static bool attr32 = false;
            if (!attr32) { cudaFuncSetAttribute(softmax_scaled_smem_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 12288 * 4); attr32 = true; }
            osb_launch((softmax_scaled_smem_kernel<float>), grid, 256, smem, st, (const float*)x, (float*)y, rows, (int)cols, scale, (const float*)mask, mask_rows);
        } else return (int)cudaErrorInvalidValue;
        return launched();
    }
    if (dtype == OSB_F16) osb_launch((softmax_scaled_kernel<__half>), grid, threads, 0, st, (const __half*)x, (__half*)y, rows, cols, scale, (const __half*)mask, mask_rows);
    else if (dtype == OSB_F32) osb_launch((softmax_scaled_kernel<float>), grid, threads, 0, st, (const float*)x, (float*)y, rows, cols, scale, (const float*)mask, mask_rows);
    else return (int)cudaErrorInvalidValue;
    return launched();
}

int osb_attention(const void* q, const void* k, const void* v, const void* mask, void* out, int64_t heads, int64_t Tq, int64_t Tk,
                  int64_t d, int64_t dv, float scale, int k_transposed, int64_t kv_group, int dtype, void* stream)
{
    if (heads * Tq * dv == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (kv_group < 1) kv_group = 1;
    {
        // long key axis, few query rows (decode): split the keys over the grid
        static const bool dec = [] { const char* e = getenv("OSB_DECODE_ATTN"); return !(e && e[0] == '0'); }();
        const int64_t rows = heads * Tq, nsplit = (Tk + DEC_KEYS - 1) / DEC_KEYS;
        const size_t dsm = (size_t)(d + 4 * dv + 8 + 128) * sizeof(float);
        if (dec && !k_transposed && Tk >= 256 && rows <= 4096 && nsplit <= 4 * dv && rows * nsplit <= 65535 * 4 && nsplit <= 65535 && rows <= 65535 && dsm <= 48 * 1024 &&
            (size_t)rows * nsplit * (dv + 2) * sizeof(float) <= OSB_WS_SPLITK_BYTES && (dtype == OSB_F16 || dtype == OSB_F32)) {
            OsbWorkspace* ws = osb_workspace(st, OSB_WS_SPLITK);
            if (ws) {
                dim3 grid((unsigned)nsplit, (unsigned)rows);
                if (dtype == OSB_F16) osb_launch((attention_decode_kernel<__half>), grid, 128, dsm, st, (const __half*)q, (const __half*)k, (const __half*)v, (const __half*)mask, (__half*)out, ws->splitk, ws->splitk_counters, Tq, Tk, (int)d, (int)dv, scale, kv_group, (int)nsplit);
                else osb_launch((attention_decode_kernel<float>), grid, 128, dsm, st, (const float*)q, (const float*)k, (const float*)v, (const float*)mask, (float*)out, ws->splitk, ws->splitk_counters, Tq, Tk, (int)d, (int)dv, scale, kv_group, (int)nsplit);
                return launched();
            }
        }
    }
    int warps = 4;
    size_t smem = (size_t)warps * (d + dv + 32) * sizeof(float);
    if (smem > 48 * 1024) return (int)cudaErrorInvalidValue;
    int grid = (int)min<int64_t>((heads * Tq + warps - 1) / warps, OSB_SMS * 8);
    if (dtype == OSB_F16) osb_launch((attention_rows_kernel<__half>), grid, warps * 32, smem, st, (const __half*)q, (const __half*)k, (const __half*)v, (const __half*)mask, (__half*)out, heads, Tq, Tk, (int)d, (int)dv, scale, k_transposed, kv_group);
    else if (dtype == OSB_F32) osb_launch((attention_rows_kernel<float>), grid, warps * 32, smem, st, (const float*)q, (const float*)k, (const float*)v, (const float*)mask, (float*)out, heads, Tq, Tk, (int)d, (int)dv, scale, k_transposed, kv_group);
    else return (int)cudaErrorInvalidValue;
    return launched();
}

// ---- launch counters -----------------------------------------------------------------------------------------
static int g_pdl = -1;
int osb_pdl_enabled(void)
{
    // opt-in (OSB_PDL=1): inside a CUDA graph PDL did not pay on this workload
    if (g_pdl < 0) { const char* e = getenv("OSB_PDL"); g_pdl = (e && e[0] == '1') ? 1 : 0; }
    return g_pdl;
}
void osb_set_pdl(int enable) { g_pdl = enable ? 1 : 0; }
static uint64_t g_launches = 0, g_tc_launches = 0;
void osb_count_launch(int tensor_core) { g_launches++; if (tensor_core) g_tc_launches++; }
uint64_t osb_launch_count(void) { return g_launches; }
uint64_t osb_tc_launch_count(void) { return g_tc_launches; }
void osb_launch_count_reset(void) { g_launches = 0; g_tc_launches = 0; }

} // extern "C"
