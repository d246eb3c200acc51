/* onnxstream_b200_kernels.h -- internal C ABI between the C++ host (engine.cpp) and the hand-written sm_90a CUDA
 * kernels.  Device pointers + explicit shapes/strides/dtype enums in, `int` status (cudaError_t value, 0 = OK) out,
 * no exceptions and no torch types across it.  Each entry point replaces one method of the reference's private
 * `class XnnPack` (src/onnxstream.cpp:657-2150) or one inline pthreadpool lambda of `Model::run()`
 * (src/onnxstream.cpp:3550-8269); the reference location is cited per function.
 *
 * All kernels are asynchronous on `stream` (a cudaStream_t passed as void*).
 */
#ifndef ONNXSTREAM_B200_KERNELS_H
#define ONNXSTREAM_B200_KERNELS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* TensorDataType order of the reference (src/onnxstream.h:147-154). */
enum { OSB_NONE = 0, OSB_U8 = 1, OSB_F16 = 2, OSB_F32 = 3, OSB_I64 = 4 };

#define OSB_MAX_DIMS 6

/* XnnPack::convert / convert_qu8 (src/onnxstream.cpp:757-834); also int64 <-> float casts (src/onnxstream.cpp:7352-7424).
 * u8 -> float: (q - zp) * scale.  float -> u8: clamp(rint(x / scale) + zp, 0, 255). */
int osb_convert(const void* src, int src_dtype, void* dst, int dst_dtype, size_t n, float scale, int zero_point, void* stream);

/* Unary elementwise: Sigmoid (src/onnxstream.cpp:1217-1280), Cos/Sin/Sqrt/Erf (4001-4139), Pow with scalar exponent
 * (5478-5604), Neg (7475-7542); plus the fused chains the engine recognises: SiLU (Sigmoid*x) and erf-GELU. */
enum { OSB_UN_SIGMOID = 0, OSB_UN_SILU, OSB_UN_ERF, OSB_UN_SQRT, OSB_UN_SIN, OSB_UN_COS, OSB_UN_POW, OSB_UN_NEG,
       OSB_UN_GELU_ERF, OSB_UN_COPY, OSB_UN_MULC, OSB_UN_ADDC, OSB_UN_RECIP_SQRT };
int osb_unary(int op, const void* x, void* y, int dtype, size_t n, float alpha, void* stream);

/* N-d broadcasting binary ops: XnnPack::add/subtract/multiply/divide (src/onnxstream.cpp:846-927, 1666-1949).
 * Shapes are right-aligned and padded to `ndim` by the caller; stride 0 marks a broadcast dimension.
 * OSB_BIN_MUL_GELU computes a * gelu_erf(b) (GEGLU gate), OSB_BIN_MUL_SIGMOID a * sigmoid(b). */
enum { OSB_BIN_ADD = 0, OSB_BIN_SUB, OSB_BIN_MUL, OSB_BIN_DIV, OSB_BIN_MUL_GELU, OSB_BIN_MUL_SIGMOID, OSB_BIN_SILU_MUL /* silu(a) * b: gated MLP */ };
int osb_binary(int op, const void* a, const int64_t* a_strides, const void* b, const int64_t* b_strides,
               void* out, const int64_t* out_shape, int ndim, int dtype, void* stream);

/* Generic strided gather-copy: out[i0..] = in[in_offset + sum_k (i_k / in_div[k]) * in_stride[k]], written at
 * out_offset + sum_k i_k * out_stride[k].  Covers XnnPack::transpose (src/onnxstream.cpp:1748-1809), Concat
 * (4140-4299), Split (5999-6119), Slice (6499-6695), Expand (7154-7351) and nearest Resize (6120-6315, in_div = scale). */
/* fp32 Conv / MatMul / Gemm on the tensor cores (replaces XnnPack::convolution / matrix_multiply for float, src/onnxstream.cpp:1035-1534):
   every fp32 operand is split into three bfloat16 parts (24 mantissa bits) and expanded 6x along K so that ONE tensor-core contraction sums the
   six significant cross products in its fp32 accumulator.  expand_cols: rows of length L -> rows of 6 L (GEMM A rows, [N][K] weights, NHWC
   pixels, OHWI taps); expand_rows: a [K][N] weight -> [6 K][N].  b_side: 0 for the A operand, 1 for the B operand (the segment orders pair up).
   The f32x launchers take the bf16 expansions and fp32 C / bias / residual; cudaErrorNotSupported (801) = shape outside the tensor-core path. */
int osb_bf16x3_expand_cols(const void* in_f32, void* out_bf16, int64_t rows, int64_t L, int64_t ld_in, int b_side, void* stream);
int osb_bf16x3_expand_rows(const void* in_f32, void* out_bf16, int64_t K, int64_t N, int b_side, void* stream);
int osb_tc_gemm_f32x_ok(int64_t M, int64_t N, int64_t K);      /* 1: osb_tc_gemm_f32x takes this fp32 problem (K = the un-expanded depth) */
int osb_tc_conv_f32x_ok(int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, int64_t Ho, int64_t Wo);
int osb_tc_gemm_f32x(const void* A6, const void* B6, void* C_f32, const void* bias_f32, const void* residual_f32, int64_t M, int64_t N, int64_t K6, int b_transposed, void* stream);
int osb_tc_conv_f32x(const void* x6, const void* w6, const void* bias_f32, const void* residual_f32, void* y_f32, int64_t H, int64_t W, int64_t Cin6, int64_t Cout,
                     int kh, int kw, int stride, int pad_top, int pad_left, int64_t Ho, int64_t Wo, void* stream);
/* Concat of two tensors along one axis in one launch (src/onnxstream.cpp Concat branch, two inputs): outer slices of a_bytes / b_bytes each.
   cudaErrorNotSupported (801) unless both slice sizes and all three pointers are multiples of 16 bytes. */
int osb_concat2(const void* a, const void* b, void* out, int64_t outer, int64_t a_bytes, int64_t b_bytes, void* stream);
int osb_strided_copy(const void* in, void* out, int elem_size, int ndim, const int64_t* shape,
                     const int64_t* in_stride, const int64_t* in_div, int64_t in_offset,
                     const int64_t* out_stride, int64_t out_offset, void* stream);

/* Tiled 2-D batched transpose [B, R, C] -> [B, C, R] (NCHW <-> NHWC relayout, src/onnxstream.cpp:2914-2955). */
int osb_transpose2d(const void* in, void* out, int elem_size, int64_t batch, int64_t rows, int64_t cols, void* stream);

/* Softmax over the last axis: XnnPack::softmax (src/onnxstream.cpp:1958-2051). */
int osb_softmax(const void* x, void* y, int dtype, int64_t rows, int64_t cols, void* stream);

/* Softmax over the last axis of (x * scale + mask[row % mask_rows]): the Mul + Softmax pair of the attention pattern
 * (src/onnxstream.cpp:6837-6887) and the mask add of the SDPA pattern; mask may be NULL. */
int osb_softmax_scaled(const void* x, void* y, int dtype, int64_t rows, int64_t cols, float scale, const void* mask, int64_t mask_rows, void* stream);
/* rows stored `ld` elements apart (ld >= cols, ld <= 256 when ld != cols); pad columns of y are zero-filled */
int osb_softmax_scaled_ld(const void* x, void* y, int dtype, int64_t rows, int64_t cols, int64_t ld, float scale, const void* mask, int64_t mask_rows, void* stream);

/* InstanceNormalization on [1, C, N] contiguous (src/onnxstream.cpp:4788-5055): two-pass mean/variance per channel
 * (the reference accumulates in double), y = scale[c] * (x - mean) / sqrt(var + eps) + bias[c]. scale/bias in `dtype`. */
int osb_instance_norm(const void* x, void* y, int dtype, int64_t channels, int64_t n_per_channel,
                      const void* scale, const void* bias, float eps, void* stream);

/* Fused GroupNorm (+SiLU): the Reshape/InstanceNormalization/Reshape/Mul/Add[/Sigmoid/Mul] chain of the diffusers export
 * (SURVEY Appendix C.1) in one pass pair. x is [1,C,H,W] in NCHW (nhwc=0) or NHWC (nhwc=1) physical order; gamma/beta [C].
 * `stats` is caller-provided device scratch of 2048 bytes, zero-initialised once by the caller (the single-launch NHWC path keeps
 * its region self-cleaning; the two-pass path clears its own region per call). */
int osb_group_norm(const void* x, void* y, int dtype, int nhwc, int64_t C, int64_t HW, int groups,
                   const void* gamma, const void* beta, float eps, int fuse_silu, void* stats, void* stream);

/* GEGLU feed-forward gate: x [rows, 2*inner] -> y [rows, inner], y = x[:, :inner] * gelu_erf(x[:, inner:]).  One pass for the
 * Slice, Slice, Div, Erf, Add, Mul, Mul, Mul group (src/onnxstream.cpp Slice 6499-6652, Erf 1950-2100, binary ops 1666-1949). */
int osb_geglu(const void* x, void* y, int dtype, int64_t rows, int64_t inner, void* stream);

/* Fused LayerNorm over the last axis (ReduceMean,Sub,Pow,ReduceMean,Add,Sqrt,Div,Mul,Add chain; src/onnxstream.cpp
 * 5237-5393 et al.).  gamma/beta may be NULL. */
int osb_layer_norm(const void* x, void* y, int dtype, int64_t rows, int64_t cols, const void* gamma, const void* beta,
                   float eps, void* stream);

/* ReduceMean over the last axis (src/onnxstream.cpp:5237-5393). */
int osb_reduce_mean(const void* x, void* y, int dtype, int64_t rows, int64_t cols, void* stream);

/* Row gather: out[i, :] = table[idx[i], :]  (Gather axis 0, src/onnxstream.cpp:6316-6498). idx is int64 on device. */
int osb_gather_rows(const void* table, const int64_t* idx, void* out, int64_t n_idx, int64_t table_rows, int64_t row_bytes, void* stream);

/* Batched GEMM  C[b] = A[b] (M x K, row-major) * B[b] (K x N, row-major) (+ bias[N]) (+ residual[b] M x N):
 * XnnPack::matrix_multiply / matrix_multiply_dynamic (src/onnxstream.cpp:929-1215) and the MatMul/Gemm branches
 * (4300-4375, 5669-5861).  stride_* are element strides between batches (0 = shared operand).
 * b_transposed: B[b] is stored N x K row-major.  Accumulation is fp32 for both dtypes.
 * `impl`: 0 = auto (tensor cores when dtype == f16 and the shape is eligible), 1 = force the CUDA-core reference kernel,
 * 2 = force the tensor-core kernel (returns an error if ineligible). */
int osb_gemm(const void* A, const void* B, void* C, const void* bias, const void* residual,
             int64_t batch, int64_t M, int64_t N, int64_t K,
             int64_t stride_a, int64_t stride_b, int64_t stride_c, int b_transposed, int dtype, int impl, void* stream);

/* `groups` (1..3) GEMMs C_g = A * B_g sharing A [M,K] and the shape, dense operands, no bias: one tensor-core launch when the
 * problem qualifies (the q/k/v MatMuls of an attention block, src/onnxstream.cpp:4343-4664 run three times), else `groups`
 * ordinary launches. */
int osb_gemm_grouped(const void* A, const void* const* B, void* const* C, int groups, int64_t M, int64_t N, int64_t K,
                     int b_transposed, int dtype, int impl, void* stream);

/* Same with explicit leading dimensions (elements between consecutive rows of A, B, C): lets the attention GEMMs read the
 * per-head slices of a [T, heads*d] projection in place -- the Reshape/Transpose/Reshape head split and merge of the exported
 * graph (SURVEY Appendix C.1) costs no copy -- and write O straight into the merged [T, heads*d] layout. */
int osb_gemm_ld(const void* A, int64_t lda, const void* B, int64_t ldb, void* C, int64_t ldc, const void* bias, const void* residual,
                int64_t batch, int64_t M, int64_t N, int64_t K, int64_t stride_a, int64_t stride_b, int64_t stride_c,
                int b_transposed, int dtype, int impl, void* stream);

/* 2-D convolution, batch 1, groups 1, dilation 1: XnnPack::convolution (src/onnxstream.cpp:1292-1534).
 * x NHWC [H,W,Cin], w OHWI [Cout,kh,kw,Cin], bias [Cout] or NULL, y NHWC [Ho,Wo,Cout]; optional residual (same shape
 * as y) added in the epilogue.  Padding follows the reference's re-symmetrisation: callers pass pad_top/pad_left
 * computed as (p0+p2)/2, (p1+p3)/2 (src/onnxstream.cpp:1315-1329). */
int osb_conv2d(const void* x, const void* w, const void* bias, const void* residual, void* y,
               int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, int pad_top, int pad_left,
               int64_t Ho, int64_t Wo, int dtype, int impl, void* stream);
/* Conv with a second per-channel addend (`bias2`: the time-embedding row a resnet adds to conv1's output, src/onnxstream.cpp:5056-5175 Add
 * on a [1,C,1,1] operand) and with the GroupNorm statistics of the output gathered in the epilogue: gn_stats = fp64 [2 * gn_groups]
 * (sum, sum of squares per group of Cout / gn_groups channels), ACCUMULATED into (the caller zeroes it); *gn_done = 1 when the kernel
 * produced them.  Both need the tensor-core path: ask osb_conv2d_fusable first. */
int osb_conv2d_ex(const void* x, const void* w, const void* bias, const void* bias2, const void* residual, void* y, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                  int kh, int kw, int stride, int pad_top, int pad_left, int64_t Ho, int64_t Wo, int dtype, int impl, void* stream,
                  void* gn_stats, int gn_groups, int* gn_done);
int osb_conv2d_fusable(const void* x, const void* w, const void* y, int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, int dtype, int impl);
/* GroupNorm(+SiLU) apply pass on an NHWC tensor whose statistics were gathered by the producing conv (osb_conv2d_ex): reads `stats`,
 * writes y = silu?((x - mean) * rstd * gamma + beta), and zeroes `clear_stats` (the buffer the NEXT producer will accumulate into). */
/* RMSNorm y = w * x / sqrt(mean(x^2) + eps) over the last axis, fp32 arithmetic, any mix of fp16 / fp32 storage (the 7-op chain Pow,
 * ReduceMean, Add, Sqrt, Div, Mul, Mul of llm.cpp's graphs; the reference keeps it in fp32 through m_requires_upcast, src/llm.cpp:385-389) */
int osb_rms_norm(const void* x, int xd, const void* w, int wd, void* y, int yd, int64_t rows, int64_t cols, float eps, void* stream);
/* rotary embedding, rotate_half form (Slice, Slice, Neg, Concat, Mul, Mul, Add): y = x * cos + rotate_half(x) * sin; cos / sin: 1 or `rows` rows of D */
int osb_rope(const void* x, const void* cs, const void* sn, void* y, int dtype, int64_t rows, int64_t D, int64_t table_rows, void* stream);
/* Decode GEMV with uint8 weights [K,N] dequantised in registers (M <= 2): y = x . ((Wq - zp) * scale rounded to `dtype`) + bias + residual.
 * The uint8-weight / float-arithmetic MatMul of the reference (weights converted at load, src/onnxstream.cpp:2885-2890) at half the HBM bytes. */
int osb_gemv_w8(const void* A, const void* Wq, void* C, const void* bias, const void* residual, int64_t M, int64_t N, int64_t K, float wscale, int wzp, int dtype, void* stream);
/* 2 or 3 GEMVs that share their input rows (q / k / v projections, gate / up of a gated MLP: consecutive MatMul nodes of llm.cpp's graphs,
   src/onnxstream.cpp:5669-5861) as one launch; wdtype OSB_U8 = uint8 weights dequantised in registers.  cudaErrorNotSupported (801) when the
   shapes are outside the grouped kernels: launch them one by one. */
int osb_gemv_grouped(const void* A, const void* const* B, void* const* C, const int64_t* N, const float* wscale, const int* wzp, int groups,
                     int64_t M, int64_t K, int wdtype, int dtype, void* stream);
/* W8A8 on the tensor cores (wgmma .u8, uint8 x uint8 -> int32): XnnPack::matrix_multiply<uint8_t,int32_t> / convolution for uint8
 * (src/onnxstream.cpp:1035-1215, 1292-1534) with XNNPACK's fp32 requantisation y = clamp(lrintf(acc * sx*sw/sy)) + zy.  The kernel multiplies raw
 * bytes and corrects with rowsum_x / colsum_w (osb_rowsum_u8: row sums of a [rows][cols] byte matrix; osb_colsum_u8: column sums of a [K][N] one);
 * a convolution runs on the image padded with the input zero point (osb_pad_sum_u8 also emits its per-pixel channel sums).  *_ok: TMA-addressable. */
int osb_qu8_tc_gemm_ok(int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C);
int osb_qu8_tc_conv_ok(int64_t Cin, int64_t Cout, int64_t Ho, int64_t Wo, int kh, int kw, int stride, const void* x, const void* w, const void* y);
int osb_rowsum_u8(const void* x, void* out, int64_t rows, int64_t cols, void* stream);
int osb_colsum_u8(const void* w, void* out, int64_t K, int64_t N, void* stream);
int osb_pad_sum_u8(const void* x, void* xp, void* psum, int64_t H, int64_t W, int64_t C, int64_t Hp, int64_t Wp, int pad_top, int pad_left, int zx, void* stream);
int osb_qu8_tc_gemm(const void* A, const void* B, void* C, const void* bias, const void* rsum, const void* csum, int64_t M, int64_t N, int64_t K, int bt,
                    int zx, float sx, int zw, float sw, int zy, float sy, void* stream);
int osb_qu8_tc_conv(const void* xp, const void* psum, const void* w, const void* bias, const void* csum, void* y, int64_t Hp, int64_t Wp, int64_t Cin, int64_t Cout,
                    int kh, int kw, int stride, int64_t Ho, int64_t Wo, int zx, float sx, int zw, float sw, int zy, float sy, void* stream);
/* XNNPACK qu8 elementwise add / multiply with N-d broadcasting (XnnPack::add / multiply for T = uint8_t, src/onnxstream.cpp:846-927, 1666-1746):
 * strides in elements (0 = broadcast) like osb_binary.  Bit-exact restatement of the library's fixed-point add and fp32-requantised multiply. */
int osb_binary_qu8(int op, const void* a, const int64_t* as, float sa, int za, const void* b, const int64_t* bs, float sb, int zb,
                   void* out, float so, int zo, const int64_t* shape, int ndim, void* stream);
/* qu8 softmax over the last axis (XnnPack::softmax for T = uint8_t, src/onnxstream.cpp:1958-2051; output scale 2^-8 / zero point 0 at 5971-5972) */
int osb_softmax_qu8(const void* x, void* y, int64_t rows, int64_t cols, float in_scale, float out_scale, int out_zp, void* stream);
/* Dynamic-quantisation range of a float tensor, Model::get_percentiles (src/onnxstream.cpp:3104-3232): per reference chunk (the tensor
 * split over `threads` pool workers, then 64 KiB buffers) the k-th smallest / largest finite value, k = (size_t)(n_chunk * from_x); min of
 * the lows, max of the highs.  out3 = DEVICE uint32[3] initialised to {0xFFFFFFFF, 0, 0}: order-preserving keys of (low, high) and the
 * number of chunks that produced a result; decode with osb_percentile_key_to_float. */
int osb_percentiles(const void* x, int dtype, size_t n, int threads, float from_left, float from_right, void* out3, void* stream);
float osb_percentile_key_to_float(unsigned key, int dtype);
/* NHWC statistics producer for osb_group_norm_apply: stats[2 * groups] += per-group (sum, sum of squares) of y = x + addv[c]; addv and
 * y both null = statistics of x.  cudaErrorInvalidValue for shapes the vector kernel does not cover. */
int osb_channel_add_stats(const void* x, const void* addv, void* y, int dtype, int64_t C, int64_t HW, int groups, void* stats, void* stream);
int osb_group_norm_apply(const void* x, void* y, int dtype, int64_t C, int64_t HW, int groups, const void* gamma, const void* beta, float eps, int fuse_silu,
                         const void* stats, void* clear_stats, void* stream);

/* Fused attention softmax(Q K^T * scale) V per head: the AttentionFusedOps branch (src/onnxstream.cpp:6696-6929).
 * q [h,Tq,d], k [h,d,Tk] when k_transposed (the diffusers export) else [h,Tk,d], v [h,Tk,d], out [h,Tq,d].
 * `mask` (optional, [Tq,Tk], additive, same dtype) and `kv_group` (query heads per kv head) cover the
 * ScaledDotProductAttention branch (src/onnxstream.cpp:7767-7882). */
int osb_attention(const void* q, const void* k, const void* v, const void* mask, void* out,
                  int64_t heads, int64_t Tq, int64_t Tk, int64_t d, int64_t dv, float scale, int k_transposed,
                  int64_t kv_group, int dtype, void* stream);

/* Fused flash-style multi-head attention on wgmma (fp16, d <= 64): q [T, heads*d] / k, v [Tk, heads*d] are read in place
 * from the projection buffers (row strides ld*), out [T, heads*d] is written in the merged layout; the score tile lives in registers.
 * Covers the MatMul/Mul/Softmax/MatMul pattern plus the head split / merge around it (src/onnxstream.cpp:3576-3633, 6696-6929). */
int osb_flash_attention_ok(int64_t T, int64_t Tk, int64_t d, int dtype);
int osb_flash_attention(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out, int64_t ldo,
                        int64_t heads, int64_t T, int64_t Tk, int64_t d, float scale, void* stream);

/* qu8 GEMM / conv with XNNPACK's requantisation (bit-exact target; SURVEY section 8c):
 * acc = sum (x - zx)(w - zw) + bias_i32; y = clamp(lrintf(acc * (sx*sw/sy)) + zy, 0, 255). */
int osb_gemm_qu8(const uint8_t* A, const uint8_t* B, uint8_t* C, const int32_t* bias, int64_t M, int64_t N, int64_t K,
                 int zx, float sx, int zw, float sw, int zy, float sy, void* stream);
int osb_conv2d_qu8(const uint8_t* x, const uint8_t* w, const int32_t* bias, uint8_t* y,
                   int64_t H, int64_t W, int64_t Cin, int64_t Cout, int kh, int kw, int stride, int pad_top, int pad_left,
                   int64_t Ho, int64_t Wo, int zx, float sx, int zw, float sw, int zy, float sy, void* stream);

/* ScatterND with full-rank indices (src/onnxstream.cpp:7939-8074): out[pos[i]] = updates[i] for 2- or 4-byte elements; `pos`
 * = host-linearised, range-checked positions, on the device. */
int osb_scatter_elems(void* out, const int64_t* pos, const void* updates, int64_t n, int elem_size, void* stream);

/* MaxPool, NHWC, dilation 1, ceil_mode 0 (XnnPack::maxpool_nhwc, src/onnxstream.cpp:1537-1664; branch 8075-8143). */
int osb_maxpool_nhwc(const void* x, void* y, int dtype, int64_t H, int64_t W, int64_t C, int kh, int kw, int stride, int pad_top,
                     int pad_left, int64_t Ho, int64_t Wo, void* stream);

/* Fill `n` bytes-worth of elements with a constant (ConstantOfShape, src/onnxstream.cpp:7543-7588). */
int osb_fill(void* dst, int dtype, size_t n, float value, void* stream);

/* 1 when the wgmma/TMA GEMM path can take this problem (used by tests and the bench to assert the fast path ran). */
int osb_gemm_tc_eligible(int64_t M, int64_t N, int64_t K, int dtype);

/* Tile decomposition of the tensor-core GEMM / conv: 0 = one CTA per 128 x 128 tile only, 1 = the default rule (single tiles: CTA pairs
 * measured slower on the H100), 2 = CTA pairs (2-CTA clusters sharing the B tile through TMA multicast) wherever the shape is
 * eligible.  Tests and A/B runs. */
void osb_tc_set_pair_mode(int mode);

/* Per-launch timing of the wgmma GEMM/conv kernel (CUDA events on the launching stream; eager mode only).
 * osb_tc_profile(1) starts recording, osb_tc_profile_read fills {launches, total ms, total FLOPs, total algorithmic bytes}. */
void osb_tc_profile(int enable);
int osb_tc_profile_read(double* out4);
int osb_tc_profile_dump(char* buf, int cap);   /* one line per launch: M N K taps batch split conv ms gflop */

/* Programmatic dependent launch for every kernel of this library (default on). */
int osb_pdl_enabled(void);
void osb_set_pdl(int enable);

/* Counters: number of kernel launches issued through this ABI since the last reset (bench.py's gpu_launches). */
uint64_t osb_launch_count(void);
void osb_launch_count_reset(void);
uint64_t osb_tc_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif
