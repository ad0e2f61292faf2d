/* b200_quant.h — internal C ABI of the one-pass e4m3 quantisers of FP8 activations (libb200_quant.so). Like
 * libb200_epilogue.so, the library has no public symbol: cuda_l2_b200/capi.py binds it (capi.INTERNAL_ABI).
 *
 * They produce the A operand and its scales for the FP8 GEMMs of the other libraries, in the layouts those read:
 *
 *   per tensor   q = e4m3(x / s), one scale s for the whole tensor (b200_fp8gemm, include/b200_hgemm.h)
 *   rowwise      one scale per row of x [rows, cols], scale [rows] (b200_fp8gemm_rowwise)
 *   1 x 128      one scale per row and 128-column block of x [(B,) M, K], written M-major into the scale_a layout of
 *                the block-scaled GEMMs (include/b200_fp8_block.h, b200_grouped_fp8.h, b200_batched_fp8.h)
 *   SwiGLU       the 1 x 128 quantiser of silu(g) * u, with g = h[..., :I] and u = h[..., I:] of h [(B,) M, 2I]
 *
 * Each element is read from device memory once (twice for the per-tensor quantiser, see below) and written once.
 * Inputs: dtype 0 fp16, 1 bf16, 2 fp32 (the SwiGLU kernel takes fp16 and bf16 only). Rows are contiguous; any length
 * is accepted (16-byte vector loads when the pointers and the row length allow them, element loads otherwise). q is
 * float8_e4m3fn, contiguous in the shape of the input. stream is a cudaStream_t (NULL = legacy default stream). The
 * calls never synchronise with the host and use no memory of their own, so they are safe on concurrent streams and in
 * CUDA-graph capture.
 *
 * Arithmetic, in fp32 with IEEE operations (no fast-math, no flush to zero), per scale group G:
 *   amax  = max over G of |x|; NaN if any element of G is NaN (torch.amax's rule)
 *   s     = fp32(amax * fp32(1 / 448)), then FLT_MIN if s < FLT_MIN (a NaN s stays NaN)
 *   q     = e4m3fn(clamp(x / s, -448, 448)), x / s an IEEE division, the clamp keeping NaN, the conversion rounding to
 *           nearest even; a NaN gives 0x7f with the sign of the quotient
 * These are the bits of the torch composition the ops layer keeps as its reference (cuda_l2_b200/ops.py): torch's CUDA
 * division of a tensor by a Python scalar multiplies by the scalar's fp32 reciprocal, which is why s is a product.
 * SwiGLU first forms p = RN(fp32(RN(g / (1 + expf(-g)))) * fp32(u)), RN being the rounding to the input type and expf
 * the full-precision one (torch's CUDA silu, then the product of two 16-bit tensors), and quantises p.
 *
 * Return value: 0 on success, < 0 a status (cuda_l2_b200_quant_strerror), > 0 a cudaError_t from the launch.
 * Launches are asynchronous. Statuses: -1 a size <= 0 (1 x 128: or more than INT_MAX tiles of 32 rows by one
 * k-block); -5 a null pointer; -6 an unknown dtype (or fp32 for SwiGLU); -10 ld_a < M or ld_a % 4 != 0; -2 a scale or
 * workspace pointer that is not 4-byte aligned. Every status comes back before any CUDA call.
 */
#ifndef CUDA_L2_B200_QUANT_H_
#define CUDA_L2_B200_QUANT_H_

#ifdef __cplusplus
extern "C" {
#endif

/* Floats of the workspace cuda_l2_b200_quant_e4m3_tensor takes. */
#define CUDA_L2_B200_QUANT_TENSOR_WORKSPACE 1024

/* Per tensor, two launches: each CTA of the first writes the amax of its share of x to workspace
 * (CUDA_L2_B200_QUANT_TENSOR_WORKSPACE floats of device memory, owned by the call until the second launch has run);
 * each CTA of the second reduces those partials to amax and quantises its share, and its first CTA writes scale[0].
 * The result does not depend on the order of the partials. */
int cuda_l2_b200_quant_e4m3_tensor(int dtype, const void* x, long long n, void* q, float* scale,
                                   float* workspace, void* stream);

/* Rowwise, one launch: scale[r] for every row r of x [rows, cols]. Up to 16384 columns (8192 for fp32) a row is held
 * on chip between its two passes; longer rows are read a second time, from L2. */
int cuda_l2_b200_quant_e4m3_rowwise(int dtype, const void* x, int rows, int cols, void* q, float* scale,
                                    void* stream);

/* 1 x 128 blocks, one launch: x [B, M, K] (B = 1 for a 2-D x), q [B, M, K], scale value (b, m, kb) at
 * scale[(b * nkb + kb) * ld_a + m], nkb = ceil(K / 128), ld_a >= M and ld_a % 4 == 0: torch's [(B,) M, nkb] view with
 * strides (nkb * ld_a, 1, ld_a), which the block-scaled GEMMs read in place. Each CTA stores the scales of 32
 * consecutive rows of one k-block with one coalesced store. masked_m (optional, NULL = every row): B int32 values in
 * device memory, read by the kernel; only rows [0, clamp(masked_m[b], 0, M)) of matrix b are read and written (q and
 * scale), the rest keep what they held. */
int cuda_l2_b200_quant_e4m3_blockwise(int dtype, const void* x, int B, int M, int K, void* q, float* scale,
                                      int ld_a, const int* masked_m, void* stream);

/* SwiGLU + 1 x 128 blocks, one launch: h [B, M, 2I] (fp16 or bf16), q [B, M, I], scale and masked_m as for
 * cuda_l2_b200_quant_e4m3_blockwise with K = I. */
int cuda_l2_b200_quant_silu_mul_e4m3_blockwise(int dtype, const void* h, int B, int M, int I, void* q,
                                               float* scale, int ld_a, const int* masked_m, void* stream);

/* Kernel launches issued by this library since load. */
unsigned long long cuda_l2_b200_quant_launch_count(void);

const char* cuda_l2_b200_quant_strerror(int status);

#ifdef __cplusplus
}
#endif
#endif /* CUDA_L2_B200_QUANT_H_ */
