/* b200_quant_dual.h — internal C ABI of the dual-orientation rowwise e4m3 quantiser (libb200_quant_dual.so). Like
 * libb200_quant.so, the library has no public symbol: cuda_l2_b200/capi.py binds it (capi.INTERNAL_ABI).
 *
 * FP8 training of a linear layer runs three rowwise-scaled GEMMs, and e4m3 wgmma reads only K-major operands, so each of
 * x, W and dY is needed twice: quantised along its rows, and transposed and quantised along its columns. This call
 * produces both from x [rows, cols] (rows contiguous):
 *
 *   q       [rows, cols]   e4m3, scale   [rows] fp32: the rowwise quantisation of x (b200_quant.h's, bit for bit)
 *   q_t     [cols, ld_t]   e4m3, scale_t [cols] fp32: the rowwise quantisation of x^T zero-padded to ld_t columns,
 *                          ld_t = rows rounded up to 16, so that q_t is a K-major operand of the FP8 GEMM (K % 16 == 0)
 *
 * The arithmetic is b200_quant.h's (shared source, b200_quant_arith.cuh): s = fp32(amax * fp32(1/448)), FLT_MIN if
 * smaller, NaN if the group holds one; q = e4m3fn(clamp(v / s, -448, 448)) with an IEEE division. A padding byte of q_t
 * is e4m3(0 / s): 0x00, or 0x7f where the column's scale is NaN. Inputs: dtype 0 fp16, 1 bf16, 2 fp32; any row length
 * (16-byte vector loads when x, q and the row length allow them, element loads otherwise). stream is a cudaStream_t
 * (NULL = legacy default stream).
 *
 * A column's amax needs every row, so the call is one memset and two launches, in stream order:
 *   1. cudaMemsetAsync of the workspace to zero;
 *   2. each CTA reduces a 128-row tile to per-row and per-column maxima of |x| and folds them into the workspace with
 *      atomicMax on the bits of |x| (for non-negative floats the unsigned order of the bits is the float order, and
 *      every NaN sorts above +Inf, which is torch.amax's NaN rule);
 *   3. each CTA reloads a 64 x 64 tile, reads its rows' and columns' maxima, stores q row-major, and stores q_t through a
 *      shared-memory transpose with 16-byte stores; the CTAs of the first tile column write scale, those of the first
 *      tile row scale_t.
 * The maxima do not depend on the order of the atomics, so the bits are deterministic. The call never synchronises
 * with the host and uses no memory of its own: the workspace is the caller's, and owned by the call until the third
 * step has run. It is therefore safe on concurrent streams (one workspace per call) and in CUDA-graph capture.
 *
 * Return value: 0 on success, < 0 a status (cuda_l2_b200_quant_dual_strerror), > 0 a cudaError_t from the memset or a
 * launch. Statuses: -1 rows or cols <= 0, or rows > INT_MAX - 15; -2 scale, scale_t or workspace not 4-byte aligned, or
 * q_t not 16-byte aligned; -5 a null pointer; -6 an unknown dtype. Every status comes back before any CUDA call.
 */
#ifndef CUDA_L2_B200_QUANT_DUAL_H_
#define CUDA_L2_B200_QUANT_DUAL_H_

#ifdef __cplusplus
extern "C" {
#endif

/* Floats of the workspace cuda_l2_b200_quant_dual_e4m3_rowwise takes for x [rows, cols]. */
#define CUDA_L2_B200_QUANT_DUAL_WORKSPACE(rows, cols) ((long long)(rows) + (long long)(cols))

/* q [rows, cols] and scale [rows]; q_t [cols, ld_t] (ld_t = (rows + 15) / 16 * 16, rows of q_t contiguous) and
 * scale_t [cols]; workspace: CUDA_L2_B200_QUANT_DUAL_WORKSPACE(rows, cols) floats of device memory. */
int cuda_l2_b200_quant_dual_e4m3_rowwise(int dtype, const void* x, int rows, int cols, void* q, float* scale,
                                         void* q_t, float* scale_t, float* workspace, void* stream);

/* Kernel launches issued by this library since load (two per call; the memset is not a launch). */
unsigned long long cuda_l2_b200_quant_dual_launch_count(void);

const char* cuda_l2_b200_quant_dual_strerror(int status);

#ifdef __cplusplus
}
#endif
#endif /* CUDA_L2_B200_QUANT_DUAL_H_ */
