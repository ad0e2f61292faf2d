/* b200_quant_block_dual.h — internal C ABI of the dual-orientation block e4m3 quantisers (libb200_quant_block_dual.so).
 * Like libb200_quant.so, the library has no public symbol: cuda_l2_b200/capi.py binds it (capi.INTERNAL_ABI).
 *
 * Blockwise FP8 training of a linear layer (the DeepSeek-V3 recipe) quantises x and dY per token and 128 channels and W
 * per 128 x 128 block, and needs each of them twice, as e4m3 wgmma reads only K-major operands: along its rows, and
 * transposed along its columns. Both orientations of a 128 x 128 tile are complete groups (each row's 128 columns,
 * each column's 128 rows), so one CTA per tile reads the tile once and writes both: one launch, no atomics, no
 * workspace.
 *
 *   1 x 128, x [rows, cols]:
 *     q       [rows, cols]  e4m3, scale   value (r, cb) at scale[cb * ld_s + r], ld_s = rows rounded up to 4 (the M-major
 *                           [ceil(cols/128), ld_s] layout of cuda_l2_b200_quant_e4m3_blockwise, b200_quant.h)
 *     q_t     [cols, ld_t]  e4m3, ld_t = rows rounded up to 16: x^T zero-padded, quantised per row and 128 columns, with
 *                           scale_t value (c, rb) at scale_t[rb * ld_st + c], ld_st = cols rounded up to 4
 *   128 x 128, w [rows, cols]:
 *     q       [rows, cols]  e4m3, scale   row-major [ceil(rows/128), ceil(cols/128)]
 *     q_t     [cols, rows]  e4m3, q^T, scale_t row-major [ceil(cols/128), ceil(rows/128)], scale^T: with 128 x 128 blocks
 *                           the quantisation of w^T is the transpose of that of w, bit for bit
 *
 * The arithmetic is b200_quant.h's (shared source, b200_quant_arith.cuh): s = fp32(amax * fp32(1/448)), FLT_MIN if
 * smaller, NaN if the group holds one; q = e4m3fn(clamp(v / s, -448, 448)) with an IEEE division; a group past the
 * tensor's edge is zero-padded. A padding byte of q_t (1 x 128) is e4m3(0 / s): 0x00, or 0x7f where the group's scale is
 * NaN. Inputs: dtype 0 fp16, 1 bf16; any row length (16-byte vector loads and 8-byte stores of q when x, q and the row
 * length allow them, element accesses otherwise); q_t is stored 16 bytes at a time where its row length is a multiple of
 * 16, a byte at a time otherwise. stream is a cudaStream_t (NULL = legacy default stream). No host synchronisation and no
 * memory of its own: safe on concurrent streams and in CUDA-graph capture.
 *
 * Return value: 0 on success, < 0 a status (cuda_l2_b200_quant_block_dual_strerror), > 0 a cudaError_t from the launch.
 * Statuses: -1 rows or cols <= 0, rows > INT_MAX - 15, or more than INT_MAX tiles of 128 x 128; -2 scale or scale_t not
 * 4-byte aligned, or q_t not 16-byte aligned; -5 a null pointer; -6 an unknown dtype. Every status comes back before any
 * CUDA call.
 */
#ifndef CUDA_L2_B200_QUANT_BLOCK_DUAL_H_
#define CUDA_L2_B200_QUANT_BLOCK_DUAL_H_

#ifdef __cplusplus
extern "C" {
#endif

/* 1 x 128 groups of x [rows, cols] and of x^T, in one launch. */
int cuda_l2_b200_quant_block_dual_e4m3_1x128(int dtype, const void* x, int rows, int cols, void* q, float* scale,
                                             void* q_t, float* scale_t, void* stream);

/* 128 x 128 blocks of w [rows, cols] and their transpose, in one launch. */
int cuda_l2_b200_quant_block_dual_e4m3_128x128(int dtype, const void* w, int rows, int cols, void* q, float* scale,
                                               void* q_t, float* scale_t, void* stream);

/* Kernel launches issued by this library since load (one per call). */
unsigned long long cuda_l2_b200_quant_block_dual_launch_count(void);

const char* cuda_l2_b200_quant_block_dual_strerror(int status);

#ifdef __cplusplus
}
#endif
#endif /* CUDA_L2_B200_QUANT_BLOCK_DUAL_H_ */
