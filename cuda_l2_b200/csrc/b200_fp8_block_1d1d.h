/* b200_fp8_block_1d1d.h — internal C ABI of the block-scaled FP8 (e4m3) GEMM with 1 x 128 scales on both operands
 * (libb200_fp8block_1d1d.so). Like libb200_quant.so, the library has no public symbol: cuda_l2_b200/capi.py binds it
 * (capi.INTERNAL_ABI), and users reach it through fp8_gemm with scale_b [N, ceil(K/128)].
 *
 *     C[M,N] (fp16 or bf16) = A[M,K] (e4m3) x Bt[N,K]^T (e4m3), one fp32 scale per (row of A, 128-element k-block) and
 *     one per (row of Bt, 128-element k-block)
 *
 * The weight gradient of blockwise FP8 training, dW = q(dY^T) q(X^T)^T: both operands are transposed activations,
 * [out, T] and [in, T], each quantised per row and per 128 tokens. Operand conventions as in include/b200_fp8_block.h:
 * A and Bt K-major (float8_e4m3fn, K contiguous), C [M,N] row-major and fully overwritten, all 16-byte aligned,
 * K % 16 == 0, N % 8 == 0; stream is a cudaStream_t (NULL = legacy default stream).
 *
 * Scales (fp32, device memory, read when the kernel runs), with nkb = ceil(K/128):
 *   scale_a   value (m, kb) at scale_a[kb * ld_a + m]: M-major, torch's [M, nkb] with strides (1, ld_a). ld_a >= M,
 *             ld_a % 4 == 0, 16-byte aligned; nkb * ld_a floats must be readable.
 *   scale_b   value (n, kb) at scale_b[kb * ld_b + n]: the same N-major form. ld_b >= N, ld_b % 4 == 0, 16-byte
 *             aligned; nkb * ld_b floats must be readable.
 * Arithmetic: p_kb[m,n] is the sum of the 128 products of k-block kb (the last block is zero-filled past K), s =
 * fp32(scale_a(m,kb) * scale_b(n,kb)). acc = fp32(p_kb0 * s) for a unit's first k-block, acc = fmaf(p_kb, s, acc) for
 * every later one in increasing kb, C = RN_out(acc). Cluster split-K (splits -2/-4/-8) sums the splits' scaled partials
 * in fixed order. This is include/b200_fp8_block.h's contract with only the index of scale_b changed: with
 * scale_b(n, kb) = that header's scale_b(n / 128, kb) the two libraries compute the same bits for the same configuration
 * and splits. Plain and cluster split-K schedules only: no scratch memory, always safe to capture in a CUDA graph.
 *
 * Return value: 0 on success, < 0 a status (cuda_l2_b200_fp8block_1d1d_strerror), > 0 a cudaError_t. Launches are
 * asynchronous. Statuses as in include/b200_fp8_block.h (-10 for a bad ld_a, null scales -5, a misaligned scale_a or
 * scale_b -2), plus -13 for ld_b < N or ld_b % 4 != 0. Every status comes back before any CUDA call.
 */
#ifndef CUDA_L2_B200_FP8_BLOCK_1D1D_H_
#define CUDA_L2_B200_FP8_BLOCK_1D1D_H_

#ifdef __cplusplus
extern "C" {
#endif

/* The dispatched call: b200_fp8gemm_blockwise_select's choice (libb200_fp8block.so's rule, unchanged). out_bf16: 0 fp16
 * output, 1 bf16 output (anything else: -6). */
int cuda_l2_b200_fp8block_1d1d_run(const void* A, const void* B_kmajor, void* C, const void* scale_a, int ld_a,
                                   const void* scale_b, int ld_b, int out_bf16, int M, int N, int K, void* stream);

/* One explicit configuration: the block-scaled ones of include/b200_fp8_block.h (m_rep * bn <= 128: 1, 2, 4, 7-17, 22,
 * 23 and 30; any other id returns -6). splits: 1 none, -2/-4/-8 cluster split-K (configurations 1 and 2); any other
 * code runs the plain schedule. */
int cuda_l2_b200_fp8block_1d1d_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                          const void* scale_a, int ld_a, const void* scale_b, int ld_b, int M, int N,
                                          int K, int group_m, int max_ctas, int splits, void* stream);

/* The dispatcher's choice (config id, rasterisation group, splits code): b200_fp8gemm_blockwise_select's. Returns 0 or
 * a negative status. */
int cuda_l2_b200_fp8block_1d1d_select(int M, int N, int K, int* config_id, int* group_m, int* splits);

/* Kernel launches issued by this library since load. */
unsigned long long cuda_l2_b200_fp8block_1d1d_launch_count(void);

const char* cuda_l2_b200_fp8block_1d1d_strerror(int status);

#ifdef __cplusplus
}
#endif
#endif /* CUDA_L2_B200_FP8_BLOCK_1D1D_H_ */
