/* b200_fp8_block.h — C ABI of the block-scaled FP8 (e4m3) GEMM (libb200_fp8block.so).
 *
 *     C[M,N] (fp16 or bf16) = A[M,K] (e4m3) x Bt[N,K]^T (e4m3), one fp32 scale per (row of A, 128-element k-block) and
 *     one per 128 x 128 block of Bt
 *
 * The scale granularity of DeepSeek-V3-style FP8 checkpoints: the weight Bt is stored with `weight_scale_inv`
 * [ceil(N/128), ceil(K/128)], the activation A is quantised per token and per 128 input channels. A library of its own,
 * next to libb200_hgemm.so (include/b200_hgemm.h), with the same operand conventions: A and Bt K-major
 * (float8_e4m3fn, K contiguous), C [M,N] row-major and fully overwritten, all of them 16-byte aligned, K % 16 == 0,
 * N % 8 == 0; stream is a cudaStream_t (NULL = legacy default stream).
 *
 * Scales (fp32, device memory, read when the kernel runs), with nkb = ceil(K/128):
 *   scale_a   value (m, kb) at scale_a[kb * ld_a + m]: M-major, torch's [M, nkb] with strides (1, ld_a). ld_a >= M,
 *             ld_a % 4 == 0, 16-byte aligned; nkb * ld_a floats must be readable.
 *   scale_b   row-major [ceil(N/128), nkb], 4-byte aligned (the checkpoint layout).
 * Arithmetic: p_kb[m,n] is the sum of the 128 products of k-block kb (the last block is zero-filled past K), s =
 * fp32(scale_a(m,kb) * scale_b(n/128,kb)). acc = fp32(p_kb0 * s) for a unit's first k-block, acc = fmaf(p_kb, s, acc)
 * for every later one in increasing kb, C = RN_out(acc). Cluster split-K (splits -2/-4/-8) sums the splits' scaled
 * partials in fixed order. There is no output scale. Only the plain and cluster split-K schedules exist for this
 * variant, so it never needs scratch memory and is always safe to capture in a CUDA graph.
 *
 * Return value: 0 on success, < 0 a status (b200_fp8block_strerror), > 0 a cudaError_t. Launches are asynchronous.
 * Statuses as in b200_hgemm.h, plus -10 for ld_a < M or ld_a % 4 != 0; null scales are -5, a misaligned scale_a /
 * scale_b -2.
 */
#ifndef B200_FP8_BLOCK_H_
#define B200_FP8_BLOCK_H_

#ifdef __cplusplus
extern "C" {
#endif

/* The dispatched call. out_bf16: 0 fp16 output, 1 bf16 output (anything else: -6). */
int b200_fp8gemm_blockwise(const void* A, const void* B_kmajor, void* C, const void* scale_a, int ld_a,
                           const void* scale_b, int out_bf16, int M, int N, int K, void* stream);

/* One explicit configuration of libb200_hgemm.so's table (b200_hgemm_config_info). Only configurations with
 * m_rep * bn <= 128 have block-scaled kernels (two accumulator sets must fit the registers): 1, 2, 4, 7-17, 22, 23 and
 * 30; any other id returns -6. splits: 1 none, -2/-4/-8 cluster split-K (configurations 1 and 2); any other code runs
 * the plain schedule. */
int b200_fp8gemm_blockwise_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                      const void* scale_a, int ld_a, const void* scale_b, int M, int N, int K,
                                      int group_m, int max_ctas, int splits, void* stream);

/* The dispatcher's choice: the e4m3 choice of b200_fp8gemm_select, its configuration mapped to the block-scaled
 * one with the same CTA group and cluster, M_REP 1 and BN min(BN, 128), a workspace split-K factor s to cluster split-K
 * of the largest of 8/4/2 not above s (where that configuration has it), stream-K to the plain schedule.
 * Returns 0 or a negative status. */
int b200_fp8gemm_blockwise_select(int M, int N, int K, int* config_id, int* group_m, int* splits);

/* Kernel launches issued by this library since load. */
unsigned long long b200_fp8block_launch_count(void);

const char* b200_fp8block_strerror(int status);

#ifdef __cplusplus
}
#endif
#endif /* B200_FP8_BLOCK_H_ */
