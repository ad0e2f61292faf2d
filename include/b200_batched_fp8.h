/* b200_batched_fp8.h — C ABI of the block-scaled FP8 (e4m3) batched GEMM with optional per-batch row counts on the
 * device (libb200_batched_fp8.so).
 *
 *     C[b][0 : rows_b] = RN_out(block-scaled product of A[b][0 : rows_b] and Bt[b]^T)    for b in [0, B)
 *
 * with rows_b = clamp(masked_m[b], 0, M), or M when masked_m is NULL. The routed experts of a mixture-of-experts layer
 * in a DeepSeek-V3-style FP8 checkpoint at decode: each local expert gets a fixed [M, K] slot of tokens and the real
 * counts live on the GPU. A [B,M,K] (float8_e4m3fn), Bt [B,N,K] (float8_e4m3fn, K-major: a stack of the experts'
 * nn.Linear weights) and C [B,M,N] (fp16 or bf16) are contiguous and 16-byte aligned, K % 16 == 0, N % 8 == 0. A
 * library of its own, next to libb200_batched.so (include/b200_batched.h) and libb200_fp8block.so
 * (include/b200_fp8_block.h): the block-scaled kernels of the configurations that have one, with 3-D tensor maps, so
 * every matrix is clipped and zero-filled at its own edges, and one persistent schedule over the tiles of all matrices.
 * stream is a cudaStream_t (NULL = legacy default stream).
 *
 * out_bf16: 0 fp16 output, 1 bf16 output; anything else returns -6.
 *
 * Scales (fp32, device memory), with nkb = ceil(K/128):
 *   scale_a   the 2-D block-scaled layout per matrix, stacked: value (batch b, row m, kb) at
 *             scale_a[(b * nkb + kb) * ld_a + m], ld_a >= M, ld_a % 4 == 0, 16-byte aligned; B * nkb * ld_a floats
 *             must be readable. Torch's [B, M, nkb] with strides (nkb * ld_a, 1, ld_a): what one quantisation of
 *             [B, M, K] per token and 128 channels produces, with no copy.
 *   scale_b   row-major [B, ceil(N/128), nkb], 4-byte aligned: each expert's weight_scale_inv, stacked.
 * Arithmetic: that of b200_fp8gemm_blockwise (include/b200_fp8_block.h) per matrix, with matrix b's block of scale_a
 * and scale_b[b]. There is no output scale.
 *
 * masked_m (optional, NULL = dense): B int32 values in device memory, 4-byte aligned. The counts, both scales and the
 * operands are read by the kernel after its grid dependency wait, never by the host, so a kernel just before on the
 * stream may write them and a CUDA-graph replay sees their current contents. No host synchronisation.
 *
 * Masked rows, as in b200_batched.h: only rows [0, rows_b) of C[b] are computed and defined; the rows past the count
 * are unspecified, except that no 16-row store box starting at or past the count is written: rows from
 * round_up(rows_b, 16) on keep what they held, and whole tiles past the count cost nothing. Rows of A[b] and of
 * matrix b's scale_a at or past rows_b may hold anything, NaN and Inf included: they reach only their own output rows.
 *
 * Bits: per matrix, the computed rows are bit-identical to b200_fp8gemm_blockwise_run_config with the same
 * configuration, group_m and splits = 1 on that matrix's rows of A, Bt[b], its rows of scale_a (any ld_a) and
 * scale_b[b]. An output row depends only on its own row of A and its own scales, so which rows share a tile does not
 * change the bits.
 *
 * Schedule: only the plain schedule exists for this variant (no split-K, no stream-K), so a launch never needs scratch
 * memory and is always safe to capture in a CUDA graph. The tile list of a configuration is the one of the 16-bit
 * batched kernel with the same id: b200_batched_schedule_units (include/b200_batched.h) describes it. Launches take no
 * L2 eviction hints.
 *
 * Return value: 0 on success, < 0 a status (b200_batched_fp8_strerror), > 0 a cudaError_t. Launches are asynchronous.
 * Statuses as in b200_batched.h and b200_fp8_block.h: -5 for a null operand or scale; -1 for B <= 0, M, N or K <= 0,
 * and more than INT_MAX tiles in all for every block-scaled configuration; -2 for a misaligned operand, scale_a,
 * scale_b or masked_m, and N % 8 != 0; -9 for K % 16 != 0; -10 for ld_a < M or ld_a % 4 != 0.
 */
#ifndef B200_BATCHED_FP8_H_
#define B200_BATCHED_FP8_H_

#ifdef __cplusplus
extern "C" {
#endif

/* The dispatched call: the configuration of b200_batched_fp8_select. */
int b200_batched_fp8_gemm(const void* A, const void* B_kmajor, void* C, const void* scale_a, int ld_a,
                          const void* scale_b, int out_bf16, const int* masked_m, int B, int M, int N, int K,
                          void* stream);

/* One explicit configuration of libb200_hgemm.so's table (b200_hgemm_config_info). Only the configurations with a
 * block-scaled kernel (m_rep * bn <= 128: 1, 2, 4, 7-17, 22, 23 and 30) have one here; any other id returns -6.
 * group_m <= 0 selects the default rasterisation width, max_ctas <= 0 all SMs. */
int b200_batched_fp8_gemm_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                     const void* scale_a, int ld_a, const void* scale_b, const int* masked_m, int B,
                                     int M, int N, int K, int group_m, int max_ctas, void* stream);

/* The dispatcher's choice: the batched rule (b200_batched_select) for e4m3 operands, its configuration mapped to the
 * block-scaled one with the same CTA group and cluster, M_REP 1 and BN min(BN, 128), as b200_fp8gemm_blockwise_select
 * maps it. Returns 0 or a negative status. */
int b200_batched_fp8_select(int B, int M, int N, int K, int* config_id, int* group_m);

/* Kernel launches issued by this library since load. */
unsigned long long b200_batched_fp8_launch_count(void);

const char* b200_batched_fp8_strerror(int status);

#ifdef __cplusplus
}
#endif
#endif /* B200_BATCHED_FP8_H_ */
