/* b200_grouped_fp8.h — C ABI of the block-scaled FP8 (e4m3) grouped GEMM over contiguous row groups
 * (libb200_grouped_fp8.so).
 *
 *     C[start_g : end_g] = RN_out(block-scaled product of A[start_g : end_g] and Bt[g]^T)    for g in [0, G)
 *
 * The routed experts of a mixture-of-experts layer in a DeepSeek-V3-style FP8 checkpoint, with the tokens sorted by
 * expert: A [T,K] (float8_e4m3fn) and C [T,N] (fp16 or bf16) hold the rows of all groups one after another, Bt [G,N,K]
 * (float8_e4m3fn, K-major: a stack of the experts' nn.Linear weights) one matrix per group. All three are contiguous
 * and 16-byte aligned, K % 16 == 0, N % 8 == 0. A library of its own, next to libb200_grouped.so (include/b200_grouped.h)
 * and libb200_fp8block.so (include/b200_fp8_block.h): the block-scaled kernels of the configurations that have one, one
 * persistent schedule over the tiles of all groups. stream is a cudaStream_t (NULL = legacy default stream).
 *
 * out_bf16: 0 fp16 output, 1 bf16 output; anything else returns -6.
 *
 * Scales (fp32, device memory), with nkb = ceil(K/128):
 *   scale_a   the 2-D block-scaled layout with M = T: value (row t, kb) at scale_a[kb * ld_a + t], ld_a >= max(T, 1),
 *             ld_a % 4 == 0, 16-byte aligned; nkb * ld_a floats must be readable. The scales of the sorted activations
 *             as one quantisation of [T, K] produces them, with no copy.
 *   scale_b   row-major [G, ceil(N/128), nkb], 4-byte aligned: each expert's weight_scale_inv, stacked.
 * Arithmetic: that of b200_fp8gemm_blockwise (include/b200_fp8_block.h) per group, with the group's rows of scale_a and
 * scale_b[g]. There is no output scale.
 *
 * offs: G int32 values in device memory, 4-byte aligned, the cumulative group ends with torch._grouped_mm's meaning.
 * The offsets and both scales are read by the kernel after its grid dependency wait, never by the host, so a kernel
 * just before on the stream may write them and a CUDA-graph replay sees their current contents. No host
 * synchronisation.
 *
 * Clamping: group g is rows [start_g, end_g) with start_0 = 0, start_g = end_{g-1} and end_g = clamp(offs[g], start_g,
 * T). Decreasing, negative or too-large offsets give empty or shortened groups; nothing outside A, Bt[0..G), the scales
 * described above or C is ever read or written.
 *
 * Exact rows: every row of C in [0, end_{G-1}) is written exactly once, by its own group; rows at or past end_{G-1}
 * keep what they held.
 *
 * Bits: per group, the result is bit-identical to b200_fp8gemm_blockwise_run_config with the same configuration,
 * group_m and splits = 1 on that group's rows of A, Bt[g], the group's rows of scale_a (any ld_a) and scale_b[g]. An
 * output row depends only on its own row of A and its own scales, so which rows share a tile does not change the bits.
 *
 * Schedule: only the plain schedule exists for this variant (no split-K, no stream-K), so a launch never needs scratch
 * memory and is always safe to capture in a CUDA graph. The tile list of a configuration is the one of the 16-bit
 * grouped kernel with the same id: b200_grouped_schedule_units (include/b200_grouped.h) describes it. Launches take no
 * L2 eviction hints. T == 0 launches nothing.
 *
 * Return value: 0 on success, < 0 a status (b200_grouped_fp8_strerror), > 0 a cudaError_t. Launches are asynchronous.
 * Statuses as in b200_grouped.h and b200_fp8_block.h: -5 for a null operand, offs or scale; -1 for G <= 0, T < 0,
 * N or K <= 0, and a worst-case tile count (ceil(T / block rows) + G) * (column blocks) past INT_MAX; -2 for a
 * misaligned operand, offs, scale_a or scale_b, and N % 8 != 0; -9 for K % 16 != 0; -10 for ld_a < max(T, 1) or
 * ld_a % 4 != 0.
 */
#ifndef B200_GROUPED_FP8_H_
#define B200_GROUPED_FP8_H_

#ifdef __cplusplus
extern "C" {
#endif

/* The dispatched call: the configuration of b200_grouped_fp8_select. */
int b200_grouped_fp8_gemm(const void* A, const void* B_kmajor, void* C, const void* scale_a, int ld_a,
                          const void* scale_b, int out_bf16, const int* offs, int G, int T, int N, int K, void* stream);

/* One explicit configuration of libb200_hgemm.so's table (b200_hgemm_config_info). Only the configurations with a
 * block-scaled kernel (m_rep * bn <= 128: 1, 2, 4, 7-17, 22, 23 and 30) have one here; any other id returns -6.
 * group_m <= 0 selects the default rasterisation width, max_ctas <= 0 all SMs. */
int b200_grouped_fp8_gemm_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                     const void* scale_a, int ld_a, const void* scale_b, const int* offs, int G, int T,
                                     int N, int K, int group_m, int max_ctas, void* stream);

/* The dispatcher's choice: the grouped rule (b200_grouped_select: the batched choice for G matrices of ceil(T / G)
 * rows) for e4m3 operands, its configuration mapped to the block-scaled one with the same CTA group and cluster, M_REP 1
 * and BN min(BN, 128), as b200_fp8gemm_blockwise_select maps it. Returns 0 or a negative status. */
int b200_grouped_fp8_select(int G, int T, int N, int K, int* config_id, int* group_m);

/* Kernel launches issued by this library since load. */
unsigned long long b200_grouped_fp8_launch_count(void);

const char* b200_grouped_fp8_strerror(int status);

#ifdef __cplusplus
}
#endif
#endif /* B200_GROUPED_FP8_H_ */
