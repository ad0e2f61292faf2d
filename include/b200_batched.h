/* b200_batched.h — C ABI of the batched 16-bit GEMM (libb200_batched.so).
 *
 *     C[b] (M x N) = A[b] (M x K) x Bt[b]^T (Bt[b]: N x K)    for b in [0, B)
 *
 * A [B,M,K], Bt [B,N,K] (K-major, like an nn.Linear weight) and C [B,M,N] are contiguous and 16-byte aligned; the
 * rules of the 2-D call (include/b200_hgemm.h) hold per matrix: K % 8 == 0, N % 8 == 0. A library of its own, next to
 * libb200_hgemm.so: the same kernels (one per configuration of b200_hgemm_config_info and type) with 3-D tensor maps,
 * so every matrix is clipped and zero-filled at its own edges, and one persistent schedule over the tiles of all
 * matrices. Per matrix, the result is bit-identical to b200_hgemm_run_config / b200_bgemm_run_config with the same
 * configuration and group_m on that matrix's operands. stream is a cudaStream_t (NULL = legacy default stream).
 *
 * variant: the data type, 0 fp16 with fp32 accumulation, 1 fp16 with fp16 accumulation, 2 bf16 (fp32 accumulation);
 * anything else returns -6.
 *
 * masked_m (optional, NULL = dense): B int32 values in device memory, 4-byte aligned, read by the kernel after its
 * grid dependency wait (never by the host), so a kernel just before on the stream may write them and a CUDA-graph
 * replay sees their current contents. Only rows [0, clamp(masked_m[b], 0, M)) of C[b] are computed and defined; the
 * rows past the count are unspecified, except that no 16-row store box starting at or past the count is written:
 * rows from round_up(count, 16) on keep what they held, and whole tiles past the count cost nothing.
 *
 * Only the plain schedule exists for this variant (no split-K, no stream-K), so a launch never needs scratch memory
 * and is always safe to capture in a CUDA graph. Launches take no L2 eviction hints.
 *
 * Return value: 0 on success, < 0 a status (b200_batched_strerror), > 0 a cudaError_t. Launches are asynchronous.
 * Statuses as in b200_hgemm.h: -1 also for B <= 0 and for more than INT_MAX tiles in all, -2 also for a misaligned
 * masked_m.
 */
#ifndef B200_BATCHED_H_
#define B200_BATCHED_H_

#ifdef __cplusplus
extern "C" {
#endif

/* The dispatched call: the configuration of b200_batched_select. */
int b200_batched_gemm(int variant, const void* A, const void* B_kmajor, void* C, const int* masked_m, int B, int M,
                      int N, int K, void* stream);

/* One explicit configuration (0 .. b200_hgemm_num_configs() - 1) of libb200_hgemm.so's table. group_m <= 0 selects the
 * default rasterisation width, max_ctas <= 0 all SMs. */
int b200_batched_gemm_run_config(int variant, int config_id, const void* A, const void* B_kmajor, void* C,
                                 const int* masked_m, int B, int M, int N, int K, int group_m, int max_ctas,
                                 void* stream);

/* The dispatcher's choice: the 2-D choice for (B * M, N, K), whose tile count is about the batched problem's, if its
 * pair / cluster fits one matrix of M x N; otherwise the 2-D choice for (M, N, K). Returns 0 or a negative status. */
int b200_batched_select(int variant, int B, int M, int N, int K, int* config_id, int* group_m);

/* Host-side view of the schedule, produced by the code the kernel runs: the tiles worker `worker` (a CTA, CTA pair or
 * cluster) of a launch on num_sms SMs computes, in order, as (batch, m-block, n-block) triples in units[3 * i ..]
 * (at most max_units are written). masked_m_host: the row counts in host memory (NULL = dense). *num_workers receives
 * the launch's worker count. Returns the number of tiles of the worker, or a negative status. */
int b200_batched_schedule_units(int config_id, int B, int M, int N, int K, const int* masked_m_host, int num_sms,
                                int worker, int* units, int max_units, int* num_workers);

/* Kernel launches issued by this library since load. */
unsigned long long b200_batched_launch_count(void);

const char* b200_batched_strerror(int status);

#ifdef __cplusplus
}
#endif
#endif /* B200_BATCHED_H_ */
