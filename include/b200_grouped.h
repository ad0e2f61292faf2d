/* b200_grouped.h — C ABI of the grouped 16-bit GEMM over contiguous row groups (libb200_grouped.so).
 *
 *     C[start_g : end_g] = A[start_g : end_g] x Bt[g]^T    for g in [0, G)
 *
 * The layout of a mixture-of-experts layer whose tokens are sorted by expert (torch._grouped_mm(A, Bt.transpose(-2, -1),
 * offs=offs)): A [T,K] and C [T,N] hold the rows of all groups one after another, Bt [G,N,K] (K-major, a stack of
 * nn.Linear weights) one matrix per group. All three are contiguous and 16-byte aligned; the rules of the 2-D call
 * (include/b200_hgemm.h) hold: K % 8 == 0, N % 8 == 0. A library of its own, next to libb200_hgemm.so: the same kernels
 * (one per configuration of b200_hgemm_config_info and type), one persistent schedule over the tiles of all groups.
 * stream is a cudaStream_t (NULL = legacy default stream).
 *
 * variant: the data type, 0 fp16 with fp32 accumulation, 1 fp16 with fp16 accumulation, 2 bf16 (fp32 accumulation);
 * anything else returns -6.
 *
 * offs: G int32 values in device memory, 4-byte aligned, the cumulative group ends with torch's meaning. They are read
 * by the kernel after its grid dependency wait, never by the host, so a kernel just before on the stream may write them
 * and a CUDA-graph replay sees their current contents. No host synchronisation.
 *
 * Clamping: group g is rows [start_g, end_g) with start_0 = 0, start_g = end_{g-1} and end_g = clamp(offs[g], start_g,
 * T). Decreasing, negative or too-large offsets give empty or shortened groups; nothing outside A, Bt[0..G) or C is
 * ever read or written.
 *
 * Exact rows: every row of C in [0, end_{G-1}) is written exactly once, by its own group; rows at or past end_{G-1}
 * keep what they held. (A 16-row store box that straddles a group's end stores only that group's rows: the rows after
 * them belong to the next group.)
 *
 * Bits: per group, the result is bit-identical to b200_hgemm_run_config / b200_bgemm_run_config with the same
 * configuration and group_m on that group's rows of A and on Bt[g]. An output row depends only on its own row of A, so
 * which rows share a tile does not change the bits.
 *
 * Schedule: only the plain schedule exists for this variant (no split-K, no stream-K), so a launch never needs scratch
 * memory and is always safe to capture in a CUDA graph. Launches take no L2 eviction hints. T == 0 launches nothing.
 *
 * Return value: 0 on success, < 0 a status (b200_grouped_strerror), > 0 a cudaError_t. Launches are asynchronous.
 * Statuses as in b200_hgemm.h: -5 also for a null offs; -1 for G <= 0, T < 0, and a worst-case tile count
 * (ceil(T / block rows) + G) * (column blocks) past INT_MAX; -2 also for a misaligned offs.
 */
#ifndef B200_GROUPED_H_
#define B200_GROUPED_H_

#ifdef __cplusplus
extern "C" {
#endif

/* The dispatched call: the configuration of b200_grouped_select. */
int b200_grouped_gemm(int variant, const void* A, const void* B_kmajor, void* C, const int* offs, int G, int T, int N,
                      int K, void* stream);

/* One explicit configuration (0 .. b200_hgemm_num_configs() - 1) of libb200_hgemm.so's table. group_m <= 0 selects the
 * default rasterisation width, max_ctas <= 0 all SMs. */
int b200_grouped_gemm_run_config(int variant, int config_id, const void* A, const void* B_kmajor, void* C,
                                 const int* offs, int G, int T, int N, int K, int group_m, int max_ctas, void* stream);

/* The dispatcher's choice: the batched library's (b200_batched_select) for G matrices of the average group,
 * M = ceil(T / G) rows. Returns 0 or a negative status. */
int b200_grouped_select(int variant, int G, int T, int N, int K, int* config_id, int* group_m);

/* Host-side view of the schedule, produced by the code the kernel runs: the tiles worker `worker` (a CTA, CTA pair or
 * cluster) of a launch on num_sms SMs computes, in order, as (group, m-block, n-block) triples in units[3 * i ..] (at
 * most max_units are written); m-blocks count cluster row blocks from the group's first row. offs_host: the G offsets in
 * host memory. *num_workers receives the launch's worker count. Returns the number of tiles of the worker, or a
 * negative status. */
int b200_grouped_schedule_units(int config_id, int G, int T, int N, int K, const int* offs_host, int num_sms,
                                int worker, int* units, int max_units, int* num_workers);

/* Kernel launches issued by this library since load. */
unsigned long long b200_grouped_launch_count(void);

const char* b200_grouped_strerror(int status);

#ifdef __cplusplus
}
#endif
#endif /* B200_GROUPED_H_ */
