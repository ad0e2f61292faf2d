/* b200_hgemm.h — C ABI of the H100-native HGEMM hot path (libb200_hgemm.so).
 *
 * This is the drop-in boundary for the one path this repository accelerates:
 *     C[M,N] (fp16) = A[M,K] (fp16) x B[K,N] (fp16), fp32 or fp16 accumulation.
 *
 * Each entry point names the reference interface it stands in for (paths relative to the
 * CUDA-L2 checkout). The reference exposes the path as a torch C++ extension; the functions here
 * take plain device pointers so that the torch binding (pybind/hgemm_b200_fp32.cc,
 * pybind/hgemm_b200_fp16.cc), ctypes (cuda_l2_b200/capi.py) or any other FFI can bind them.
 *
 * Conventions (same as the reference's kernels, kernels/a100_F32F16F16F32/4096_4096_4096.cu:292-310):
 *   A          [M,K] row-major fp16 (K contiguous)
 *   B_rowmajor [K,N] row-major fp16 (N contiguous), the layout of torch.matmul(a, b). Read only when B_kmajor is
 *              NULL: the drop-in calls below then run the row-major B (NN) kernels of libb200_nn.so, which the
 *              library loads from its own directory on the first such call (status -11 if it is missing). Same
 *              rules and dispatcher choice as K-major B (a BN = 32 configuration maps to a BN = 64 one); the result
 *              is bit-identical to the K-major call on a transposed copy. NULL otherwise (ignored when B_kmajor is set).
 *   B_kmajor   B transposed in memory: [N,K] row-major (K contiguous) — the harness's `b_col_major`
 *              (tools/utils.py:110-115). Takes precedence over B_rowmajor; both NULL is status -5.
 *   C          [M,N] row-major fp16, fully overwritten (alpha = 1, beta = 0), nothing else is written
 *   stream     a cudaStream_t (NULL = the legacy default stream the reference launches on)
 * All pointers are device pointers, 16-byte aligned; K % 8 == 0 and N % 8 == 0 (TMA stride rule).
 * Any M, N, K > 0 meeting that rule is accepted: edges are handled in-kernel, no padding needed.
 * Return value: 0 on success, < 0 a b200_hgemm status, > 0 a cudaError_t. Launches are asynchronous.
 */
#ifndef B200_HGEMM_H_
#define B200_HGEMM_H_

#ifdef __cplusplus
extern "C" {
#endif

/* Replaces cuda_l2_{a100,h100,3090}_fp32(a, b, b_col_major, c)
 * (kernels/a100_F32F16F16F32/4096_4096_4096.cu:292-310, pybind/hgemm_a100_fp32.cc:27,51):
 * fp16 x fp16 products, fp32 accumulation, one round-to-nearest conversion to fp16. */
int b200_hgemm_f32acc(const void* A, const void* B_rowmajor, const void* B_kmajor, void* C,
                      int M, int N, int K, void* stream);

/* Replaces cuda_l2_a100_fp16(a, b, b_col_major, c)
 * (kernels/a100_F16F16F16F16/8192_8192_8192.cu:290-303, pybind/hgemm_a100_fp16.cc:27,51):
 * same, with fp16 accumulation in the tensor core. */
int b200_hgemm_f16acc(const void* A, const void* B_rowmajor, const void* B_kmajor, void* C,
                      int M, int N, int K, void* stream);

/* bf16 variant (README.md:73 lists further data types as future work; no reference kernel exists for it): bf16 x bf16
 * products, fp32 accumulation, one round-to-nearest-even conversion to bf16. Same layouts, same dispatcher (the fp32-
 * accumulate table), same pipeline — the MMA instruction descriptor names bf16 operands and the epilogue converts with
 * cvt.rn.bf16x2.f32. b200_bgemm_run_config is b200_hgemm_run_config for this data type. */
int b200_bgemm_f32acc(const void* A, const void* B_rowmajor, const void* B_kmajor, void* C,
                      int M, int N, int K, void* stream);
int b200_bgemm_run_config(int config_id, const void* A, const void* B_kmajor, void* C,
                          int M, int N, int K, int group_m, int max_ctas, int splits, void* stream);

/* FP8 variant (no reference kernel exists for it): A [M,K] and B_kmajor [N,K] hold float8_e4m3fn values (one byte
 * each, K contiguous); C [M,N] is fp16 (out_bf16 = 0) or bf16 (out_bf16 = 1), row-major, fully overwritten:
 *     C = RN_out( (sum_k A[m,k] * B_kmajor[n,k]) * fp32(scale_a * scale_b) )
 * The sum is accumulated by the tensor core in fp32 (one accumulator per element, the equivalent of fast accumulation:
 * Hopper's FP8 MMA keeps fewer than 23 mantissa bits in its running sum); the scale is applied once, to the finished sum,
 * right before the one rounding to the output type, in every K-mode. scale_a and scale_b point to one fp32 value each in
 * DEVICE memory (4-byte aligned) and are read when the kernel runs, after the stream's preceding work: a graph replay
 * sees their current contents. The same as torch._scaled_mm(A, B_kmajor.t(), scale_a, scale_b, out_dtype) with
 * per-tensor scales. Requires K % 16 == 0 (16-byte row strides; status -9 otherwise), N % 8 == 0 and 16-byte aligned A,
 * B_kmajor and C. The dispatcher takes the fp32-accumulate table's choice for (M, N, K / 2), the fp16 problem that moves
 * the same bytes per k-block. b200_fp8gemm_run_config is b200_hgemm_run_config for this data type (same `splits`
 * codes); b200_fp8gemm_select reports the dispatcher's choice. */
int b200_fp8gemm(const void* A, const void* B_kmajor, void* C, const void* scale_a, const void* scale_b, int out_bf16,
                 int M, int N, int K, void* stream);
int b200_fp8gemm_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                            const void* scale_a, const void* scale_b, int M, int N, int K, int group_m, int max_ctas,
                            int splits, void* stream);
int b200_fp8gemm_select(int M, int N, int K, int* config_id, int* group_m, int* splits);

/* FP8 with rowwise scales (per token x per output channel): the same operands, output, kernels and dispatcher choice as
 * b200_fp8gemm, but scale_a points to M fp32 values (one per row of A) and scale_b to N fp32 values (one per row of
 * B_kmajor, i.e. per output column), both in DEVICE memory and 16-byte aligned (status -2 otherwise, -5 if NULL):
 *     C[m,n] = RN_out( fp32( fp32(acc[m,n] * scale_b[n]) * scale_a[m] ) ),   acc[m,n] = sum_k A[m,k] * B_kmajor[n,k]
 * The column scale is applied first, then the row scale, each product rounded to fp32, then the one rounding to the
 * output type, in every K-mode. The vectors are read when the kernel runs (a graph replay sees their current contents).
 * The same as torch._scaled_mm(A, B_kmajor.t(), scale_a[M,1], scale_b[1,N], out_dtype) with rowwise scales.
 * b200_fp8gemm_rowwise_run_config is b200_fp8gemm_run_config for these scales (same `splits` codes). */
int b200_fp8gemm_rowwise(const void* A, const void* B_kmajor, void* C, const void* scale_a, const void* scale_b,
                         int out_bf16, int M, int N, int K, void* stream);
int b200_fp8gemm_rowwise_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                    const void* scale_a, const void* scale_b, int M, int N, int K, int group_m,
                                    int max_ctas, int splits, void* stream);

/* The reference fixes tile/stage/swizzle per (M,N,K) at compile time inside each
 * kernels/<dev>/<M>_<N>_<K>.cu (e.g. a100_F32F16F16F32/4096_4096_4096.cu:185-200,305-309). Here the
 * per-shape choice is a table lookup; these calls expose it for the tuner and the tests. */
int b200_hgemm_num_configs(void);
/* BN = tile N, stages = the shared-memory ring depth the kernel runs with, cta_group = 1 (128xBN per CTA) or 2
 * (a 2-CTA cluster of 256xBN sharing its B tile). */
int b200_hgemm_config_info(int config_id, int* bn, int* stages, int* cta_group);
/* The ring depth the configuration table requests; the kernel caps it at what fits in shared memory (the value
 * config_info reports). The per-shape sources under kernels/ name this value. Negative status for an unknown id. */
int b200_hgemm_config_stages_requested(int config_id);
/* TMA-multicast cluster shape of a configuration (1 x 1 = none): cluster_m x cluster_n single-CTA groups work on
 * adjacent tiles; A tiles are shared along N, B tiles along M. */
int b200_hgemm_config_cluster(int config_id, int* cluster_m, int* cluster_n);
/* 128-row blocks per CTA: 1, or 2 for the configurations whose CTAs own 256 rows (two MMAs per k-step that share the
 * B tile in shared memory); the tile is then 128 * m_rep * cta_group rows. Negative status for an unknown id. */
int b200_hgemm_config_m_rep(int config_id);
/* The configuration the dispatcher uses for this problem (acc_bits = 32 or 16). */
int b200_hgemm_select_config(int acc_bits, int M, int N, int K);
/* Same, also reporting the rasterisation group (0 = kernel default) and the split-K factor (1 = none).
 * Returns 0 or a negative status. */
int b200_hgemm_select(int acc_bits, int M, int N, int K, int* config_id, int* group_m, int* splits);
/* Run one explicit configuration. group_m <= 0 and max_ctas <= 0 select the defaults; splits > 1 asks for
 * split-K through a lazily allocated per-stream fp32 workspace (cta_group 1 configurations only; clamped so
 * that tiles x splits fits the SMs); splits = -2, -4 or -8 asks for split-K inside a thread-block cluster of that
 * many CTAs, reduced through distributed shared memory (no workspace); splits = 100 asks for stream-K over the tiles of
 * the partial last wave, 101 for stream-K over that tail plus one full wave (both through the workspace; cta_group 1
 * and 2, no multicast cluster; ignored when the tile count already fills the last wave). All reductions are
 * deterministic. */
int b200_hgemm_run_config(int acc_bits, int config_id, const void* A, const void* B_kmajor, void* C,
                          int M, int N, int K, int group_m, int max_ctas, int splits, void* stream);

/* Host-only view of the kernel's schedule (no device needed): the work units worker `worker` runs, in order, on a
 * device with num_sms SMs, as triples (tile, first k-block, end k-block) written to units[3 * max_units]. The plan
 * is the one b200_hgemm_run_config makes for this `splits` request. Also reports the number of workers (CTAs, CTA
 * pairs or clusters) of the launch, the stream-K tile count, the K-mode the request runs in (0 plain, 1 workspace
 * split-K, 2 cluster split-K, 3 stream-K), and per unit the number of contributor units an owner unit waits for
 * (each NULL to skip). Returns the worker's unit count (possibly > max_units) or a negative status. The same code
 * walks the schedule inside the kernel. */
int b200_hgemm_schedule_units(int config_id, int M, int N, int K, int splits, int num_sms, int worker, int* units,
                              int max_units, int* num_workers, int* sk_tiles, int* mode, int* contributors);

/* End-to-end form with HOST buffers (pageable or pinned): copies A and B_kmajor to the device,
 * runs the GEMM and copies C back, synchronising before it returns. This is the call bench.py
 * times for its "e2e" figure; it stands where the reference harness's host loop stands
 * (benchmarking_utils.py:12-33, which also brackets one call with device synchronisation). */
int b200_hgemm_host(int acc_bits, const void* hA, const void* hB_kmajor, void* hC, int M, int N, int K);

/* Resource management. The library keeps, per (device, stream) that ever ran a workspace split-K or stream-K launch,
 * 21 MB of device scratch (first use allocates with cudaMalloc — illegal inside a CUDA-graph capture, where the launch
 * then quietly runs the undivided schedule instead), and per device the staging buffers / streams of b200_hgemm_host.
 * The reference kernels allocate such state per call (torch::zeros scratch, kernels/a100_F32F16F16F32/64_256_16384.cu:233-248;
 * cudaMalloc of the CUTLASS workspace, kernels/h100_F32F16F16F32/4096_4096_4096.cu:148-149).
 *   b200_hgemm_prewarm(stream)  allocate the scratch of (current device, stream) now — call it before capturing a graph;
 *   b200_hgemm_release()        free everything the library holds on every device. No launch of this library may be
 *                               in flight or issued concurrently. Later calls re-allocate on demand.
 * Both return 0 or a status / cudaError_t.
 * Split-K / stream-K launches wait for sibling CTAs of their own grid; they are launched cooperatively, so the driver
 * starts such a grid only when all of it fits on the device (it may therefore wait for other kernels to drain). */
int b200_hgemm_prewarm(void* stream);
int b200_hgemm_release(void);

/* Kernel launches issued by this library since load (the bench's `gpu_launches` evidence). */
unsigned long long b200_hgemm_launch_count(void);

const char* b200_hgemm_strerror(int status);

#ifdef __cplusplus
}
#endif
#endif /* B200_HGEMM_H_ */
