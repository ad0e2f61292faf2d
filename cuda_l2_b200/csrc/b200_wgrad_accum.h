// libb200_wgrad_accum.so — weight gradients added into fp32 main-grad buffers (AccumF32<> configurations,
// hgemm_sm90.cuh). Not a public ABI: nothing under include/ declares these functions, and their names do not start with
// b200_. cuda_l2_b200/capi.py binds them.
//
// For every element (m, n) of the product's output, in fp32:
//   C32[m, n] = fp32(C32[m, n] + s(m, n))     (one round-to-nearest-even addition, after the whole reduction)
// where s is exactly the fp32 value the wrapped library's call of the same configuration and K-mode rounds to its
// 16-bit output: the fp32 sum of the K-grouped product (libb200_grouped_bwd.so's cuda_l2_b200_grouped_bwd_wgrad),
// fp32(fp32(acc * sb[n]) * sa[m]) for rowwise e4m3 scales (b200_fp8gemm_rowwise), or the promoted sum for 1 x 128 scales
// on both operands (libb200_fp8block_1d1d.so). Split-K partials are summed in their fixed order first, and no split or
// stream-K contributor adds on its own, so the result is deterministic. With C32 all -0.0 beforehand, C32 afterwards is
// s itself, and C32 rounded to fp16 / bf16 is the wrapped call's output bit for bit. Nothing outside the [M, N] matrix
// (K-grouped: [G, M, N]) is written; an empty group leaves its matrix as it is, bits included, and T == 0 launches
// nothing (cuBLAS's k = 0 with beta = 1).
//
// C32: fp32, row-major, contiguous, 16-byte aligned. Statuses are those of b200_hgemm_strerror; every argument status
// comes back before any CUDA call.
#pragma once
#include "hgemm_host.cuh"

extern "C" {

// The K-grouped product added into C32 [G, M, N]: C32[g] += A[start_g : end_g]^T B[start_g : end_g] for g < G, with
// A [T, M], B [T, N] (fp16 or bf16: `variant` 0 or 2, the GemmType index) and the int32 group ends `offs` [G] in device
// memory, as for cuda_l2_b200_grouped_bwd_wgrad. config_id < 0: that library's dispatched choice
// (cuda_l2_b200_grouped_bwd_wgrad_select); otherwise configuration config_id (one with BN >= 64), with group_m and
// max_ctas as for it. The 2-D weight gradient dW += dY^T X of a [T, N] x [N, K] layer is the case G = 1, offs = {T}.
int cuda_l2_b200_wgrad_accum_grouped(int variant, int config_id, const void* A, const void* B, float* C32,
                                     const int* offs, int G, int T, int M, int N, int group_m, int max_ctas,
                                     void* stream);

// The e4m3 product A [M, K] x B_kmajor [N, K]^T added into C32 [M, N]. `form` names the scales: 1 rowwise (scale_a M
// values, scale_b N values, 16-byte aligned; ld_a and ld_b unused) or 3, 1 x 128 scales on both operands (scale_a
// [ceil(K/128), ld_a] and scale_b [ceil(K/128), ld_b], as for cuda_l2_b200_fp8block_1d1d_run). Per-tensor (0) and
// 128 x 128 (2) scales have no accumulating kernel: kBadConfig. config_id < 0: the wrapped library's dispatched choice
// (b200_fp8gemm_select, or cuda_l2_b200_fp8block_1d1d_select); otherwise configuration config_id with group_m,
// max_ctas and splits as for b200_fp8gemm_rowwise_run_config / cuda_l2_b200_fp8block_1d1d_run_config.
int cuda_l2_b200_wgrad_accum_fp8(int form, int config_id, const void* A, const void* B_kmajor, float* C32,
                                 const void* scale_a, int ld_a, const void* scale_b, int ld_b, int M, int N, int K,
                                 int group_m, int max_ctas, int splits, void* stream);

// The dispatched calls' choices, into the optional out-parameters.
int cuda_l2_b200_wgrad_accum_grouped_select(int variant, int G, int T, int M, int N, int* config_id, int* group_m);
int cuda_l2_b200_wgrad_accum_fp8_select(int form, int M, int N, int K, int* config_id, int* group_m, int* splits);

// The library's own split-K / stream-K scratch (as b200_hgemm_prewarm / b200_hgemm_release for libb200_hgemm.so): a
// first split-K or stream-K call inside a CUDA-graph capture without a prewarm runs undivided.
int cuda_l2_b200_wgrad_accum_prewarm(void* stream);
int cuda_l2_b200_wgrad_accum_release(void);

// Kernel launches of the library.
unsigned long long cuda_l2_b200_wgrad_accum_launch_count(void);

const char* cuda_l2_b200_wgrad_accum_strerror(int status);

}  // extern "C"
