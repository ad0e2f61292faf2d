// libb200_epilogue.so — the 2-D GEMM with a fused bias + activation epilogue (BiasAct<> configurations,
// hgemm_sm90.cuh). Not a public ABI: nothing under include/ declares these functions, and their names do not start with
// b200_. cuda_l2_b200/capi.py binds them.
//
// For output element (m, n), in fp32, then one rounding to the output type:
//   z = s(m, n) + fp32(bias[n])      (one FADD; none when bias is null)
//   C[m, n] = RN_out(act(z))
// where s is what the library's TN call of the same variant rounds: the fp32 sum (fp16, bf16), fp32(acc * fp32(sa * sb))
// (e4m3 per tensor) or fp32(fp32(acc * sb[n]) * sa[m]) (e4m3 rowwise). act is 0 none, 1 relu (max(z, +0.0)), 2 gelu_tanh
// (0.5 z (1 + tanhf(sqrt(2/pi) (z + 0.044715 z^3))), each step in fp32, tanhf CUDA's full-precision one: torch's tanh
// form). With bias all -0.0 and act 0, C is the TN call's output bit for bit.
//
// `variant` is the GemmType index: 0 fp16, 2 bf16 (fp32 accumulation), 3 e4m3 with fp16 output, 4 e4m3 with bf16
// output. The fp16-accumulating variant (1) and the block-scaled ones (5, 6) have no bias kernel: kBadConfig. A, B_kmajor
// and C as for b200_hgemm_f32acc / b200_fp8gemm (TN: A [M, K], B_kmajor [N, K], C [M, N], all contiguous and 16-byte
// aligned). scale_a / scale_b: e4m3 only, per tensor (one fp32 value each, rowwise = 0) or rowwise (M and N fp32
// values, 16-byte aligned, rowwise = 1); ignored by the 16-bit variants. bias: null, or N values of the output type,
// 16-byte aligned (kBadAlignment otherwise). An unknown act is kBadActivation (-12). Statuses are those of
// b200_hgemm_strerror.
#pragma once
#include "hgemm_host.cuh"

extern "C" {

// The dispatched call: the choice of the library's TN call of the same variant (tuned table, B200_HGEMM_TABLE,
// B200_HGEMM_FORCE), unchanged.
int cuda_l2_b200_epilogue_run(int variant, const void* A, const void* B_kmajor, void* C, const void* scale_a,
                              const void* scale_b, int rowwise, const void* bias, int act, int M, int N, int K,
                              void* stream);

// Configuration `config_id` (0 .. b200_hgemm_num_configs() - 1; all have a bias kernel in every K-mode), with group_m,
// max_ctas and splits as for b200_hgemm_run_config.
int cuda_l2_b200_epilogue_run_config(int variant, int config_id, const void* A, const void* B_kmajor, void* C,
                                     const void* scale_a, const void* scale_b, int rowwise, const void* bias, int act,
                                     int M, int N, int K, int group_m, int max_ctas, int splits, void* stream);

// The dispatched call's choice for variant `variant` (b200_hgemm_select / b200_fp8gemm_select's), into the optional
// out-parameters.
int cuda_l2_b200_epilogue_select(int variant, int M, int N, int K, int* config_id, int* group_m, int* splits);

// The library's own split-K / stream-K scratch (as b200_hgemm_prewarm / b200_hgemm_release for libb200_hgemm.so): a
// first split-K or stream-K call inside a CUDA-graph capture without a prewarm runs undivided.
int cuda_l2_b200_epilogue_prewarm(void* stream);
int cuda_l2_b200_epilogue_release(void);

// Kernel launches of the library.
unsigned long long cuda_l2_b200_epilogue_launch_count(void);

const char* cuda_l2_b200_epilogue_strerror(int status);

}  // extern "C"
