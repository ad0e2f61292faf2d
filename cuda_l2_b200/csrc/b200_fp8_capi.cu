// libb200_hgemm.so, e4m3 part: C[M,N] (fp16 or bf16) = (A[M,K] (e4m3) * Bt[N,K]^T (e4m3)) scaled, fp32 accumulation,
// per-tensor or rowwise (per-row of A x per-row of Bt) fp32 scales in device memory. A translation unit of its own so
// that its 92 kernels compile in parallel with the 16-bit ones (b200_hgemm_capi.cu); both are linked into the one
// library. Both scale granularities run the same 92 kernels: the granularity travels in Scales.
#include "../../include/b200_hgemm.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

using b200::host::GemmType;

namespace {

// The epilogue operands of a call: the per-tensor or rowwise scales.
b200::host::EpiOperands scales_of(const void* scale_a, const void* scale_b, bool rowwise) {
  return {b200::Scales{static_cast<const float*>(scale_a), static_cast<const float*>(scale_b), rowwise}};
}

int fp8_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                   const b200::host::EpiOperands& op, int M, int N, int K, int group_m, int max_ctas, int splits,
                   void* stream) {
  if (out_bf16 == 0)
    return b200::run_config<GemmType::kE4M3F16>(config_id, A, B_kmajor, C, M, N, K, group_m, max_ctas, splits, stream, op);
  if (out_bf16 == 1)
    return b200::run_config<GemmType::kE4M3BF16>(config_id, A, B_kmajor, C, M, N, K, group_m, max_ctas, splits, stream, op);
  return b200::host::kBadConfig;
}

int fp8_gemm(const void* A, const void* B_kmajor, void* C, const b200::host::EpiOperands& op, int out_bf16, int M, int N,
             int K, void* stream) {
  if (out_bf16 == 0) return b200::dispatch::gemm<GemmType::kE4M3F16>(A, B_kmajor, C, M, N, K, stream, op);
  if (out_bf16 == 1) return b200::dispatch::gemm<GemmType::kE4M3BF16>(A, B_kmajor, C, M, N, K, stream, op);
  return b200::host::kBadConfig;
}

}  // namespace

extern "C" {

int b200_fp8gemm_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                            const void* scale_a, const void* scale_b, int M, int N, int K, int group_m, int max_ctas,
                            int splits, void* stream) {
  return fp8_run_config(config_id, out_bf16, A, B_kmajor, C, scales_of(scale_a, scale_b, false), M, N, K, group_m,
                        max_ctas, splits, stream);
}

int b200_fp8gemm_rowwise_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                    const void* scale_a, const void* scale_b, int M, int N, int K, int group_m,
                                    int max_ctas, int splits, void* stream) {
  return fp8_run_config(config_id, out_bf16, A, B_kmajor, C, scales_of(scale_a, scale_b, true), M, N, K, group_m,
                        max_ctas, splits, stream);
}

int b200_fp8gemm_select(int M, int N, int K, int* config_id, int* group_m, int* splits) {
  if (M <= 0 || N <= 0 || K <= 0) return b200::host::kBadShape;
  const b200::dispatch::Choice ch = b200::dispatch::select(GemmType::kE4M3F16, M, N, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  if (splits) *splits = ch.splits;
  return 0;
}

int b200_fp8gemm(const void* A, const void* B_kmajor, void* C, const void* scale_a, const void* scale_b, int out_bf16,
                 int M, int N, int K, void* stream) {
  return fp8_gemm(A, B_kmajor, C, scales_of(scale_a, scale_b, false), out_bf16, M, N, K, stream);
}

int b200_fp8gemm_rowwise(const void* A, const void* B_kmajor, void* C, const void* scale_a, const void* scale_b,
                         int out_bf16, int M, int N, int K, void* stream) {
  return fp8_gemm(A, B_kmajor, C, scales_of(scale_a, scale_b, true), out_bf16, M, N, K, stream);
}

}  // extern "C"
