// libb200_hgemm.so, e4m3 part: C[M,N] (fp16 or bf16) = (A[M,K] (e4m3) * Bt[N,K]^T (e4m3)) * scale_a * scale_b, fp32
// accumulation, per-tensor fp32 scales in device memory. A translation unit of its own so that its 92 kernels compile in
// parallel with the 16-bit ones (b200_hgemm_capi.cu); both are linked into the one library.
#include "../../include/b200_hgemm.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

using b200::host::GemmType;

extern "C" {

int b200_fp8gemm_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                            const void* scale_a, const void* scale_b, int M, int N, int K, int group_m, int max_ctas,
                            int splits, void* stream) {
  const b200::Scales sc{static_cast<const float*>(scale_a), static_cast<const float*>(scale_b)};
  if (out_bf16 == 0)
    return b200::run_config<GemmType::kE4M3F16>(config_id, A, B_kmajor, C, sc, M, N, K, group_m, max_ctas, splits, stream);
  if (out_bf16 == 1)
    return b200::run_config<GemmType::kE4M3BF16>(config_id, A, B_kmajor, C, sc, M, N, K, group_m, max_ctas, splits, stream);
  return b200::host::kBadConfig;
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
  const b200::Scales sc{static_cast<const float*>(scale_a), static_cast<const float*>(scale_b)};
  if (out_bf16 == 0) return b200::dispatch::gemm<GemmType::kE4M3F16>(A, B_kmajor, C, sc, M, N, K, stream);
  if (out_bf16 == 1) return b200::dispatch::gemm<GemmType::kE4M3BF16>(A, B_kmajor, C, sc, M, N, K, stream);
  return b200::host::kBadConfig;
}

}  // extern "C"
