// libb200_hgemm.so, e4m3 part: C[M,N] (fp16 or bf16) = (A[M,K] (e4m3) * Bt[N,K]^T (e4m3)) * scale_a * scale_b, fp32
// accumulation, per-tensor fp32 scales in device memory. A translation unit of its own so that its 90 kernels compile in
// parallel with the 16-bit ones (b200_hgemm_capi.cu); both are linked into the one library.
#include "../../include/b200_hgemm.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

namespace b200 {
void count_launch();   // b200_hgemm_capi.cu
}

namespace {

template <bool kOutBf16>
int run_fp8(int id, const void* A, const void* Bt, void* C, const float* scale_a, const float* scale_b, int M, int N,
            int K, int group_m, int max_ctas, int splits, cudaStream_t s) {
  using namespace b200;
  const Scales scales{scale_a, scale_b};
  int st;
  switch (id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                      \
  case ID:                                                                                                         \
    st = host::launch<Config<BN, STAGES, CG, true, CM, CN, MR, kOutBf16, true>>(A, Bt, C, M, N, K, s, group_m, max_ctas, \
                                                                             splits, scales);                     \
    break;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      return host::kBadConfig;
  }
  if (st == host::kOk) count_launch();
  return st;
}

// An e4m3 problem (M, N, K) moves the bytes of, and issues as many wgmma per tile as, the fp16 problem (M, N, K / 2):
// it takes that problem's entry of the fp32-accumulate table.
b200::dispatch::Choice select_fp8(int M, int N, int K) { return b200::dispatch::select(32, M, N, K / 2 > 0 ? K / 2 : 1); }

}  // namespace

extern "C" {

int b200_fp8gemm_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                            const void* scale_a, const void* scale_b, int M, int N, int K, int group_m, int max_ctas,
                            int splits, void* stream) {
  const float* sa = static_cast<const float*>(scale_a);
  const float* sb = static_cast<const float*>(scale_b);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (out_bf16 == 0) return run_fp8<false>(config_id, A, B_kmajor, C, sa, sb, M, N, K, group_m, max_ctas, splits, s);
  if (out_bf16 == 1) return run_fp8<true>(config_id, A, B_kmajor, C, sa, sb, M, N, K, group_m, max_ctas, splits, s);
  return b200::host::kBadConfig;
}

int b200_fp8gemm_select(int M, int N, int K, int* config_id, int* group_m, int* splits) {
  if (M <= 0 || N <= 0 || K <= 0) return b200::host::kBadShape;
  const b200::dispatch::Choice ch = select_fp8(M, N, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  if (splits) *splits = ch.splits;
  return 0;
}

int b200_fp8gemm(const void* A, const void* B_kmajor, void* C, const void* scale_a, const void* scale_b, int out_bf16,
                 int M, int N, int K, void* stream) {
  if (out_bf16 != 0 && out_bf16 != 1) return b200::host::kBadConfig;
  int st = b200::host::validate_fp8(A, B_kmajor, C, static_cast<const float*>(scale_a), static_cast<const float*>(scale_b),
                                    M, N, K);
  if (st) return st;
  const b200::dispatch::Choice ch = select_fp8(M, N, K);
  return b200_fp8gemm_run_config(ch.config_id, out_bf16, A, B_kmajor, C, scale_a, scale_b, M, N, K, ch.group_m, 0,
                                 ch.splits, stream);
}

}  // extern "C"
