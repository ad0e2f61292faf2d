// libb200_nn.so — the row-major B (NN) kernels (RowMajorB<> configurations, hgemm_sm90.cuh) behind the one internal
// entry point of b200_nn.h. A library of its own, so that the device code of libb200_hgemm.so stays as it is. The
// source is compiled once per 16-bit variant (-DB200_VARIANT = 0, 1, 2), in parallel; the object of variant 0 also
// holds the entry point.
#include "b200_nn.h"
#include "hgemm_configs.cuh"

#ifndef B200_VARIANT
#error "compile once per variant with -DB200_VARIANT=0, 1 or 2"
#endif

namespace b200 {
namespace nn {

// Configuration `id` of variant T on row-major B. A configuration without an NN kernel (BN = 32) is kBadConfig.
template <host::GemmType T>
int run_config(int id, const void* A, const void* B, void* C, int M, int N, int K, int group_m, int max_ctas,
               int splits, host::ScratchFn scratch, cudaStream_t s) {
  constexpr host::GemmTypeTraits t = host::traits(T);
  static_assert(!t.scaled, "row-major B: the 16-bit variants only");
  int st = host::kBadConfig;
  switch (id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                   \
  case ID:                                                                                                      \
    if constexpr (has_kernel(ID))                                                                               \
      st = host::launch<RowMajorB<Config<BN, STAGES, CG, t.acc_f32, CM, CN, MR, t.bf16()>>>(                    \
          A, B, C, M, N, K, s, group_m, max_ctas, splits, Scales{nullptr, nullptr}, 0, scratch);                 \
    break;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      break;
  }
  return st;
}

#define B200_NN_RUN(T)                                                                                           \
  int run_config<T>(int, const void*, const void*, void*, int, int, int, int, int, int, host::ScratchFn, cudaStream_t)
extern template B200_NN_RUN(host::GemmType::kF16Acc32);
extern template B200_NN_RUN(host::GemmType::kF16Acc16);
extern template B200_NN_RUN(host::GemmType::kBF16);
template B200_NN_RUN(host::GemmType(B200_VARIANT));
#undef B200_NN_RUN

}  // namespace nn
}  // namespace b200

#if B200_VARIANT == 0
extern "C" int cuda_l2_b200_nn_run_config(int variant, int config_id, const void* A, const void* B_rowmajor, void* C,
                                          int M, int N, int K, int group_m, int max_ctas, int splits,
                                          b200::host::ScratchFn scratch, void* stream) {
  using b200::host::GemmType;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (variant) {
    case 0:
      return b200::nn::run_config<GemmType::kF16Acc32>(config_id, A, B_rowmajor, C, M, N, K, group_m, max_ctas, splits,
                                                       scratch, s);
    case 1:
      return b200::nn::run_config<GemmType::kF16Acc16>(config_id, A, B_rowmajor, C, M, N, K, group_m, max_ctas, splits,
                                                       scratch, s);
    case 2:
      return b200::nn::run_config<GemmType::kBF16>(config_id, A, B_rowmajor, C, M, N, K, group_m, max_ctas, splits,
                                                   scratch, s);
    default:
      return b200::host::kBadConfig;
  }
}
#endif
