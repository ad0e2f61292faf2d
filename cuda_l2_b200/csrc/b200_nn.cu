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

extern template B200_RUN(host::GemmType::kF16Acc32, RowMajorB);
extern template B200_RUN(host::GemmType::kF16Acc16, RowMajorB);
extern template B200_RUN(host::GemmType::kBF16, RowMajorB);
template B200_RUN(host::GemmType(B200_VARIANT), RowMajorB);

}  // namespace b200

#if B200_VARIANT == 0
extern "C" int cuda_l2_b200_nn_run_config(int variant, int config_id, const void* A, const void* B_rowmajor, void* C,
                                          int M, int N, int K, int group_m, int max_ctas, int splits,
                                          b200::host::ScratchFn scratch, void* stream) {
  using b200::host::GemmType;
  using b200::RowMajorB;
  switch (variant) {
    case 0:
      return b200::run_config<GemmType::kF16Acc32, RowMajorB>(config_id, A, B_rowmajor, C, M, N, K, group_m, max_ctas,
                                                              splits, stream, {}, scratch);
    case 1:
      return b200::run_config<GemmType::kF16Acc16, RowMajorB>(config_id, A, B_rowmajor, C, M, N, K, group_m, max_ctas,
                                                              splits, stream, {}, scratch);
    case 2:
      return b200::run_config<GemmType::kBF16, RowMajorB>(config_id, A, B_rowmajor, C, M, N, K, group_m, max_ctas,
                                                          splits, stream, {}, scratch);
    default:
      return b200::host::kBadConfig;
  }
}
#endif
