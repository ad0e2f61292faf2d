// libb200_epilogue.so — the BiasAct<> kernels (hgemm_sm90.cuh) of every configuration and K-mode, behind the internal
// entry points of b200_epilogue.h. A library of its own, so that the device code of the other libraries stays as it
// is. build.py compiles this file once per variant (-DB200_VARIANT = 0, 2, 3 or 4), in parallel; the object of variant 0
// also holds the entry points.
#include "b200_epilogue.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_VARIANT
#error "compile once per variant with -DB200_VARIANT=0, 2, 3 or 4"
#endif

namespace b200 {

extern template B200_RUN(host::GemmType::kF16Acc32, BiasAct);
extern template B200_RUN(host::GemmType::kBF16, BiasAct);
extern template B200_RUN(host::GemmType::kE4M3F16, BiasAct);
extern template B200_RUN(host::GemmType::kE4M3BF16, BiasAct);
template B200_RUN(host::GemmType(B200_VARIANT), BiasAct);

}  // namespace b200

#if B200_VARIANT == 0

namespace {

using b200::host::GemmType;

bool known_variant(int v) {
  return v == int(GemmType::kF16Acc32) || v == int(GemmType::kBF16) || v == int(GemmType::kE4M3F16) ||
         v == int(GemmType::kE4M3BF16);
}

// The epilogue operands of a call: the scales of an e4m3 variant, the bias and the activation code.
b200::host::EpiOperands operands(int variant, const void* scale_a, const void* scale_b, int rowwise, const void* bias,
                                 int act) {
  const b200::Scales sc = b200::host::traits(GemmType(variant)).scaled
      ? b200::Scales{static_cast<const float*>(scale_a), static_cast<const float*>(scale_b), rowwise != 0}
      : b200::Scales{nullptr, nullptr};
  return {sc, 0, 0, bias, act};
}

// Split-K scratch comes from this library's own pool (host::splitk_scratch, run_config's default).
int run_config(int variant, int config_id, const void* A, const void* Bt, void* C, const b200::host::EpiOperands& op,
               int M, int N, int K, int group_m, int max_ctas, int splits, void* stream) {
  using b200::BiasAct;
  using b200::run_config;
  switch (GemmType(variant)) {
    case GemmType::kF16Acc32:
      return run_config<GemmType::kF16Acc32, BiasAct>(config_id, A, Bt, C, M, N, K, group_m, max_ctas, splits, stream,
                                                      op);
    case GemmType::kBF16:
      return run_config<GemmType::kBF16, BiasAct>(config_id, A, Bt, C, M, N, K, group_m, max_ctas, splits, stream, op);
    case GemmType::kE4M3F16:
      return run_config<GemmType::kE4M3F16, BiasAct>(config_id, A, Bt, C, M, N, K, group_m, max_ctas, splits, stream,
                                                     op);
    case GemmType::kE4M3BF16:
      return run_config<GemmType::kE4M3BF16, BiasAct>(config_id, A, Bt, C, M, N, K, group_m, max_ctas, splits, stream,
                                                      op);
    default:
      return b200::host::kBadConfig;
  }
}

}  // namespace

extern "C" {

int cuda_l2_b200_epilogue_run(int variant, const void* A, const void* B_kmajor, void* C, const void* scale_a,
                              const void* scale_b, int rowwise, const void* bias, int act, int M, int N, int K,
                              void* stream) {
  using namespace b200;
  if (!known_variant(variant)) return host::kBadConfig;
  // the argument rules before the lookup, which wants a valid shape
  const host::EpiOperands op = operands(variant, scale_a, scale_b, rowwise, bias, act);
  if (const int st = host::validate(GemmType(variant), A, B_kmajor, C, op, M, N, K)) return st;
  if (const int st = host::validate_bias_act(bias, act)) return st;
  const dispatch::Choice ch = dispatch::select(GemmType(variant), M, N, K);
  return run_config(variant, ch.config_id, A, B_kmajor, C, op, M, N, K, ch.group_m, 0, ch.splits, stream);
}

int cuda_l2_b200_epilogue_run_config(int variant, int config_id, const void* A, const void* B_kmajor, void* C,
                                     const void* scale_a, const void* scale_b, int rowwise, const void* bias, int act,
                                     int M, int N, int K, int group_m, int max_ctas, int splits, void* stream) {
  if (!known_variant(variant)) return b200::host::kBadConfig;
  return run_config(variant, config_id, A, B_kmajor, C, operands(variant, scale_a, scale_b, rowwise, bias, act), M, N,
                    K, group_m, max_ctas, splits, stream);
}

int cuda_l2_b200_epilogue_select(int variant, int M, int N, int K, int* config_id, int* group_m, int* splits) {
  using namespace b200;
  if (!known_variant(variant)) return host::kBadConfig;
  if (M <= 0 || N <= 0 || K <= 0) return host::kBadShape;
  const dispatch::Choice ch = dispatch::select(GemmType(variant), M, N, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  if (splits) *splits = ch.splits;
  return host::kOk;
}

int cuda_l2_b200_epilogue_prewarm(void* stream) {
  int dev = 0;
  const cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return int(e);
  b200::host::SplitKScratch* sk = nullptr;
  return b200::host::splitk_scratch(dev, static_cast<cudaStream_t>(stream), &sk);
}

int cuda_l2_b200_epilogue_release(void) {
  b200::host::release_scratch();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : int(e);
}

unsigned long long cuda_l2_b200_epilogue_launch_count(void) {
  return b200::g_launches.load(std::memory_order_relaxed);
}

const char* cuda_l2_b200_epilogue_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_VARIANT == 0
