// libb200_fp8block_1d1d.so — the block-scaled e4m3 GEMM with 1 x 128 scales on both operands (b200_fp8_block_1d1d.h):
// the BlockScaled1D1D<> kernels (hgemm_sm90.cuh) of the block-scaled configurations. A library of its own, so that the
// device code of the others stays as it is. build.py compiles this file once per output type (-DB200_VARIANT = 7, fp16,
// or 8, bf16: the GemmType index), in parallel; the object of variant 7 also holds the entry points.
#include "b200_fp8_block_1d1d.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_VARIANT
#error "compile once per output type with -DB200_VARIANT=7 or 8"
#endif

namespace b200 {

extern template B200_RUN(host::GemmType::kE4M3F16Block1D1D, BlockScaled1D1D);
extern template B200_RUN(host::GemmType::kE4M3BF16Block1D1D, BlockScaled1D1D);
template B200_RUN(host::GemmType(B200_VARIANT), BlockScaled1D1D);

}  // namespace b200

#if B200_VARIANT == 7

namespace {

using b200::host::GemmType;

// The epilogue operands of a call: both operands' 1 x 128 scales and their row strides.
b200::host::EpiOperands operands(const void* scale_a, int ld_a, const void* scale_b, int ld_b) {
  return {b200::Scales{static_cast<const float*>(scale_a), static_cast<const float*>(scale_b)}, ld_a, ld_b};
}

int run(int config_id, int out_bf16, const void* A, const void* Bt, void* C, const b200::host::EpiOperands& op, int M,
        int N, int K, int group_m, int max_ctas, int splits, void* stream) {
  using b200::BlockScaled1D1D;
  using b200::run_config;
  if (out_bf16 == 0)
    return run_config<GemmType::kE4M3F16Block1D1D, BlockScaled1D1D>(config_id, A, Bt, C, M, N, K, group_m, max_ctas,
                                                                    splits, stream, op);
  if (out_bf16 == 1)
    return run_config<GemmType::kE4M3BF16Block1D1D, BlockScaled1D1D>(config_id, A, Bt, C, M, N, K, group_m, max_ctas,
                                                                     splits, stream, op);
  return b200::host::kBadConfig;
}

}  // namespace

extern "C" {

int cuda_l2_b200_fp8block_1d1d_run(const void* A, const void* B_kmajor, void* C, const void* scale_a, int ld_a,
                                   const void* scale_b, int ld_b, int out_bf16, int M, int N, int K, void* stream) {
  using namespace b200;
  if (out_bf16 != 0 && out_bf16 != 1) return host::kBadConfig;
  // the argument rules before the lookup, which wants a valid shape
  const host::EpiOperands op = operands(scale_a, ld_a, scale_b, ld_b);
  if (const int st = host::validate(GemmType::kE4M3F16Block1D1D, A, B_kmajor, C, op, M, N, K)) return st;
  if (ld_b < N || ld_b % 4) return host::kBadScaleLdB;
  const dispatch::Choice ch = block::select(M, N, K);
  return run(ch.config_id, out_bf16, A, B_kmajor, C, op, M, N, K, ch.group_m, 0, ch.splits, stream);
}

int cuda_l2_b200_fp8block_1d1d_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                          const void* scale_a, int ld_a, const void* scale_b, int ld_b, int M, int N,
                                          int K, int group_m, int max_ctas, int splits, void* stream) {
  return run(config_id, out_bf16, A, B_kmajor, C, operands(scale_a, ld_a, scale_b, ld_b), M, N, K, group_m, max_ctas,
             splits, stream);
}

int cuda_l2_b200_fp8block_1d1d_select(int M, int N, int K, int* config_id, int* group_m, int* splits) {
  if (M <= 0 || N <= 0 || K <= 0) return b200::host::kBadShape;
  const b200::dispatch::Choice ch = b200::block::select(M, N, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  if (splits) *splits = ch.splits;
  return 0;
}

unsigned long long cuda_l2_b200_fp8block_1d1d_launch_count(void) {
  return b200::g_launches.load(std::memory_order_relaxed);
}

const char* cuda_l2_b200_fp8block_1d1d_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_VARIANT == 7
