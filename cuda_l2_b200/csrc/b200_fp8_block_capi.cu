// libb200_fp8block.so: the block-scaled e4m3 GEMM (include/b200_fp8_block.h). The kernels are the family's pipeline
// with BlockScaled<> configurations (hgemm_sm90.cuh): every k-block's sum is promoted into a second fp32 accumulator
// with its scales. A library of its own, so that libb200_hgemm.so's device code stays as it is.
#include "../../include/b200_fp8_block.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

using b200::host::GemmType;

namespace b200 {
namespace block {

// (eligible(), sibling() and kModes are in hgemm_configs.cuh, select() in hgemm_dispatch.cuh.)

// The epilogue operands of a call: the block scales and the row stride of A's.
host::EpiOperands operands(const void* scale_a, int ld_a, const void* scale_b) {
  return {Scales{static_cast<const float*>(scale_a), static_cast<const float*>(scale_b)}, ld_a};
}

int run(int config_id, int out_bf16, const void* A, const void* Bt, void* C, const host::EpiOperands& op, int M, int N,
        int K, int group_m, int max_ctas, int splits, void* stream) {
  if (out_bf16 == 0)
    return run_config<GemmType::kE4M3F16Block, BlockScaled>(config_id, A, Bt, C, M, N, K, group_m, max_ctas, splits,
                                                            stream, op);
  if (out_bf16 == 1)
    return run_config<GemmType::kE4M3BF16Block, BlockScaled>(config_id, A, Bt, C, M, N, K, group_m, max_ctas, splits,
                                                             stream, op);
  return host::kBadConfig;
}

}  // namespace block
}  // namespace b200

extern "C" {

int b200_fp8gemm_blockwise(const void* A, const void* B_kmajor, void* C, const void* scale_a, int ld_a,
                           const void* scale_b, int out_bf16, int M, int N, int K, void* stream) {
  using namespace b200;
  if (out_bf16 != 0 && out_bf16 != 1) return host::kBadConfig;
  const host::EpiOperands op = block::operands(scale_a, ld_a, scale_b);
  if (const int st = host::validate(GemmType::kE4M3F16Block, A, B_kmajor, C, op, M, N, K)) return st;
  const dispatch::Choice ch = block::select(M, N, K);
  return block::run(ch.config_id, out_bf16, A, B_kmajor, C, op, M, N, K, ch.group_m, 0, ch.splits, stream);
}

int b200_fp8gemm_blockwise_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                      const void* scale_a, int ld_a, const void* scale_b, int M, int N, int K,
                                      int group_m, int max_ctas, int splits, void* stream) {
  return b200::block::run(config_id, out_bf16, A, B_kmajor, C, b200::block::operands(scale_a, ld_a, scale_b), M, N,
                          K, group_m, max_ctas, splits, stream);
}

int b200_fp8gemm_blockwise_select(int M, int N, int K, int* config_id, int* group_m, int* splits) {
  if (M <= 0 || N <= 0 || K <= 0) return b200::host::kBadShape;
  const b200::dispatch::Choice ch = b200::block::select(M, N, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  if (splits) *splits = ch.splits;
  return 0;
}

unsigned long long b200_fp8block_launch_count(void) {
  return b200::g_launches.load(std::memory_order_relaxed);
}

const char* b200_fp8block_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"
