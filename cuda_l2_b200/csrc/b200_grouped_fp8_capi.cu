// libb200_grouped_fp8.so: the block-scaled e4m3 grouped GEMM over contiguous row groups (include/b200_grouped_fp8.h).
// The kernels are the family's pipeline with Grouped<BlockScaled<>> configurations (hgemm_sm90.cuh): the grouped tile
// list and maps of libb200_grouped.so, the per-k-block promotion of libb200_fp8block.so. A library of its own, so that
// the device code and kernel counts of those two stay as they are. The core is tile_list (hgemm_configs.cuh,
// hgemm_dispatch.cuh), shared with libb200_batched_fp8.so; build.py compiles this file once per output type
// (B200_VARIANT = 5: fp16, 6: bf16, the GemmType index).
#include "../../include/b200_grouped_fp8.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_VARIANT
#error "compile once per output type with -DB200_VARIANT=5 or 6 (cuda_l2_b200/build.py does)"
#endif

namespace b200 {
namespace tile_list {
B200_BLOCK_LIST_OBJECT(Grouped);
}  // namespace tile_list
}  // namespace b200

#if B200_VARIANT == 5

using b200::host::GemmType;

extern "C" {

int b200_grouped_fp8_gemm(const void* A, const void* B_kmajor, void* C, const void* scale_a, int ld_a,
                          const void* scale_b, int out_bf16, const int* offs, int G, int T, int N, int K, void* stream) {
  using namespace b200;
  if (out_bf16 != 0 && out_bf16 != 1) return host::kBadConfig;
  // the argument rules before the lookup, which wants a valid shape (the tile count is checked with the configuration)
  const Scales sc{static_cast<const float*>(scale_a), static_cast<const float*>(scale_b)};
  if (const int st = host::validate_grouped(GemmType::kE4M3F16Block, A, B_kmajor, C, offs, G, T, N, K, 1, sc, ld_a))
    return st;
  if (T == 0) return host::kOk;
  if (tile_list::fewest_tiles<Grouped>(G, T, N, true) > 0x7fffffffLL) return host::kBadShape;
  const dispatch::Choice ch = tile_list::select_block<Grouped>(G, T, N, K);
  return tile_list::run_block<Grouped>(ch.config_id, out_bf16, A, B_kmajor, C, scale_a, ld_a, scale_b, offs, G, T, N, K,
                                       ch.group_m, 0, stream);
}

int b200_grouped_fp8_gemm_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                     const void* scale_a, int ld_a, const void* scale_b, const int* offs, int G, int T,
                                     int N, int K, int group_m, int max_ctas, void* stream) {
  return b200::tile_list::run_block<b200::Grouped>(config_id, out_bf16, A, B_kmajor, C, scale_a, ld_a, scale_b, offs, G,
                                                   T, N, K, group_m, max_ctas, stream);
}

int b200_grouped_fp8_select(int G, int T, int N, int K, int* config_id, int* group_m) {
  if (G <= 0 || T <= 0 || N <= 0 || K <= 0) return b200::host::kBadShape;
  const b200::dispatch::Choice ch = b200::tile_list::select_block<b200::Grouped>(G, T, N, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  return 0;
}

unsigned long long b200_grouped_fp8_launch_count(void) {
  return b200::tile_list::g_list_launches.load(std::memory_order_relaxed);
}

const char* b200_grouped_fp8_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_VARIANT == 5
