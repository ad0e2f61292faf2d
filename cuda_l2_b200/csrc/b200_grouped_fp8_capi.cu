// libb200_grouped_fp8.so: the block-scaled e4m3 grouped GEMM over contiguous row groups (include/b200_grouped_fp8.h).
// The kernels are the family's pipeline with Grouped<BlockScaled<>> configurations (hgemm_sm90.cuh): the grouped tile
// list and maps of libb200_grouped.so, the per-k-block promotion of libb200_fp8block.so. A library of its own, so that
// the device code and kernel counts of those two stay as they are. The core is tile_list (hgemm_configs.cuh); build.py
// compiles this file once per output type (B200_VARIANT = 5: fp16, 6: bf16, the GemmType index).
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

namespace {

b200::Scales scales_of(const void* scale_a, const void* scale_b) {
  return b200::Scales{static_cast<const float*>(scale_a), static_cast<const float*>(scale_b)};
}

int run(int config_id, int out_bf16, const void* A, const void* Bt, void* C, const void* scale_a, int ld_a,
        const void* scale_b, const int* offs, int G, int T, int N, int K, int group_m, int max_ctas, void* stream) {
  using namespace b200;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const Scales sc = scales_of(scale_a, scale_b);
  if (out_bf16 == 0)
    return tile_list::run_config<Grouped, GemmType::kE4M3F16Block>(config_id, A, Bt, C, offs, G, T, N, K, group_m,
                                                                   max_ctas, s, sc, ld_a);
  if (out_bf16 == 1)
    return tile_list::run_config<Grouped, GemmType::kE4M3BF16Block>(config_id, A, Bt, C, offs, G, T, N, K, group_m,
                                                                    max_ctas, s, sc, ld_a);
  return host::kBadConfig;
}

// The grouped rule for e4m3 operands, mapped to the block-scaled sibling (group_m kept; there is no split here).
b200::dispatch::Choice select(int G, int T, int N, int K) {
  b200::dispatch::Choice ch = b200::dispatch::select_grouped(GemmType::kE4M3F16Block, G, T, N, K);
  ch.config_id = b200::block::sibling(ch.config_id);
  ch.splits = 1;
  return ch;
}

}  // namespace

extern "C" {

int b200_grouped_fp8_gemm(const void* A, const void* B_kmajor, void* C, const void* scale_a, int ld_a,
                          const void* scale_b, int out_bf16, const int* offs, int G, int T, int N, int K, void* stream) {
  using namespace b200;
  if (out_bf16 != 0 && out_bf16 != 1) return host::kBadConfig;
  // the argument rules before the lookup, which wants a valid shape (the tile count is checked with the configuration)
  if (const int st = host::validate_grouped(GemmType::kE4M3F16Block, A, B_kmajor, C, offs, G, T, N, K, 1,
                                            scales_of(scale_a, scale_b), ld_a))
    return st;
  if (T == 0) return host::kOk;
  if (tile_list::fewest_tiles<Grouped>(G, T, N, true) > 0x7fffffffLL) return host::kBadShape;
  const dispatch::Choice ch = select(G, T, N, K);
  return run(ch.config_id, out_bf16, A, B_kmajor, C, scale_a, ld_a, scale_b, offs, G, T, N, K, ch.group_m, 0, stream);
}

int b200_grouped_fp8_gemm_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                     const void* scale_a, int ld_a, const void* scale_b, const int* offs, int G, int T,
                                     int N, int K, int group_m, int max_ctas, void* stream) {
  return run(config_id, out_bf16, A, B_kmajor, C, scale_a, ld_a, scale_b, offs, G, T, N, K, group_m, max_ctas, stream);
}

int b200_grouped_fp8_select(int G, int T, int N, int K, int* config_id, int* group_m) {
  if (G <= 0 || T <= 0 || N <= 0 || K <= 0) return b200::host::kBadShape;
  const b200::dispatch::Choice ch = select(G, T, N, K);
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
