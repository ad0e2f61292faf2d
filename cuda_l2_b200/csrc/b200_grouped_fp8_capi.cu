// libb200_grouped_fp8.so: the block-scaled e4m3 grouped GEMM over contiguous row groups (include/b200_grouped_fp8.h).
// The kernels are the family's pipeline with Grouped<BlockScaled<>> configurations (hgemm_sm90.cuh): the grouped tile
// list and maps of libb200_grouped.so, the per-k-block promotion of libb200_fp8block.so. A library of its own, so that
// the device code and kernel counts of those two stay as they are. The core is tile_list (hgemm_configs.cuh,
// hgemm_dispatch.cuh), shared by the four tile-list libraries; build.py compiles this file once per output type
// (B200_VARIANT = 5: fp16, 6: bf16, the GemmType index).
#include "../../include/b200_grouped_fp8.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_VARIANT
#error "compile once per output type with -DB200_VARIANT=5 or 6 (cuda_l2_b200/build.py does)"
#endif

namespace b200 {
namespace tile_list {
B200_LIST_OBJECT(Library, Grouped, B200_BLOCK_LIST_TYPES);
}  // namespace tile_list
}  // namespace b200

#if B200_VARIANT == 5

using b200::host::GemmType;

extern "C" {

int b200_grouped_fp8_gemm(const void* A, const void* B_kmajor, void* C, const void* scale_a, int ld_a,
                          const void* scale_b, int out_bf16, const int* offs, int G, int T, int N, int K, void* stream) {
  using namespace b200;
  if (!tile_list::known_out(out_bf16)) return host::kBadConfig;
  return tile_list::gemm(tile_list::Library{}, tile_list::block_type(out_bf16), A, B_kmajor, C, offs, G, T, N, K, stream,
                         tile_list::block_operands(scale_a, ld_a, scale_b));
}

int b200_grouped_fp8_gemm_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                     const void* scale_a, int ld_a, const void* scale_b, const int* offs, int G, int T,
                                     int N, int K, int group_m, int max_ctas, void* stream) {
  using namespace b200;
  if (!tile_list::known_out(out_bf16)) return host::kBadConfig;
  return tile_list::run(tile_list::Library{}, tile_list::block_type(out_bf16), config_id, A, B_kmajor, C, offs, G, T, N,
                        K, group_m, max_ctas, stream, tile_list::block_operands(scale_a, ld_a, scale_b));
}

int b200_grouped_fp8_select(int G, int T, int N, int K, int* config_id, int* group_m) {
  return b200::tile_list::select_into<b200::Grouped>(GemmType::kE4M3F16Block, G, T, N, K, config_id, group_m);
}

unsigned long long b200_grouped_fp8_launch_count(void) {
  return b200::tile_list::g_list_launches.load(std::memory_order_relaxed);
}

const char* b200_grouped_fp8_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_VARIANT == 5
