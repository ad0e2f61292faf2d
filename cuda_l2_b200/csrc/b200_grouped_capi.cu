// libb200_grouped.so: the grouped 16-bit GEMM over contiguous row groups (include/b200_grouped.h). The kernels are the
// family's pipeline with Grouped<> configurations (hgemm_sm90.cuh): a 2-D map over A [T, K] and C [T, N], the batched
// 3-D map over Bt [G, N, K], and one flat tile list over the groups' own rows. A library of its own, so that the device
// code of libb200_hgemm.so and libb200_batched.so stays as it is. The library's core is tile_list (hgemm_configs.cuh,
// hgemm_dispatch.cuh), shared by the four tile-list libraries; build.py compiles this file once per data type (B200_VARIANT).
#include "../../include/b200_grouped.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_VARIANT
#error "compile once per data type with -DB200_VARIANT=0, 1 or 2 (cuda_l2_b200/build.py does)"
#endif

namespace b200 {
namespace tile_list {
B200_LIST_OBJECT(Library, Grouped, B200_LIST_TYPES);
}  // namespace tile_list
}  // namespace b200

#if B200_VARIANT == 0

using b200::host::GemmType;

extern "C" {

int b200_grouped_gemm(int variant, const void* A, const void* B_kmajor, void* C, const int* offs, int G, int T, int N,
                      int K, void* stream) {
  using namespace b200;
  if (!tile_list::holds(tile_list::Library{}, variant)) return host::kBadConfig;
  return tile_list::gemm(tile_list::Library{}, GemmType(variant), A, B_kmajor, C, offs, G, T, N, K, stream);
}

int b200_grouped_gemm_run_config(int variant, int config_id, const void* A, const void* B_kmajor, void* C,
                                 const int* offs, int G, int T, int N, int K, int group_m, int max_ctas, void* stream) {
  using namespace b200;
  return tile_list::run(tile_list::Library{}, GemmType(variant), config_id, A, B_kmajor, C, offs, G, T, N, K, group_m,
                        max_ctas, stream);
}

int b200_grouped_select(int variant, int G, int T, int N, int K, int* config_id, int* group_m) {
  if (!b200::tile_list::holds(b200::tile_list::Library{}, variant)) return b200::host::kBadConfig;
  return b200::tile_list::select_into<b200::Grouped>(GemmType(variant), G, T, N, K, config_id, group_m);
}

int b200_grouped_schedule_units(int config_id, int G, int T, int N, int K, const int* offs_host, int num_sms,
                                int worker, int* units, int max_units, int* num_workers) {
  if (G <= 0 || T <= 0 || N <= 0 || K <= 0 || num_sms <= 0 || !offs_host) return b200::host::kBadShape;
  return b200::tile_list::schedule_config<b200::Grouped>(config_id, G, T, N, K, offs_host, num_sms, worker, units,
                                                         max_units, num_workers);
}

unsigned long long b200_grouped_launch_count(void) {
  return b200::tile_list::g_list_launches.load(std::memory_order_relaxed);
}

const char* b200_grouped_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_VARIANT == 0
