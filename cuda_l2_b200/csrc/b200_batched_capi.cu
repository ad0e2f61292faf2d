// libb200_batched.so: the batched 16-bit GEMM (include/b200_batched.h). The kernels are the family's pipeline with
// Batched<> configurations (hgemm_sm90.cuh): 3-D tensor maps and one flat tile list over all matrices. A library of its
// own, so that libb200_hgemm.so's device code stays as it is. The library's core is tile_list (hgemm_configs.cuh,
// hgemm_dispatch.cuh), shared by the four tile-list libraries; build.py compiles this file once per data type (B200_VARIANT).
#include "../../include/b200_batched.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_VARIANT
#error "compile once per data type with -DB200_VARIANT=0, 1 or 2 (cuda_l2_b200/build.py does)"
#endif

namespace b200 {
namespace tile_list {
B200_LIST_OBJECT(Library, Batched, B200_LIST_TYPES);
}  // namespace tile_list
}  // namespace b200

#if B200_VARIANT == 0

using b200::host::GemmType;

extern "C" {

int b200_batched_gemm(int variant, const void* A, const void* B_kmajor, void* C, const int* masked_m, int B, int M,
                      int N, int K, void* stream) {
  using namespace b200;
  if (!tile_list::holds(tile_list::Library{}, variant)) return host::kBadConfig;
  return tile_list::gemm(tile_list::Library{}, GemmType(variant), A, B_kmajor, C, masked_m, B, M, N, K, stream);
}

int b200_batched_gemm_run_config(int variant, int config_id, const void* A, const void* B_kmajor, void* C,
                                 const int* masked_m, int B, int M, int N, int K, int group_m, int max_ctas,
                                 void* stream) {
  using namespace b200;
  return tile_list::run(tile_list::Library{}, GemmType(variant), config_id, A, B_kmajor, C, masked_m, B, M, N, K,
                        group_m, max_ctas, stream);
}

int b200_batched_select(int variant, int B, int M, int N, int K, int* config_id, int* group_m) {
  if (!b200::tile_list::holds(b200::tile_list::Library{}, variant)) return b200::host::kBadConfig;
  return b200::tile_list::select_into<b200::Batched>(GemmType(variant), B, M, N, K, config_id, group_m);
}

int b200_batched_schedule_units(int config_id, int B, int M, int N, int K, const int* masked_m_host, int num_sms,
                                int worker, int* units, int max_units, int* num_workers) {
  if (B <= 0 || M <= 0 || N <= 0 || K <= 0 || num_sms <= 0) return b200::host::kBadShape;
  return b200::tile_list::schedule_config<b200::Batched>(config_id, B, M, N, K, masked_m_host, num_sms, worker, units,
                                                         max_units, num_workers);
}

unsigned long long b200_batched_launch_count(void) {
  return b200::tile_list::g_list_launches.load(std::memory_order_relaxed);
}

const char* b200_batched_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_VARIANT == 0
