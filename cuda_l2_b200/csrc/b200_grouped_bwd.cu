// libb200_grouped_bwd.so — the backward of the grouped 16-bit product (b200_grouped_bwd.h): Grouped<RowMajorB<>>
// (the input gradient) and GroupedK<RowMajorB<>> (the weight gradient) kernels of every configuration with a row-major
// B kernel (nn::has_kernel), launched through tile_list (hgemm_configs.cuh, hgemm_dispatch.cuh) like the other
// tile-list libraries. A library of its own, so that the device code of the other libraries stays as it is. build.py
// compiles this file once per variant (-DB200_VARIANT = 0 or 2); the object of variant 0 also holds the entry points.
#include "b200_grouped_bwd.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_VARIANT
#error "compile once per variant with -DB200_VARIANT=0 or 2"
#endif

namespace b200 {
namespace tile_list {

template <class Cfg>
using GroupedRowMajorB = Grouped<RowMajorB<Cfg>>;
template <class Cfg>
using GroupedKRowMajorB = GroupedK<RowMajorB<Cfg>>;

// fp16 and bf16, both with fp32 accumulation
#define B200_BWD_TYPES(X, W) X(W, host::GemmType::kF16Acc32) X(W, host::GemmType::kBF16)
B200_LIST_OBJECT(NNLibrary, GroupedRowMajorB, B200_BWD_TYPES);
B200_LIST_OBJECT(WgradLibrary, GroupedKRowMajorB, B200_BWD_TYPES);
#undef B200_BWD_TYPES

}  // namespace tile_list
}  // namespace b200

#if B200_VARIANT == 0

using b200::host::GemmType;

extern "C" {

int cuda_l2_b200_grouped_bwd_nn(int variant, int config_id, const void* A, const void* B_rowmajor, void* C,
                                const int* offs, int G, int T, int N, int K, int group_m, int max_ctas, void* stream) {
  using namespace b200;
  const tile_list::NNLibrary lib;
  if (!tile_list::holds(lib, variant)) return host::kBadConfig;
  if (config_id < 0) return tile_list::gemm(lib, GemmType(variant), A, B_rowmajor, C, offs, G, T, N, K, stream);
  return tile_list::run(lib, GemmType(variant), config_id, A, B_rowmajor, C, offs, G, T, N, K, group_m, max_ctas, stream);
}

// The K-grouped list: `count` = G matrices of `rows` = M rows by N columns, a reduction over K = T rows.
int cuda_l2_b200_grouped_bwd_wgrad(int variant, int config_id, const void* A, const void* B, void* C, const int* offs,
                                   int G, int T, int M, int N, int group_m, int max_ctas, void* stream) {
  using namespace b200;
  const tile_list::WgradLibrary lib;
  if (!tile_list::holds(lib, variant)) return host::kBadConfig;
  if (config_id < 0) return tile_list::gemm(lib, GemmType(variant), A, B, C, offs, G, M, N, T, stream);
  return tile_list::run(lib, GemmType(variant), config_id, A, B, C, offs, G, M, N, T, group_m, max_ctas, stream);
}

int cuda_l2_b200_grouped_bwd_nn_select(int variant, int G, int T, int N, int K, int* config_id, int* group_m) {
  using namespace b200;
  if (!tile_list::holds(tile_list::NNLibrary{}, variant)) return host::kBadConfig;
  return tile_list::select_into<tile_list::GroupedRowMajorB>(GemmType(variant), G, T, N, K, config_id, group_m);
}

int cuda_l2_b200_grouped_bwd_wgrad_select(int variant, int G, int T, int M, int N, int* config_id, int* group_m) {
  using namespace b200;
  if (!tile_list::holds(tile_list::WgradLibrary{}, variant)) return host::kBadConfig;
  return tile_list::select_into<tile_list::GroupedKRowMajorB>(GemmType(variant), G, M, N, T, config_id, group_m);
}

int cuda_l2_b200_grouped_bwd_wgrad_schedule(int config_id, int G, int T, int M, int N, const int* offs_host,
                                            int num_sms, int worker, int* units, int max_units, int* num_workers) {
  using namespace b200;
  if (G <= 0 || T < 0 || M <= 0 || N <= 0 || num_sms <= 0 || !offs_host) return host::kBadShape;
  return tile_list::schedule_config<tile_list::GroupedKRowMajorB>(config_id, G, M, N, T, offs_host, num_sms, worker,
                                                                  units, max_units, num_workers);
}

unsigned long long cuda_l2_b200_grouped_bwd_launch_count(void) {
  return b200::tile_list::g_list_launches.load(std::memory_order_relaxed);
}

const char* cuda_l2_b200_grouped_bwd_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_VARIANT == 0
