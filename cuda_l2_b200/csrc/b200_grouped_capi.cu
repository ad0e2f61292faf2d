// libb200_grouped.so: the grouped 16-bit GEMM over contiguous row groups (include/b200_grouped.h). The kernels are the
// family's pipeline with Grouped<> configurations (hgemm_sm90.cuh): a 2-D map over A [T, K] and C [T, N], the batched
// 3-D map over Bt [G, N, K], and one flat tile list over the groups' own rows. A library of its own, so that the device
// code of libb200_hgemm.so and libb200_batched.so stays as it is.
//
// build.py compiles this file once per data type (-DB200_GROUPED_VARIANT = 0, 1, 2: the GemmType index), in parallel;
// each object instantiates the 31 kernels of its type, and the object of variant 0 also holds the C entry points.
#include "../../include/b200_grouped.h"

#include <climits>

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_GROUPED_VARIANT
#error "compile once per data type with -DB200_GROUPED_VARIANT=0, 1 or 2 (cuda_l2_b200/build.py does)"
#endif

using b200::host::GemmType;

namespace b200 {
namespace gmm {

// Kernel launches of this library (b200_grouped_launch_count): one counter for its three objects.
__attribute__((visibility("hidden"))) inline std::atomic<unsigned long long> g_grouped_launches{0};

template <GemmType T>
int run_config(int id, const void* A, const void* Bt, void* C, const int* offs, int G, int rows, int N, int K,
               int group_m, int max_ctas, cudaStream_t s) {
  constexpr host::GemmTypeTraits t = host::traits(T);
  static_assert(!t.e4m3() && !t.scaled, "16-bit variants only");
  int st;
  switch (id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                  \
  case ID:                                                                                                     \
    st = host::launch_grouped<Grouped<Config<BN, STAGES, CG, t.acc_f32, CM, CN, MR, t.bf16()>>>(               \
        A, Bt, C, offs, G, rows, N, K, s, group_m, max_ctas);                                                   \
    break;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      return host::kBadConfig;
  }
  if (st == host::kOk && rows > 0) g_grouped_launches.fetch_add(1, std::memory_order_relaxed);
  return st;
}

// Each object instantiates its own variant's kernels; the calls of the other objects' variants link against theirs.
#define B200_GROUPED_RUN(T)                                                                                    \
  int run_config<T>(int, const void*, const void*, void*, const int*, int, int, int, int, int, int, cudaStream_t)
extern template B200_GROUPED_RUN(GemmType::kF16Acc32);
extern template B200_GROUPED_RUN(GemmType::kF16Acc16);
extern template B200_GROUPED_RUN(GemmType::kBF16);
template B200_GROUPED_RUN(GemmType(B200_GROUPED_VARIANT));
#undef B200_GROUPED_RUN

}  // namespace gmm
}  // namespace b200

#if B200_GROUPED_VARIANT == 0

namespace b200 {
namespace gmm {

bool known_variant(int v) { return v >= 0 && v <= 2; }

int run(int variant, int config_id, const void* A, const void* Bt, void* C, const int* offs, int G, int T, int N, int K,
        int group_m, int max_ctas, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (variant) {
    case 0: return run_config<GemmType::kF16Acc32>(config_id, A, Bt, C, offs, G, T, N, K, group_m, max_ctas, s);
    case 1: return run_config<GemmType::kF16Acc16>(config_id, A, Bt, C, offs, G, T, N, K, group_m, max_ctas, s);
    case 2: return run_config<GemmType::kBF16>(config_id, A, Bt, C, offs, G, T, N, K, group_m, max_ctas, s);
    default: return host::kBadConfig;
  }
}

// The batched rule with B = G matrices of the average group, ceil(T / G) rows.
dispatch::Choice select(int variant, int G, int T, int N, int K) {
  return dispatch::select_batched(GemmType(variant), G, (T + G - 1) / G, N, K);
}

template <class Cfg>
int schedule_units(int G, int T, int N, int K, const int* offs, int num_sms, int worker, int* units, int max_units,
                   int* num_workers) {
  if (host::grouped_worst_tiles<Cfg>(G, T, N) > INT_MAX) return host::kBadShape;
  // every cluster resident: the launcher's plan on a device of num_sms SMs, with its default group_m
  const int max_workers = num_sms / Cfg::CLUSTER_CTAS;
  const host::Plan p = host::grouped_plan<Cfg>(G, T, N, K, max_workers, [=] { return max_workers; });
  if (num_workers) *num_workers = p.workers;
  if (worker < 0 || worker >= p.workers) return host::kBadShape;
  const int n_blocks = (N + Cfg::BN * Cfg::CLUSTER_N - 1) / (Cfg::BN * Cfg::CLUSTER_N);
  GroupCursor groups(offs, G, T, Cfg::TILE_M * Cfg::CLUSTER_M, n_blocks, Cfg::CTA_GROUP == 2 ? 8 : 16);
  WorkIter it(worker, p.workers, groups.total(), p.nkb, 1, 0);
  WorkUnit u;
  int n = 0;
  while (it.next(u)) {
    const BatchTile gt = groups.locate(u.tile);
    if (n < max_units && units) {
      units[3 * n] = gt.batch; units[3 * n + 1] = gt.tc.m_blk; units[3 * n + 2] = gt.tc.n_blk;
    }
    ++n;
  }
  return n;
}

}  // namespace gmm
}  // namespace b200

extern "C" {

int b200_grouped_gemm(int variant, const void* A, const void* B_kmajor, void* C, const int* offs, int G, int T, int N,
                      int K, void* stream) {
  using namespace b200;
  if (!gmm::known_variant(variant)) return host::kBadConfig;
  // the argument rules before the lookup, which wants a valid shape (the tile count is checked with the configuration)
  if (const int st = host::validate_grouped(GemmType(variant), A, B_kmajor, C, offs, G, T, N, K, 1)) return st;
  if (T == 0) return host::kOk;
  const dispatch::Choice ch = gmm::select(variant, G, T, N, K);
  return gmm::run(variant, ch.config_id, A, B_kmajor, C, offs, G, T, N, K, ch.group_m, 0, stream);
}

int b200_grouped_gemm_run_config(int variant, int config_id, const void* A, const void* B_kmajor, void* C,
                                 const int* offs, int G, int T, int N, int K, int group_m, int max_ctas, void* stream) {
  return b200::gmm::run(variant, config_id, A, B_kmajor, C, offs, G, T, N, K, group_m, max_ctas, stream);
}

int b200_grouped_select(int variant, int G, int T, int N, int K, int* config_id, int* group_m) {
  if (!b200::gmm::known_variant(variant)) return b200::host::kBadConfig;
  if (G <= 0 || T <= 0 || N <= 0 || K <= 0) return b200::host::kBadShape;
  const b200::dispatch::Choice ch = b200::gmm::select(variant, G, T, N, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  return 0;
}

int b200_grouped_schedule_units(int config_id, int G, int T, int N, int K, const int* offs_host, int num_sms,
                                int worker, int* units, int max_units, int* num_workers) {
  if (G <= 0 || T <= 0 || N <= 0 || K <= 0 || num_sms <= 0 || !offs_host) return b200::host::kBadShape;
  switch (config_id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                 \
  case ID:                                                                                                      \
    return b200::gmm::schedule_units<b200::Grouped<b200::Config<BN, STAGES, CG, true, CM, CN, MR>>>(          \
        G, T, N, K, offs_host, num_sms, worker, units, max_units, num_workers);
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      return b200::host::kBadConfig;
  }
}

unsigned long long b200_grouped_launch_count(void) {
  return b200::gmm::g_grouped_launches.load(std::memory_order_relaxed);
}

const char* b200_grouped_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_GROUPED_VARIANT == 0
