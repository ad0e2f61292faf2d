// libb200_batched.so: the batched 16-bit GEMM (include/b200_batched.h). The kernels are the family's pipeline with
// Batched<> configurations (hgemm_sm90.cuh): 3-D tensor maps and one flat tile list over all matrices. A library of its
// own, so that libb200_hgemm.so's device code stays as it is.
//
// build.py compiles this file once per data type (-DB200_BATCHED_VARIANT = 0, 1, 2: the GemmType index), in parallel;
// each object instantiates the 31 kernels of its type, and the object of variant 0 also holds the C entry points.
#include "../../include/b200_batched.h"

#include <climits>

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_BATCHED_VARIANT
#error "compile once per data type with -DB200_BATCHED_VARIANT=0, 1 or 2 (cuda_l2_b200/build.py does)"
#endif

using b200::host::GemmType;

namespace b200 {
namespace bmm {

// Kernel launches of this library (b200_batched_launch_count): one counter for its three objects.
__attribute__((visibility("hidden"))) inline std::atomic<unsigned long long> g_batched_launches{0};

template <GemmType T>
int run_config(int id, const void* A, const void* Bt, void* C, const int* masked_m, int B, int M, int N, int K,
               int group_m, int max_ctas, cudaStream_t s) {
  constexpr host::GemmTypeTraits t = host::traits(T);
  static_assert(!t.e4m3() && !t.scaled, "16-bit variants only");
  int st;
  switch (id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                  \
  case ID:                                                                                                     \
    st = host::launch_batched<Batched<Config<BN, STAGES, CG, t.acc_f32, CM, CN, MR, t.bf16()>>>(               \
        A, Bt, C, masked_m, B, M, N, K, s, group_m, max_ctas);                                                  \
    break;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      return host::kBadConfig;
  }
  if (st == host::kOk) g_batched_launches.fetch_add(1, std::memory_order_relaxed);
  return st;
}

// Each object instantiates its own variant's kernels; the calls of the other objects' variants link against theirs.
#define B200_BATCHED_RUN(T)                                                                                    \
  int run_config<T>(int, const void*, const void*, void*, const int*, int, int, int, int, int, int, cudaStream_t)
extern template B200_BATCHED_RUN(GemmType::kF16Acc32);
extern template B200_BATCHED_RUN(GemmType::kF16Acc16);
extern template B200_BATCHED_RUN(GemmType::kBF16);
template B200_BATCHED_RUN(GemmType(B200_BATCHED_VARIANT));
#undef B200_BATCHED_RUN

}  // namespace bmm
}  // namespace b200

#if B200_BATCHED_VARIANT == 0

namespace b200 {
namespace bmm {

bool known_variant(int v) { return v >= 0 && v <= 2; }

int run(int variant, int config_id, const void* A, const void* Bt, void* C, const int* masked_m, int B, int M, int N,
        int K, int group_m, int max_ctas, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (variant) {
    case 0: return run_config<GemmType::kF16Acc32>(config_id, A, Bt, C, masked_m, B, M, N, K, group_m, max_ctas, s);
    case 1: return run_config<GemmType::kF16Acc16>(config_id, A, Bt, C, masked_m, B, M, N, K, group_m, max_ctas, s);
    case 2: return run_config<GemmType::kBF16>(config_id, A, Bt, C, masked_m, B, M, N, K, group_m, max_ctas, s);
    default: return host::kBadConfig;
  }
}

dispatch::Choice select(int variant, int B, int M, int N, int K) {
  return dispatch::select_batched(GemmType(variant), B, M, N, K);
}

template <class Cfg>
int schedule_units(int B, int M, int N, int K, const int* masked_m, int num_sms, int worker, int* units, int max_units,
                   int* num_workers) {
  if ((long long)B * host::batch_tiles<Cfg>(M, N) > INT_MAX) return host::kBadShape;
  // every cluster resident: the launcher's plan on a device of num_sms SMs, with its default group_m
  const int max_workers = num_sms / Cfg::CLUSTER_CTAS;
  const host::Plan p = host::batched_plan<Cfg>(B, M, N, K, max_workers, [=] { return max_workers; });
  if (num_workers) *num_workers = p.workers;
  if (worker < 0 || worker >= p.workers) return host::kBadShape;
  const int n_blocks = (N + Cfg::BN * Cfg::CLUSTER_N - 1) / (Cfg::BN * Cfg::CLUSTER_N);
  BatchCursor batches(masked_m, B, M, Cfg::TILE_M * Cfg::CLUSTER_M, n_blocks, Cfg::CTA_GROUP == 2 ? 8 : 16);
  WorkIter it(worker, p.workers, batches.total(), p.nkb, 1, 0);
  WorkUnit u;
  int n = 0;
  while (it.next(u)) {
    const BatchTile bt = batches.locate(u.tile);
    if (n < max_units && units) {
      units[3 * n] = bt.batch; units[3 * n + 1] = bt.tc.m_blk; units[3 * n + 2] = bt.tc.n_blk;
    }
    ++n;
  }
  return n;
}

}  // namespace bmm
}  // namespace b200

extern "C" {

int b200_batched_gemm(int variant, const void* A, const void* B_kmajor, void* C, const int* masked_m, int B, int M,
                      int N, int K, void* stream) {
  using namespace b200;
  if (!bmm::known_variant(variant)) return host::kBadConfig;
  // the argument rules before the lookup, which wants a valid shape (the tile count is checked with the configuration)
  if (const int st = host::validate(GemmType(variant), A, B_kmajor, C, Scales{nullptr, nullptr}, M, N, K, 0, B, 1,
                                    masked_m))
    return st;
  const dispatch::Choice ch = bmm::select(variant, B, M, N, K);
  return bmm::run(variant, ch.config_id, A, B_kmajor, C, masked_m, B, M, N, K, ch.group_m, 0, stream);
}

int b200_batched_gemm_run_config(int variant, int config_id, const void* A, const void* B_kmajor, void* C,
                                 const int* masked_m, int B, int M, int N, int K, int group_m, int max_ctas,
                                 void* stream) {
  return b200::bmm::run(variant, config_id, A, B_kmajor, C, masked_m, B, M, N, K, group_m, max_ctas, stream);
}

int b200_batched_select(int variant, int B, int M, int N, int K, int* config_id, int* group_m) {
  if (!b200::bmm::known_variant(variant)) return b200::host::kBadConfig;
  if (B <= 0 || M <= 0 || N <= 0 || K <= 0) return b200::host::kBadShape;
  const b200::dispatch::Choice ch = b200::bmm::select(variant, B, M, N, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  return 0;
}

int b200_batched_schedule_units(int config_id, int B, int M, int N, int K, const int* masked_m_host, int num_sms,
                                int worker, int* units, int max_units, int* num_workers) {
  if (B <= 0 || M <= 0 || N <= 0 || K <= 0 || num_sms <= 0) return b200::host::kBadShape;
  switch (config_id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                 \
  case ID:                                                                                                      \
    return b200::bmm::schedule_units<b200::Batched<b200::Config<BN, STAGES, CG, true, CM, CN, MR>>>(          \
        B, M, N, K, masked_m_host, num_sms, worker, units, max_units, num_workers);
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      return b200::host::kBadConfig;
  }
}

unsigned long long b200_batched_launch_count(void) {
  return b200::bmm::g_batched_launches.load(std::memory_order_relaxed);
}

const char* b200_batched_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_BATCHED_VARIANT == 0
