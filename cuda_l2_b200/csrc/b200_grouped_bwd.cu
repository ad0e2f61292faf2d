// libb200_grouped_bwd.so — the backward of the grouped 16-bit product (b200_grouped_bwd.h): Grouped<RowMajorB<>>
// (the input gradient) and GroupedK<RowMajorB<>> (the weight gradient) kernels of every configuration with a row-major
// B kernel (nn::has_kernel), launched by host::launch_list. A library of its own, so that the device code of the other
// libraries stays as it is. build.py compiles this file once per variant (-DB200_VARIANT = 0 or 2); the object of
// variant 0 also holds the entry points.
#include "b200_grouped_bwd.h"

#include <climits>

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_VARIANT
#error "compile once per variant with -DB200_VARIANT=0 or 2"
#endif

namespace b200 {
namespace grouped_bwd {

enum Kind : int { kNN = 0, kWgrad = 1 };

// Kernel launches of the library (one counter for both objects; hidden, like g_launches).
__attribute__((visibility("hidden"))) inline std::atomic<unsigned long long> g_bwd_launches{0};

inline bool known_variant(int v) { return v == int(host::GemmType::kF16Acc32) || v == int(host::GemmType::kBF16); }

// Configuration `id` of variant T for `kind`: kNN over (count = G, rows = T, N, K), kWgrad over (count = G, rows = M,
// N, K = T). A configuration without a row-major B kernel is kBadConfig.
template <host::GemmType T>
int run_config(int kind, int id, const void* A, const void* B, void* C, const int* offs, int count, int rows, int N,
               int K, int group_m, int max_ctas, cudaStream_t s) {
  constexpr host::GemmTypeTraits t = host::traits(T);
  static_assert(!t.scaled && t.acc_f32, "the backward kernels: 16-bit operands, fp32 accumulation");
  int st = host::kBadConfig;
  switch (id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                   \
  case ID:                                                                                                      \
    if constexpr (nn::has_kernel(ID)) {                                                                         \
      using Cfg = RowMajorB<Config<BN, STAGES, CG, true, CM, CN, MR, t.bf16()>>;                                \
      if (kind == kNN)                                                                                          \
        st = host::launch_list<Grouped<Cfg>>(A, B, C, offs, count, rows, N, K, s, group_m, max_ctas);           \
      else                                                                                                      \
        st = host::launch_list<GroupedK<Cfg>>(A, B, C, offs, count, rows, N, K, s, group_m, max_ctas);          \
    }                                                                                                           \
    break;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      break;
  }
  // no launch for an empty problem: no row of the input gradient, no row to reduce over for the weight gradient
  if (st == host::kOk && (kind == kNN ? rows : K) > 0) g_bwd_launches.fetch_add(1, std::memory_order_relaxed);
  return st;
}

#define B200_BWD_RUN(T)                                                                                          \
  int run_config<T>(int, int, const void*, const void*, void*, const int*, int, int, int, int, int, int, cudaStream_t)
extern template B200_BWD_RUN(host::GemmType::kF16Acc32);
extern template B200_BWD_RUN(host::GemmType::kBF16);
template B200_BWD_RUN(host::GemmType(B200_VARIANT));
#undef B200_BWD_RUN

}  // namespace grouped_bwd
}  // namespace b200

#if B200_VARIANT == 0

namespace b200 {
namespace grouped_bwd {

int run(int variant, int kind, int config_id, const void* A, const void* B, void* C, const int* offs, int count,
        int rows, int N, int K, int group_m, int max_ctas, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (variant == int(host::GemmType::kF16Acc32))
    return run_config<host::GemmType::kF16Acc32>(kind, config_id, A, B, C, offs, count, rows, N, K, group_m, max_ctas, s);
  if (variant == int(host::GemmType::kBF16))
    return run_config<host::GemmType::kBF16>(kind, config_id, A, B, C, offs, count, rows, N, K, group_m, max_ctas, s);
  return host::kBadConfig;
}

// The input gradient's choice: the grouped forward's rule for G groups over T rows with N output columns and a
// reduction over K, mapped to the row-major B sibling (there is no tuned table for either kind).
dispatch::Choice select_nn(host::GemmType type, int G, int T, int N, int K) {
  dispatch::Choice ch = tile_list::select<Grouped>(type, G, T, N, K);
  ch.config_id = nn::sibling(ch.config_id);
  ch.splits = 1;
  return ch;
}

// The weight gradient's choice: the batched rule for G matrices of M x N with the average group's ceil(T / G) rows
// (at least one) as the reduction, mapped to the row-major B sibling.
dispatch::Choice select_wgrad(host::GemmType type, int G, int T, int M, int N) {
  const int k = int(std::max<long long>(1, (T + (G - 1LL)) / G));
  dispatch::Choice ch = dispatch::select_batched(type, G, M, N, k);
  ch.config_id = nn::sibling(ch.config_id);
  ch.splits = 1;
  return ch;
}

// The K-grouped schedule of Cfg (fp32-accumulating fp16: the schedule does not depend on the variant), walked with
// the kernel's own cursor and work iterator.
template <class Cfg>
int wgrad_schedule(int G, int T, int M, int N, const int* offs, int num_sms, int worker, int* units, int max_units,
                   int* num_workers) {
  const long long tiles = Cfg::Cursor::template max_tiles<Cfg>(G, M, N);
  if (tiles > 0x7fffffffLL) return host::kBadShape;
  const int max_workers = num_sms / Cfg::CLUSTER_CTAS;
  const host::Plan p = host::list_plan<Cfg>(tiles, T, max_workers, [=] { return max_workers; });
  if (num_workers) *num_workers = p.workers;
  if (worker < 0 || worker >= p.workers) return host::kBadShape;
  const int n_blocks = (N + Cfg::BN * Cfg::CLUSTER_N - 1) / (Cfg::BN * Cfg::CLUSTER_N);
  typename Cfg::Cursor cursor = make_cursor<Cfg>(offs, G, M, T, Cfg::TILE_M * Cfg::CLUSTER_M, n_blocks,
                                                 host::default_group_m<Cfg>());
  WorkIter it(worker, p.workers, cursor.total(), p.nkb, 1, 0);
  WorkUnit u;
  int n = 0;
  while (it.next(u)) {
    const BatchTile bt = cursor.unit(u);
    if (n < max_units && units) {
      units[4 * n] = bt.batch; units[4 * n + 1] = bt.tc.m_blk; units[4 * n + 2] = bt.tc.n_blk;
      units[4 * n + 3] = u.kb1 - u.kb0;
    }
    ++n;
  }
  return n;
}

}  // namespace grouped_bwd
}  // namespace b200

using b200::host::GemmType;
namespace gb = b200::grouped_bwd;

extern "C" {

int cuda_l2_b200_grouped_bwd_nn(int variant, int config_id, const void* A, const void* B_rowmajor, void* C,
                                const int* offs, int G, int T, int N, int K, int group_m, int max_ctas, void* stream) {
  using namespace b200;
  if (!gb::known_variant(variant)) return host::kBadConfig;
  if (config_id < 0) {
    if (const int st = host::validate_grouped(GemmType(variant), A, B_rowmajor, C, offs, G, T, N, K, 1)) return st;
    if (T == 0) return host::kOk;
    const dispatch::Choice ch = gb::select_nn(GemmType(variant), G, T, N, K);
    config_id = ch.config_id; group_m = ch.group_m; max_ctas = 0;
  }
  return gb::run(variant, gb::kNN, config_id, A, B_rowmajor, C, offs, G, T, N, K, group_m, max_ctas, stream);
}

int cuda_l2_b200_grouped_bwd_wgrad(int variant, int config_id, const void* A, const void* B, void* C, const int* offs,
                                   int G, int T, int M, int N, int group_m, int max_ctas, void* stream) {
  using namespace b200;
  if (!gb::known_variant(variant)) return host::kBadConfig;
  if (config_id < 0) {
    if (const int st = host::validate_k_grouped(GemmType(variant), A, B, C, offs, G, T, M, N, 1)) return st;
    const dispatch::Choice ch = gb::select_wgrad(GemmType(variant), G, T, M, N);
    config_id = ch.config_id; group_m = ch.group_m; max_ctas = 0;
  }
  return gb::run(variant, gb::kWgrad, config_id, A, B, C, offs, G, M, N, T, group_m, max_ctas, stream);
}

int cuda_l2_b200_grouped_bwd_nn_select(int variant, int G, int T, int N, int K, int* config_id, int* group_m) {
  using namespace b200;
  if (!gb::known_variant(variant)) return host::kBadConfig;
  if (G <= 0 || T <= 0 || N <= 0 || K <= 0) return host::kBadShape;
  const dispatch::Choice ch = gb::select_nn(GemmType(variant), G, T, N, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  return host::kOk;
}

int cuda_l2_b200_grouped_bwd_wgrad_select(int variant, int G, int T, int M, int N, int* config_id, int* group_m) {
  using namespace b200;
  if (!gb::known_variant(variant)) return host::kBadConfig;
  if (G <= 0 || T < 0 || M <= 0 || N <= 0) return host::kBadShape;
  const dispatch::Choice ch = gb::select_wgrad(GemmType(variant), G, T, M, N);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  return host::kOk;
}

int cuda_l2_b200_grouped_bwd_wgrad_schedule(int config_id, int G, int T, int M, int N, const int* offs_host,
                                            int num_sms, int worker, int* units, int max_units, int* num_workers) {
  using namespace b200;
  if (G <= 0 || T < 0 || M <= 0 || N <= 0 || num_sms <= 0 || !offs_host) return host::kBadShape;
  switch (config_id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                  \
  case ID:                                                                                                     \
    if constexpr (nn::has_kernel(ID))                                                                          \
      return gb::wgrad_schedule<GroupedK<RowMajorB<Config<BN, STAGES, CG, true, CM, CN, MR>>>>(                \
          G, T, M, N, offs_host, num_sms, worker, units, max_units, num_workers);                               \
    return host::kBadConfig;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      return host::kBadConfig;
  }
}

unsigned long long cuda_l2_b200_grouped_bwd_launch_count(void) {
  return gb::g_bwd_launches.load(std::memory_order_relaxed);
}

const char* cuda_l2_b200_grouped_bwd_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_VARIANT == 0
