// The family of kernel configurations compiled into libb200_hgemm.so and referenced by the
// generated per-shape translation units (kernels/b200_*/<M>_<N>_<K>.cu).
//   X(id, BN, STAGES, CTA_GROUP, CLUSTER_M, CLUSTER_N, M_REP)
// STAGES is the requested ring depth; Config caps it at what fits the 227 KB of shared memory next to the 16 KB
// epilogue staging area (every CTA of a pair holds the whole B tile, so pairs with BN >= 128 run shallower rings).
// CTA_GROUP = 2: two CTAs of a cluster on adjacent 128-row tiles that multicast their shared B tile.
// M_REP = 2: 256 rows per CTA (two wgmmas per k-step sharing the B tile): config 26 is a 512 x 128 tile per CTA pair,
// 27 / 28 two such pairs sharing B / A by multicast. Register accumulators limit these to BN = 128.
// 29 / 30: four CTA pairs in a 2 x 2 multicast cluster (8 CTAs: both operands fetched from L2 once per two pairs).
// CLUSTER_M x CLUSTER_N > 1: TMA-multicast clusters of groups (single CTAs or CTA pairs): A shared along N, B along M.
#pragma once
#include <atomic>
#include <type_traits>

#include "hgemm_host.cuh"

#define B200_HGEMM_CONFIGS(X) \
  X(0, 256, 4, 1, 1, 1, 1)       \
  X(1, 128, 6, 1, 1, 1, 1)       \
  X(2, 64, 8, 1, 1, 1, 1)        \
  X(3, 256, 6, 2, 1, 1, 1)       \
  X(4, 128, 8, 2, 1, 1, 1)       \
  X(5, 192, 4, 1, 1, 1, 1)       \
  X(6, 192, 6, 2, 1, 1, 1)       \
  X(7, 64, 8, 1, 1, 2, 1)        \
  X(8, 64, 8, 1, 1, 4, 1)        \
  X(9, 64, 8, 1, 2, 2, 1)        \
  X(10, 128, 6, 1, 1, 2, 1)      \
  X(11, 128, 6, 1, 2, 2, 1)      \
  X(12, 32, 9, 1, 1, 1, 1)       \
  X(13, 32, 9, 1, 1, 4, 1)       \
  X(14, 32, 9, 1, 1, 8, 1)       \
  X(15, 64, 8, 1, 2, 1, 1)       \
  X(16, 64, 8, 1, 4, 1, 1)       \
  X(17, 128, 6, 1, 2, 1, 1)      \
  X(18, 256, 4, 1, 1, 2, 1)      \
  X(19, 256, 4, 1, 2, 1, 1)      \
  X(20, 256, 6, 2, 1, 2, 1)      \
  X(21, 256, 6, 2, 2, 1, 1)      \
  X(22, 128, 8, 2, 1, 2, 1)      \
  X(23, 128, 8, 2, 2, 1, 1)      \
  X(24, 192, 6, 2, 1, 2, 1)      \
  X(25, 192, 6, 2, 2, 1, 1)     \
  X(26, 128, 4, 2, 1, 1, 2)      \
  X(27, 128, 4, 2, 2, 1, 2)      \
  X(28, 128, 4, 2, 1, 2, 2)      \
  X(29, 256, 6, 2, 2, 2, 1)      \
  X(30, 128, 8, 2, 2, 2, 1)

namespace b200 {
constexpr int kNumConfigs = 31;

// What the host needs to know about a configuration, as Config<> derives it: tile and ring shape, cluster layout, and
// which K-decompositions its kernels carry. The accumulator and operand type change none of these.
struct ConfigDesc {
  int bn, stages, stages_requested, cta_group, cluster_m, cluster_n, m_rep;
  bool split_k, stream_k;
};
template <class Cfg>
constexpr ConfigDesc describe(int stages_requested) {
  return ConfigDesc{Cfg::BN, Cfg::STAGES, stages_requested, Cfg::CTA_GROUP, Cfg::CLUSTER_M, Cfg::CLUSTER_N, Cfg::M_REP,
                    Cfg::SPLIT_K, Cfg::STREAM_K};
}
constexpr ConfigDesc kConfigs[kNumConfigs] = {
#define B200_DESC(ID, BN, STAGES, CG, CM, CN, MR) describe<Config<BN, STAGES, CG, true, CM, CN, MR>>(STAGES),
    B200_HGEMM_CONFIGS(B200_DESC)
#undef B200_DESC
};

// The block-scaled configurations (libb200_fp8block.so, libb200_batched_fp8.so, libb200_grouped_fp8.so). Host code:
// the three libraries map the dispatcher's choice through the same rule.
namespace block {

// Two accumulator sets (the running sum and the k-block's wgmma target) fit the registers for M_REP * BN <= 128.
constexpr bool eligible(int id) { return kConfigs[id].m_rep * kConfigs[id].bn <= 128; }

// The block-scaled stand-in of configuration `id`: the same CTA group and cluster, M_REP = 1, BN = min(BN, 128).
constexpr int sibling(int id) {
  const ConfigDesc& c = kConfigs[id];
  const int bn = c.bn < 128 ? c.bn : 128;
  for (int j = 0; j < kNumConfigs; ++j) {
    const ConfigDesc& d = kConfigs[j];
    if (d.cta_group == c.cta_group && d.cluster_m == c.cluster_m && d.cluster_n == c.cluster_n && d.m_rep == 1 &&
        d.bn == bn)
      return j;
  }
  return -1;
}
constexpr bool every_config_has_an_eligible_sibling() {
  for (int id = 0; id < kNumConfigs; ++id) {
    const int s = sibling(id);
    if (s < 0 || !eligible(s) || (eligible(id) && s != id)) return false;
  }
  return true;
}
static_assert(every_config_has_an_eligible_sibling(), "the configuration table lost a block-scaled sibling");

// Workspace split-K and stream-K are not compiled for the block-scaled kernels: plan() runs such requests plain.
constexpr unsigned kModes = (1u << kPlain) | (1u << kClusterSplitK);

}  // namespace block

// The row-major B (NN) configurations (libb200_nn.so, RowMajorB<>). Host code: libb200_hgemm.so maps the dispatcher's
// choice through this rule before it calls the NN library.
namespace nn {

// An MN-major B stage is whole 64-column atom columns: every configuration but the BN = 32 ones has an NN kernel.
constexpr bool has_kernel(int id) { return kConfigs[id].bn % 64 == 0; }

// The NN stand-in of configuration `id`: itself if it has an NN kernel; otherwise the BN = 64 configuration with the
// same CTA group, cluster_m and M_REP and the widest cluster_n up to its own (the same cluster where there is one).
constexpr int sibling(int id) {
  const ConfigDesc& c = kConfigs[id];
  if (has_kernel(id)) return id;
  int best = -1;
  for (int j = 0; j < kNumConfigs; ++j) {
    const ConfigDesc& d = kConfigs[j];
    if (d.bn == 64 && d.cta_group == c.cta_group && d.cluster_m == c.cluster_m && d.m_rep == c.m_rep &&
        d.cluster_n <= c.cluster_n && (best < 0 || d.cluster_n > kConfigs[best].cluster_n))
      best = j;
  }
  return best;
}
constexpr bool every_config_has_a_sibling() {
  for (int id = 0; id < kNumConfigs; ++id) {
    const int s = sibling(id);
    if (s < 0 || !has_kernel(s) || (has_kernel(id) && s != id)) return false;
  }
  return true;
}
static_assert(every_config_has_a_sibling(), "the configuration table lost a row-major B sibling");

}  // namespace nn

// The SwiGLU configurations (libb200_swiglu.so, Gated<>). Host code: the library maps the dispatcher's TN choice through
// this rule.
namespace gated {

// A gate / up pair is two 64-column chunks of one tile: BN = 128 and 256 have a gated kernel.
constexpr bool has_kernel(int id) { return kConfigs[id].bn == 128 || kConfigs[id].bn == 256; }

// The gated stand-in of configuration `id`: itself if it has a gated kernel; otherwise (BN = 32, 64, 192) the BN = 128
// configuration with the same CTA group and M_REP and the largest cluster no wider in M or N than its own.
constexpr int sibling(int id) {
  const ConfigDesc& c = kConfigs[id];
  if (has_kernel(id)) return id;
  int best = -1;
  for (int j = 0; j < kNumConfigs; ++j) {
    const ConfigDesc& d = kConfigs[j];
    if (d.bn == 128 && d.cta_group == c.cta_group && d.m_rep == c.m_rep && d.cluster_m <= c.cluster_m &&
        d.cluster_n <= c.cluster_n &&
        (best < 0 || d.cluster_m * d.cluster_n > kConfigs[best].cluster_m * kConfigs[best].cluster_n))
      best = j;
  }
  return best;
}
constexpr bool every_config_has_a_sibling() {
  for (int id = 0; id < kNumConfigs; ++id) {
    const int s = sibling(id);
    if (s < 0 || !has_kernel(s) || (has_kernel(id) && s != id)) return false;
  }
  return true;
}
static_assert(every_config_has_a_sibling(), "the configuration table lost a SwiGLU sibling");

// Only the plain schedule is compiled for the gated kernels: plan() runs split-K and stream-K requests plain.
constexpr unsigned kModes = 1u << kPlain;

}  // namespace gated

// What the kernels of a configuration wrapper cover, read from Probe, the wrapper's type of configuration 1 (BN = 128,
// one CTA, no cluster), which every wrapper compiles: block-scaled kernels exist for the block::eligible
// configurations and carry block::kModes, row-major B ones exist for the nn::has_kernel configurations, gated ones for
// the gated::has_kernel configurations with gated::kModes; every other wrapper has every configuration in every K-mode.
template <class Probe>
constexpr bool has_kernel(int id) {
  return block_scaled<Probe>() ? block::eligible(id)
         : row_major_b<Probe>() ? nn::has_kernel(id)
         : is_gated<Probe>()    ? gated::has_kernel(id)
                                : true;
}
template <class Probe>
constexpr unsigned k_modes() { return block_scaled<Probe>() ? block::kModes : is_gated<Probe>() ? gated::kModes : 0xFu; }

// The wrapper of the TN, per-tensor and rowwise configurations: none.
template <class Cfg>
using Unwrapped = Cfg;

// Kernel launches the library has issued (b200_hgemm_launch_count, b200_fp8block_launch_count). One counter for every
// translation unit of the library; hidden, so that no other shared object's copy is bound to it.
__attribute__((visibility("hidden"))) inline std::atomic<unsigned long long> g_launches{0};

// Launch configuration `id` of variant T in Wrapper (Unwrapped, BlockScaled, BlockScaled1D1D, RowMajorB, BiasAct,
// AccumF32 or Gated), with the epilogue operands and the split-K scratch source of host::launch. A configuration
// without a kernel is kBadConfig. An instantiation compiles the kernels of all configurations for T, so each translation
// unit of a library instantiates only the variants it exports (B200_RUN).
template <host::GemmType T, template <class> class Wrapper = Unwrapped>
int run_config(int id, const void* A, const void* Bt, void* C, int M, int N, int K, int group_m, int max_ctas,
               int splits, void* stream, const host::EpiOperands& op = {},
               host::ScratchFn scratch = host::splitk_scratch) {
  constexpr host::GemmTypeTraits t = host::traits(T);
  using Probe = Wrapper<Config<128, 6, 1, t.acc_f32, 1, 1, 1, t.bf16(), t.e4m3()>>;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int st = host::kBadConfig;
  switch (id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                  \
  case ID:                                                                                                     \
    if constexpr (has_kernel<Probe>(ID))                                                                       \
      st = host::launch<Wrapper<Config<BN, STAGES, CG, t.acc_f32, CM, CN, MR, t.bf16(), t.e4m3()>>,            \
                        k_modes<Probe>()>(A, Bt, C, M, N, K, s, group_m, max_ctas, splits, op, scratch);   \
    break;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      break;
  }
  if (st == host::kOk) g_launches.fetch_add(1, std::memory_order_relaxed);
  return st;
}

// The explicit instantiation of run_config<T, W>: a library compiled once per variant declares the other objects'
// `extern template B200_RUN(T, W);` and instantiates its own with `template B200_RUN(T, W);`.
#define B200_RUN(T, W)                                                                                        \
  int run_config<T, W>(int, const void*, const void*, void*, int, int, int, int, int, int, void*,              \
                       const host::EpiOperands&, host::ScratchFn)

// The tile-list libraries (libb200_batched.so, libb200_grouped.so): the 16-bit variants 0, 1, 2 (the GemmType index) of
// every configuration, wrapped in Wrapper (Batched or Grouped), launched by host::launch_list. libb200_batched_fp8.so,
// libb200_grouped_fp8.so: the block-scaled e4m3 variants 5, 6 of the block-scaled configurations,
// Wrapper<BlockScaled<...>>, with their scales. libb200_grouped_bwd.so: variants 0 and 2 of the configurations with a
// row-major B kernel, wrapped in Grouped<RowMajorB<>> or GroupedK<RowMajorB<>>. libb200_wgrad_accum.so:
// AccumF32<GroupedK<RowMajorB<>>>. libb200_grouped_swiglu.so: the gated configurations in Gated<Grouped<>>.
namespace tile_list {

// The C entry points' selectors: a block-scaled library's `out_bf16` (0: fp16, 1: bf16 output) names GemmType
// 5 + out_bf16, and its scales arrive as untyped pointers (block_operands: with the row stride of A's); the other
// libraries' `variant` is the GemmType index.
inline bool known_out(int out_bf16) { return out_bf16 == 0 || out_bf16 == 1; }
inline host::GemmType block_type(int out_bf16) { return host::GemmType(int(host::GemmType::kE4M3F16Block) + out_bf16); }
inline host::EpiOperands block_operands(const void* a, int ld_a, const void* b) {
  return {Scales{static_cast<const float*>(a), static_cast<const float*>(b)}, ld_a};
}

// Kernel launches of the library that holds it (b200_batched_launch_count, b200_grouped_launch_count,
// b200_batched_fp8_launch_count, b200_grouped_fp8_launch_count, cuda_l2_b200_grouped_bwd_launch_count): one counter
// for the library's objects; hidden, like g_launches.
__attribute__((visibility("hidden"))) inline std::atomic<unsigned long long> g_list_launches{0};

// The configuration Cfg of variant T in a tile-list library: a block-scaled variant's configurations are BlockScaled<>.
template <host::GemmType T, class Cfg>
using Variant = std::conditional_t<host::traits(T).block, BlockScaled<Cfg>, Cfg>;

// A configuration without a kernel of Wrapper and T (has_kernel) returns kBadConfig.
template <template <class> class Wrapper, host::GemmType T>
int run_config(int id, const void* A, const void* Bt, void* C, const int* list, int count, int rows, int N, int K,
               int group_m, int max_ctas, cudaStream_t s, const host::EpiOperands& op) {
  constexpr host::GemmTypeTraits t = host::traits(T);
  static_assert(!t.scaled || t.block, "16-bit or block-scaled variants");
  using Probe = Wrapper<Variant<T, Config<128, 6, 1, t.acc_f32, 1, 1, 1, t.bf16(), t.e4m3()>>>;
  int st = host::kBadConfig;
  switch (id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                  \
  case ID:                                                                                                     \
    if constexpr (has_kernel<Probe>(ID))                                                                       \
      st = host::launch_list<Wrapper<Variant<T, Config<BN, STAGES, CG, t.acc_f32, CM, CN, MR, t.bf16(), t.e4m3()>>>>( \
          A, Bt, C, list, count, rows, N, K, s, group_m, max_ctas, op);                                        \
    break;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      break;
  }
  // no launch for an empty problem: no rows, or no reduction (the K-grouped T == 0, which only zero-fills C)
  if (st == host::kOk && rows > 0 && K > 0) g_list_launches.fetch_add(1, std::memory_order_relaxed);
  return st;
}

// A tile-list library: its wrapper (Batched, Grouped, or a row-major B alias) and its variants, the tag that run() and
// gemm() take.
template <template <class> class Wrapper, host::GemmType... Types>
struct ListLibrary {};

// Whether `variant` (a GemmType index) is one of the library's.
template <template <class> class Wrapper, host::GemmType... Types>
constexpr bool holds(ListLibrary<Wrapper, Types...>, int variant) {
  return ((variant == int(Types)) || ...);
}

// The wrapper's fp16 configuration 1 (BN = 128, one CTA, no cluster), which every tile-list wrapper compiles: what
// does not depend on the variant (the kind of list, has_kernel of the 16-bit variants) is read from it.
template <template <class> class Wrapper>
using ListProbe = Wrapper<Config<128, 6, 1, true>>;

// The variants of each kind of tile-list library, listed once as X(W, T): the 16-bit libraries hold variants 0, 1, 2
// (the GemmType index), the block-scaled e4m3 ones 5, 6.
#define B200_LIST_TYPES(X, W) X(W, host::GemmType::kF16Acc32) X(W, host::GemmType::kF16Acc16) X(W, host::GemmType::kBF16)
#define B200_BLOCK_LIST_TYPES(X, W) X(W, host::GemmType::kE4M3F16Block) X(W, host::GemmType::kE4M3BF16Block)

// A library compiles its source once per variant (-DB200_VARIANT), in parallel: each object instantiates its own
// variant's kernels, and the calls of the other objects' variants link against theirs. B200_LIST_OBJECT(NAME, W, TYPES)
// declares this and names the library NAME (W and the variants of TYPES), so that run() can launch no other variant's
// kernels. The first variant's object also holds the C entry points.
#define B200_LIST_RUN(W, T)                                                                                    \
  int run_config<W, T>(int, const void*, const void*, void*, const int*, int, int, int, int, int, int, cudaStream_t, \
                       const host::EpiOperands&)
#define B200_LIST_EXTERN(W, T) extern template B200_LIST_RUN(W, T);
#define B200_LIST_ARG(W, T) , T
#define B200_LIST_OBJECT(NAME, W, TYPES)                                                                       \
  TYPES(B200_LIST_EXTERN, W)                                                                                   \
  template B200_LIST_RUN(W, host::GemmType(B200_VARIANT));                                                     \
  using NAME = ListLibrary<W TYPES(B200_LIST_ARG, W)>

// Configuration `config_id` of variant `type`, with the epilogue operands of host::launch_list (a block-scaled
// variant's scales and ld_a, Gated<Grouped<>>'s y). A variant that is not the library's own is kBadConfig.
template <template <class> class Wrapper, host::GemmType... Types>
int run(ListLibrary<Wrapper, Types...>, host::GemmType type, int config_id, const void* A, const void* Bt, void* C,
        const int* list, int count, int rows, int N, int K, int group_m, int max_ctas, void* stream,
        const host::EpiOperands& op = {}) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int st = host::kBadConfig;
  (void)((type == Types && (st = run_config<Wrapper, Types>(config_id, A, Bt, C, list, count, rows, N, K, group_m,
                                                            max_ctas, s, op), true)) || ...);
  return st;
}

// Host view of worker `worker`'s tiles, with the launcher's plan on a device of num_sms SMs (every cluster resident)
// and its default group_m: (index, m_block, n_block) per tile into `units` (at most max_units), and for a K-grouped
// configuration a fourth value, the tile's k-blocks; returns the count.
template <class Cfg>
int schedule_units(int count, int rows, int N, int K, const int* list, int num_sms, int worker, int* units,
                   int max_units, int* num_workers) {
  const long long tiles = Cfg::Cursor::template max_tiles<Cfg>(count, rows, N);
  if (tiles > 0x7fffffffLL) return host::kBadShape;
  const int max_workers = num_sms / Cfg::CLUSTER_CTAS;
  const host::Plan p = host::list_plan<Cfg>(tiles, K, max_workers, [=] { return max_workers; });
  if (num_workers) *num_workers = p.workers;
  if (worker < 0 || worker >= p.workers) return host::kBadShape;
  const int n_blocks = (N + Cfg::BN * Cfg::CLUSTER_N - 1) / (Cfg::BN * Cfg::CLUSTER_N);
  typename Cfg::Cursor cursor = make_cursor<Cfg>(list, count, rows, K, Cfg::TILE_M * Cfg::CLUSTER_M, n_blocks,
                                                 host::default_group_m<Cfg>());
  constexpr int kInts = k_grouped<Cfg>() ? 4 : 3;
  WorkIter it(worker, p.workers, cursor.total(), p.nkb, 1, 0);
  WorkUnit u;
  int n = 0;
  while (it.next(u)) {
    BatchTile bt;
    if constexpr (k_grouped<Cfg>()) bt = cursor.unit(u);   // bounds u's k-range to the tile's group
    else bt = cursor.locate(u.tile);
    if (n < max_units && units) {
      int* v = units + kInts * n;
      v[0] = bt.batch; v[1] = bt.tc.m_blk; v[2] = bt.tc.n_blk;
      if constexpr (k_grouped<Cfg>()) v[3] = u.kb1 - u.kb0;
    }
    ++n;
  }
  return n;
}

// The shortest worst-case tile list (Cursor::max_tiles) of any configuration with a kernel (block_only: of any
// block::eligible one). When it passes INT_MAX, every configuration refuses the shape, so the dispatched call refuses
// it before the lookup.
template <template <class> class Wrapper>
long long fewest_tiles(int count, int rows, int N, bool block_only = false) {
  long long fewest = 0x7fffffffffffffffLL;
#define B200_TILES(ID, BN, STAGES, CG, CM, CN, MR)                                                               \
  if constexpr (has_kernel<ListProbe<Wrapper>>(ID)) {                                                           \
    using W = Wrapper<Config<BN, STAGES, CG, true, CM, CN, MR>>;                                                \
    if (!block_only || block::eligible(ID))                                                                     \
      fewest = std::min(fewest, W::Cursor::template max_tiles<W>(count, rows, N));                              \
  }
  B200_HGEMM_CONFIGS(B200_TILES)
#undef B200_TILES
  return fewest;
}

// The same for configuration `config_id` (fp32-accumulating fp16: the schedule does not depend on the variant). A
// configuration without a kernel is kBadConfig.
template <template <class> class Wrapper>
int schedule_config(int config_id, int count, int rows, int N, int K, const int* list, int num_sms, int worker,
                    int* units, int max_units, int* num_workers) {
  switch (config_id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                 \
  case ID:                                                                                                      \
    if constexpr (has_kernel<ListProbe<Wrapper>>(ID))                                                           \
      return schedule_units<Wrapper<Config<BN, STAGES, CG, true, CM, CN, MR>>>(count, rows, N, K, list, num_sms, \
                                                                               worker, units, max_units,        \
                                                                               num_workers);                    \
    break;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      break;
  }
  return host::kBadConfig;
}

}  // namespace tile_list
}  // namespace b200
