// libb200_wgrad_accum.so — the AccumF32<> kernels (hgemm_sm90.cuh) behind the internal entry points of
// b200_wgrad_accum.h: AccumF32<GroupedK<RowMajorB<>>> of every configuration with a row-major B kernel (fp16 and bf16,
// launched through tile_list like libb200_grouped_bwd.so), AccumF32<> of the 2-D e4m3 configurations in every K-mode
// (rowwise scales, as libb200_hgemm.so's), and AccumF32<BlockScaled1D1D<>> of the block-scaled ones (as
// libb200_fp8block_1d1d.so's). The output type is fp32 whatever the 16-bit flavour, so each e4m3 family is compiled
// once (its fp16-output Config<>). A library of its own, so that the device code of the other libraries stays as it
// is. build.py compiles this file once per family (-DB200_VARIANT = 0, 2: the K-grouped fp16 / bf16 kernels; 3: the
// rowwise e4m3 ones; 7: the 1 x 128 ones), in parallel; the object of variant 0 also holds the entry points.
#include "b200_wgrad_accum.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_VARIANT
#error "compile once per kernel family with -DB200_VARIANT=0, 2, 3 or 7"
#endif

namespace b200 {

template <class Cfg>
using Accum1D1D = AccumF32<BlockScaled1D1D<Cfg>>;

extern template B200_RUN(host::GemmType::kE4M3F16, AccumF32);
extern template B200_RUN(host::GemmType::kE4M3F16Block1D1D, Accum1D1D);
#if B200_VARIANT == 3
template B200_RUN(host::GemmType::kE4M3F16, AccumF32);
#elif B200_VARIANT == 7
template B200_RUN(host::GemmType::kE4M3F16Block1D1D, Accum1D1D);
#endif

namespace tile_list {

template <class Cfg>
using AccumGroupedK = AccumF32<GroupedK<RowMajorB<Cfg>>>;

B200_LIST_EXTERN(AccumGroupedK, host::GemmType::kF16Acc32)
B200_LIST_EXTERN(AccumGroupedK, host::GemmType::kBF16)
#if B200_VARIANT == 0 || B200_VARIANT == 2
template B200_LIST_RUN(AccumGroupedK, host::GemmType(B200_VARIANT));
#endif
using AccumWgradLibrary = ListLibrary<AccumGroupedK, host::GemmType::kF16Acc32, host::GemmType::kBF16>;

}  // namespace tile_list
}  // namespace b200

#if B200_VARIANT == 0

namespace {

using b200::host::GemmType;

constexpr int kFormRowwise = 1, kForm1D1D = 3;   // the scale forms with an accumulating kernel

// The dispatched choice of the wrapped library for `form` (a known one).
b200::dispatch::Choice fp8_select(int form, int M, int N, int K) {
  return form == kFormRowwise ? b200::dispatch::select(GemmType::kE4M3F16, M, N, K) : b200::block::select(M, N, K);
}

// The epilogue operands of `form`: rowwise scales, or 1 x 128 scales of both operands with their row strides.
b200::host::EpiOperands operands(int form, const void* scale_a, int ld_a, const void* scale_b, int ld_b) {
  const b200::Scales sc{static_cast<const float*>(scale_a), static_cast<const float*>(scale_b), form == kFormRowwise};
  if (form == kFormRowwise) return {sc};
  return {sc, ld_a, ld_b};
}

// Split-K scratch comes from this library's own pool (host::splitk_scratch, run_config's default).
int run_fp8(int form, int config_id, const void* A, const void* Bt, float* C32, const b200::host::EpiOperands& op,
            int M, int N, int K, int group_m, int max_ctas, int splits, void* stream) {
  using namespace b200;
  if (form == kFormRowwise)
    return run_config<GemmType::kE4M3F16, AccumF32>(config_id, A, Bt, C32, M, N, K, group_m, max_ctas, splits, stream,
                                                    op);
  return run_config<GemmType::kE4M3F16Block1D1D, Accum1D1D>(config_id, A, Bt, C32, M, N, K, group_m, max_ctas, splits,
                                                            stream, op);
}

}  // namespace

extern "C" {

int cuda_l2_b200_wgrad_accum_grouped(int variant, int config_id, const void* A, const void* B, float* C32,
                                     const int* offs, int G, int T, int M, int N, int group_m, int max_ctas,
                                     void* stream) {
  using namespace b200;
  const tile_list::AccumWgradLibrary lib;
  if (!tile_list::holds(lib, variant)) return host::kBadConfig;
  if (config_id < 0) return tile_list::gemm(lib, GemmType(variant), A, B, C32, offs, G, M, N, T, stream);
  return tile_list::run(lib, GemmType(variant), config_id, A, B, C32, offs, G, M, N, T, group_m, max_ctas, stream);
}

int cuda_l2_b200_wgrad_accum_fp8(int form, int config_id, const void* A, const void* B_kmajor, float* C32,
                                 const void* scale_a, int ld_a, const void* scale_b, int ld_b, int M, int N, int K,
                                 int group_m, int max_ctas, int splits, void* stream) {
  using namespace b200;
  if (form != kFormRowwise && form != kForm1D1D) return host::kBadConfig;
  const host::EpiOperands op = operands(form, scale_a, ld_a, scale_b, ld_b);
  if (config_id < 0) {
    // the argument rules before the lookup, which wants a valid shape
    const GemmType type = form == kFormRowwise ? GemmType::kE4M3F16 : GemmType::kE4M3F16Block1D1D;
    if (const int st = host::validate(type, A, B_kmajor, C32, op, M, N, K)) return st;
    if (form == kForm1D1D && (ld_b < N || ld_b % 4)) return host::kBadScaleLdB;
    const dispatch::Choice ch = fp8_select(form, M, N, K);
    config_id = ch.config_id;
    group_m = ch.group_m;
    max_ctas = 0;
    splits = ch.splits;
  }
  return run_fp8(form, config_id, A, B_kmajor, C32, op, M, N, K, group_m, max_ctas, splits, stream);
}

int cuda_l2_b200_wgrad_accum_grouped_select(int variant, int G, int T, int M, int N, int* config_id, int* group_m) {
  using namespace b200;
  if (!tile_list::holds(tile_list::AccumWgradLibrary{}, variant)) return host::kBadConfig;
  return tile_list::select_into<tile_list::AccumGroupedK>(GemmType(variant), G, M, N, T, config_id, group_m);
}

int cuda_l2_b200_wgrad_accum_fp8_select(int form, int M, int N, int K, int* config_id, int* group_m, int* splits) {
  using namespace b200;
  if (form != kFormRowwise && form != kForm1D1D) return host::kBadConfig;
  if (M <= 0 || N <= 0 || K <= 0) return host::kBadShape;
  const dispatch::Choice ch = fp8_select(form, M, N, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  if (splits) *splits = ch.splits;
  return host::kOk;
}

int cuda_l2_b200_wgrad_accum_prewarm(void* stream) {
  int dev = 0;
  const cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return int(e);
  b200::host::SplitKScratch* sk = nullptr;
  return b200::host::splitk_scratch(dev, static_cast<cudaStream_t>(stream), &sk);
}

int cuda_l2_b200_wgrad_accum_release(void) {
  b200::host::release_scratch();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : int(e);
}

unsigned long long cuda_l2_b200_wgrad_accum_launch_count(void) {
  return b200::g_launches.load(std::memory_order_relaxed) +
         b200::tile_list::g_list_launches.load(std::memory_order_relaxed);
}

const char* cuda_l2_b200_wgrad_accum_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_VARIANT == 0
