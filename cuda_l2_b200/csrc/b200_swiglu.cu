// libb200_swiglu.so — the Gated<> kernels (hgemm_sm90.cuh) of every configuration with a gated kernel, and the SwiGLU
// backward, behind the internal entry points of b200_swiglu.h. A library of its own, so that the device code of the
// other libraries stays as it is. build.py compiles this file once per variant (-DB200_VARIANT = 0 or 2), in parallel;
// the object of variant 0 also holds the entry points and the backward kernel.
#include "b200_swiglu.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"
#include "swiglu_backward.cuh"

#ifndef B200_VARIANT
#error "compile once per variant with -DB200_VARIANT=0 or 2"
#endif

namespace b200 {
extern template B200_RUN(host::GemmType::kF16Acc32, Gated);
extern template B200_RUN(host::GemmType::kBF16, Gated);
template B200_RUN(host::GemmType(B200_VARIANT), Gated);
}  // namespace b200

#if B200_VARIANT == 0

namespace b200 {
namespace swiglu {

// dh = swiglu_grad(dy, h) over all M rows, M * I / 8 vectors.
template <typename T>
__global__ void __launch_bounds__(kBwdThreads) swiglu_backward_kernel(const T* __restrict__ dy, const T* __restrict__ h,
                                                                       T* __restrict__ dh, long long vectors, int I) {
  backward_vectors(dy, h, dh, vectors, I);
}

// The argument rules shared by the forward entry points, before any CUDA call.
int validate(int variant, const void* x, const void* w, const void* h, const void* y, int M, int I, int K) {
  if (variant != int(host::GemmType::kF16Acc32) && variant != int(host::GemmType::kBF16)) return kSwigluBadDtype;
  if (!x || !w || !y) return host::kNullPointer;
  if (M <= 0 || I <= 0 || K <= 0) return host::kBadShape;
  if (I % 64) return kSwigluBadWidth;
  if (K % 8 || ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(h) |
                 reinterpret_cast<uintptr_t>(y)) & 15))
    return host::kBadAlignment;
  if (2LL * I > 0x7fffffffLL) return host::kBadShape;
  return host::kOk;
}

// The TN choice for (M, 2I, K) mapped to its gated sibling, on the plain schedule (gated::kModes).
dispatch::Choice select(int variant, int M, int I, int K) {
  dispatch::Choice ch = dispatch::select(host::GemmType(variant), M, 2 * I, K);
  ch.config_id = gated::sibling(ch.config_id);
  ch.splits = 1;
  return ch;
}

// Configuration `config_id` of `variant` wrapped in Gated<>: h (may be null) and y, N = 2I. A configuration without a
// gated kernel is kBadConfig.
int run(int variant, int config_id, const void* x, const void* w, void* h, void* y, int M, int I, int K, int group_m,
        int splits, int max_ctas, void* stream) {
  host::EpiOperands op;
  op.y = y;
  if (variant == int(host::GemmType::kBF16))
    return run_config<host::GemmType::kBF16, Gated>(config_id, x, w, h, M, 2 * I, K, group_m, max_ctas, splits, stream,
                                                    op);
  return run_config<host::GemmType::kF16Acc32, Gated>(config_id, x, w, h, M, 2 * I, K, group_m, max_ctas, splits,
                                                      stream, op);
}

template <typename T>
int backward(const void* dy, const void* h, void* dh, int M, int I, cudaStream_t s) {
  const long long vectors = (long long)M * (I / 8);
  const int ctas = int(std::min<long long>((vectors + kBwdThreads - 1) / kBwdThreads, kBwdMaxCtas));
  swiglu_backward_kernel<T><<<ctas, kBwdThreads, 0, s>>>(static_cast<const T*>(dy), static_cast<const T*>(h),
                                                         static_cast<T*>(dh), vectors, I);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return int(e);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return host::kOk;
}

}  // namespace swiglu
}  // namespace b200

extern "C" {

int cuda_l2_b200_swiglu_run(int variant, const void* x, const void* w_gu, void* h, void* y, int M, int I, int K,
                            void* stream) {
  using namespace b200;
  if (const int st = swiglu::validate(variant, x, w_gu, h, y, M, I, K)) return st;
  const dispatch::Choice ch = swiglu::select(variant, M, I, K);
  return swiglu::run(variant, ch.config_id, x, w_gu, h, y, M, I, K, ch.group_m, ch.splits, 0, stream);
}

int cuda_l2_b200_swiglu_run_config(int variant, int config_id, const void* x, const void* w_gu, void* h, void* y, int M,
                                   int I, int K, int group_m, int splits, int max_ctas, void* stream) {
  using namespace b200;
  if (const int st = swiglu::validate(variant, x, w_gu, h, y, M, I, K)) return st;
  return swiglu::run(variant, config_id, x, w_gu, h, y, M, I, K, group_m, splits, max_ctas, stream);
}

int cuda_l2_b200_swiglu_select(int variant, int M, int I, int K, int* config_id, int* group_m, int* splits) {
  using namespace b200;
  if (variant != int(host::GemmType::kF16Acc32) && variant != int(host::GemmType::kBF16)) return kSwigluBadDtype;
  if (M <= 0 || I <= 0 || K <= 0 || 2LL * I > 0x7fffffffLL) return host::kBadShape;
  if (I % 64) return kSwigluBadWidth;
  const dispatch::Choice ch = swiglu::select(variant, M, I, K);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  if (splits) *splits = ch.splits;
  return host::kOk;
}

int cuda_l2_b200_swiglu_backward(int variant, const void* dy, const void* h, void* dh, int M, int I, void* stream) {
  using namespace b200;
  if (variant != int(host::GemmType::kF16Acc32) && variant != int(host::GemmType::kBF16)) return kSwigluBadDtype;
  if (!dy || !h || !dh) return host::kNullPointer;
  if (M < 0 || I <= 0 || 2LL * I > 0x7fffffffLL) return host::kBadShape;
  if (I % 64) return kSwigluBadWidth;
  if ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(dh)) & 15)
    return host::kBadAlignment;
  if (M == 0) return host::kOk;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  return variant == int(host::GemmType::kBF16) ? swiglu::backward<__nv_bfloat16>(dy, h, dh, M, I, s)
                                               : swiglu::backward<__half>(dy, h, dh, M, I, s);
}

unsigned long long cuda_l2_b200_swiglu_launch_count(void) { return b200::g_launches.load(std::memory_order_relaxed); }

const char* cuda_l2_b200_swiglu_strerror(int status) {
  switch (status) {
    case kSwigluBadWidth: return "the intermediate size I must be a multiple of 64 (whole 64-row gate / up blocks)";
    case kSwigluBadDtype: return "variant must be 0 (fp16) or 2 (bf16), with fp32 accumulation";
    default: return b200::host::status_string(status);
  }
}

}  // extern "C"

#endif  // B200_VARIANT == 0
