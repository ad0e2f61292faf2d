// libb200_swiglu.so — the Gated<> kernels (hgemm_sm90.cuh) of every configuration with a gated kernel, and the SwiGLU
// backward, behind the internal entry points of b200_swiglu.h. A library of its own, so that the device code of the
// other libraries stays as it is. build.py compiles this file once per variant (-DB200_VARIANT = 0 or 2), in parallel;
// the object of variant 0 also holds the entry points and the backward kernel.
#include "b200_swiglu.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"
#include "swiglu_arith.cuh"

#ifndef B200_VARIANT
#error "compile once per variant with -DB200_VARIANT=0 or 2"
#endif

namespace b200 {
namespace swiglu {

// Configuration `id` of variant T wrapped in Gated<>: h (C, may be null) and y, N = 2I. A configuration without a
// gated kernel is kBadConfig.
template <host::GemmType T>
int run_config(int id, const void* x, const void* w, void* h, void* y, int M, int N, int K, int group_m, int max_ctas,
               int splits, void* stream) {
  constexpr host::GemmTypeTraits t = host::traits(T);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int st = host::kBadConfig;
  switch (id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                  \
  case ID:                                                                                                     \
    if constexpr (gated::has_kernel(ID))                                                                       \
      st = host::launch<Gated<Config<BN, STAGES, CG, t.acc_f32, CM, CN, MR, t.bf16()>>, gated::kModes>(        \
          x, w, h, M, N, K, s, group_m, max_ctas, splits, Scales{nullptr, nullptr}, 0, host::splitk_scratch,   \
          nullptr, kActNone, 0, y);                                                                            \
    break;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      break;
  }
  if (st == host::kOk) g_launches.fetch_add(1, std::memory_order_relaxed);
  return st;
}

#define B200_SWIGLU_RUN(T) \
  int run_config<T>(int, const void*, const void*, void*, void*, int, int, int, int, int, int, void*)
extern template B200_SWIGLU_RUN(host::GemmType::kF16Acc32);
extern template B200_SWIGLU_RUN(host::GemmType::kBF16);
template B200_SWIGLU_RUN(host::GemmType(B200_VARIANT));
#undef B200_SWIGLU_RUN

}  // namespace swiglu
}  // namespace b200

#if B200_VARIANT == 0

namespace b200 {
namespace swiglu {

constexpr int kBwdThreads = 256;
constexpr int kBwdMaxCtas = 132 * 16;   // grid-stride beyond this: enough 16-byte requests in flight to fill HBM

__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

// One 16-byte vector of eight 16-bit values as fp32, and back (RN: the values are 16-bit values already)
template <typename T>
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const T* e = reinterpret_cast<const T*>(&v);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = to_f32(e[j]);
}

template <typename T>
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 v;
  uint32_t* w = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) w[j] = ptx::pack_out_x2_rn<std::is_same_v<T, __nv_bfloat16>>(f[2 * j], f[2 * j + 1]);
  return v;
}

// dh = swiglu_grad(dy, h): one thread per eight consecutive columns of y (one 16-byte vector of dy, of g, of u, of dg and
// of du), grid-stride over the M * I / 8 vectors. I % 64 == 0: the eight columns lie in one 64-column gate / up block.
template <typename T>
__global__ void __launch_bounds__(kBwdThreads) swiglu_backward_kernel(const T* __restrict__ dy, const T* __restrict__ h,
                                                                       T* __restrict__ dh, long long vectors, int I) {
  const int per_row = I / 8;
  for (long long i = blockIdx.x * (long long)kBwdThreads + threadIdx.x; i < vectors;
       i += (long long)gridDim.x * kBwdThreads) {
    const long long row = i / per_row;
    const int col = int(i - row * per_row) * 8;                      // y's column
    const size_t hg = size_t(row) * 2 * I + size_t(col / 64) * 128 + col % 64, hu = hg + 64;
    float d[8], g[8], u[8], dg[8], du[8];
    unpack8<T>(__ldg(reinterpret_cast<const uint4*>(dy + size_t(row) * I + col)), d);
    unpack8<T>(__ldg(reinterpret_cast<const uint4*>(h + hg)), g);
    unpack8<T>(__ldg(reinterpret_cast<const uint4*>(h + hu)), u);
#pragma unroll
    for (int j = 0; j < 8; ++j) swiglu_grad<T>(d[j], g[j], u[j], dg[j], du[j]);
    *reinterpret_cast<uint4*>(dh + hg) = pack8<T>(dg);
    *reinterpret_cast<uint4*>(dh + hu) = pack8<T>(du);
  }
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

int run(int variant, int config_id, const void* x, const void* w, void* h, void* y, int M, int I, int K, int group_m,
        int splits, int max_ctas, void* stream) {
  if (variant == int(host::GemmType::kBF16))
    return run_config<host::GemmType::kBF16>(config_id, x, w, h, y, M, 2 * I, K, group_m, max_ctas, splits, stream);
  return run_config<host::GemmType::kF16Acc32>(config_id, x, w, h, y, M, 2 * I, K, group_m, max_ctas, splits, stream);
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
