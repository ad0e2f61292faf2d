// libb200_grouped_swiglu.so — the Gated<Grouped<>> kernels (hgemm_sm90.cuh) of every configuration with a gated kernel,
// and the SwiGLU backward over contiguous row groups, behind the internal entry points of b200_grouped_swiglu.h. A
// library of its own, so that the device code of the other libraries (libb200_swiglu.so's included) stays as it is.
// build.py compiles this file once per variant (-DB200_VARIANT = 0 or 2), in parallel; the object of variant 0 also
// holds the entry points and the backward kernels.
#include "b200_grouped_swiglu.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"
#include "swiglu_backward.cuh"

#ifndef B200_VARIANT
#error "compile once per variant with -DB200_VARIANT=0 or 2"
#endif

namespace b200 {
namespace tile_list {

template <class Cfg>
using GatedGrouped = Gated<Grouped<Cfg>>;

// fp16 and bf16, both with fp32 accumulation
#define B200_SWIGLU_TYPES(X, W) X(W, host::GemmType::kF16Acc32) X(W, host::GemmType::kBF16)
B200_LIST_OBJECT(Library, GatedGrouped, B200_SWIGLU_TYPES);
#undef B200_SWIGLU_TYPES

}  // namespace tile_list
}  // namespace b200

#if B200_VARIANT == 0

namespace b200 {
namespace grouped_swiglu {

using swiglu::kBwdMaxCtas;
using swiglu::kBwdThreads;

// The groups' last end as GroupCursor clamps them: end_g = clamp(offs[g], end_{g-1}, T) from end_{-1} = 0 is
// min(max(0, offs[0], ..., offs[g]), T), so the last one is the largest offset clamped to [0, T]. Warp 0 of the block
// reduces the G offsets (read after the grid dependency: a preceding kernel may have just written them) and hands the
// end to the block through shared memory.
__device__ __forceinline__ int groups_end(const int* __restrict__ offs, int G, int T) {
  __shared__ int s_end;
  if (threadIdx.x < 32) {
    int e = 0;
    for (int g = int(threadIdx.x); g < G; g += 32) e = max(e, offs[g]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) e = max(e, __shfl_xor_sync(0xffffffffu, e, o));
    if (threadIdx.x == 0) s_end = min(e, T);
  }
  __syncthreads();
  return s_end;
}

// dh = swiglu_grad(dy, h) for the rows below the groups' last end: libb200_swiglu.so's backward over those rows.
template <typename T>
__global__ void __launch_bounds__(kBwdThreads)
grouped_swiglu_backward_kernel(const T* __restrict__ dy, const T* __restrict__ h, T* __restrict__ dh,
                               const int* __restrict__ offs, int G, int rows, int I) {
  swiglu::backward_vectors(dy, h, dh, (long long)groups_end(offs, G, rows) * (I / 8), I);
}

inline bool known_variant(int variant) {
  return variant == int(host::GemmType::kF16Acc32) || variant == int(host::GemmType::kBF16);
}

// The argument rules of the forward entry points, before any CUDA call.
int validate(int variant, const void* x, const void* w, const void* h, const void* y, const int* offs, int G, int T,
             int I, int H) {
  if (!known_variant(variant)) return kSwigluBadDtype;
  if (!x || !w || !y || !offs) return host::kNullPointer;
  if (T < 0 || G < 1 || I <= 0 || H <= 0 || 2LL * I > 0x7fffffffLL) return host::kBadShape;
  if (I % 64) return kSwigluBadWidth;
  if (H % 8 || ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(h) |
                 reinterpret_cast<uintptr_t>(y)) & 15))
    return host::kBadAlignment;
  if (reinterpret_cast<uintptr_t>(offs) & 3) return host::kBadAlignment;
  // the shortest worst-case tile list of the gated configurations: past INT_MAX every configuration refuses the shape
  if (tile_list::fewest_tiles<tile_list::GatedGrouped>(G, T > 0 ? T : 1, 2 * I) > 0x7fffffffLL) return host::kBadShape;
  return host::kOk;
}

// The grouped choice for (G, T, 2I, H) mapped to its gated sibling (tile_list::select).
dispatch::Choice select(int variant, int G, int T, int I, int H) {
  return tile_list::select<tile_list::GatedGrouped>(host::GemmType(variant), G, T, 2 * I, H);
}

// Configuration `config_id` of `variant` wrapped in Gated<Grouped<>>: h (may be null) and y over the groups of `offs`,
// N = 2I. A configuration without a gated kernel is kBadConfig; T == 0 launches nothing.
int run(int variant, int config_id, const void* x, const void* w, void* h, void* y, const int* offs, int G, int T,
        int I, int H, int group_m, int max_ctas, void* stream) {
  host::EpiOperands op;
  op.y = y;
  return tile_list::run(tile_list::Library{}, host::GemmType(variant), config_id, x, w, h, offs, G, T, 2 * I, H, group_m,
                        max_ctas, stream, op);
}

template <typename T>
int backward(const void* dy, const void* h, void* dh, const int* offs, int G, int rows, int I, cudaStream_t s) {
  const long long vectors = (long long)rows * (I / 8);   // the most the groups can hold: the kernel bounds it on device
  const int ctas = int(std::min<long long>((vectors + kBwdThreads - 1) / kBwdThreads, kBwdMaxCtas));
  grouped_swiglu_backward_kernel<T><<<ctas, kBwdThreads, 0, s>>>(static_cast<const T*>(dy), static_cast<const T*>(h),
                                                                 static_cast<T*>(dh), offs, G, rows, I);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return int(e);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return host::kOk;
}

}  // namespace grouped_swiglu
}  // namespace b200

extern "C" {

int cuda_l2_b200_grouped_swiglu_run(int variant, const void* x, const void* w_gu, void* h, void* y, const int* offs,
                                    int G, int T, int I, int H, void* stream) {
  using namespace b200;
  if (const int st = grouped_swiglu::validate(variant, x, w_gu, h, y, offs, G, T, I, H)) return st;
  if (T == 0) return host::kOk;
  const dispatch::Choice ch = grouped_swiglu::select(variant, G, T, I, H);
  return grouped_swiglu::run(variant, ch.config_id, x, w_gu, h, y, offs, G, T, I, H, ch.group_m, 0, stream);
}

int cuda_l2_b200_grouped_swiglu_run_config(int variant, int config_id, const void* x, const void* w_gu, void* h,
                                           void* y, const int* offs, int G, int T, int I, int H, int group_m,
                                           int max_ctas, void* stream) {
  using namespace b200;
  if (const int st = grouped_swiglu::validate(variant, x, w_gu, h, y, offs, G, T, I, H)) return st;
  return grouped_swiglu::run(variant, config_id, x, w_gu, h, y, offs, G, T, I, H, group_m, max_ctas, stream);
}

int cuda_l2_b200_grouped_swiglu_select(int variant, int G, int T, int I, int H, int* config_id, int* group_m) {
  using namespace b200;
  if (!grouped_swiglu::known_variant(variant)) return kSwigluBadDtype;
  if (G < 1 || T <= 0 || I <= 0 || H <= 0 || 2LL * I > 0x7fffffffLL) return host::kBadShape;
  if (I % 64) return kSwigluBadWidth;
  const dispatch::Choice ch = grouped_swiglu::select(variant, G, T, I, H);
  if (config_id) *config_id = ch.config_id;
  if (group_m) *group_m = ch.group_m;
  return host::kOk;
}

int cuda_l2_b200_grouped_swiglu_backward(int variant, const void* dy, const void* h, void* dh, const int* offs, int G,
                                         int T, int I, void* stream) {
  using namespace b200;
  if (!grouped_swiglu::known_variant(variant)) return kSwigluBadDtype;
  if (!offs || (T != 0 && (!dy || !h || !dh))) return host::kNullPointer;   // T == 0: nothing is read or written
  if (T < 0 || G < 1 || I <= 0 || 2LL * I > 0x7fffffffLL) return host::kBadShape;
  if (I % 64) return kSwigluBadWidth;
  if ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(dh)) & 15)
    return host::kBadAlignment;
  if (reinterpret_cast<uintptr_t>(offs) & 3) return host::kBadAlignment;
  if (T == 0) return host::kOk;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  return variant == int(host::GemmType::kBF16)
             ? grouped_swiglu::backward<__nv_bfloat16>(dy, h, dh, offs, G, T, I, s)
             : grouped_swiglu::backward<__half>(dy, h, dh, offs, G, T, I, s);
}

unsigned long long cuda_l2_b200_grouped_swiglu_launch_count(void) {
  return b200::g_launches.load(std::memory_order_relaxed) +
         b200::tile_list::g_list_launches.load(std::memory_order_relaxed);
}

const char* cuda_l2_b200_grouped_swiglu_strerror(int status) {
  switch (status) {
    case kSwigluBadWidth: return "the intermediate size I must be a multiple of 64 (whole 64-row gate / up blocks)";
    case kSwigluBadDtype: return "variant must be 0 (fp16) or 2 (bf16), with fp32 accumulation";
    default: return b200::host::status_string(status);
  }
}

}  // extern "C"

#endif  // B200_VARIANT == 0
