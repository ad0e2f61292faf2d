// libb200_grouped_swiglu.so — the Gated<Grouped<>> kernels (hgemm_sm90.cuh) of every configuration with a gated kernel,
// and the SwiGLU backward over contiguous row groups, behind the internal entry points of b200_grouped_swiglu.h. A
// library of its own, so that the device code of the other libraries (libb200_swiglu.so's included) stays as it is.
// build.py compiles this file once per variant (-DB200_VARIANT = 0 or 2), in parallel; the object of variant 0 also
// holds the entry points and the backward kernels.
#include "b200_grouped_swiglu.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"
#include "swiglu_arith.cuh"

#ifndef B200_VARIANT
#error "compile once per variant with -DB200_VARIANT=0 or 2"
#endif

namespace b200 {
namespace grouped_swiglu {

// Configuration `id` of variant T wrapped in Gated<Grouped<>>: h (C, may be null) and y over the groups of `offs`,
// N = 2I. A configuration without a gated kernel is kBadConfig; T == 0 launches nothing.
template <host::GemmType T>
int run_config(int id, const void* x, const void* w, void* h, void* y, const int* offs, int G, int rows, int N, int K,
               int group_m, int max_ctas, void* stream) {
  constexpr host::GemmTypeTraits t = host::traits(T);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int st = host::kBadConfig;
  switch (id) {
#define B200_CASE(ID, BN, STAGES, CG, CM, CN, MR)                                                                  \
  case ID:                                                                                                     \
    if constexpr (gated::has_kernel(ID))                                                                       \
      st = host::launch_list<Gated<Grouped<Config<BN, STAGES, CG, t.acc_f32, CM, CN, MR, t.bf16()>>>>(         \
          x, w, h, offs, G, rows, N, K, s, group_m, max_ctas, Scales{nullptr, nullptr}, 0, y);                 \
    break;
    B200_HGEMM_CONFIGS(B200_CASE)
#undef B200_CASE
    default:
      break;
  }
  if (st == host::kOk && rows > 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  return st;
}

#define B200_GROUPED_SWIGLU_RUN(T)                                                                           \
  int run_config<T>(int, const void*, const void*, void*, void*, const int*, int, int, int, int, int, int, void*)
extern template B200_GROUPED_SWIGLU_RUN(host::GemmType::kF16Acc32);
extern template B200_GROUPED_SWIGLU_RUN(host::GemmType::kBF16);
template B200_GROUPED_SWIGLU_RUN(host::GemmType(B200_VARIANT));
#undef B200_GROUPED_SWIGLU_RUN

}  // namespace grouped_swiglu
}  // namespace b200

#if B200_VARIANT == 0

namespace b200 {
namespace grouped_swiglu {

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

// dh = swiglu_grad(dy, h) for the rows below the groups' last end: one thread per eight consecutive columns of y (one
// 16-byte vector of dy, of g, of u, of dg and of du), grid-stride over those rows' vectors. I % 64 == 0: the eight
// columns lie in one 64-column gate / up block. The arithmetic is libb200_swiglu.so's backward, element for element.
template <typename T>
__global__ void __launch_bounds__(kBwdThreads)
grouped_swiglu_backward_kernel(const T* __restrict__ dy, const T* __restrict__ h, T* __restrict__ dh,
                               const int* __restrict__ offs, int G, int rows, int I) {
  const int per_row = I / 8;
  const long long vectors = (long long)groups_end(offs, G, rows) * per_row;
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

inline bool known_variant(int variant) {
  return variant == int(host::GemmType::kF16Acc32) || variant == int(host::GemmType::kBF16);
}

// The shortest worst-case tile list (GroupCursor::max_tiles) of any configuration with a gated kernel: when it passes
// INT_MAX, every configuration refuses the shape, so the dispatched call refuses it before the lookup. The list is
// Grouped<>'s of the same configuration.
inline long long fewest_tiles(int G, int T, int N) {
  long long fewest = 0x7fffffffffffffffLL;
#define B200_TILES(ID, BN, STAGES, CG, CM, CN, MR)                                                               \
  if constexpr (gated::has_kernel(ID)) {                                                                        \
    using W = Grouped<Config<BN, STAGES, CG, true, CM, CN, MR>>;                                                 \
    fewest = std::min(fewest, W::Cursor::template max_tiles<W>(G, T, N));                                       \
  }
  B200_HGEMM_CONFIGS(B200_TILES)
#undef B200_TILES
  return fewest;
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
  if (fewest_tiles(G, T > 0 ? T : 1, 2 * I) > 0x7fffffffLL) return host::kBadShape;
  return host::kOk;
}

// The grouped choice for (G, T, 2I, H) mapped to its gated sibling (the plain schedule is the only one of tile lists).
dispatch::Choice select(int variant, int G, int T, int I, int H) {
  dispatch::Choice ch = tile_list::select<Grouped>(host::GemmType(variant), G, T, 2 * I, H);
  ch.config_id = gated::sibling(ch.config_id);
  ch.splits = 1;
  return ch;
}

int run(int variant, int config_id, const void* x, const void* w, void* h, void* y, const int* offs, int G, int T,
        int I, int H, int group_m, int max_ctas, void* stream) {
  if (variant == int(host::GemmType::kBF16))
    return run_config<host::GemmType::kBF16>(config_id, x, w, h, y, offs, G, T, 2 * I, H, group_m, max_ctas, stream);
  return run_config<host::GemmType::kF16Acc32>(config_id, x, w, h, y, offs, G, T, 2 * I, H, group_m, max_ctas, stream);
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
  return b200::g_launches.load(std::memory_order_relaxed);
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
