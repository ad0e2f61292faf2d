// libb200_quant.so — the one-pass e4m3 quantisers of FP8 activations (b200_quant.h). Memory-bound kernels:
// every element is loaded once into registers, its group's amax is reduced on chip, and the quantised bytes are stored
// from the same registers. A library of its own, so that the device code of the GEMM libraries stays as it is. The
// element arithmetic is in b200_quant_arith.cuh, shared with libb200_quant_dual.so.
#include "b200_quant.h"
#include "b200_quant_arith.cuh"
#include "swiglu_arith.cuh"

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cfloat>
#include <climits>
#include <cstdint>

namespace b200 {
namespace quant {

enum Status : int {
  kOk = 0,
  kBadShape = -1,
  kBadAlignment = -2,
  kNullPointer = -5,
  kBadDtype = -6,
  kBadScaleLd = -10,
};

constexpr int kBlock = 128;   // the 1 x 128 scale block

// ------------------------------------------------------------------------------------------------ SwiGLU
// the SwiGLU product p = RN(fp32(RN(silu(g))) * fp32(u)) of torch's `F.silu(g) * u` on 16-bit tensors: silu_mul of
// swiglu_arith.cuh, which the gated GEMM epilogue shares

// ------------------------------------------------------------------------------------------------ 1 x 128 blocks
// One CTA of 128 threads quantises 32 rows of one k-block. A row's 128 columns are spread over LPR = 128 / EPL lanes
// of a warp (16 for 16-bit vectors, 32 otherwise); a warp holds 8 rows, 32 / LPR per pass, every pass's loads issued
// before any is used. The scales of the 32 rows go out as one coalesced 128-byte store along M.
constexpr int kRowsPerCta = 32, kBlockThreads = 128;

struct BlockTile {
  int b, m0, kb, rows;   // matrix, first row, k-block, rows of this matrix that are read and written
};

__device__ __forceinline__ BlockTile block_tile(int B, int M, int nkb, const int* masked_m) {
  const int mtiles = (M + kRowsPerCta - 1) / kRowsPerCta;
  const long long t = blockIdx.x;
  BlockTile bt;
  bt.kb = int(t % nkb);
  bt.m0 = int((t / nkb) % mtiles) * kRowsPerCta;
  bt.b = int(t / (static_cast<long long>(nkb) * mtiles));
  bt.rows = M;
  if (masked_m != nullptr) bt.rows = min(max(masked_m[bt.b], 0), M);
  return bt;
}

// Src::load(row, col, valid, v) fills v with the EPL values at (row, col..col+EPL) of the quantised matrix
template <int EPL, bool kVec, class Src>
__device__ __forceinline__ void blockwise_body(const Src& src, int M, int K, uint8_t* __restrict__ q,
                                               float* __restrict__ scale, int ld_a, const int* masked_m, int B) {
  constexpr int LPR = kBlock / EPL;          // lanes per row
  constexpr int RPP = 32 / LPR;              // rows per warp pass
  constexpr int PASSES = kRowsPerCta / (kBlockThreads / 32) / RPP;
  const int nkb = (K + kBlock - 1) / kBlock;
  const BlockTile t = block_tile(B, M, nkb, masked_m);
  if (t.m0 >= t.rows) return;
  __shared__ float s_tile[kRowsPerCta];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int col = t.kb * kBlock + (lane % LPR) * EPL;
  const int valid = min(max(K - col, 0), EPL);
  float v[PASSES][EPL];
  int r[PASSES];
#pragma unroll
  for (int p = 0; p < PASSES; ++p) {
    r[p] = warp * (kRowsPerCta / 4) + p * RPP + lane / LPR;   // row within the tile
    const int row = t.m0 + r[p];
    if (row < t.rows && valid > 0) {
      src.template load<EPL, kVec>(static_cast<long long>(t.b) * M + row, col, valid, v[p]);
    } else {
#pragma unroll
      for (int j = 0; j < EPL; ++j) v[p][j] = 0.0f;
    }
  }
#pragma unroll
  for (int p = 0; p < PASSES; ++p) {
    float m = 0.0f;
#pragma unroll
    for (int j = 0; j < EPL; ++j) m = nan_max(m, fabsf(v[p][j]));
    const float s = scale_of(group_amax<LPR>(m));
    const int row = t.m0 + r[p];
    if (row < t.rows && valid > 0)
      store_e4m3<EPL, kVec>(q + (static_cast<long long>(t.b) * M + row) * K + col, valid, v[p], s);
    if (lane % LPR == 0) s_tile[r[p]] = s;
  }
  __syncthreads();
  if (threadIdx.x < kRowsPerCta && t.m0 + int(threadIdx.x) < t.rows)
    scale[(static_cast<long long>(t.b) * nkb + t.kb) * ld_a + t.m0 + threadIdx.x] = s_tile[threadIdx.x];
}

template <typename T>
struct PlainSrc {   // x [B * M, K]
  const T* x;
  int K;
  template <int EPL, bool kVec>
  __device__ __forceinline__ void load(long long row, int col, int valid, float (&v)[EPL]) const {
    load_f32<T, EPL, kVec>(x + row * K + col, valid, v);
  }
};

template <typename T>
struct SiluMulSrc {   // h [B * M, 2I]: silu(h[:, :I]) * h[:, I:]
  const T* h;
  int I;
  template <int EPL, bool kVec>
  __device__ __forceinline__ void load(long long row, int col, int valid, float (&v)[EPL]) const {
    const T* g = h + row * 2 * I + col;
    float gv[EPL], uv[EPL];
    load_f32<T, EPL, kVec>(g, valid, gv);
    load_f32<T, EPL, kVec>(g + I, valid, uv);
#pragma unroll
    for (int j = 0; j < EPL; ++j) v[j] = silu_mul<T>(gv[j], uv[j]);
  }
};

template <typename T, int EPL, bool kVec>
__global__ void __launch_bounds__(kBlockThreads) b200_quant_blockwise_kernel(
    const T* __restrict__ x, int B, int M, int K, uint8_t* __restrict__ q, float* __restrict__ scale, int ld_a,
    const int* __restrict__ masked_m) {
  blockwise_body<EPL, kVec>(PlainSrc<T>{x, K}, M, K, q, scale, ld_a, masked_m, B);
}

template <typename T, int EPL, bool kVec>
__global__ void __launch_bounds__(kBlockThreads) b200_quant_silu_mul_blockwise_kernel(
    const T* __restrict__ h, int B, int M, int I, uint8_t* __restrict__ q, float* __restrict__ scale, int ld_a,
    const int* __restrict__ masked_m) {
  blockwise_body<EPL, kVec>(SiluMulSrc<T>{h, I}, M, I, q, scale, ld_a, masked_m, B);
}

// ------------------------------------------------------------------------------------------------ rowwise
// One CTA per row. Each thread's first kCached chunks of EPL elements stay in registers between the amax and the
// quantisation; chunks past them (rows longer than THREADS * kCached * EPL) are loaded again, from L2.
constexpr int kRowThreads = 512, kCached = 4;

template <typename T, int EPL, bool kVec>
__global__ void __launch_bounds__(kRowThreads) b200_quant_rowwise_kernel(const T* __restrict__ x, int cols,
                                                                          uint8_t* __restrict__ q,
                                                                          float* __restrict__ scale) {
  __shared__ float red[kRowThreads / 32];
  const long long row = blockIdx.x;
  const T* xr = x + row * cols;
  uint8_t* qr = q + row * cols;
  const int chunks = (cols + EPL - 1) / EPL;
  float v[kCached][EPL];
  float m = 0.0f;
#pragma unroll
  for (int j = 0; j < kCached; ++j) {
    const int c = (threadIdx.x + j * blockDim.x) * EPL;
    if (c < cols) {
      load_f32<T, EPL, kVec>(xr + c, min(cols - c, EPL), v[j]);
    } else {
#pragma unroll
      for (int e = 0; e < EPL; ++e) v[j][e] = 0.0f;
    }
  }
#pragma unroll
  for (int j = 0; j < kCached; ++j)
#pragma unroll
    for (int e = 0; e < EPL; ++e) m = nan_max(m, fabsf(v[j][e]));
  for (int i = threadIdx.x + kCached * blockDim.x; i < chunks; i += blockDim.x) {
    float w[EPL];
    load_f32<T, EPL, kVec>(xr + i * EPL, min(cols - i * EPL, EPL), w);
#pragma unroll
    for (int e = 0; e < EPL; ++e) m = nan_max(m, fabsf(w[e]));
  }
  const float s = scale_of(cta_amax(m, red));
#pragma unroll
  for (int j = 0; j < kCached; ++j) {
    const int c = (threadIdx.x + j * blockDim.x) * EPL;
    if (c < cols) store_e4m3<EPL, kVec>(qr + c, min(cols - c, EPL), v[j], s);
  }
  for (int i = threadIdx.x + kCached * blockDim.x; i < chunks; i += blockDim.x) {
    float w[EPL];
    load_f32<T, EPL, kVec>(xr + i * EPL, min(cols - i * EPL, EPL), w);
    store_e4m3<EPL, kVec>(qr + i * EPL, min(cols - i * EPL, EPL), w, s);
  }
  if (threadIdx.x == 0) scale[row] = s;
}

// ------------------------------------------------------------------------------------------------ per tensor
// Two launches over a grid of at most CUDA_L2_B200_QUANT_TENSOR_WORKSPACE CTAs, each taking a grid-stride share of the
// EPL-element chunks (CTA 0 also the last n % EPL elements): the first writes each CTA's amax to the workspace, the
// second reduces the workspace in every CTA (a few KiB from L2), quantises its share and, in CTA 0, writes the scale.
constexpr int kTensorThreads = 256, kTensorUnroll = 4;

template <typename T, int EPL, bool kVec>
__global__ void __launch_bounds__(kTensorThreads) b200_quant_tensor_amax_kernel(const T* __restrict__ x, long long n,
                                                                                float* __restrict__ workspace) {
  __shared__ float red[kTensorThreads / 32];
  const long long chunks = n / EPL, stride = static_cast<long long>(gridDim.x) * blockDim.x;
  float m = 0.0f;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i + (kTensorUnroll - 1) * stride < chunks; i += kTensorUnroll * stride) {
    float v[kTensorUnroll][EPL];
#pragma unroll
    for (int u = 0; u < kTensorUnroll; ++u) load_f32<T, EPL, kVec>(x + (i + u * stride) * EPL, EPL, v[u]);
#pragma unroll
    for (int u = 0; u < kTensorUnroll; ++u)
#pragma unroll
      for (int e = 0; e < EPL; ++e) m = nan_max(m, fabsf(v[u][e]));
  }
  for (; i < chunks; i += stride) {
    float v[EPL];
    load_f32<T, EPL, kVec>(x + i * EPL, EPL, v);
#pragma unroll
    for (int e = 0; e < EPL; ++e) m = nan_max(m, fabsf(v[e]));
  }
  if (blockIdx.x == 0 && threadIdx.x < n - chunks * EPL) {   // the last n % EPL elements, one per thread
    float v[1];
    load_f32<T, 1, false>(x + chunks * EPL + threadIdx.x, 1, v);
    m = nan_max(m, fabsf(v[0]));
  }
  m = cta_amax(m, red);
  if (threadIdx.x == 0) workspace[blockIdx.x] = m;
}

template <typename T, int EPL, bool kVec>
__global__ void __launch_bounds__(kTensorThreads) b200_quant_tensor_kernel(const T* __restrict__ x, long long n,
                                                                           uint8_t* __restrict__ q,
                                                                           float* __restrict__ scale,
                                                                           const float* __restrict__ workspace,
                                                                           int partials) {
  __shared__ float red[kTensorThreads / 32];
  float m = 0.0f;
  for (int i = threadIdx.x; i < partials; i += blockDim.x) m = nan_max(m, workspace[i]);
  const float s = scale_of(cta_amax(m, red));
  if (blockIdx.x == 0 && threadIdx.x == 0) scale[0] = s;
  const long long chunks = n / EPL, stride = static_cast<long long>(gridDim.x) * blockDim.x;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i + (kTensorUnroll - 1) * stride < chunks; i += kTensorUnroll * stride) {
    float v[kTensorUnroll][EPL];
#pragma unroll
    for (int u = 0; u < kTensorUnroll; ++u) load_f32<T, EPL, kVec>(x + (i + u * stride) * EPL, EPL, v[u]);
#pragma unroll
    for (int u = 0; u < kTensorUnroll; ++u) store_e4m3<EPL, kVec>(q + (i + u * stride) * EPL, EPL, v[u], s);
  }
  for (; i < chunks; i += stride) {
    float v[EPL];
    load_f32<T, EPL, kVec>(x + i * EPL, EPL, v);
    store_e4m3<EPL, kVec>(q + i * EPL, EPL, v, s);
  }
  if (blockIdx.x == 0 && threadIdx.x < n - chunks * EPL) {
    float v[1];
    load_f32<T, 1, false>(x + chunks * EPL + threadIdx.x, 1, v);
    store_e4m3<1, false>(q + chunks * EPL + threadIdx.x, 1, v, s);
  }
}

}  // namespace quant
}  // namespace b200

namespace {

using namespace b200::quant;

std::atomic<unsigned long long> g_launches{0};

// ------------------------------------------------------------------------------------------------ host side
bool aligned(const void* p, unsigned bytes) { return reinterpret_cast<uintptr_t>(p) % bytes == 0; }

int launched(cudaError_t e) {
  if (e != cudaSuccess) return int(e);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return kOk;
}

// Calls l.template run<T, EPL, kVec>() for dtype: 16-byte vectors of EPL = 16 / sizeof(T) elements when `vec(EPL)`
// says the pointers and row length allow them, four elements by element loads otherwise.
template <class L>
int by_dtype(int dtype, const L& l) {
  switch (dtype) {
    case 0: return l.vec(8) ? l.template run<__half, 8, true>() : l.template run<__half, 4, false>();
    case 1: return l.vec(8) ? l.template run<__nv_bfloat16, 8, true>() : l.template run<__nv_bfloat16, 4, false>();
    case 2: return l.vec(4) ? l.template run<float, 4, true>() : l.template run<float, 4, false>();
    default: return kBadDtype;
  }
}

int check_blockwise(int dtype, const void* x, int B, int M, int K, const void* q, const float* scale, int ld_a) {
  if (dtype < 0 || dtype > 2) return kBadDtype;
  if (x == nullptr || q == nullptr || scale == nullptr) return kNullPointer;
  if (B <= 0 || M <= 0 || K <= 0) return kBadShape;
  const long long ctas =
      static_cast<long long>(B) * ((M + kRowsPerCta - 1) / kRowsPerCta) * ((K + kBlock - 1) / kBlock);
  if (ctas > INT_MAX) return kBadShape;   // one CTA per 32 rows and k-block, in a 1-D grid
  if (!aligned(scale, 4)) return kBadAlignment;
  if (ld_a < M || ld_a % 4 != 0) return kBadScaleLd;
  return kOk;
}


struct TensorLaunch {
  const void* x;
  long long n;
  void* q;
  float* scale;
  float* workspace;
  cudaStream_t st;
  bool vec(int epl) const { return aligned(x, 16) && aligned(q, epl); }
  template <typename T, int EPL, bool kVec>
  int run() const {
    const long long per_cta = static_cast<long long>(EPL) * kTensorThreads * kTensorUnroll;
    const long long want = (n + per_cta - 1) / per_cta;
    const int grid = int(want < CUDA_L2_B200_QUANT_TENSOR_WORKSPACE ? want : CUDA_L2_B200_QUANT_TENSOR_WORKSPACE);
    b200::quant::b200_quant_tensor_amax_kernel<T, EPL, kVec>
        <<<grid, kTensorThreads, 0, st>>>(static_cast<const T*>(x), n, workspace);
    if (const int e = launched(cudaGetLastError())) return e;
    b200::quant::b200_quant_tensor_kernel<T, EPL, kVec><<<grid, kTensorThreads, 0, st>>>(
        static_cast<const T*>(x), n, static_cast<uint8_t*>(q), scale, workspace, grid);
    return launched(cudaGetLastError());
  }
};

struct RowwiseLaunch {
  const void* x;
  int rows, cols;
  void* q;
  float* scale;
  cudaStream_t st;
  bool vec(int epl) const { return aligned(x, 16) && aligned(q, epl) && cols % epl == 0; }
  template <typename T, int EPL, bool kVec>
  int run() const {
    const int chunks = (cols + EPL - 1) / EPL;
    const int per = (chunks + kCached - 1) / kCached;   // threads that hold the whole row in registers
    const int threads = per >= kRowThreads ? kRowThreads : (per <= 32 ? 32 : (per + 31) / 32 * 32);
    b200::quant::b200_quant_rowwise_kernel<T, EPL, kVec>
        <<<rows, threads, 0, st>>>(static_cast<const T*>(x), cols, static_cast<uint8_t*>(q), scale);
    return launched(cudaGetLastError());
  }
};

template <bool kSiluMul>
struct BlockwiseLaunch {   // x [B, M, K], or h [B, M, 2K] for the SwiGLU product
  const void* x;
  int B, M, K;
  void* q;
  float* scale;
  int ld_a;
  const int* masked_m;
  cudaStream_t st;
  bool vec(int epl) const { return aligned(x, 16) && aligned(q, epl) && K % epl == 0; }
  template <typename T, int EPL, bool kVec>
  int run() const {
    const long long ctas =
        static_cast<long long>(B) * ((M + kRowsPerCta - 1) / kRowsPerCta) * ((K + kBlock - 1) / kBlock);
    if constexpr (kSiluMul) {
      if constexpr (sizeof(T) == 4) {
        return kBadDtype;
      } else {
        b200::quant::b200_quant_silu_mul_blockwise_kernel<T, EPL, kVec><<<ctas, kBlockThreads, 0, st>>>(
            static_cast<const T*>(x), B, M, K, static_cast<uint8_t*>(q), scale, ld_a, masked_m);
      }
    } else {
      b200::quant::b200_quant_blockwise_kernel<T, EPL, kVec><<<ctas, kBlockThreads, 0, st>>>(
          static_cast<const T*>(x), B, M, K, static_cast<uint8_t*>(q), scale, ld_a, masked_m);
    }
    return launched(cudaGetLastError());
  }
};

}  // namespace

extern "C" {

int cuda_l2_b200_quant_e4m3_tensor(int dtype, const void* x, long long n, void* q, float* scale,
                                   float* workspace, void* stream) {
  if (dtype < 0 || dtype > 2) return kBadDtype;
  if (x == nullptr || q == nullptr || scale == nullptr || workspace == nullptr) return kNullPointer;
  if (n <= 0) return kBadShape;
  if (!aligned(scale, 4) || !aligned(workspace, 4)) return kBadAlignment;
  return by_dtype(dtype, TensorLaunch{x, n, q, scale, workspace, static_cast<cudaStream_t>(stream)});
}

int cuda_l2_b200_quant_e4m3_rowwise(int dtype, const void* x, int rows, int cols, void* q, float* scale,
                                    void* stream) {
  if (dtype < 0 || dtype > 2) return kBadDtype;
  if (x == nullptr || q == nullptr || scale == nullptr) return kNullPointer;
  if (rows <= 0 || cols <= 0) return kBadShape;
  if (!aligned(scale, 4)) return kBadAlignment;
  return by_dtype(dtype, RowwiseLaunch{x, rows, cols, q, scale, static_cast<cudaStream_t>(stream)});
}

int cuda_l2_b200_quant_e4m3_blockwise(int dtype, const void* x, int B, int M, int K, void* q, float* scale,
                                      int ld_a, const int* masked_m, void* stream) {
  if (const int e = check_blockwise(dtype, x, B, M, K, q, scale, ld_a)) return e;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return by_dtype(dtype, BlockwiseLaunch<false>{x, B, M, K, q, scale, ld_a, masked_m, st});
}

int cuda_l2_b200_quant_silu_mul_e4m3_blockwise(int dtype, const void* h, int B, int M, int I, void* q,
                                               float* scale, int ld_a, const int* masked_m, void* stream) {
  if (const int e = check_blockwise(dtype, h, B, M, I, q, scale, ld_a)) return e;
  if (dtype == 2) return kBadDtype;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return by_dtype(dtype, BlockwiseLaunch<true>{h, B, M, I, q, scale, ld_a, masked_m, st});
}

unsigned long long cuda_l2_b200_quant_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

const char* cuda_l2_b200_quant_strerror(int status) {
  switch (status) {
    case kOk: return "ok";
    case kBadShape: return "every size must be positive";
    case kBadAlignment: return "scale and workspace pointers must be 4-byte aligned";
    case kNullPointer: return "null pointer";
    case kBadDtype: return "unknown input dtype (0 fp16, 1 bf16, 2 fp32; SwiGLU takes fp16 and bf16 only)";
    case kBadScaleLd: return "ld_a must be >= M and a multiple of 4";
    default: return status > 0 ? cudaGetErrorString(static_cast<cudaError_t>(status)) : "unknown status";
  }
}

}  // extern "C"
