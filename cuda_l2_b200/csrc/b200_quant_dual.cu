// libb200_quant_dual.so — the dual-orientation rowwise e4m3 quantiser (b200_quant_dual.h): from one tensor x, its
// rowwise quantisation and that of x^T, the two K-major operands an FP8 linear layer's training step needs of it.
// Memory-bound: x is read twice (the column maxima need every row before any column can be quantised) and each
// e4m3 byte is written once. A library of its own, so that libb200_quant.so stays as it is; the element arithmetic is
// shared with it (b200_quant_arith.cuh).
#include "b200_quant_dual.h"
#include "b200_quant_arith.cuh"

#include <atomic>
#include <climits>

namespace b200 {
namespace quant {

enum DualStatus : int {
  kDualOk = 0,
  kDualBadShape = -1,
  kDualBadAlignment = -2,
  kDualNullPointer = -5,
  kDualBadDtype = -6,
};

// |x| as ordered bits: with the sign cleared, the unsigned order of a float's bits is its order, and a NaN sorts above
// +Inf, so an unsigned max is torch.amax's NaN-keeping max of |x|
__device__ __forceinline__ unsigned abs_bits(float v) { return __float_as_uint(v) & 0x7fffffffu; }

// ------------------------------------------------------------------------------------------------ pass 1: maxima
// One CTA of 256 threads per tile of kAmaxRows rows by 32 * EPL columns (one EPL-wide chunk per lane). Each warp takes
// kAmaxRows / 8 rows, kBatch of them loaded before any is reduced; a row's maximum is reduced across the warp and
// folded into row_amax by lane 0, and the column maxima are reduced across the warps in shared memory and folded into
// col_amax, one atomic per column.
constexpr int kAmaxThreads = 256, kAmaxRows = 128, kBatch = 8;

template <typename T, int EPL, bool kVec>
__global__ void __launch_bounds__(kAmaxThreads) b200_quant_dual_amax_kernel(const T* __restrict__ x, int rows,
                                                                            int cols, int col_tiles,
                                                                            unsigned* __restrict__ row_amax,
                                                                            unsigned* __restrict__ col_amax) {
  constexpr int kCols = 32 * EPL, kWarps = kAmaxThreads / 32, kWarpRows = kAmaxRows / kWarps;
  __shared__ unsigned s_col[kWarps][kCols];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int r0 = (blockIdx.x / col_tiles) * kAmaxRows + warp * kWarpRows;
  const int c0 = (blockIdx.x % col_tiles) * kCols;
  const int col = c0 + lane * EPL;
  const int valid = min(max(cols - col, 0), EPL);
  unsigned cm[EPL];
#pragma unroll
  for (int j = 0; j < EPL; ++j) cm[j] = 0u;
#pragma unroll
  for (int b = 0; b < kWarpRows; b += kBatch) {
    float v[kBatch][EPL];
#pragma unroll
    for (int i = 0; i < kBatch; ++i) {
      const int row = r0 + b + i;
      if (row < rows && valid > 0) {
        load_f32<T, EPL, kVec>(x + static_cast<long long>(row) * cols + col, valid, v[i]);
      } else {
#pragma unroll
        for (int j = 0; j < EPL; ++j) v[i][j] = 0.0f;
      }
    }
#pragma unroll
    for (int i = 0; i < kBatch; ++i) {
      unsigned m = 0u;
#pragma unroll
      for (int j = 0; j < EPL; ++j) {
        const unsigned a = abs_bits(v[i][j]);
        m = max(m, a);
        cm[j] = max(cm[j], a);
      }
      m = __reduce_max_sync(0xffffffffu, m);
      const int row = r0 + b + i;
      if (lane == 0 && row < rows) atomicMax(row_amax + row, m);
    }
  }
#pragma unroll
  for (int j = 0; j < EPL; ++j) s_col[warp][lane * EPL + j] = cm[j];
  __syncthreads();
  for (int c = threadIdx.x; c < kCols; c += kAmaxThreads) {
    unsigned m = 0u;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) m = max(m, s_col[w][c]);
    if (c0 + c < cols) atomicMax(col_amax + c0 + c, m);
  }
}

// ------------------------------------------------------------------------------------------------ pass 2: quantise
// One CTA of 128 threads per kTile x kTile tile. A tile row's kTile columns are spread over LPR = kTile / EPL lanes;
// every pass's loads are issued before any is used. The row-major bytes are stored from registers with the row scale;
// the tile goes to shared memory as fp32 (rows past `rows` as 0, the padding of q_t), and each thread then quantises
// 32 rows of one column with the column's scale and stores them as two 16-byte vectors of q_t.
constexpr int kTile = 64, kDualThreads = 128;

template <typename T, int EPL, bool kVec>
__global__ void __launch_bounds__(kDualThreads) b200_quant_dual_kernel(
    const T* __restrict__ x, int rows, int cols, int col_tiles, int ld_t, uint8_t* __restrict__ q,
    float* __restrict__ scale, uint8_t* __restrict__ q_t, float* __restrict__ scale_t,
    const unsigned* __restrict__ row_amax, const unsigned* __restrict__ col_amax) {
  constexpr int LPR = kTile / EPL;            // lanes per tile row
  constexpr int RPP = kDualThreads / LPR;     // tile rows per pass
  constexpr int PASSES = kTile / RPP;
  static_assert(kDualThreads == 2 * kTile, "two threads per column of the transposed store");
  __shared__ float s_x[kTile][kTile + 1];
  const int r0 = (blockIdx.x / col_tiles) * kTile, c0 = (blockIdx.x % col_tiles) * kTile;
  const int lc = (threadIdx.x % LPR) * EPL, col = c0 + lc;
  const int valid = min(max(cols - col, 0), EPL);
  float v[PASSES][EPL];
#pragma unroll
  for (int p = 0; p < PASSES; ++p) {
    const int row = r0 + p * RPP + threadIdx.x / LPR;
    if (row < rows && valid > 0) {
      load_f32<T, EPL, kVec>(x + static_cast<long long>(row) * cols + col, valid, v[p]);
    } else {
#pragma unroll
      for (int j = 0; j < EPL; ++j) v[p][j] = 0.0f;
    }
  }
#pragma unroll
  for (int p = 0; p < PASSES; ++p) {
    const int r = p * RPP + threadIdx.x / LPR, row = r0 + r;
#pragma unroll
    for (int j = 0; j < EPL; ++j) s_x[r][lc + j] = v[p][j];
    if (row < rows && valid > 0)
      store_e4m3<EPL, kVec>(q + static_cast<long long>(row) * cols + col, valid, v[p],
                            scale_of(__uint_as_float(row_amax[row])));
  }
  if (c0 == 0)
    for (int r = threadIdx.x; r < kTile && r0 + r < rows; r += kDualThreads)
      scale[r0 + r] = scale_of(__uint_as_float(row_amax[r0 + r]));
  if (r0 == 0)
    for (int c = threadIdx.x; c < kTile && c0 + c < cols; c += kDualThreads)
      scale_t[c0 + c] = scale_of(__uint_as_float(col_amax[c0 + c]));
  __syncthreads();
  const int c = threadIdx.x % kTile, h = threadIdx.x / kTile;
  if (c0 + c >= cols) return;
  const float s = scale_of(__uint_as_float(col_amax[c0 + c]));
  uint8_t* dst = q_t + static_cast<long long>(c0 + c) * ld_t + r0;
#pragma unroll
  for (int v16 = 0; v16 < 2; ++v16) {
    const int r = h * 32 + v16 * 16;
    if (r0 + r >= ld_t) break;   // ld_t % 16 == 0: a 16-row vector is all padding-or-data, or past the end
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      w[k] = e4m3x2(quotient(s_x[r + 4 * k][c], s), quotient(s_x[r + 4 * k + 1][c], s)) |
             (e4m3x2(quotient(s_x[r + 4 * k + 2][c], s), quotient(s_x[r + 4 * k + 3][c], s)) << 16);
    *reinterpret_cast<uint4*>(dst + r) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

}  // namespace quant
}  // namespace b200

namespace {

using namespace b200::quant;

std::atomic<unsigned long long> g_launches{0};

bool aligned(const void* p, unsigned bytes) { return reinterpret_cast<uintptr_t>(p) % bytes == 0; }

int launched(cudaError_t e) {
  if (e != cudaSuccess) return int(e);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return kDualOk;
}

long long tiles(int rows, int cols, int tile_rows, int tile_cols) {
  return static_cast<long long>((rows + tile_rows - 1) / tile_rows) * ((cols + tile_cols - 1) / tile_cols);
}

struct DualLaunch {
  const void* x;
  int rows, cols;
  void* q;
  float* scale;
  void* q_t;
  float* scale_t;
  float* workspace;
  cudaStream_t st;
  bool vec(int epl) const { return aligned(x, 16) && aligned(q, epl) && cols % epl == 0; }
  template <typename T, int EPL, bool kVec>
  int run() const {
    unsigned* row_amax = reinterpret_cast<unsigned*>(workspace);
    unsigned* col_amax = row_amax + rows;
    const cudaError_t e = cudaMemsetAsync(workspace, 0, sizeof(float) * CUDA_L2_B200_QUANT_DUAL_WORKSPACE(rows, cols),
                                          st);
    if (e != cudaSuccess) return int(e);
    const int amax_col_tiles = (cols + 32 * EPL - 1) / (32 * EPL);
    b200::quant::b200_quant_dual_amax_kernel<T, EPL, kVec>
        <<<int(tiles(rows, cols, kAmaxRows, 32 * EPL)), kAmaxThreads, 0, st>>>(static_cast<const T*>(x), rows, cols,
                                                                               amax_col_tiles, row_amax, col_amax);
    if (const int err = launched(cudaGetLastError())) return err;
    const int col_tiles = (cols + kTile - 1) / kTile;
    b200::quant::b200_quant_dual_kernel<T, EPL, kVec><<<int(tiles(rows, cols, kTile, kTile)), kDualThreads, 0, st>>>(
        static_cast<const T*>(x), rows, cols, col_tiles, (rows + 15) / 16 * 16, static_cast<uint8_t*>(q), scale,
        static_cast<uint8_t*>(q_t), scale_t, row_amax, col_amax);
    return launched(cudaGetLastError());
  }
};

}  // namespace

extern "C" {

int cuda_l2_b200_quant_dual_e4m3_rowwise(int dtype, const void* x, int rows, int cols, void* q, float* scale,
                                         void* q_t, float* scale_t, float* workspace, void* stream) {
  if (dtype < 0 || dtype > 2) return kDualBadDtype;
  if (x == nullptr || q == nullptr || scale == nullptr || q_t == nullptr || scale_t == nullptr || workspace == nullptr)
    return kDualNullPointer;
  if (rows <= 0 || cols <= 0 || rows > INT_MAX - 15) return kDualBadShape;
  if (tiles(rows, cols, kTile, kTile) > INT_MAX) return kDualBadShape;   // one CTA per 64 x 64 tile, in a 1-D grid
  if (!aligned(scale, 4) || !aligned(scale_t, 4) || !aligned(workspace, 4) || !aligned(q_t, 16))
    return kDualBadAlignment;
  const DualLaunch l{x, rows, cols, q, scale, q_t, scale_t, workspace, static_cast<cudaStream_t>(stream)};
  switch (dtype) {
    case 0: return l.vec(8) ? l.run<__half, 8, true>() : l.run<__half, 4, false>();
    case 1: return l.vec(8) ? l.run<__nv_bfloat16, 8, true>() : l.run<__nv_bfloat16, 4, false>();
    default: return l.vec(4) ? l.run<float, 4, true>() : l.run<float, 4, false>();
  }
}

unsigned long long cuda_l2_b200_quant_dual_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

const char* cuda_l2_b200_quant_dual_strerror(int status) {
  switch (status) {
    case kDualOk: return "ok";
    case kDualBadShape: return "rows and cols must be positive, rows at most INT_MAX - 15";
    case kDualBadAlignment: return "scale, scale_t and workspace must be 4-byte aligned, q_t 16-byte aligned";
    case kDualNullPointer: return "null pointer";
    case kDualBadDtype: return "unknown input dtype (0 fp16, 1 bf16, 2 fp32)";
    default: return status > 0 ? cudaGetErrorString(static_cast<cudaError_t>(status)) : "unknown status";
  }
}

}  // extern "C"
