// libb200_quant_block_dual.so — the dual-orientation block e4m3 quantisers (b200_quant_block_dual.h): from one tensor,
// its 1 x 128 (or 128 x 128) quantisation and that of its transpose, the two K-major operands blockwise FP8 training
// needs of x, dY and W. One CTA per 128 x 128 tile, which holds complete groups in both orientations: x is read once,
// each e4m3 byte written once, no atomics and no workspace. A library of its own, so that libb200_quant.so and
// libb200_quant_dual.so stay as they are; the element arithmetic is shared with them (b200_quant_arith.cuh).
#include "b200_quant_block_dual.h"
#include "b200_quant_arith.cuh"

#include <atomic>
#include <climits>

namespace b200 {
namespace quant {

enum BlockDualStatus : int {
  kBlockDualOk = 0,
  kBlockDualBadShape = -1,
  kBlockDualBadAlignment = -2,
  kBlockDualNullPointer = -5,
  kBlockDualBadDtype = -6,
};

constexpr int kTile = 128, kThreads = 256;
constexpr int kEPL = 8;                          // elements per lane and pass: one 16-byte load of a 16-bit row
constexpr int kLPR = kTile / kEPL;               // lanes per tile row (a half-warp)
constexpr int kRPP = kThreads / kLPR;            // tile rows per pass
constexpr int kPasses = kTile / kRPP;
constexpr int kWarps = kThreads / 32;
constexpr int kStageLd = kTile + 2;              // halves per staged row: rows 16 apart fall in different banks

template <typename T>
__device__ __forceinline__ float from_bits(uint16_t b) {
  return to_f32(*reinterpret_cast<const T*>(&b));
}

// One CTA per 128 x 128 tile of x [rows, cols] (fp16 or bf16). kBlock128: one scale for the tile (128 x 128 blocks);
// otherwise one per tile row (q's 1 x 128 groups) and one per tile column (q_t's). The tile is loaded once, row-major
// (a half-warp per row, 16 bytes per lane and pass), into registers and, as its 16-bit bits, into shared memory; rows
// and columns past x's edge are +0.0. q is stored from registers with the row scales; q_t from shared memory, each
// thread quantising 16 rows of one column with the column's scale into one 16-byte store (two lanes per column, so a
// warp writes whole 32-byte sectors), or byte stores where q_t's row length ld_t is no multiple of 16.
template <typename T, bool kVec, bool kBlock128>
__global__ void __launch_bounds__(kThreads) b200_quant_block_dual_kernel(
    const T* __restrict__ x, int rows, int cols, int col_tiles, uint8_t* __restrict__ q, float* __restrict__ scale,
    int ld_s, uint8_t* __restrict__ q_t, int ld_t, float* __restrict__ scale_t, int ld_st) {
  static_assert(sizeof(T) == 2, "16-bit inputs");
  __shared__ uint16_t s_x[kTile][kStageLd];
  __shared__ float s_cmax[kWarps][kTile];   // per warp: the column maxima of its rows
  __shared__ float s_cscale[kTile];         // the scale of each tile column (q_t's groups)
  __shared__ float s_red[kWarps];
  const int rb = blockIdx.x / col_tiles, cb = blockIdx.x % col_tiles;
  const int r0 = rb * kTile, c0 = cb * kTile;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int lc = (threadIdx.x % kLPR) * kEPL, col = c0 + lc;
  const int valid = min(max(cols - col, 0), kEPL);
  float v[kPasses][kEPL];
#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    const int r = p * kRPP + threadIdx.x / kLPR, row = r0 + r;
    uint16_t raw[kEPL];
    if (row < rows && valid > 0) {
      const uint16_t* src = reinterpret_cast<const uint16_t*>(x) + static_cast<long long>(row) * cols + col;
      if constexpr (kVec) {
        const uint4 w = __ldg(reinterpret_cast<const uint4*>(src));
        const uint16_t* e = reinterpret_cast<const uint16_t*>(&w);
#pragma unroll
        for (int j = 0; j < kEPL; ++j) raw[j] = e[j];
      } else {
#pragma unroll
        for (int j = 0; j < kEPL; ++j) raw[j] = j < valid ? src[j] : uint16_t(0);
      }
    } else {
#pragma unroll
      for (int j = 0; j < kEPL; ++j) raw[j] = 0;
    }
#pragma unroll
    for (int j = 0; j < kEPL; ++j) v[p][j] = from_bits<T>(raw[j]);
    uint32_t* srow = reinterpret_cast<uint32_t*>(&s_x[r][lc]);   // kStageLd and lc are even: 4-byte aligned pairs
#pragma unroll
    for (int j = 0; j < kEPL / 2; ++j) srow[j] = uint32_t(raw[2 * j]) | (uint32_t(raw[2 * j + 1]) << 16);
  }
  // the maxima of |x|: per row (across the half-warp), per column (over the passes, the two half-warps, the warps)
  float rmax[kPasses], cmax[kEPL];
#pragma unroll
  for (int j = 0; j < kEPL; ++j) cmax[j] = 0.0f;
#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    float m = 0.0f;
#pragma unroll
    for (int j = 0; j < kEPL; ++j) {
      const float a = fabsf(v[p][j]);
      m = nan_max(m, a);
      cmax[j] = nan_max(cmax[j], a);
    }
    rmax[p] = group_amax<kLPR>(m);
  }
  if constexpr (kBlock128) {
    float m = 0.0f;
#pragma unroll
    for (int p = 0; p < kPasses; ++p) m = nan_max(m, rmax[p]);
    const float s = scale_of(cta_amax(m, s_red));   // every thread: the tile's scale
#pragma unroll
    for (int p = 0; p < kPasses; ++p) rmax[p] = s;
    if (threadIdx.x < kTile) s_cscale[threadIdx.x] = s;
    if (threadIdx.x == 0) {
      const int row_tiles = (rows + kTile - 1) / kTile;
      scale[rb * col_tiles + cb] = s;
      scale_t[cb * row_tiles + rb] = s;
    }
  } else {
#pragma unroll
    for (int j = 0; j < kEPL; ++j) {
      cmax[j] = nan_max(cmax[j], __shfl_xor_sync(0xffffffffu, cmax[j], 16));
      if (lane < kLPR) s_cmax[warp][lc + j] = cmax[j];
    }
#pragma unroll
    for (int p = 0; p < kPasses; ++p) {
      rmax[p] = scale_of(rmax[p]);
      const int row = r0 + p * kRPP + threadIdx.x / kLPR;
      if (threadIdx.x % kLPR == 0 && row < rows) scale[static_cast<long long>(cb) * ld_s + row] = rmax[p];
    }
  }
  // q, row-major from registers (rmax now holds each row's scale)
#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    const int row = r0 + p * kRPP + threadIdx.x / kLPR;
    if (row < rows && valid > 0)
      store_e4m3<kEPL, kVec>(q + static_cast<long long>(row) * cols + col, valid, v[p], rmax[p]);
  }
  __syncthreads();
  if constexpr (!kBlock128) {
    if (threadIdx.x < kTile) {
      float m = 0.0f;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) m = nan_max(m, s_cmax[w][threadIdx.x]);
      const float s = scale_of(m);
      s_cscale[threadIdx.x] = s;
      if (c0 + int(threadIdx.x) < cols) scale_t[static_cast<long long>(rb) * ld_st + c0 + threadIdx.x] = s;
    }
    __syncthreads();
  }
  // q_t: rows c0 + c of q_t, columns r0 + 16 k .. + 15; lanes 2i and 2i + 1 take one column's adjacent 16-row chunks
#pragma unroll
  for (int i = 0; i < kTile * (kTile / 16) / kThreads; ++i) {
    const int c = threadIdx.x / 2, k = 2 * i + (threadIdx.x & 1);
    const int r = 16 * k;
    if (c0 + c >= cols || r0 + r >= ld_t) continue;
    const float s = s_cscale[c];
    uint8_t* dst = q_t + static_cast<long long>(c0 + c) * ld_t + r0 + r;
    if ((ld_t & 15) == 0) {   // a 16-row chunk lies wholly inside ld_t
      uint32_t w[4];
#pragma unroll
      for (int e = 0; e < 4; ++e)
        w[e] = e4m3x2(quotient(from_bits<T>(s_x[r + 4 * e][c]), s), quotient(from_bits<T>(s_x[r + 4 * e + 1][c]), s)) |
               (e4m3x2(quotient(from_bits<T>(s_x[r + 4 * e + 2][c]), s),
                       quotient(from_bits<T>(s_x[r + 4 * e + 3][c]), s)) << 16);
      *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
      for (int e = 0; e < 16 && r0 + r + e < ld_t; ++e) dst[e] = e4m3(quotient(from_bits<T>(s_x[r + e][c]), s));
    }
  }
}

}  // namespace quant
}  // namespace b200

namespace {

using namespace b200::quant;

std::atomic<unsigned long long> g_launches{0};

bool aligned(const void* p, unsigned bytes) { return reinterpret_cast<uintptr_t>(p) % bytes == 0; }

long long tiles(int rows, int cols) {
  return static_cast<long long>((rows + kTile - 1) / kTile) * ((cols + kTile - 1) / kTile);
}

// The argument rules of both entry points, before any CUDA call.
int check(int dtype, const void* x, int rows, int cols, const void* q, const float* scale, const void* q_t,
          const float* scale_t) {
  if (dtype != 0 && dtype != 1) return kBlockDualBadDtype;
  if (!x || !q || !scale || !q_t || !scale_t) return kBlockDualNullPointer;
  if (rows <= 0 || cols <= 0 || rows > INT_MAX - 15 || tiles(rows, cols) > INT_MAX) return kBlockDualBadShape;
  if (!aligned(scale, 4) || !aligned(scale_t, 4) || !aligned(q_t, 16)) return kBlockDualBadAlignment;
  return kBlockDualOk;
}

template <bool kBlock128>
int launch(int dtype, const void* x, int rows, int cols, void* q, float* scale, void* q_t, int ld_t, float* scale_t,
           void* stream) {
  const int col_tiles = (cols + kTile - 1) / kTile;
  const int ld_s = (rows + 3) / 4 * 4, ld_st = (cols + 3) / 4 * 4;
  const bool vec = aligned(x, 16) && aligned(q, 8) && cols % kEPL == 0;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto go = [&](auto kernel, auto* xt) {
    kernel<<<int(tiles(rows, cols)), kThreads, 0, st>>>(xt, rows, cols, col_tiles, static_cast<uint8_t*>(q), scale,
                                                         ld_s, static_cast<uint8_t*>(q_t), ld_t, scale_t, ld_st);
  };
  if (dtype == 0) {
    const __half* xt = static_cast<const __half*>(x);
    if (vec) go(b200_quant_block_dual_kernel<__half, true, kBlock128>, xt);
    else go(b200_quant_block_dual_kernel<__half, false, kBlock128>, xt);
  } else {
    const __nv_bfloat16* xt = static_cast<const __nv_bfloat16*>(x);
    if (vec) go(b200_quant_block_dual_kernel<__nv_bfloat16, true, kBlock128>, xt);
    else go(b200_quant_block_dual_kernel<__nv_bfloat16, false, kBlock128>, xt);
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return int(e);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return kBlockDualOk;
}

}  // namespace

extern "C" {

int cuda_l2_b200_quant_block_dual_e4m3_1x128(int dtype, const void* x, int rows, int cols, void* q, float* scale,
                                             void* q_t, float* scale_t, void* stream) {
  if (const int st = check(dtype, x, rows, cols, q, scale, q_t, scale_t)) return st;
  return launch<false>(dtype, x, rows, cols, q, scale, q_t, (rows + 15) / 16 * 16, scale_t, stream);
}

int cuda_l2_b200_quant_block_dual_e4m3_128x128(int dtype, const void* w, int rows, int cols, void* q, float* scale,
                                               void* q_t, float* scale_t, void* stream) {
  if (const int st = check(dtype, w, rows, cols, q, scale, q_t, scale_t)) return st;
  return launch<true>(dtype, w, rows, cols, q, scale, q_t, rows, scale_t, stream);
}

unsigned long long cuda_l2_b200_quant_block_dual_launch_count(void) {
  return g_launches.load(std::memory_order_relaxed);
}

const char* cuda_l2_b200_quant_block_dual_strerror(int status) {
  switch (status) {
    case kBlockDualOk: return "ok";
    case kBlockDualBadShape: return "rows and cols must be positive, rows at most INT_MAX - 15, at most INT_MAX tiles";
    case kBlockDualBadAlignment: return "scale and scale_t must be 4-byte aligned, q_t 16-byte aligned";
    case kBlockDualNullPointer: return "null pointer";
    case kBlockDualBadDtype: return "unknown input dtype (0 fp16, 1 bf16)";
    default: return status > 0 ? cudaGetErrorString(static_cast<cudaError_t>(status)) : "unknown status";
  }
}

}  // extern "C"
