// b200_quant_arith.cuh — the element arithmetic the e4m3 quantisers share (libb200_quant.so, libb200_quant_dual.so):
// torch.amax's NaN-keeping max, the scale, the IEEE quotient, e4m3 rounding, and the vector loads and stores. The rule
// they implement is stated in b200_quant.h; both libraries produce the same bits because they compile this one text.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>

namespace b200 {
namespace quant {

constexpr float kE4M3Max = 448.0f;
// torch's CUDA `tensor / 448.0` multiplies by the fp32 reciprocal of the scalar (see b200_quant.h)
constexpr float kInvE4M3Max = 1.0f / 448.0f;

// ------------------------------------------------------------------------------------------------ element arithmetic
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_f32(float v) { return v; }

// max that keeps a NaN once it has seen one (torch.amax), unlike fmaxf
__device__ __forceinline__ float nan_max(float m, float a) { return (a > m || a != a) ? a : m; }

__device__ __forceinline__ float scale_of(float amax) {
  const float s = amax * kInvE4M3Max;
  return s < FLT_MIN ? FLT_MIN : s;   // clamp_min(FLT_MIN); NaN stays NaN
}

// clamp(x / s, -448, 448) with an IEEE division; a NaN quotient passes the clamp unchanged
__device__ __forceinline__ float quotient(float x, float s) {
  const float v = __fdiv_rn(x, s);
  return v != v ? v : fminf(fmaxf(v, -kE4M3Max), kE4M3Max);
}

// e4m3fn bytes of two clamped quotients, lo in bits 0-7: round to nearest even; NaN is 0x7f with the input's sign
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  unsigned short r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  uint32_t out = r;
  if (lo != lo) out = (out & 0xff00u) | 0x7fu | ((__float_as_uint(lo) >> 24) & 0x80u);
  if (hi != hi) out = (out & 0x00ffu) | ((0x7fu | ((__float_as_uint(hi) >> 24) & 0x80u)) << 8);
  return out;
}

__device__ __forceinline__ uint8_t e4m3(float v) { return uint8_t(e4m3x2(v, 0.0f)); }

// EPL consecutive elements from p, as fp32: one 16-byte load when kVec, EPL element loads otherwise (only the first
// `valid` of them are read; the rest are 0)
template <typename T, int EPL, bool kVec>
__device__ __forceinline__ void load_f32(const T* p, int valid, float (&v)[EPL]) {
  if constexpr (kVec) {
    static_assert(EPL * sizeof(T) == 16, "one 16-byte vector");
    const uint4 raw = __ldg(reinterpret_cast<const uint4*>(p));
    const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int j = 0; j < EPL; ++j) v[j] = to_f32(e[j]);
  } else {
#pragma unroll
    for (int j = 0; j < EPL; ++j) v[j] = j < valid ? to_f32(p[j]) : 0.0f;
  }
}

// EPL quantised bytes to q: one 4- or 8-byte store when kVec, byte stores of the first `valid` otherwise
template <int EPL, bool kVec>
__device__ __forceinline__ void store_e4m3(uint8_t* q, int valid, const float (&v)[EPL], float s) {
  if constexpr (kVec) {
    uint32_t w[EPL / 4];
#pragma unroll
    for (int j = 0; j < EPL / 4; ++j)
      w[j] = e4m3x2(quotient(v[4 * j], s), quotient(v[4 * j + 1], s)) |
             (e4m3x2(quotient(v[4 * j + 2], s), quotient(v[4 * j + 3], s)) << 16);
    if constexpr (EPL == 8)
      *reinterpret_cast<uint2*>(q) = make_uint2(w[0], w[1]);
    else
      *reinterpret_cast<uint32_t*>(q) = w[0];
  } else {
#pragma unroll
    for (int j = 0; j < EPL; ++j)
      if (j < valid) q[j] = e4m3(quotient(v[j], s));
  }
}

template <int LANES>
__device__ __forceinline__ float group_amax(float m) {   // over aligned groups of LANES lanes
#pragma unroll
  for (int off = LANES / 2; off > 0; off /= 2) m = nan_max(m, __shfl_xor_sync(0xffffffffu, m, off));
  return m;
}

// every thread gets the CTA's amax; red holds a float per warp of the CTA (blockDim.x a multiple of 32)
__device__ __forceinline__ float cta_amax(float m, float* red) {
  m = group_amax<32>(m);
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  __syncthreads();   // red may still be read from an earlier call
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = lane < int(blockDim.x / 32) ? red[lane] : 0.0f;
  return group_amax<32>(m);
}

}  // namespace quant
}  // namespace b200
