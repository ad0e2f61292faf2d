// The body of the SwiGLU backward, dh = swiglu_grad(dy, h), shared by libb200_swiglu.so's kernel and
// libb200_grouped_swiglu.so's, which differ only in how many rows they cover. Only those two libraries include it.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstdint>
#include <type_traits>

#include "ptx_sm90.cuh"
#include "swiglu_arith.cuh"

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

// dh = swiglu_grad(dy, h) over the first `vectors` / (I / 8) rows: one thread per eight consecutive columns of y (one
// 16-byte vector of dy, of g, of u, of dg and of du), grid-stride over the vectors of a kBwdThreads-thread block.
// I % 64 == 0: the eight columns lie in one 64-column gate / up block.
template <typename T>
__device__ __forceinline__ void backward_vectors(const T* __restrict__ dy, const T* __restrict__ h, T* __restrict__ dh,
                                                 long long vectors, int I) {
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

}  // namespace swiglu
}  // namespace b200
