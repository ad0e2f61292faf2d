// swiglu_arith.cuh — the SwiGLU element arithmetic of torch's `F.silu(g) * u` on 16-bit tensors, shared by the SwiGLU
// quantiser (libb200_quant.so), the gated GEMM epilogue (Gated<>, hgemm_sm90.cuh) and the SwiGLU backward
// (libb200_swiglu.so), so that all three produce torch's bits from one text. Every step is an IEEE fp32 operation,
// expf is CUDA's full-precision one, and RN is round-to-nearest-even to the 16-bit type T.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace b200 {

// RN to the 16-bit type of the second argument, back as fp32 (exact)
__device__ __forceinline__ float round_to(float v, __half) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ float round_to(float v, __nv_bfloat16) { return __bfloat162float(__float2bfloat16_rn(v)); }

// torch's silu, x / (1 + exp(-x)) in fp32, rounded to T: the tensor `F.silu(g)` holds
template <typename T>
__device__ __forceinline__ float silu_rn(float g) { return round_to(__fdiv_rn(g, 1.0f + expf(-g)), T()); }

// the SwiGLU product p = RN(fp32(RN(silu(g))) * fp32(u)) of torch's `F.silu(g) * u` on 16-bit tensors
template <typename T>
__device__ __forceinline__ float silu_mul(float g, float u) {
  const float s = silu_rn<T>(g);
  return round_to(s * u, T());
}

// The gradient torch's autograd computes for y = F.silu(g) * u on 16-bit tensors, from the output gradient dy and the
// 16-bit g and u (all as fp32):
//   s   = RN(g / (1 + expf(-g)))                       the saved silu output (silu_rn)
//   du  = RN(dy * s)                                   mul's gradient of u
//   t   = RN(dy * u)                                   mul's gradient of s, a 16-bit tensor
//   sig = 1 / (1 + expf(-g))                           IEEE quotient
//   dg  = RN((t * sig) * fmaf(g, 1 - sig, 1))          silu_backward's dy * sig * (1 + x * (1 - sig)), evaluated left to
//                                                      right with x * (1 - sig) + 1 contracted into one FMA
template <typename T>
__device__ __forceinline__ void swiglu_grad(float dy, float g, float u, float& dg, float& du) {
  du = round_to(__fmul_rn(dy, silu_rn<T>(g)), T());
  const float t = round_to(__fmul_rn(dy, u), T());
  const float sig = __fdiv_rn(1.0f, 1.0f + expf(-g));   // the denominator as silu_rn writes it (torch's text too)
  dg = round_to(__fmul_rn(__fmul_rn(t, sig), __fmaf_rn(g, __fsub_rn(1.0f, sig), 1.0f)), T());
}

}  // namespace b200
