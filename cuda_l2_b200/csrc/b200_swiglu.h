// libb200_swiglu.so — the gate / up projection of a SwiGLU MLP with its activation fused into the GEMM epilogue
// (Gated<> configurations, hgemm_sm90.cuh), and the one-pass SwiGLU backward. Not a public ABI: nothing under include/
// declares these functions, and their names do not start with b200_. cuda_l2_b200/capi.py binds them.
//
// Layout: the weight w_gu [2I, K] holds the gate and up weights interleaved in 64-row blocks: rows [128 b, 128 b + 64)
// are gate rows [64 b, 64 b + 64), rows [128 b + 64, 128 b + 128) the matching up rows. The product h = x w_gu^T [M, 2I]
// is then [g | u] per 128 columns, and for y column j = 64 b + c: g = h[:, 128 b + c], u = h[:, 128 b + 64 + c].
//
// Forward, per element of y [M, I], with s(m, n) the fp32 sum of the TN call of the same variant and configuration:
//   y = RN(fp32(RN(silu(RN(g)))) * fp32(RN(u)))     silu(v) = v / (1 + expf(-v)) in fp32 (swiglu_arith.cuh)
// which is torch's `F.silu(g) * u` on the 16-bit h, bit for bit. h itself, when requested, is the TN call's output bit
// for bit (the unchanged store path).
//
// Backward, per element, from dy [M, I] and the 16-bit h (swiglu_grad of swiglu_arith.cuh, the steps of torch's
// autograd through `F.silu(g) * u`):
//   du = RN(dy * RN(silu(g)))
//   dg = RN((RN(dy * u) * sig) * fmaf(g, 1 - sig, 1)),   sig = 1 / (1 + expf(-g))
// each product and quotient one IEEE fp32 operation, written into dh [M, 2I] in h's interleaved layout.
//
// `variant` is the GemmType index: 0 fp16, 2 bf16 (fp32 accumulation). x [M, K], w_gu [2I, K], h [M, 2I], y [M, I],
// dy [M, I] and dh [M, 2I] are contiguous and 16-byte aligned; K % 8 == 0 and I % 64 == 0. h may be null in the forward
// (y only). The argument rules are checked before any CUDA call, in this order: the variant, null pointers, the shape,
// I's multiple of 64, then alignment.
#pragma once
#include "hgemm_host.cuh"

// The library's own statuses, beyond those of b200_hgemm_strerror (cuda_l2_b200_swiglu_strerror decodes both).
enum SwigluStatus : int {
  kSwigluBadWidth = -14,   // I must be a multiple of 64 (whole 64-row gate / up blocks)
  kSwigluBadDtype = -15,   // variant must be 0 (fp16) or 2 (bf16)
};

extern "C" {

// The dispatched call: the TN dispatcher's choice for (M, 2I, K) of the same variant, mapped through gated::sibling and
// run on the plain schedule (cuda_l2_b200_swiglu_select).
int cuda_l2_b200_swiglu_run(int variant, const void* x, const void* w_gu, void* h, void* y, int M, int I, int K,
                            void* stream);

// Configuration `config_id` (gated::has_kernel: BN = 128 or 256; others are kBadConfig), with group_m and max_ctas as
// for b200_hgemm_run_config; every `splits` code runs the plain schedule.
int cuda_l2_b200_swiglu_run_config(int variant, int config_id, const void* x, const void* w_gu, void* h, void* y, int M,
                                   int I, int K, int group_m, int splits, int max_ctas, void* stream);

// The dispatched call's choice, into the optional out-parameters (splits is always 1: the plain schedule).
int cuda_l2_b200_swiglu_select(int variant, int M, int I, int K, int* config_id, int* group_m, int* splits);

// dh [M, 2I] = the SwiGLU gradient of dy [M, I] at h [M, 2I] (above). M == 0 launches nothing.
int cuda_l2_b200_swiglu_backward(int variant, const void* dy, const void* h, void* dh, int M, int I, void* stream);

// Kernel launches of the library (forward and backward).
unsigned long long cuda_l2_b200_swiglu_launch_count(void);

const char* cuda_l2_b200_swiglu_strerror(int status);

}  // extern "C"
