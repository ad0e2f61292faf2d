// libb200_grouped_swiglu.so — the gate / up projection of the SwiGLU experts of a mixture-of-experts layer, over
// contiguous row groups, with the activation fused into the GEMM epilogue (Gated<Grouped<>> configurations,
// hgemm_sm90.cuh), and the one-pass SwiGLU backward over the groups' rows. Not a public ABI: nothing under include/
// declares these functions, and their names do not start with b200_. cuda_l2_b200/capi.py binds them.
//
// Layout: the tokens x [T, H] are sorted by expert; group g owns rows [start_g, end_g) with start_0 = 0,
// start_g = end_{g-1} and end_g = clamp(offs[g], start_g, T), the rule of include/b200_grouped.h. The weight stack
// w_gu [G, 2I, H] holds one fused gate / up weight per expert in libb200_swiglu.so's layout (csrc/b200_swiglu.h): rows
// [128 b, 128 b + 64) of expert g are its gate rows [64 b, 64 b + 64), the next 64 its matching up rows. The product
// h [T, 2I] (rows of group g: x[rows] w_gu[g]^T) is then [g | u] per 128 columns.
//
// Forward, per element of y [T, I] below the last group's end: y = silu_mul(RN(g), RN(u)), torch's `F.silu(g) * u` on
// the 16-bit h, bit for bit. h itself, when requested, is libb200_grouped.so's output with the same configuration, bit
// for bit. Rows of h and y at or past the last group's end are never written.
//
// Backward, per element below `end`, the groups' last end (clamp(offs[G-1], 0, T) for non-decreasing offsets; the
// largest end of the clamped groups in general), read on the device: the SwiGLU gradient of libb200_swiglu.so
// (swiglu_grad of swiglu_arith.cuh) into dh [T, 2I] in h's layout. Rows of dy and h at or past `end` are never read,
// and rows of dh there never written, so capacity padding past the routed tokens costs nothing and needs no host
// synchronisation.
//
// `variant` is the GemmType index: 0 fp16, 2 bf16 (fp32 accumulation). x, w_gu, h, y, dy and dh are contiguous and
// 16-byte aligned, offs (G int32 values, device memory) 4-byte aligned; H % 8 == 0 and I % 64 == 0. h may be null in
// the forward (y only). T == 0 is an empty problem: it launches nothing. The argument rules are checked before any CUDA
// call, in this order: the variant, null pointers, the shape (T >= 0, G >= 1, I > 0, H > 0), I's multiple of 64,
// alignment (H % 8, then the pointers, then the offsets), and the worst-case tile list (GroupCursor::max_tiles) of at
// most INT_MAX tiles.
#pragma once
#include "b200_swiglu.h"   // the SwiGLU statuses kSwigluBadWidth and kSwigluBadDtype, which this library shares

extern "C" {

// The dispatched call: the grouped dispatcher's choice for (G, T, 2I, H) of the same variant (tile_list::select),
// mapped through gated::sibling (cuda_l2_b200_grouped_swiglu_select).
int cuda_l2_b200_grouped_swiglu_run(int variant, const void* x, const void* w_gu, void* h, void* y, const int* offs,
                                    int G, int T, int I, int H, void* stream);

// Configuration `config_id` (gated::has_kernel: BN = 128 or 256; others are kBadConfig), with group_m and max_ctas as
// for b200_grouped_gemm_run_config.
int cuda_l2_b200_grouped_swiglu_run_config(int variant, int config_id, const void* x, const void* w_gu, void* h,
                                           void* y, const int* offs, int G, int T, int I, int H, int group_m,
                                           int max_ctas, void* stream);

// The dispatched call's choice, into the optional out-parameters.
int cuda_l2_b200_grouped_swiglu_select(int variant, int G, int T, int I, int H, int* config_id, int* group_m);

// dh [T, 2I] = the SwiGLU gradient of dy [T, I] at h [T, 2I] (above), rows below the groups' last end only. T == 0
// launches nothing, and dy, h and dh may then be null (torch's pointer for a tensor without elements).
int cuda_l2_b200_grouped_swiglu_backward(int variant, const void* dy, const void* h, void* dh, const int* offs, int G,
                                         int T, int I, void* stream);

// Kernel launches of the library (forward and backward).
unsigned long long cuda_l2_b200_grouped_swiglu_launch_count(void);

const char* cuda_l2_b200_grouped_swiglu_strerror(int status);

}  // extern "C"
