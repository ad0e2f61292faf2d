// libb200_grouped_bwd.so — the backward of the grouped product of libb200_grouped.so (the MoE experts' training
// step), fp16 or bf16 operands with fp32 accumulation. Not a public ABI: nothing under include/ declares these
// functions, and their names do not start with b200_. cuda_l2_b200/capi.py binds them.
//
// With the forward Y[start_g : end_g] = X[start_g : end_g] W[g]^T (X [T, K_model], W [G, N_model, K_model]) and the
// groups of include/b200_grouped.h (start_0 = 0, start_g = end_{g-1}, end_g = clamp(offs[g], start_g, T)):
//   input gradient   dX[start_g : end_g] = dY[start_g : end_g] W[g]          the grouped row-major B (NN) product
//   weight gradient  dW[g] = dY[start_g : end_g]^T X[start_g : end_g]        the K-grouped product
// Below, M, N and K are each product's own names. `variant` is the GemmType index: 0 fp16 or 2 bf16 (fp32
// accumulation; the output has the operands' type). Statuses are those of b200_hgemm_strerror.
#pragma once
#include "hgemm_host.cuh"

extern "C" {

// Grouped row-major B: C[start_g : end_g] = A[start_g : end_g] B[g] for g < G, A [T, K], B [G, K, N] row-major (N
// contiguous: the weight stack [G, N_model, K_model] read in place), C [T, N], all contiguous. Rows of C at or past
// end_{G-1} are not written. `offs` (G int32 values, device memory) is read by the kernel. config_id < 0: the
// dispatcher's choice (group_m and max_ctas are then ignored); otherwise that configuration (one with a row-major B
// kernel, BN >= 64), group_m <= 0 its default rasterisation, max_ctas <= 0 all SMs. K % 8 and N % 8 == 0, G >= 1,
// T >= 0 (T == 0 launches nothing).
int cuda_l2_b200_grouped_bwd_nn(int variant, int config_id, const void* A, const void* B_rowmajor, void* C,
                                const int* offs, int G, int T, int N, int K, int group_m, int max_ctas, void* stream);

// K-grouped: C[g] = A[start_g : end_g]^T B[start_g : end_g] for g < G, A [T, M] and B [T, N] row-major, C [G, M, N],
// all contiguous. Every matrix of C is written; an empty group's is +0.0, and T == 0 zero-fills C on the stream
// without a launch. Rows of A and B at or past end_{G-1} do not reach C. config_id, group_m and max_ctas as above.
// M % 8 and N % 8 == 0, G >= 1, T >= 0; with T == 0, A and B are not read and may be null.
int cuda_l2_b200_grouped_bwd_wgrad(int variant, int config_id, const void* A, const void* B, void* C, const int* offs,
                                   int G, int T, int M, int N, int group_m, int max_ctas, void* stream);

// The dispatcher's choice for each kind (no tuned table: the forward's rules, mapped to a configuration with a
// row-major B kernel), into the optional out-parameters.
int cuda_l2_b200_grouped_bwd_nn_select(int variant, int G, int T, int N, int K, int* config_id, int* group_m);
int cuda_l2_b200_grouped_bwd_wgrad_select(int variant, int G, int T, int M, int N, int* config_id, int* group_m);

// Host view of worker `worker`'s tiles of a K-grouped launch of configuration `config_id` with the host copy
// `offs_host` of the offsets, on a device of num_sms SMs (every cluster resident) with the default rasterisation:
// (group, m_block, n_block, k-blocks) per tile into `units` (at most max_units). Returns the tile count, or a status.
int cuda_l2_b200_grouped_bwd_wgrad_schedule(int config_id, int G, int T, int M, int N, const int* offs_host,
                                            int num_sms, int worker, int* units, int max_units, int* num_workers);

// Kernel launches of the library.
unsigned long long cuda_l2_b200_grouped_bwd_launch_count(void);

const char* cuda_l2_b200_grouped_bwd_strerror(int status);

}  // extern "C"
