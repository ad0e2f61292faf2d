// libb200_nn.so — the row-major B (NN) kernels, C[M,N] = A[M,K] B[K,N] with B row-major (N contiguous): the
// RowMajorB<> configurations of the three 16-bit variants. Not a public ABI. The drop-in entry points of
// libb200_hgemm.so (include/b200_hgemm.h) reach it when they get B_rowmajor and no B_kmajor: they check the arguments,
// take the dispatcher's choice, load this library next to themselves on the first such call and call the one function
// below, which they resolve by name. Its name does not start with b200_, so that no public symbol is added.
#pragma once
#include "hgemm_host.cuh"

extern "C" {

// Configuration `config_id` (one with an NN kernel: nn::has_kernel) of variant `variant` (the GemmType index: 0 fp16
// with fp32 accumulation, 1 fp16 with fp16 accumulation, 2 bf16), with the arguments of b200_hgemm_run_config and
// B_rowmajor [K,N] in place of B_kmajor. The workspace of a split-K or stream-K launch comes from `scratch` (the pool of
// the calling library). Returns kBadConfig for an unknown variant or a configuration without an NN kernel.
int cuda_l2_b200_nn_run_config(int variant, int config_id, const void* A, const void* B_rowmajor, void* C, int M, int N,
                               int K, int group_m, int max_ctas, int splits, b200::host::ScratchFn scratch,
                               void* stream);

}  // extern "C"

namespace b200 {
namespace nn {
using RunConfigFn = decltype(&cuda_l2_b200_nn_run_config);
constexpr const char* kLibrary = "libb200_nn.so";
constexpr const char* kRunConfigSymbol = "cuda_l2_b200_nn_run_config";
}  // namespace nn
}  // namespace b200
