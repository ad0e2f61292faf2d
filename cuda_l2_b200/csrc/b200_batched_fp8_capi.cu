// libb200_batched_fp8.so: the block-scaled e4m3 batched GEMM with optional per-batch row counts on the device
// (include/b200_batched_fp8.h), the MoE decode layout of an FP8 checkpoint. The kernels are the family's pipeline with
// Batched<BlockScaled<>> configurations (hgemm_sm90.cuh): the 3-D maps, tile list and masked store of
// libb200_batched.so, the per-k-block promotion of libb200_fp8block.so. A library of its own, so that the device code
// and kernel counts of those two stay as they are. The core is tile_list (hgemm_configs.cuh, hgemm_dispatch.cuh),
// shared by the four tile-list libraries; build.py compiles this file once per output type (B200_VARIANT = 5: fp16, 6:
// bf16, the GemmType index).
#include "../../include/b200_batched_fp8.h"

#include "hgemm_configs.cuh"
#include "hgemm_dispatch.cuh"

#ifndef B200_VARIANT
#error "compile once per output type with -DB200_VARIANT=5 or 6 (cuda_l2_b200/build.py does)"
#endif

namespace b200 {
namespace tile_list {
B200_LIST_OBJECT(Library, Batched, B200_BLOCK_LIST_TYPES);

// The batched wrapper keeps BlockScaled<>'s scale stage, ring depth and shared memory in every configuration that has a
// block-scaled kernel, so that each batched kernel runs the 2-D block-scaled kernel's pipeline.
template <int ID, class Cfg>
constexpr bool same_ring() {
  if constexpr (!block::eligible(ID)) {
    return true;
  } else {
    using B = BlockScaled<Cfg>;
    using W = Batched<B>;
    return W::SA_WINDOW_BYTES == B::SA_WINDOW_BYTES && W::SCALE_STAGE_BYTES == B::SCALE_STAGE_BYTES &&
           W::STAGES == B::STAGES && W::SMEM_BYTES == B::SMEM_BYTES;
  }
}
#define B200_SAME_RING(ID, BN, STAGES, CG, CM, CN, MR)                                                           \
  ok = ok && same_ring<ID, Config<BN, STAGES, CG, true, CM, CN, MR, false, true>>() &&                          \
       same_ring<ID, Config<BN, STAGES, CG, true, CM, CN, MR, true, true>>();
constexpr bool every_batched_ring_is_the_2d_ring() {
  bool ok = true;
  B200_HGEMM_CONFIGS(B200_SAME_RING)
  return ok;
}
#undef B200_SAME_RING
static_assert(every_batched_ring_is_the_2d_ring(), "Batched<BlockScaled<>> changed a block-scaled ring");
}  // namespace tile_list
}  // namespace b200

#if B200_VARIANT == 5

using b200::host::GemmType;

extern "C" {

int b200_batched_fp8_gemm(const void* A, const void* B_kmajor, void* C, const void* scale_a, int ld_a,
                          const void* scale_b, int out_bf16, const int* masked_m, int B, int M, int N, int K,
                          void* stream) {
  using namespace b200;
  if (!tile_list::known_out(out_bf16)) return host::kBadConfig;
  return tile_list::gemm(tile_list::Library{}, tile_list::block_type(out_bf16), A, B_kmajor, C, masked_m, B, M, N, K,
                         stream, tile_list::block_operands(scale_a, ld_a, scale_b));
}

int b200_batched_fp8_gemm_run_config(int config_id, int out_bf16, const void* A, const void* B_kmajor, void* C,
                                     const void* scale_a, int ld_a, const void* scale_b, const int* masked_m, int B,
                                     int M, int N, int K, int group_m, int max_ctas, void* stream) {
  using namespace b200;
  if (!tile_list::known_out(out_bf16)) return host::kBadConfig;
  return tile_list::run(tile_list::Library{}, tile_list::block_type(out_bf16), config_id, A, B_kmajor, C, masked_m, B,
                        M, N, K, group_m, max_ctas, stream, tile_list::block_operands(scale_a, ld_a, scale_b));
}

int b200_batched_fp8_select(int B, int M, int N, int K, int* config_id, int* group_m) {
  return b200::tile_list::select_into<b200::Batched>(GemmType::kE4M3F16Block, B, M, N, K, config_id, group_m);
}

unsigned long long b200_batched_fp8_launch_count(void) {
  return b200::tile_list::g_list_launches.load(std::memory_order_relaxed);
}

const char* b200_batched_fp8_strerror(int status) { return b200::host::status_string(status); }

}  // extern "C"

#endif  // B200_VARIANT == 5
