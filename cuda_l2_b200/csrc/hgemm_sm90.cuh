// H100 (sm_90a) HGEMM:  C[M,N] (fp16) = A[M,K] (fp16, K-contiguous) * Bt[N,K]^T (fp16, K-contiguous)
// with fp32 (F32F16F16F32) or fp16 (F16F16F16F16) accumulation in registers. The same pipeline also runs bf16 operands
// (bf16 out) and e4m3 operands with per-tensor or rowwise scales (fp16 or bf16 out), both with fp32 accumulation.
//
// Replaces, for this repository's device type, the per-shape kernels the reference ships
// (reference: kernels/a100_F32F16F16F32/4096_4096_4096.cu:22-177 mainloop+epilogue, :179-279 launcher;
//  kernels/h100_F32F16F16F32/4096_4096_4096.cu:21-80 for the TMA/wgmma flavour). Same contract:
// TN operands (A row-major, B supplied K-major as `b_col_major`, tools/utils.py:110-115), C row-major
// fully overwritten, one round-to-nearest fp32->fp16 conversion at the end.
//
// Design (nothing below is translated from the reference):
//   * persistent CTAs (one per SM), static tile schedule with grouped rasterisation for L2 reuse;
//   * warp-specialised: warpgroup 0 is the producer (warp 0 issues TMA, one elected lane), warpgroups 1 and 2
//     consume: each issues wgmma.mma_async on its half of the CTA's rows (64 or 128 rows x BN), accumulates in
//     registers, and runs its own epilogue (registers -> swizzled smem -> TMA store, one 16-row box per warp).
//     setmaxnreg moves registers from the producer to the consumers;
//   * operands land in 128B-swizzled smem via cp.async.bulk.tensor (OOB rows/cols zero-filled, so no
//     harness padding is ever needed), consumed in place by wgmma through smem descriptors;
//   * a STAGES-deep full/empty mbarrier ring between TMA and the consumers; a consumer warp releases a stage
//     as soon as the wgmma group that read it has completed (one group stays in flight; none in the stream-K kernels);
//   * CTA_GROUP == 2 ("CTA pair"): two CTAs of a cluster on vertically adjacent 128-row tiles share their B tile —
//     each loads half of it and TMA-multicasts it to both, so L2->SM traffic for B halves;
//   * CLUSTER_M x CLUSTER_N > 1: thread-block clusters of such groups on adjacent tiles. The CTAs of a cluster row
//     need the same A tile, those of a cluster column the same B tile: each CTA loads only a 1/CLUSTER_N slice of
//     A and a 1/(CTA_GROUP * CLUSTER_M) slice of B and TMA-multicasts it to the CTAs that need it. A stage is
//     released by an mbarrier arrive at every CTA of the consumer's cluster row and column;
//   * split-K for problems with few output tiles and long K, two flavours, both deterministic: partial tiles
//     through an fp32 global workspace with a distributed reduction (up to 32 splits), or the splits of a tile
//     form a cluster and reduce through distributed shared memory (2/4/8 splits, no workspace);
//   * stream-K for tile counts that leave the last wave partly empty: the first tiles of the schedule are cut along
//     K into one equal slice per worker (hgemm_schedule.cuh), the partial sums of a tile meet in its owner's
//     registers through the same workspace, in fixed k order.
#pragma once
#include <cuda.h>          // CUtensorMap (type only; the encoder is fetched at run time)
#include <cuda_runtime.h>
#include <cstdint>
#include <type_traits>

#include "hgemm_schedule.cuh"
#include "ptx_sm90.cuh"
#include "swiglu_arith.cuh"
#include "wgmma_sm90.cuh"


namespace b200 {

constexpr int kBlockKBytes = 128;    // one k-block = one 128-byte swizzle row: 64 16-bit or 128 8-bit elements
constexpr int kBlockK = 64;          // 64 fp16 = 128 B = one swizzle row
constexpr int kWgmmaK = 16;          // K per wgmma.mma_async (16-bit operands; k32 = the same 32 bytes for 8-bit ones)
constexpr int kBlockM = 128;         // rows per CTA (per 128-row block: two consumer warpgroups x 64 rows)
constexpr int kNumThreads = 384;     // warpgroup 0: producer (warp 0 issues), warpgroups 1-2: MMA + epilogue
constexpr int kEpiWarp0 = 4;         // first consumer warp
constexpr int kConsumerThreads = 256;
constexpr int kProducerRegs = 40;    // setmaxnreg budgets: 128 x 40 + 256 x 232 <= 64K registers
constexpr int kConsumerRegs = 232;
constexpr int kSmemLimit = 232448;   // 227 KB of dynamic shared memory per block on sm_90
// How a launch divides K. The kernel is compiled once per (configuration, mode), so that the plain schedule — nearly
// every launch — carries none of the three other epilogues.
enum KMode : int { kPlain = 0, kWorkspaceSplitK = 1, kClusterSplitK = 2, kStreamK = 3 };
struct Scales;   // the epilogue arguments of every configuration but BiasAct<>'s and BlockScaled1D1D<>'s (below)
struct Block1D1DArgs;

template <int BN_, int STAGES_, int CTA_GROUP_, bool ACC_F32_, int CLUSTER_M_ = 1, int CLUSTER_N_ = 1, int M_REP_ = 1, bool BF16_ = false,
          bool E4M3_ = false>
struct Config {
  static constexpr int BN = BN_;               // tile N (= wgmma N)
  static constexpr int CTA_GROUP = CTA_GROUP_; // 1: one CTA per 128-row tile; 2: a pair of CTAs sharing the B tile
  static constexpr bool ACC_F32 = ACC_F32_;
  // bf16 operands and bf16 output instead of fp16 (README.md:73 "denser configurations" territory): same pipeline, the
  // wgmma type and the epilogue's convert differ. bf16 products accumulate in fp32 only.
  static constexpr bool BF16 = BF16_;
  static_assert(!BF16_ || ACC_F32_, "bf16 operands accumulate in fp32");
  // e4m3 operands (float8_e4m3fn): the operand type is then separate from the output type, which BF16 names (fp16 or
  // bf16). The k-block stays 128 bytes, now 128 elements; stage sizes, descriptors and the wgmma count per k-block are
  // unchanged. The per-tensor scales multiply the finished fp32 sum once, just before the one rounding to the output.
  static constexpr bool E4M3 = E4M3_;
  static_assert(!E4M3_ || ACC_F32_, "e4m3 operands accumulate in fp32");
  static constexpr int OP_BYTES = E4M3_ ? 1 : 2;             // bytes per operand element
  static constexpr int BLOCK_K = kBlockKBytes / OP_BYTES;    // operand elements per k-block
  // Multicast cluster: CLUSTER_M x CLUSTER_N groups (single CTAs or CTA pairs) work on a block of adjacent tiles.
  // On sm_90 a CTA pair is two CTAs along M that multicast B between them, so the cluster is MCAST_M x CLUSTER_N
  // CTAs, cluster rank = mi + MCAST_M * cn with mi = cm * CTA_GROUP + (position inside the pair).
  static constexpr int CLUSTER_M = CLUSTER_M_;
  static constexpr int CLUSTER_N = CLUSTER_N_;
  static constexpr int MCAST_CTAS = CLUSTER_M * CLUSTER_N;
  static constexpr int MCAST_M = CTA_GROUP * CLUSTER_M;
  static constexpr int CLUSTER_CTAS = MCAST_M * CLUSTER_N;
  // M_REP = 2: every CTA owns 256 rows — each consumer warpgroup issues two 64-row wgmmas per k-step that share the B
  // tile in shared memory, so each B byte fetched from L2 feeds twice the MMA work. Accumulators are registers:
  // M_REP * BN <= 256 keeps them within a consumer thread's budget. No split-K / stream-K in this mode.
  static constexpr int M_REP = M_REP_;
  static constexpr int CTA_M = kBlockM * M_REP;             // rows per CTA
  static constexpr int TILE_M = CTA_M * CTA_GROUP;
  static constexpr int A_BOX_ROWS = CTA_M / CLUSTER_N;      // A rows each CTA loads per stage
  static constexpr int B_BOX_ROWS = BN / MCAST_M;           // B rows each CTA loads per stage
  static constexpr int A_STAGE_BYTES = CTA_M * kBlockK * 2;
  static constexpr int B_STAGE_BYTES = BN * kBlockK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int EPI_N = BN < 64 ? BN : 64;            // columns per epilogue step / TMA store box
  static constexpr int EPI_CHUNKS = BN / EPI_N;
  static constexpr int EPI_ROWS = 16;                        // rows of one warp's share of a 64-row wgmma tile
  static constexpr int NUM_THREADS = kNumThreads;
  // which K-decompositions this configuration's kernel carries
  static constexpr bool STREAM_K = CLUSTER_M_ * CLUSTER_N_ == 1 && BN_ >= 64 && M_REP_ == 1;
  static constexpr bool SPLIT_K = STREAM_K && CTA_GROUP_ == 1;
  // the variant wrappers below (BlockScaled<>, BlockScaled1D1D<>, Batched<>, Grouped<>, RowMajorB<>, GroupedK<>,
  // BiasAct<>, AccumF32<>) override these
  static constexpr bool BLOCK_SCALED = false, BATCHED = false, GROUPED = false, ROW_MAJOR_B = false, K_GROUPED = false,
                        BIAS_ACT = false, BLOCK_1D1D = false, ACCUM_F32 = false;
  using Cursor = NoBatches;   // the flat tile list the kernel walks (hgemm_schedule.cuh): none
  using EpiArgs = Scales;     // the kernel's last parameter
  static constexpr int EPI_BYTES = 8 * EPI_ROWS * 64 * 2;    // 8 consumer warps x one staging buffer (sized for EPI_N = 64)
  static constexpr int BAR_BYTES = 256;
  // STAGES_ is the requested ring depth; on sm_90 every CTA of a pair holds the whole B tile, so the depth is capped
  // by what fits next to the epilogue staging area.
  static constexpr int MAX_STAGES = (kSmemLimit - 1024 - EPI_BYTES - BAR_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_ < MAX_STAGES ? STAGES_ : MAX_STAGES;
  static constexpr int SMEM_BYTES = 1024 /*align slack*/ + STAGES * STAGE_BYTES + EPI_BYTES + BAR_BYTES;
  static_assert(BN == 32 || BN % 64 == 0, "tile N is 32 or a multiple of 64");
  static_assert(BN >= 32 && BN <= 256, "wgmma N constraints");
  static_assert(M_REP * BN <= 256, "register accumulators: at most 256 columns x 128 rows per consumer warpgroup");
  static_assert(CLUSTER_CTAS <= 8, "portable cluster size");
  static_assert(A_BOX_ROWS % 8 == 0 && B_BOX_ROWS % 8 == 0, "slices must cover whole 8-row swizzle atoms");
  static_assert(M_REP == 1 || M_REP == 2, "one or two 128-row blocks per CTA");
  static_assert(A_BOX_ROWS <= 256 && B_BOX_ROWS <= 256, "TMA box dimension limit");
  static_assert(STAGES >= 2, "the ring needs two stages");
  static_assert(SMEM_BYTES <= kSmemLimit, "exceeds 227 KB of shared memory");
  static_assert(A_STAGE_BYTES % 1024 == 0 && B_STAGE_BYTES % 1024 == 0, "swizzle-128B tiles need 1 KB alignment");
  static_assert(8 * (2 * STAGES + 1) <= BAR_BYTES, "barrier block too small");
};

constexpr int kMaxSplitTiles = 256;   // split-K is only used when tiles * splits <= #SMs

// Block-scaled e4m3 (the layout of DeepSeek-V3-style FP8 checkpoints): one fp32 scale per (row of A, 128-element
// k-block) and one per 128 x 128 block of Bt. Every k-block's wgmma sum is scaled and added into a separate fp32
// accumulator, so the kernel holds two accumulator sets: only tiles with M_REP * BN <= 128 qualify, and a BN <= 128 tile
// lies inside one 128-column scale block of Bt. Each ring stage carries its k-block's scales next to the operands:
// CTA_M values of A's scales (one 1-D bulk copy, counted in the stage's transaction bytes) and the tile's one value of
// Bt's (written by the producer before its arrive), 16 bytes of padding keeping the next stage's slice aligned.
// A wrapper, so that the Config<> instantiations of the other variants, and with them their kernels' names, stay as
// they are; block_scaled<Cfg>() reads the flag.
template <class Base>
struct BlockScaled : Base {
  static constexpr bool BLOCK_SCALED = true;
  static_assert(Base::E4M3 && Base::M_REP * Base::BN <= 128, "block scales: e4m3, and room for two accumulator sets");
  static constexpr int SA_WINDOW_BYTES = Base::CTA_M * 4;   // A's scales of a stage; Bt's one value follows them
  static constexpr int SCALE_STAGE_BYTES = SA_WINDOW_BYTES + 16;
  static constexpr int MAX_STAGES =
      (kSmemLimit - 1024 - Base::EPI_BYTES - Base::BAR_BYTES) / (Base::STAGE_BYTES + SCALE_STAGE_BYTES);
  static constexpr int STAGES = Base::STAGES < MAX_STAGES ? Base::STAGES : MAX_STAGES;
  static constexpr int SMEM_BYTES = Base::SMEM_BYTES + STAGES * SCALE_STAGE_BYTES - (Base::STAGES - STAGES) * Base::STAGE_BYTES;
  static_assert(STAGES >= 2 && SMEM_BYTES <= kSmemLimit, "block-scaled ring does not fit");
};
template <class Cfg>
__host__ __device__ constexpr bool block_scaled() { return Cfg::BLOCK_SCALED; }

// Block-scaled e4m3 with 1 x 128 scales on both operands (libb200_fp8block_1d1d.so, the weight gradient of blockwise
// FP8 training, dW = q(dY^T) q(X^T)^T, whose two operands are transposed activations): Bt's scales are one per (row of
// Bt, 128-element k-block), N-major like A's, value (n, kb) at b[kb * ld_b + n]. BlockScaled<>'s main loop and
// schedules; the promotion forms s = fp32(sa(m, kb) * sb(n, kb)) per element. Each ring stage's scale slice holds
// CTA_M values of A's scales and then BN of Bt's, each one 1-D bulk copy counted in the stage's transaction bytes (rows
// clamped at ld_a / ld_b, so a CTA past them loads none); the ring depth is recomputed for the larger stage. ld_b
// travels in the kernel's Block1D1DArgs (hgemm_block_1d1d_kernel), not in Scales. A wrapper of its own, so that
// BlockScaled<>'s kernels, and the other variants', stay as they are.
template <class Base>
struct BlockScaled1D1D : BlockScaled<Base> {
  static constexpr bool BLOCK_1D1D = true;
  using EpiArgs = Block1D1DArgs;
  static constexpr int SA_WINDOW_BYTES = Base::CTA_M * 4;   // A's scales of a stage; Bt's BN values follow them
  static constexpr int SCALE_STAGE_BYTES = SA_WINDOW_BYTES + Base::BN * 4;
  static constexpr int MAX_STAGES =
      (kSmemLimit - 1024 - Base::EPI_BYTES - Base::BAR_BYTES) / (Base::STAGE_BYTES + SCALE_STAGE_BYTES);
  static constexpr int STAGES = Base::STAGES < MAX_STAGES ? Base::STAGES : MAX_STAGES;
  static constexpr int SMEM_BYTES = Base::SMEM_BYTES + STAGES * SCALE_STAGE_BYTES - (Base::STAGES - STAGES) * Base::STAGE_BYTES;
  static_assert(STAGES >= 2 && SMEM_BYTES <= kSmemLimit, "1D1D block-scaled ring does not fit");
  static_assert(SA_WINDOW_BYTES % 16 == 0 && SCALE_STAGE_BYTES % 16 == 0, "bulk copies need 16-byte aligned slices");
};
template <class Cfg>
__host__ __device__ constexpr bool block_1d1d() { return Cfg::BLOCK_1D1D; }

// Batched 16-bit GEMM, C[b] = A[b] Bt[b]^T (libb200_batched.so): A, Bt and C are 3-D tensor maps whose third
// coordinate is the batch, so a tile's loads are zero-filled and its stores clipped at its own matrix's edge, and a
// cluster block never crosses a batch (multicast is kept). The flat tile list of BatchCursor (hgemm_schedule.cuh),
// plain schedule only. A plain launch reads neither splits_arg nor splitk_ctr, so these carry the batch count and the
// optional per-batch row counts (int32, device memory, read after the grid dependency wait). A wrapper, like
// BlockScaled<>, so that the other kernels and their names stay as they are.
template <class Base>
struct Batched : Base {
  static constexpr bool BATCHED = true;
  using Cursor = BatchCursor;
  static_assert(!Base::E4M3, "batched: 16-bit operands, or block-scaled e4m3 (Batched<BlockScaled<...>>)");
};
// Batched block-scaled e4m3 (libb200_batched_fp8.so, the MoE decode layout of an FP8 checkpoint): the batched kernel
// with BlockScaled<>'s main loop. A's scales are one [ceil(K/128), ld_a] block per matrix, stacked, and Bt's one
// [ceil(N/128), ceil(K/128)] matrix per batch. A CTA's first row inside its matrix is a multiple of CTA_M, so the bulk
// copy of A's scales is aligned as in 2-D: the scale stage, the ring depth and the shared memory are BlockScaled<>'s.
template <class Base>
struct Batched<BlockScaled<Base>> : BlockScaled<Base> {
  static constexpr bool BATCHED = true;
  using Cursor = BatchCursor;
};
template <class Cfg>
__host__ __device__ constexpr bool batched() { return Cfg::BATCHED; }

// Grouped 16-bit GEMM over contiguous row groups, C[start_g : end_g] = A[start_g : end_g] Bt[g]^T (the MoE prefill
// layout, libb200_grouped.so): A [T, K] and C [T, N] are 2-D tensor maps, Bt [G, N, K] the batched 3-D map. The flat
// tile list of GroupCursor (hgemm_schedule.cuh), plain schedule only; a cluster block never crosses a group, so
// multicast is kept. splits_arg carries the group count and splitk_ctr the int32 offsets (device memory, read after
// the grid dependency wait). A group starts at any row, so the rows of a box past the group's end belong to the next
// group: they are multiplied but never stored. A 16-row store box wholly inside the group is a TMA store; one that
// straddles the group's end stores only the group's rows, with 16-byte generic stores from the staging buffer.
template <class Base>
struct Grouped : Base {
  static constexpr bool GROUPED = true;
  using Cursor = GroupCursor;
  static_assert(!Base::E4M3, "grouped: 16-bit operands, or block-scaled e4m3 (Grouped<BlockScaled<...>>)");
};
// Grouped block-scaled e4m3 (libb200_grouped_fp8.so): the grouped kernel with BlockScaled<>'s main loop, Bt's scales
// [G, ceil(N/128), ceil(K/128)] read at the group's own matrix. A CTA's first row r0 = start_g + (its row block) * CTA_M
// is any row, but the bulk copy of A's scales needs a 16-byte aligned source and size: the stage holds the aligned
// window [r0 & ~3, min(round_up(r0 + CTA_M, 4), ld_a)), up to CTA_M + 4 values, and the consumers read row i at
// (start_g & 3) + i (CTA_M % 4 == 0, so the shift is the group's). 16 more bytes per scale stage than BlockScaled<>,
// whose own layout stays as it is; the ring depth is recomputed with the larger stage.
template <class Base>
struct Grouped<BlockScaled<Base>> : BlockScaled<Base> {
  static constexpr bool GROUPED = true;
  using Cursor = GroupCursor;
  static constexpr int SA_WINDOW_BYTES = Base::CTA_M * 4 + 16;
  static constexpr int SCALE_STAGE_BYTES = SA_WINDOW_BYTES + 16;
  static constexpr int MAX_STAGES =
      (kSmemLimit - 1024 - Base::EPI_BYTES - Base::BAR_BYTES) / (Base::STAGE_BYTES + SCALE_STAGE_BYTES);
  static constexpr int STAGES = Base::STAGES < MAX_STAGES ? Base::STAGES : MAX_STAGES;
  static constexpr int SMEM_BYTES = Base::SMEM_BYTES + STAGES * SCALE_STAGE_BYTES - (Base::STAGES - STAGES) * Base::STAGE_BYTES;
  static_assert(STAGES >= 2 && SMEM_BYTES <= kSmemLimit, "grouped block-scaled ring does not fit");
  static_assert(Base::CTA_M % 4 == 0, "the scale window's shift is the group's");
};
template <class Cfg>
__host__ __device__ constexpr bool grouped() { return Cfg::GROUPED; }

// Row-major B (NN, libb200_nn.so): C = A B with B [K, N] row-major (N contiguous), the layout of torch.matmul(a, b),
// read in place instead of through a transposed copy. wgmma reads a 16-bit B operand MN-major (imm-trans-b = 1), so
// only the B load and the B descriptor change. A B stage holds BN / 64 MN-major SW128 atom columns, each 64 N x 64 K
// rows of 128 B (8 KB, the descriptor's LBO), 8-row K groups 1024 B apart (SBO); a k16 step advances 16 K rows. TMA
// loads a {64 N, rows} box of B's {N, K} map into an atom column, zero-filling past K and N as for Bt. Multicast is
// sliced along K: each of the MCAST_M CTAs loads K rows [mi * B_K_ROWS, (mi + 1) * B_K_ROWS) of every atom column, so
// every slice is whole 8-row swizzle groups (1 KB aligned) and any per-CTA N extent works. e4m3 wgmma takes K-major
// operands only, and a BN = 32 tile has no 128-byte N row: those configurations have no NN kernel (nn::sibling). A
// wrapper, like BlockScaled<>, so that the other kernels and their names stay as they are.
template <class Base>
struct RowMajorB : Base {
  static constexpr bool ROW_MAJOR_B = true;
  static_assert(!Base::E4M3 && !Base::BLOCK_SCALED && !Base::BATCHED && !Base::GROUPED,
                "row-major B: the 2-D 16-bit kernels only");
  static_assert(Base::BN % 64 == 0, "row-major B: whole 64-column atom columns");
  static constexpr int B_ATOMS = Base::BN / 64;                       // atom columns per stage
  static constexpr int B_ATOM_BYTES = 64 * kBlockK * 2;               // one atom column: 64 K rows of 128 B
  static constexpr int B_K_ROWS = kBlockK / Base::MCAST_M;            // K rows of each atom column this CTA loads
  static_assert(B_K_ROWS % 8 == 0, "K slices of whole 8-row swizzle groups");
  static_assert(B_ATOMS * B_ATOM_BYTES == Base::B_STAGE_BYTES, "the stage holds the same bytes as the K-major one");
};
template <class Cfg>
__host__ __device__ constexpr bool row_major_b() { return Cfg::ROW_MAJOR_B; }

// Grouped<RowMajorB<...>> (libb200_grouped_bwd.so, the input gradient of the grouped product): C[start_g : end_g] =
// A[start_g : end_g] B[g] with B [G, K, N] row-major, one expert's weight [N_model, K_model] read in place. A and the
// epilogue are Grouped<>'s; B is RowMajorB<>'s atom columns, loaded from the 3-D map {N, K, G}, so each expert's
// matrix clips its own boxes and K is zero-filled per expert as in 2-D. Nothing else changes: the partial
// specialisation only names the combination (RowMajorB<> itself still refuses a grouped, batched or e4m3 base).
template <class Base>
struct Grouped<RowMajorB<Base>> : RowMajorB<Base> {
  static constexpr bool GROUPED = true;
  using Cursor = GroupCursor;
};

// K-grouped row-major operands (libb200_grouped_bwd.so, the weight gradient of the grouped product):
// C[g] = A[start_g : end_g]^T B[start_g : end_g] for g < G, A [T, M] and B [T, N] row-major, C [G, M, N]. The reduction
// runs over the group's own rows (GroupKCursor), so both operands are MN-major: A is read with imm-trans-a = 1 in
// CTA_M / 64 SW128 atom columns of 64 M x 64 K rows (8 KB each, the same bytes as the K-major stage), loaded as
// {64, A_K_ROWS} boxes of A's {M, T} map; the CTAs of a cluster row multicast A sliced along K, A_K_ROWS rows each,
// as RowMajorB<> does for B along the cluster column. B is RowMajorB<>'s over B's {N, T} map, C the batched 3-D map
// {N, M, G}. A group's last k-block may hold r < 64 of its rows; rows [r, 64) of that stage belong to the next group
// (or lie past T, already zero), and the consumers zero them in both operands before the wgmma reads them (0 * Inf
// is NaN). A group without rows gives a tile of +0.0. Plain schedule, fp32 accumulation.
template <class Base>
struct GroupedK : Base {
  static constexpr bool K_GROUPED = true;
  using Cursor = GroupKCursor;
  static_assert(Base::ROW_MAJOR_B && !Base::GROUPED && Base::ACC_F32, "K-grouped: RowMajorB<> 16-bit configurations, fp32 accumulation");
  static constexpr int A_ATOMS = Base::CTA_M / 64;                    // atom columns of an A stage
  static constexpr int A_K_ROWS = kBlockK / Base::CLUSTER_N;          // K rows of each atom column this CTA loads
  static_assert(A_K_ROWS % 8 == 0, "K slices of whole 8-row swizzle groups");
  static_assert(A_ATOMS * Base::B_ATOM_BYTES == Base::A_STAGE_BYTES, "the stage holds the same bytes as the K-major one");
};
template <class Cfg>
__host__ __device__ constexpr bool k_grouped() { return Cfg::K_GROUPED; }

// The tile list a kernel of Cfg walks (Cfg::Cursor) over `count` matrices or groups; the K-grouped list also needs the
// reduction's rows, K.
template <class Cfg>
__host__ __device__ __forceinline__ typename Cfg::Cursor make_cursor(const int* list, int count, int M, int K,
                                                                     int block_rows, int n_blocks, int group_m) {
  if constexpr (k_grouped<Cfg>()) return typename Cfg::Cursor(list, count, M, K, block_rows, n_blocks, group_m);
  else return typename Cfg::Cursor(list, count, M, block_rows, n_blocks, group_m);
}

// Scales of an e4m3 launch, in device memory (null for the 16-bit operand types). Per tensor: one fp32 value each.
// Rowwise: `a` holds M values (one per row of A and C), `b` N values (one per row of Bt, i.e. per column of C), both
// 16-byte aligned; C[m,n] = RN_out(fp32(fp32(acc * b[n]) * a[m])). The granularity is a run-time property of the
// same kernels. Block-scaled kernels (BlockScaled<>): value (m, kb) of `a` at a[kb * ld_a + m] (16-byte aligned,
// ld_a % 4 == 0; batched: one [nkb, ld_a] block per matrix), `b` row-major [ceil(N/128), ceil(K/128)] (batched /
// grouped: one such matrix per batch or group). ld_a travels in the
// kernel's aux_arg, not here: a member added to this struct, even in its padding, changes the code ptxas emits for the
// other e4m3 kernels.
struct Scales { const float* a; const float* b; bool rowwise = false; };

// Fused bias + activation epilogue (libb200_epilogue.so): C[m,n] = RN_out(act(s(m,n) + fp32(bias[n]))), fp32 throughout
// and one rounding, where s is what the wrapped kernel rounds (the fp32 sum; e4m3: the sum after its per-tensor or
// rowwise scales). `bias` has the output's type, N values, 16-byte aligned; null adds nothing (the kernel then adds
// -0.0, which leaves every value, -0.0 included, as it is). The activation code is a run-time value, the same for the
// whole launch, so one kernel serves all three. Only the finished sum sees either: partial tiles, DSMEM tiles and
// stream-K register images are those of the wrapped kernel. The 2-D kernels with fp32 accumulation (fp16, bf16, e4m3
// per-tensor and rowwise) in every K-mode; fp16 accumulation and block scales have no bias kernel. A wrapper, like
// BlockScaled<>, so that the other kernels and their names stay as they are; the kernel takes BiasActArgs as its last
// parameter (hgemm_bias_act_kernel) where the others take Scales.
enum Activation : int { kActNone = 0, kActRelu = 1, kActGeluTanh = 2 };
constexpr int kNumActivations = 3;
struct BiasActArgs { Scales scales; const void* bias; int act; };
template <class Base>
struct BiasAct : Base {
  static constexpr bool BIAS_ACT = true;
  using EpiArgs = BiasActArgs;
  static_assert(Base::ACC_F32 && !Base::BLOCK_SCALED && !Base::BATCHED && !Base::GROUPED && !Base::ROW_MAJOR_B &&
                    !Base::K_GROUPED,
                "bias + activation: the 2-D TN kernels with fp32 accumulation only");
};
template <class Cfg>
__host__ __device__ constexpr bool bias_act() { return Cfg::BIAS_ACT; }
__host__ __device__ __forceinline__ const Scales& scales_of(const Scales& s) { return s; }
__host__ __device__ __forceinline__ const Scales& scales_of(const BiasActArgs& e) { return e.scales; }

// The epilogue arguments of the BlockScaled1D1D<> kernels (hgemm_block_1d1d_kernel): the scales, and the row stride of
// Bt's (ld_b >= N, ld_b % 4 == 0, `scales.b` 16-byte aligned).
struct Block1D1DArgs { Scales scales; int ld_b; };
__host__ __device__ __forceinline__ const Scales& scales_of(const Block1D1DArgs& e) { return e.scales; }
// ld_b of a kernel's EpiArgs: 0 for the kernels without it
template <class E>
__host__ __device__ __forceinline__ int ld_b_of(const E& e) {
  if constexpr (std::is_same_v<E, Block1D1DArgs>) return e.ld_b;
  else return 0;
}

// fp32 accumulation of the finished sum (libb200_wgrad_accum.so, the weight gradient into an fp32 main-grad buffer):
// C32[m,n] = fp32(C32[m,n] + s(m,n)), one round-to-nearest-even addition per element, where s is exactly the fp32 value
// the wrapped kernel rounds to its 16-bit output (the fp32 sum; e4m3 rowwise: fp32(fp32(acc * sb[n]) * sa[m]); 1 x 128
// scales: the promoted sum). Only the finished sum is added, once: split-K partials, DSMEM tiles and stream-K register
// images are those of the wrapped kernel, summed in their fixed order first. Nothing outside [M, N] (K-grouped:
// [G, M, N]) is read or written, and an empty group of a K-grouped kernel leaves its matrix untouched. The final
// writers read and write C32 directly from registers (or the reductions' float4s), 8 bytes per fragment pair: a quad of
// lanes covers 32 contiguous bytes. Wraps the 16-bit K-grouped kernels (GroupedK<RowMajorB<>>), the 2-D e4m3 kernels
// (rowwise scales) and the 1 x 128 block-scaled ones (BlockScaled1D1D<>). A wrapper, like BiasAct<>, so that the other
// kernels and their names stay as they are; the kernel takes AccumArgs as its last parameter (hgemm_accum_kernel).
template <class E>
struct AccumArgs { E base; float* c32; };
template <class Base>
struct AccumF32 : Base {
  static constexpr bool ACCUM_F32 = true;
  using AccumBase = Base;
  using EpiArgs = AccumArgs<typename Base::EpiArgs>;
  static_assert(Base::ACC_F32 && !Base::BIAS_ACT && !Base::BATCHED && !Base::GROUPED &&
                    (Base::K_GROUPED || (Base::E4M3 && !Base::ROW_MAJOR_B)) && (!Base::BLOCK_SCALED || Base::BLOCK_1D1D),
                "fp32 accumulation: the K-grouped 16-bit kernels, the 2-D e4m3 ones and the 1 x 128 block-scaled ones");
};
template <class Cfg>
__host__ __device__ constexpr bool accum_f32() { return Cfg::ACCUM_F32; }
template <class E>
__host__ __device__ __forceinline__ const Scales& scales_of(const AccumArgs<E>& e) { return scales_of(e.base); }
template <class E>
__host__ __device__ __forceinline__ int ld_b_of(const AccumArgs<E>& e) { return ld_b_of(e.base); }
// The fp32 C of a kernel's EpiArgs: null for the kernels without one
template <class E>
__host__ __device__ __forceinline__ float* c32_of(const E&) { return nullptr; }
template <class E>
__host__ __device__ __forceinline__ float* c32_of(const AccumArgs<E>& e) { return e.c32; }

// Fused SwiGLU epilogue (libb200_swiglu.so): h = A Bt^T over a gate / up weight Bt [2I, K] whose rows are interleaved in
// 64-row blocks (rows [128 b, 128 b + 64) gate rows [64 b, 64 b + 64), the next 64 the matching up rows), so that h's
// columns are [g | u] per 128. The epilogue writes y [M, I] = silu_mul(RN(g), RN(u)) (swiglu_arith.cuh), torch's
// `F.silu(g) * u` on the 16-bit h, and, when `store_h` is set, h [M, 2I] itself through the unchanged store path (the
// bits of the wrapped kernel's output). Chunk J (even) and chunk J + 1 of a 64-row block are one gate / up pair: in the
// wgmma accumulator layout the thread that holds column c of chunk J holds column c of chunk J + 1 for the same rows, so
// every pair is in one thread's registers. y's chunk goes out through the warp's staging buffer with a TMA store of its
// own map, `y_map` ([M, I], box {64, 16}). The 2-D 16-bit TN kernels with fp32 accumulation and BN = 128 or 256 (whole
// pairs per tile), plain schedule only. A wrapper, like BiasAct<>, so that the other kernels and their names stay as
// they are; the kernel takes GatedArgs as its last parameter (hgemm_gated_kernel).
struct GatedArgs { CUtensorMap y_map; int store_h; };
template <class Base>
struct Gated : Base {
  using EpiArgs = GatedArgs;
  static_assert(Base::ACC_F32 && !Base::E4M3 && !Base::BLOCK_SCALED && !Base::BATCHED && !Base::GROUPED &&
                    !Base::ROW_MAJOR_B && !Base::K_GROUPED && !Base::BIAS_ACT && !Base::ACCUM_F32,
                "SwiGLU: the 2-D 16-bit TN kernels with fp32 accumulation only");
  static_assert(Base::BN == 128 || Base::BN == 256, "SwiGLU: whole gate / up pairs of 64-column chunks per tile");
};
// Gated<Grouped<...>> (libb200_grouped_swiglu.so, the gate / up projection of MoE experts): Grouped<>'s main loop and
// tile list over w_gu [G, 2I, K], each expert's matrix interleaved as above, with Gated<>'s epilogue. h goes through
// Grouped<>'s store path (rows from the group's first row, a box that straddles the group's end stored row by row with
// generic stores), and so does y: a 16-row box of y wholly inside the group is a TMA store of y_map ([T, I]), one that
// straddles the group's end stores only the group's rows from the staging buffer to `y` [T, I] (the next group's CTA
// owns the rest). Its own argument type, so that GatedArgs and the 2-D kernels stay as they are; the kernel is
// hgemm_grouped_gated_kernel.
struct GroupedGatedArgs : GatedArgs { __half* y; };
template <class Base>
struct Gated<Grouped<Base>> : Grouped<Base> {
  using EpiArgs = GroupedGatedArgs;
  static_assert(Base::ACC_F32 && !Base::E4M3 && !Base::BLOCK_SCALED && !Base::BATCHED && !Base::GROUPED &&
                    !Base::ROW_MAJOR_B && !Base::K_GROUPED && !Base::BIAS_ACT && !Base::ACCUM_F32,
                "grouped SwiGLU: the grouped 16-bit TN kernels with fp32 accumulation only");
  static_assert(Base::BN == 128 || Base::BN == 256, "SwiGLU: whole gate / up pairs of 64-column chunks per tile");
};
template <class Cfg>
__host__ __device__ constexpr bool is_gated() {
  return std::is_same_v<typename Cfg::EpiArgs, GatedArgs> || std::is_same_v<typename Cfg::EpiArgs, GroupedGatedArgs>;
}
// y's pointer of a kernel's EpiArgs: null for the kernels without one
template <class E>
__host__ __device__ __forceinline__ __half* y_of(const E&) { return nullptr; }
__host__ __device__ __forceinline__ __half* y_of(const GroupedGatedArgs& e) { return e.y; }

// act(z) in fp32; `act` is warp-uniform. relu: max(z, +0.0) (+0.0 for -0.0 and NaN). gelu_tanh: 0.5 z (1 + tanhf(u)),
// u = sqrt(2/pi) (z + 0.044715 z^3), torch's tanh approximation (F.gelu(approximate="tanh"), _addmm_activation), each
// step one IEEE fp32 operation and tanhf CUDA's full-precision one (no tanh.approx.f32). Where tanh(u) nears -1 (z below
// about -3) 1 + tanhf(u) keeps few bits: there the result carries an absolute error of a few 2^-24 |z|, as fp32 torch's
// does, and is -0.0 once tanhf(u) rounds to -1 (z below about -5.2).
__device__ __forceinline__ float activate(float z, int act) {
  if (act == kActRelu) return z > 0.f ? z : 0.f;
  if (act == kActGeluTanh) {
    const float inner = __fadd_rn(z, __fmul_rn(0.044715f, __fmul_rn(__fmul_rn(z, z), z)));
    const float u = __fmul_rn(0.7978845608028654f, inner);
    return __fmul_rn(__fmul_rn(0.5f, z), __fadd_rn(1.f, tanhf(u)));
  }
  return z;
}
// Two 16-bit bias values of the output type (low half: the lower column) as fp32.
template <class Cfg>
__device__ __forceinline__ float2 unpack_out_x2(uint32_t v) {
  if constexpr (Cfg::BF16) return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u));
  else {
    const __half2 h = *reinterpret_cast<const __half2*>(&v);
    return make_float2(__low2float(h), __high2float(h));
  }
}
constexpr uint32_t kNegZeroPair = 0x80008000u;   // -0.0 in both halves, fp16 and bf16: the bias of a null pointer

// The uniform factor applied to the finished fp32 sum before it is rounded to the output type: fp32(scale_a * scale_b)
// for per-tensor e4m3 scales, read where it is used (after the grid dependency wait, so a preceding kernel may have just
// written it). Rowwise launches scale per element instead (scale_quad, the plain epilogue) and do not read it; block-
// scaled sums are scaled in the main loop, so their epilogues only round.
template <class Cfg>
__device__ __forceinline__ float output_scale(const Scales& s) {
  if constexpr (Cfg::E4M3 && !block_scaled<Cfg>()) return s.rowwise ? 1.f : __fmul_rn(*s.a, *s.b);
  else return 1.f;
}

// One finished float4 of the split-K reductions, output row gm, columns gn .. gn+3 (gn % 4 == 0, in bounds), scaled
// before its rounding: by the uniform factor, or (rowwise) by b[gn..gn+3] (one 16-byte load) and then a[gm].
template <class Cfg>
__device__ __forceinline__ void scale_quad(float4& acc, float scale, const Scales& s, int gm, int gn) {
  if constexpr (Cfg::E4M3 && !block_scaled<Cfg>()) {
    if (s.rowwise) {
      const float sa = s.a[gm];
      const float4 sb = *reinterpret_cast<const float4*>(s.b + gn);
      acc.x = __fmul_rn(__fmul_rn(acc.x, sb.x), sa); acc.y = __fmul_rn(__fmul_rn(acc.y, sb.y), sa);
      acc.z = __fmul_rn(__fmul_rn(acc.z, sb.z), sa); acc.w = __fmul_rn(__fmul_rn(acc.w, sb.w), sa);
    } else {
      acc.x = __fmul_rn(acc.x, scale); acc.y = __fmul_rn(acc.y, scale);
      acc.z = __fmul_rn(acc.z, scale); acc.w = __fmul_rn(acc.w, scale);
    }
  }
}

// The bias and the activation of one finished, scaled float4 of the split-K reductions (BiasAct<> kernels only): one
// 8-byte load of the bias at columns gn .. gn+3.
template <class Cfg>
__device__ __forceinline__ void bias_act_quad(float4& acc, const typename Cfg::EpiArgs& epi, int gn) {
  if constexpr (bias_act<Cfg>()) {
    uint2 bv = make_uint2(kNegZeroPair, kNegZeroPair);
    if (epi.bias) bv = *reinterpret_cast<const uint2*>(static_cast<const uint16_t*>(epi.bias) + gn);
    const float2 lo = unpack_out_x2<Cfg>(bv.x), hi = unpack_out_x2<Cfg>(bv.y);
    acc.x = activate(__fadd_rn(acc.x, lo.x), epi.act); acc.y = activate(__fadd_rn(acc.y, lo.y), epi.act);
    acc.z = activate(__fadd_rn(acc.z, hi.x), epi.act); acc.w = activate(__fadd_rn(acc.w, hi.y), epi.act);
  }
}

// The rowwise scales one thread's share of a 64-row block needs in the plain epilogue: its two row scales (rows
// l/4 and l/4 + 8 of its warp's 16, 0 past M) and the column-scale vector, read one float2 per column pair where used.
struct RowwiseEpi { float sa_lo, sa_hi; const float* sb; };

// Where an accumulator register lands in the 64-row tile of its warpgroup: packed pair p (two adjacent columns) of
// warp w, lane l sits at row 16w + l/4 + 8(p%2), columns 8(p/2) + 2(l%4) + {0,1} (wgmma_sm90.cuh).
__device__ __forceinline__ int frag_row(int lane, int p) { return (lane >> 2) + 8 * (p & 1); }
__device__ __forceinline__ int frag_col(int lane, int p) { return (p >> 1) * 8 + (lane & 3) * 2; }

// The accumulator of one 64-row block as fp32 pairs / packed output pairs.
template <class Cfg, class Reg, int NR>
__device__ __forceinline__ float2 acc_pair(const Reg (&d)[NR], int p) {
  if constexpr (Cfg::ACC_F32) {
    return make_float2(d[2 * p], d[2 * p + 1]);
  } else {
    const uint32_t v = d[p];
    const __half2 h = *reinterpret_cast<const __half2*>(&v);
    return make_float2(__low2float(h), __high2float(h));
  }
}
template <class Cfg, class Reg, int NR>
__device__ __forceinline__ uint32_t acc_packed(const Reg (&d)[NR], int p) {
  if constexpr (Cfg::ACC_F32) return ptx::pack_out_x2_rn<Cfg::BF16>(d[2 * p], d[2 * p + 1]);
  else return d[p];   // fp16 accumulators are already the output format
}

// BiasAct<> kernels: the unit's bias, column scales and (rowwise) row scales, prefetched into L1 by one warp as the
// unit starts, so that bias_in_place, which reads them one at a time where they are used, finds them there rather than
// waiting on L2 for each. A prefetch holds no register. n0: the tile's first column; m0: the warpgroup's first row.
template <class Cfg>
__device__ __forceinline__ void bias_act_prefetch(const BiasActArgs& epi, int m0, int n0, int M, int N, int lane) {
  constexpr int kLine = 128;
  const int cols = min(Cfg::BN, N - n0), rows = min(64 * Cfg::M_REP, M - m0);
  if (cols <= 0) return;
  auto fetch = [&](const void* base, int bytes, int first_line) {
    const int i = lane - first_line;   // the lanes [first_line, first_line + lines) each take one line
    if (i >= 0 && i * kLine < bytes) asm volatile("prefetch.global.L1 [%0];" ::"l"(static_cast<const char*>(base) + i * kLine));
  };
  // up to 4 lines of bias (lanes 0-3), 8 of column scales (4-11) and 2 of row scales per 64 rows (12-15)
  if (epi.bias) fetch(static_cast<const uint16_t*>(epi.bias) + n0, cols * 2, 0);
  if constexpr (Cfg::E4M3) {
    if (epi.scales.rowwise) {
      fetch(epi.scales.b + n0, cols * 4, 4);
      if (rows > 0) fetch(epi.scales.a + m0, rows * 4, 12);
    }
  }
}

// BiasAct<> kernels, plain epilogue: the finished sums of the warpgroup's MR 64-row blocks (this warp's rows m_row0 +
// 64 r .. + 15, columns n0 ..), in place, scaled as the wrapped kernel scales them (e4m3 per tensor:
// fp32(acc * fp32(sa * sb)); rowwise: fp32(fp32(acc * sb[n]) * sa[m])) and then biased (one fp32 addition; -0.0 for a
// null bias). The loop runs over the thread's column pairs. The bias and the column scales are read where they are used
// (from L1: bias_act_prefetch), once per column pair for all its rows, so that nothing is held across the accumulators;
// the store (epilogue_store_chunk) then only adds the activation's temporaries to them.
template <class Cfg, class Reg, int MR, int NR>
__device__ __forceinline__ void bias_in_place(Reg (&d)[MR][NR], int lane, int m_row0, int n0, int M, int N,
                                              const BiasActArgs& epi) {
  const uint32_t* bias = static_cast<const uint32_t*>(epi.bias);
  [[maybe_unused]] const float scale = output_scale<Cfg>(epi.scales);
  // rowwise, one 64-row block: its two row scales stay in registers; with two blocks (M_REP = 2) there is no room for
  // their four next to the accumulators, and each is read where it is used
  [[maybe_unused]] float sa_held[2] = {0.f, 0.f};
  if constexpr (Cfg::E4M3 && MR == 1) {
    if (epi.scales.rowwise) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m_row0 + frag_row(lane, h);
        sa_held[h] = m < M ? epi.scales.a[m] : 0.f;
      }
    }
  }
#pragma unroll
  for (int c = 0; c < NR / 4; ++c) {   // pairs 2c (rows l/4) and 2c + 1 (rows l/4 + 8) of every block share two columns
    const int n = n0 + frag_col(lane, 2 * c);   // even, and N % 8 == 0: n < N covers n + 1; past N nothing is stored
    const float2 b = unpack_out_x2<Cfg>(bias && n < N ? __ldg(bias + n / 2) : kNegZeroPair);
    [[maybe_unused]] float2 sb = make_float2(0.f, 0.f);
    if constexpr (Cfg::E4M3) {
      if (epi.scales.rowwise && n < N) sb = __ldg(reinterpret_cast<const float2*>(epi.scales.b + n));
    }
#pragma unroll
    for (int r = 0; r < MR; ++r) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int p = 2 * c + h;
        float x = d[r][2 * p], y = d[r][2 * p + 1];
        if constexpr (Cfg::E4M3) {
          if (epi.scales.rowwise) {   // warp-uniform
            float sa = sa_held[h];
            if constexpr (MR > 1) {
              const int m = m_row0 + 64 * r + frag_row(lane, p);
              sa = m < M ? __ldg(epi.scales.a + m) : 0.f;
            }
            x = __fmul_rn(__fmul_rn(x, sb.x), sa);
            y = __fmul_rn(__fmul_rn(y, sb.y), sa);
          } else {
            x = __fmul_rn(x, scale);
            y = __fmul_rn(y, scale);
          }
        }
        d[r][2 * p] = __fadd_rn(x, b.x);
        d[r][2 * p + 1] = __fadd_rn(y, b.y);
      }
    }
  }
}

// The packed, activated values of one store chunk into the staging buffer (epilogue_store_chunk, BiasAct<> kernels), one
// loop per activation, so that each is straight-line code.
template <class Cfg, int ACT, class Reg, int NR>
__device__ __forceinline__ void store_activated(const Reg (&d)[NR], int chunk, uint32_t epi_buf, int lane) {
  constexpr int EN = Cfg::EPI_N;
  constexpr int PER_CHUNK = EN / 4;
#pragma unroll
  for (int q = 0; q < PER_CHUNK; ++q) {
    uint32_t off = uint32_t(frag_row(lane, q) * (EN * 2) + frag_col(lane, q) * 2);
    off ^= (EN == 64 ? ((off >> 7) & 7u) : ((off >> 7) & 3u)) << 4;
    const float2 v = acc_pair<Cfg>(d, chunk * PER_CHUNK + q);
    ptx::st_shared_b32(epi_buf + off, ptx::pack_out_x2_rn<Cfg::BF16>(activate(v.x, ACT), activate(v.y, ACT)));
  }
}

// registers -> swizzled staging buffer -> TMA store of one EPI_ROWS x EPI_N chunk of this warp. Grouped kernels: M is
// the end row of the tile's group, and a box that straddles it is copied out row by row instead (c_raw: C [., N]).
// With rowwise e4m3 scales
// (`rw` non-null) each fp32 pair is scaled by its column scales, then its row scale, right before the rounding. The
// column scales of a chunk are loaded here, after the previous chunk's store wait, one float2 (one column pair) per
// lane, and reach the lanes that need them by shuffle: two registers per thread instead of the chunk's 16, which the
// 128 accumulators of a BN = 256 (or M_REP = 2) tile leave no room for. BiasAct<> kernels (`epi`: their BiasActArgs)
// find their scales and bias applied (bias_in_place) and apply the activation as they pack.
template <class Cfg, class Reg, int NR>
__device__ __forceinline__ void epilogue_store_chunk(const Reg (&d)[NR], int chunk, uint32_t epi_buf, int lane,
                                                     const CUtensorMap* tmap_c, int col0, int row0, int M, int N,
                                                     const RowwiseEpi* rw = nullptr, int batch = 0,
                                                     __half* __restrict__ c_raw = nullptr,
                                                     const typename Cfg::EpiArgs* epi = nullptr) {
  using namespace ptx;
  constexpr int EN = Cfg::EPI_N;
  constexpr int PER_CHUNK = EN / 4;   // packed pairs of one chunk per thread
  // Gated<Grouped<>> kernels: the lane is hidden from the compiler, so that each chunk computes its staging offsets
  // anew. Otherwise ptxas holds them across the SwiGLU epilogue and, next to the group's cursor, spills them to the
  // stack in configuration 0. The other kernels are compiled as before.
  if constexpr (is_gated<Cfg>() && grouped<Cfg>()) asm volatile("" : "+r"(lane));
  // the previous store from this warp's staging buffer must have finished reading it
  if (lane == 0) tma_store_wait_read<0>();
  __syncwarp();
  [[maybe_unused]] float2 sb_lane = make_float2(0.f, 0.f);   // rowwise: chunk columns 2 lane, 2 lane + 1
  [[maybe_unused]] float sbx = 0.f, sby = 0.f;                 // rowwise: the column scales of pairs q, q + 1 (q even)
  if constexpr (Cfg::E4M3) {
    const int n = col0 + 2 * lane;   // even, and N % 8 == 0: n < N covers n + 1
    if (rw && 2 * lane < EN && n < N) sb_lane = *reinterpret_cast<const float2*>(rw->sb + n);
  }
  if constexpr (bias_act<Cfg>()) {
    // the values are scaled and biased already (bias_in_place): the activation, then the one rounding
    if (epi->act == kActGeluTanh) store_activated<Cfg, kActGeluTanh>(d, chunk, epi_buf, lane);
    else if (epi->act == kActRelu) store_activated<Cfg, kActRelu>(d, chunk, epi_buf, lane);
    else store_activated<Cfg, kActNone>(d, chunk, epi_buf, lane);
  } else {
#pragma unroll
  for (int q = 0; q < PER_CHUNK; ++q) {
    uint32_t off = uint32_t(frag_row(lane, q) * (EN * 2) + frag_col(lane, q) * 2);
    // 128-byte rows use the 128B swizzle (16-byte chunk ^= row % 8), 64-byte rows the 64B one (chunk ^= (row / 2) % 4)
    off ^= (EN == 64 ? ((off >> 7) & 7u) : ((off >> 7) & 3u)) << 4;
    if constexpr (Cfg::E4M3) {
      if (rw) {   // warp-uniform
        if ((q & 1) == 0) {   // pairs q and q + 1 share their columns (rows l/4 and l/4 + 8)
          const int src = frag_col(lane, q) / 2;   // the lane holding them
          sbx = __shfl_sync(0xffffffffu, sb_lane.x, src);
          sby = __shfl_sync(0xffffffffu, sb_lane.y, src);
        }
        const float sa = (q & 1) ? rw->sa_hi : rw->sa_lo;
        const float2 v = acc_pair<Cfg>(d, chunk * PER_CHUNK + q);
        st_shared_b32(epi_buf + off, pack_out_x2_rn<Cfg::BF16>(__fmul_rn(__fmul_rn(v.x, sbx), sa),
                                                               __fmul_rn(__fmul_rn(v.y, sby), sa)));
        continue;
      }
    }
    st_shared_b32(epi_buf + off, acc_packed<Cfg>(d, chunk * PER_CHUNK + q));
  }
  }
  fence_proxy_async_smem();
  __syncwarp();
  if constexpr (grouped<Cfg>()) {
    // A box that straddles the group's end (warp-uniform): the rows past it belong to the next group, which another
    // CTA is storing, so only the rows below M leave, one 16-byte chunk per lane and step, read through the same
    // swizzle. N % 8 == 0: a chunk is wholly inside or wholly outside the columns. A box at or past M stores nothing.
    if (row0 + Cfg::EPI_ROWS > M) {
      constexpr int CPR = EN * 2 / 16;   // 16-byte chunks per staged row
#pragma unroll 1
      for (int i = lane; i < Cfg::EPI_ROWS * CPR; i += 32) {
        const int r = i / CPR, c = i % CPR;
        if (row0 + r < M && col0 + 8 * c < N) {
          uint32_t off = uint32_t(r * (EN * 2) + c * 16);
          off ^= (EN == 64 ? ((off >> 7) & 7u) : ((off >> 7) & 3u)) << 4;
          *reinterpret_cast<uint4*>(c_raw + size_t(row0 + r) * N + col0 + 8 * c) = ld_shared_v4_b32(epi_buf + off);
        }
      }
      return;
    }
  }
  if (lane == 0) {
    if (row0 < M && col0 < N) {   // rows/cols past the edge are clipped by the tensor map
      if constexpr (batched<Cfg>() || k_grouped<Cfg>()) tma_store_3d(tmap_c, epi_buf, col0, row0, batch);
      else tma_store_2d(tmap_c, epi_buf, col0, row0);
    }
    tma_store_commit();
  }
}

// The plain epilogue of a BiasAct<> unit: the scales and the bias in place (bias_in_place), then for every 64-row block R
// of the warpgroup (rows m_row0 + 64 R ..) its store chunks J. The blocks and chunks are unrolled by recursion rather
// than by loop pragmas, which the compiler declines for bodies of this size: a chunk index that is not a constant would
// move the accumulators to local memory.
template <class Cfg, int R = 0, int J = 0, class Reg, int MR, int NR>
__device__ __forceinline__ void bias_act_epilogue(Reg (&acc)[MR][NR], uint32_t epi_buf, int lane, const CUtensorMap* tmap_c,
                                                  int m_row0, int n0, int M, int N, const BiasActArgs& epi) {
  if constexpr (R < MR) {
    const int row0 = m_row0 + R * 64;
    if constexpr (R == 0 && J == 0) {
      bias_in_place<Cfg>(acc, lane, m_row0, n0, M, N, epi);
#pragma unroll
      for (int r = 0; r < MR; ++r) ptx::reg_fence(acc[r]);
    }
    if constexpr (J < Cfg::EPI_CHUNKS) {
      epilogue_store_chunk<Cfg>(acc[R], J, epi_buf, lane, tmap_c, n0 + J * Cfg::EPI_N, row0, M, N, nullptr, 0, nullptr,
                                &epi);
      bias_act_epilogue<Cfg, R, J + 1>(acc, epi_buf, lane, tmap_c, m_row0, n0, M, N, epi);
    } else {
      bias_act_epilogue<Cfg, R + 1, 0>(acc, epi_buf, lane, tmap_c, m_row0, n0, M, N, epi);
    }
  }
}

// Gated<> kernels: y of one gate / up pair of store chunks (J = chunk, J + 1) of this warp's 16 rows into the staging
// buffer, then its TMA store at y's column col0 = (n0 + 64 J) / 2 and row row0. g and u are rounded to the output type
// as the h store packs them (RN), so y is silu_mul of the 16-bit h. Rows past M are clipped by the map; I % 64 == 0, so
// a pair is wholly inside or wholly outside y's columns. Grouped kernels: M is the end row of the tile's group, and a
// box that straddles it is copied out row by row to y_raw [., I] instead, as epilogue_store_chunk does for C.
template <class Cfg, class Reg, int NR>
__device__ __forceinline__ void gated_store_chunk(const Reg (&d)[NR], int chunk, uint32_t epi_buf, int lane,
                                                  const CUtensorMap* tmap_y, int col0, int row0, int M, int I,
                                                  __half* __restrict__ y_raw = nullptr) {
  using namespace ptx;
  using T = std::conditional_t<Cfg::BF16, __nv_bfloat16, __half>;
  constexpr int EN = Cfg::EPI_N;
  constexpr int PER_CHUNK = EN / 4;
  static_assert(EN == 64, "64-column chunks");
  if constexpr (grouped<Cfg>()) asm volatile("" : "+r"(lane));   // see epilogue_store_chunk
  if (lane == 0) tma_store_wait_read<0>();
  __syncwarp();
#pragma unroll
  for (int q = 0; q < PER_CHUNK; ++q) {
    uint32_t off = uint32_t(frag_row(lane, q) * (EN * 2) + frag_col(lane, q) * 2);
    off ^= ((off >> 7) & 7u) << 4;
    const float2 g = acc_pair<Cfg>(d, chunk * PER_CHUNK + q), u = acc_pair<Cfg>(d, (chunk + 1) * PER_CHUNK + q);
    const float y0 = silu_mul<T>(round_to(g.x, T()), round_to(u.x, T()));
    const float y1 = silu_mul<T>(round_to(g.y, T()), round_to(u.y, T()));
    st_shared_b32(epi_buf + off, pack_out_x2_rn<Cfg::BF16>(y0, y1));   // exact: both are 16-bit values already
  }
  fence_proxy_async_smem();
  __syncwarp();
  if constexpr (grouped<Cfg>()) {
    // a box that straddles the group's end (warp-uniform): only the rows below M, one 16-byte chunk per lane and step
    if (row0 + Cfg::EPI_ROWS > M) {
      constexpr int CPR = EN * 2 / 16;   // 16-byte chunks per staged row
#pragma unroll 1
      for (int i = lane; i < Cfg::EPI_ROWS * CPR; i += 32) {
        const int r = i / CPR, c = i % CPR;
        if (row0 + r < M && col0 + 8 * c < I) {
          uint32_t off = uint32_t(r * (EN * 2) + c * 16);
          off ^= ((off >> 7) & 7u) << 4;
          *reinterpret_cast<uint4*>(y_raw + size_t(row0 + r) * I + col0 + 8 * c) = ld_shared_v4_b32(epi_buf + off);
        }
      }
      return;
    }
  }
  if (lane == 0) {
    if (row0 < M && col0 < I) tma_store_2d(tmap_y, epi_buf, col0, row0);
    tma_store_commit();
  }
}

// The plain epilogue of a Gated<> unit: for every 64-row block R of the warpgroup (rows m_row0 + 64 R ..) and every
// gate / up pair of chunks (J, J + 1), h's two chunks when the launch stores h (epilogue_store_chunk, the wrapped
// kernel's bits), then y's chunk (gated_store_chunk). Unrolled by recursion, as bias_act_epilogue is. Grouped kernels:
// m_row0 counts from the group's first row, M is the group's end, and h_raw / y_raw take the rows of a box that
// straddles it.
template <class Cfg, int R = 0, int J = 0, class Reg, int MR, int NR>
__device__ __forceinline__ void gated_epilogue(const Reg (&acc)[MR][NR], uint32_t epi_buf, int lane,
                                               const CUtensorMap* tmap_h, const GatedArgs& epi, int m_row0, int n0,
                                               int M, int N, __half* __restrict__ h_raw = nullptr,
                                               __half* __restrict__ y_raw = nullptr) {
  if constexpr (R < MR) {
    const int row0 = m_row0 + R * 64;
    if constexpr (J < Cfg::EPI_CHUNKS) {
      if (epi.store_h) {
        epilogue_store_chunk<Cfg>(acc[R], J, epi_buf, lane, tmap_h, n0 + J * Cfg::EPI_N, row0, M, N, nullptr, 0, h_raw);
        epilogue_store_chunk<Cfg>(acc[R], J + 1, epi_buf, lane, tmap_h, n0 + (J + 1) * Cfg::EPI_N, row0, M, N, nullptr,
                                  0, h_raw);
      }
      gated_store_chunk<Cfg>(acc[R], J, epi_buf, lane, &epi.y_map, (n0 + J * Cfg::EPI_N) / 2, row0, M, N / 2, y_raw);
      gated_epilogue<Cfg, R, J + 2>(acc, epi_buf, lane, tmap_h, epi, m_row0, n0, M, N, h_raw, y_raw);
    } else {
      gated_epilogue<Cfg, R + 1, 0>(acc, epi_buf, lane, tmap_h, epi, m_row0, n0, M, N, h_raw, y_raw);
    }
  }
}

// The tile of an empty group of a K-grouped kernel (GroupedK<>): +0.0 in this warp's MR x 16 rows from row0 (of
// matrix `batch` of C [., M, N]) and BN columns from col0, clipped at M and N, with 16-byte generic stores.
template <class Cfg>
__device__ __forceinline__ void zero_tile_store(__half* __restrict__ c, int batch, int row0, int col0, int M, int N,
                                                int lane) {
  constexpr int CPR = Cfg::BN / 8;   // 16-byte chunks per row
#pragma unroll 1
  for (int r = 0; r < Cfg::M_REP; ++r) {
#pragma unroll 1
    for (int i = lane; i < Cfg::EPI_ROWS * CPR; i += 32) {
      const int gm = row0 + r * 64 + i / CPR, gn = col0 + 8 * (i % CPR);
      if (gm < M && gn < N) *reinterpret_cast<uint4*>(c + (size_t(batch) * M + gm) * N + gn) = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

// One finished float4 of the split-K reductions added in place into C32 (AccumF32<> kernels), at a 16-byte aligned
// address.
__device__ __forceinline__ void accum_quad(float* __restrict__ dst, const float4& v) {
  float4* p = reinterpret_cast<float4*>(dst);
  float4 o = *p;
  o.x = __fadd_rn(o.x, v.x); o.y = __fadd_rn(o.y, v.y);
  o.z = __fadd_rn(o.z, v.z); o.w = __fadd_rn(o.w, v.w);
  *p = o;
}

// One 64-row block of the plain (and stream-K owner) epilogue of an AccumF32<> unit: the finished sums of this warp's
// rows row0 .. row0 + 15 and columns n0 .., scaled as the wrapped kernel scales them before its rounding (e4m3 rowwise:
// fp32(fp32(acc * sb[n]) * sa[m]); per tensor: fp32(acc * fp32(sa * sb))), added into c32 [M, N] (the unit's own
// matrix) straight from the registers. Rows at or past M and columns at or past N are not touched (N % 8 == 0: n < N
// covers n + 1). The column scales are read where they are used, one float2 per column pair, so that nothing is held
// across the accumulators. The pairs of a row go in groups of G: the group's G loads of C32 are issued back to back,
// then its G additions and stores. Pair by pair, every load would wait for the previous pair's store (the compiler
// cannot prove that they do not alias), one dependent global round trip per pair.
template <class Cfg, class Reg, int NR>
__device__ __forceinline__ void accum_block(const Reg (&d)[NR], int lane, int row0, int n0, int M, int N,
                                           float* __restrict__ c32, const Scales& s, float scale) {
  constexpr int PAIRS = NR / 4;                  // column pairs of one row
  // pairs in flight, 2 G registers next to the accumulators; the rowwise e4m3 kernels also hold the column scales
  constexpr int G_MAX = (Cfg::E4M3 && !block_scaled<Cfg>()) ? 2 : 8;
  constexpr int G = PAIRS < G_MAX ? PAIRS : G_MAX;
  static_assert(PAIRS % G == 0, "whole groups");
#pragma unroll
  for (int h = 0; h < 2; ++h) {   // pairs 2c + h share row l/4 + 8h
    const int m = row0 + frag_row(lane, h);
    if (m >= M) continue;
    [[maybe_unused]] float sa = 0.f;
    if constexpr (Cfg::E4M3 && !block_scaled<Cfg>()) {
      if (s.rowwise) sa = __ldg(s.a + m);
    }
    float* row = c32 + size_t(m) * N;
#pragma unroll
    for (int c0 = 0; c0 < PAIRS; c0 += G) {
      float2 old[G];
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const int n = n0 + frag_col(lane, 2 * (c0 + j) + h);
        old[j] = n < N ? *reinterpret_cast<const float2*>(row + n) : make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const int p = 2 * (c0 + j) + h;
        const int n = n0 + frag_col(lane, p);
        if (n >= N) continue;
        float x = d[2 * p], y = d[2 * p + 1];
        if constexpr (Cfg::E4M3 && !block_scaled<Cfg>()) {
          if (s.rowwise) {   // warp-uniform
            const float2 sb = __ldg(reinterpret_cast<const float2*>(s.b + n));
            x = __fmul_rn(__fmul_rn(x, sb.x), sa);
            y = __fmul_rn(__fmul_rn(y, sb.y), sa);
          } else {
            x = __fmul_rn(x, scale);
            y = __fmul_rn(y, scale);
          }
        }
        *reinterpret_cast<float2*>(row + n) = make_float2(__fadd_rn(old[j].x, x), __fadd_rn(old[j].y, y));
      }
    }
  }
}

// The plain (and stream-K owner) epilogue of an AccumF32<> unit: accum_block for each of the warpgroup's MR 64-row blocks
// (this warp's rows m_row0 + 64 r ..). The blocks are separate calls rather than a loop, which the compiler declines to
// unroll around a body of this size: a block index that is not a constant would move the accumulators to local memory.
template <class Cfg, class Reg, int MR, int NR>
__device__ __forceinline__ void accum_epilogue(const Reg (&d)[MR][NR], int lane, int m_row0, int n0, int M, int N,
                                               float* __restrict__ c32, const Scales& s) {
  static_assert(MR == 1 || MR == 2, "one or two 64-row blocks per warpgroup");
  const float scale = output_scale<Cfg>(s);
  accum_block<Cfg>(d[0], lane, m_row0, n0, M, N, c32, s, scale);
  if constexpr (MR == 2) accum_block<Cfg>(d[1], lane, m_row0 + 64, n0, M, N, c32, s, scale);
}

// Split-K epilogue (CTA_GROUP == 1, one (tile, split) unit per CTA, all units resident at once).
//   phase 1  every split writes its 128 x BN fp32 partial tile to the workspace slot (tile, split);
//   barrier  a per-tile arrival counter in global memory (release/acquire at gpu scope);
//   phase 2  split s sums a contiguous 1/splits slice of the tile's rows over ALL partials in the fixed
//            order s' = 0..splits-1 (deterministic), scales it (e4m3), rounds once to fp16 and stores to C.
// The last split to finish phase 2 zeroes both counters, so the next launch on the stream starts clean.
template <class Cfg, class Reg, int NR>
__device__ __forceinline__ void splitk_epilogue(const Reg (&d)[NR], int e, int row_base, int lane, int tile, int split,
                                                int splits, int m_base, int n0, int M, int N, float* __restrict__ ws,
                                                unsigned* __restrict__ ctr, __half* __restrict__ C,
                                                uint32_t red_smem, uint32_t red_bar,
                                                const typename Cfg::EpiArgs& epi) {
  using namespace ptx;
  constexpr int BN = Cfg::BN;
  const Scales& scales = scales_of(epi);
  float* slot = ws + (size_t(tile) * splits + split) * (kBlockM * BN);
#pragma unroll
  for (int p = 0; p < NR * (Cfg::ACC_F32 ? 1 : 2) / 2; ++p) {
    const float2 v = acc_pair<Cfg>(d, p);
    __stcg(reinterpret_cast<float2*>(slot + size_t(row_base + frag_row(lane, p)) * BN + frag_col(lane, p)), v);
  }
  // publish the partial, then wait until every split of this tile has published its own
  __threadfence();
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
  if (e == 0) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr + tile) : "memory");
    unsigned seen = 0, spins = 0;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(ctr + tile) : "memory");
      if (seen < unsigned(splits)) {
        __nanosleep(64);
        if (++spins > (1u << 24)) __trap();   // watchdog: a sibling split never arrived
      }
    } while (seen < unsigned(splits));
  }
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
  // phase 2: rows [r0, r1) of the tile belong to this split. Their slices of all `splits` partials are pulled
  // into the (now idle) pipeline smem with 1-D bulk copies — one contiguous slice per partial — and summed there.
  const int rows_per = (kBlockM + splits - 1) / splits;
  const int r0 = split * rows_per;
  const int r1 = min(kBlockM, r0 + rows_per);
  if (r0 < r1) {
    const uint32_t slice_bytes = uint32_t(r1 - r0) * BN * 4u;
    const float* tile_ws = ws + size_t(tile) * splits * (kBlockM * BN) + size_t(r0) * BN;
    if (e == 0) {
      fence_proxy_async_all();   // the partials were written through the generic proxy by other CTAs
      mbar_arrive_expect_tx(red_bar, slice_bytes * uint32_t(splits));
      for (int sp = 0; sp < splits; ++sp)
        bulk_load_1d(red_smem + uint32_t(sp) * slice_bytes, tile_ws + size_t(sp) * (kBlockM * BN), slice_bytes, red_bar);
    }
    mbar_wait(red_bar, 0);
    const float scale = output_scale<Cfg>(scales);
    constexpr int V = BN / 4;      // float4 per row
    for (int i = e; i < (r1 - r0) * V; i += kConsumerThreads) {
      const int r = r0 + i / V, c4 = i % V;
      const int gm = m_base + r, gn = n0 + c4 * 4;
      if (gm >= M || gn >= N) continue;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int sp = 0; sp < splits; ++sp) {   // fixed order: deterministic
        const float4 p = ld_shared_v4f(red_smem + uint32_t(sp) * slice_bytes + uint32_t(i) * 16u);
        acc.x += p.x; acc.y += p.y; acc.z += p.z; acc.w += p.w;
      }
      scale_quad<Cfg>(acc, scale, scales, gm, gn);
      bias_act_quad<Cfg>(acc, epi, gn);
      if constexpr (accum_f32<Cfg>()) {
        accum_quad(epi.c32 + size_t(gm) * N + gn, acc);
        continue;
      }
      uint2 out;
      out.x = pack_out_x2_rn<Cfg::BF16>(acc.x, acc.y);
      out.y = pack_out_x2_rn<Cfg::BF16>(acc.z, acc.w);
      *reinterpret_cast<uint2*>(C + size_t(gm) * N + gn) = out;
    }
  }
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
  if (e == 0) {
    unsigned old;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(old) : "l"(ctr + kMaxSplitTiles + tile) : "memory");
    if (old == unsigned(splits - 1)) {   // everyone is past the arrival wait: safe to reset for the next launch
      ctr[tile] = 0;
      ctr[kMaxSplitTiles + tile] = 0;
      __threadfence();
    }
  }
}

// Cluster split-K (CTA_GROUP == 1): the `splits` CTAs of a thread-block cluster share one output tile, each
// accumulating its own k-range. Phase 1 parks the fp32 partial tile in the CTA's own (now idle) pipeline smem;
// after a cluster barrier, CTA r sums rows [r*128/splits, (r+1)*128/splits) over all peers through distributed
// shared memory in fixed order (deterministic), rounds once and stores to C. No global workspace, no atomics.
__host__ __device__ constexpr uint32_t cluster_partial_row_bytes(int bn) { return uint32_t(bn) * 4u + 16u; }   // +16 B: conflict-free rows

template <class Cfg, class Reg, int NR>
__device__ __forceinline__ void cluster_splitk_park(const Reg (&d)[NR], int row_base, int lane, uint32_t part_smem) {
  using namespace ptx;
#pragma unroll
  for (int p = 0; p < NR * (Cfg::ACC_F32 ? 1 : 2) / 2; ++p) {
    const float2 v = acc_pair<Cfg>(d, p);
    st_shared_v2f(part_smem + uint32_t(row_base + frag_row(lane, p)) * cluster_partial_row_bytes(Cfg::BN) +
                      uint32_t(frag_col(lane, p)) * 4u, v.x, v.y);
  }
}

template <class Cfg>
__device__ __forceinline__ void cluster_splitk_reduce(int e, int split, int splits, int m_base, int n0, int M, int N,
                                                      uint32_t part_smem, __half* __restrict__ C,
                                                      const typename Cfg::EpiArgs& epi) {
  using namespace ptx;
  const Scales& scales = scales_of(epi);
  constexpr int BN = Cfg::BN;
  constexpr int V = BN / 4;
  const float scale = output_scale<Cfg>(scales);
  const int rows_per = kBlockM / splits;            // splits is 2, 4 or 8
  const int r0 = split * rows_per;
  uint32_t peer[8];
#pragma unroll
  for (int p = 0; p < 8; ++p) peer[p] = (p < splits) ? mapa(part_smem, uint32_t(p)) : 0u;
  for (int i = e; i < rows_per * V; i += kConsumerThreads) {
    const int r = r0 + i / V, c4 = i % V;
    const int gm = m_base + r, gn = n0 + c4 * 4;
    if (gm >= M || gn >= N) continue;
    const uint32_t off = uint32_t(r) * cluster_partial_row_bytes(BN) + uint32_t(c4) * 16u;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      if (p < splits) {
        const float4 v = ld_dsmem_v4f(peer[p] + off);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
    scale_quad<Cfg>(acc, scale, scales, gm, gn);
    bias_act_quad<Cfg>(acc, epi, gn);
    if constexpr (accum_f32<Cfg>()) {
      accum_quad(epi.c32 + size_t(gm) * N + gn, acc);
      continue;
    }
    uint2 out;
    out.x = pack_out_x2_rn<Cfg::BF16>(acc.x, acc.y);
    out.y = pack_out_x2_rn<Cfg::BF16>(acc.z, acc.w);
    *reinterpret_cast<uint2*>(C + size_t(gm) * N + gn) = out;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Stream-K (hgemm_schedule.cuh). Partial tiles travel through the global workspace as REGISTER IMAGES: consumer
// thread t writes its accumulator registers, four at a time, to uint4 (i, t) of its CTA's slot, and the owner's
// thread t reads them back the same way, so both directions are fully coalesced and no thread ever needs another
// thread's element. One flag per (CTA slot, consumer warp): raised by the contributor warp after its image is
// written, polled and lowered again by the owner warp, so the flags are zero again when the grid ends.
constexpr int kMaxStreamKSlots = 160;   // CTAs of a launch (>= 132 SMs), one partial-tile slot each
constexpr int kStreamKFlagsPerSlot = 8; // consumer warps

template <class Cfg>
struct StreamK {
  static constexpr int REGS = Cfg::ACC_F32 ? Cfg::BN / 2 : Cfg::BN / 4;   // 32-bit accumulator registers per thread
  static constexpr int R4 = REGS / 4;
  static constexpr int SLOT_U4 = R4 * kConsumerThreads;                    // one CTA: 128 rows x BN columns
  static_assert(REGS % 4 == 0, "register images move in uint4");
};

template <class Cfg, class Reg, int NR>
__device__ __forceinline__ void streamk_contribute(const Reg (&d)[NR], int t, int ew, int lane, uint4* __restrict__ ws,
                                                   unsigned* __restrict__ flags, int slot) {
  using namespace ptx;
  using SK = StreamK<Cfg>;
  uint4* base = ws + size_t(slot) * SK::SLOT_U4 + t;
#pragma unroll
  for (int i = 0; i < SK::R4; ++i) {
    uint32_t x[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if constexpr (Cfg::ACC_F32) x[c] = __float_as_uint(d[4 * i + c]);
      else x[c] = d[4 * i + c];
    }
    st_global_cg_v4(base + i * kConsumerThreads, x[0], x[1], x[2], x[3]);
  }
  __threadfence();   // every lane's stores are visible at gpu scope before lane 0 publishes the flag
  __syncwarp();
  if (lane == 0) st_release_gpu(flags + slot * kStreamKFlagsPerSlot + ew, 1u);
}

// Owner: the partials of `n` contributors (slots slot0, slot0 + slot_stride, ... — increasing k) added to the own
// accumulator in fp32 in that fixed order; fp16 accumulators are widened, summed and rounded once. The images are
// unscaled: an e4m3 owner's plain epilogue applies the scales to the finished sum. The flags are
// lowered afterwards (this warp is their only reader, and the next writer is a later launch).
template <class Cfg, class Reg, int NR>
__device__ __forceinline__ void streamk_own(Reg (&d)[NR], int t, int ew, int lane, const uint4* __restrict__ ws,
                                            unsigned* __restrict__ flags, int slot0, int slot_stride, int n) {
  using namespace ptx;
  using SK = StreamK<Cfg>;
  if (lane == 0) {
    for (int p = 0; p < n; ++p) {
      const unsigned* f = flags + (slot0 + p * slot_stride) * kStreamKFlagsPerSlot + ew;
      unsigned spins = 0;
      while (ld_acquire_gpu(f) == 0u) {
        __nanosleep(64);
        if (++spins > (1u << 24)) __trap();   // watchdog: a contributor never raised its flag
      }
    }
  }
  __syncwarp();
#pragma unroll
  for (int i = 0; i < SK::R4; ++i) {
    float f[Cfg::ACC_F32 ? 4 : 8];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if constexpr (Cfg::ACC_F32) {
        f[c] = d[4 * i + c];
      } else {
        const uint32_t v = d[4 * i + c];
        const __half2 h = *reinterpret_cast<const __half2*>(&v);
        f[2 * c] = __low2float(h); f[2 * c + 1] = __high2float(h);
      }
    }
    for (int p = 0; p < n; ++p) {
      const uint4 v = ld_global_cg_v4(ws + size_t(slot0 + p * slot_stride) * SK::SLOT_U4 + size_t(i) * kConsumerThreads + t);
      const uint32_t x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if constexpr (Cfg::ACC_F32) {
          f[c] += __uint_as_float(x[c]);
        } else {
          const __half2 h = *reinterpret_cast<const __half2*>(&x[c]);
          f[2 * c] += __low2float(h); f[2 * c + 1] += __high2float(h);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if constexpr (Cfg::ACC_F32) d[4 * i + c] = f[c];
      else d[4 * i + c] = pack_out_x2_rn<false>(f[2 * c], f[2 * c + 1]);   // the one rounding of the fp16 output
    }
  }
  __syncwarp();
  if (lane == 0)
    for (int p = 0; p < n; ++p) flags[(slot0 + p * slot_stride) * kStreamKFlagsPerSlot + ew] = 0u;
}

// The kernel: hgemm_tn_kernel for every configuration but BiasAct<>'s, hgemm_bias_act_kernel for those. They differ in
// their last parameter only (Cfg::EpiArgs) and share their body, hgemm_tn_kernel_body.inc, which reads the scales as
// `scales` and hands the epilogues `epi`, the kernel's EpiArgs.
template <class Cfg, int KMODE = kPlain>
__global__ void __launch_bounds__(kNumThreads, 1)
hgemm_tn_kernel(const __grid_constant__ CUtensorMap tmap_a,   // A  [M,K]  box {BLOCK_K, A_BOX_ROWS}
                const __grid_constant__ CUtensorMap tmap_b,   // Bt [N,K]  box {BLOCK_K, B_BOX_ROWS}; row-major
                                                              // B (RowMajorB<>): B [K,N] box {64, B_K_ROWS}
                const __grid_constant__ CUtensorMap tmap_c,   // C  [M,N]  box {EPI_N, EPI_ROWS}
                int M, int N, int K, int group_m,
                int splits_arg,                   // split-K factor (modes kWorkspaceSplitK / kClusterSplitK: one unit per CTA);
                                                  // batched kernels (plain only): the batch count; grouped: G
                int aux_arg,                      // mode kStreamK: sk_tiles, the first tiles, cut along K across all
                                                  // workers; block-scaled kernels (no stream-K): ld_a of scales.a
                float* __restrict__ splitk_ws,    // [units][128][BN] fp32 partial tiles (workspace split-K) / stream-K slots
                unsigned* __restrict__ splitk_ctr,   // [2][kMaxSplitTiles] split-K arrive / done counters, then the
                                                     // stream-K flags; all zero between launches. Batched kernels:
                                                     // the int32 row counts per batch, or null (dense);
                                                     // grouped: the G int32 offsets (cumulative group ends)
                __half* __restrict__ c_raw,       // C base pointer, used by the split-K reductions' direct stores
                uint64_t hint_a, uint64_t hint_b, // L2 eviction priority of the A / B loads (ptx::kL2Evict*)
                Scales scales                     /* e4m3: the per-tensor scales (not read by the 16-bit kernels) */) {
  static_assert(!bias_act<Cfg>() && !block_1d1d<Cfg>(), "BiasAct<> and BlockScaled1D1D<>: kernels of their own");
  const Scales& epi = scales;
#include "hgemm_tn_kernel_body.inc"
}

// The same with a bias and an activation (BiasAct<>): the parameters of hgemm_tn_kernel, BiasActArgs last.
template <class Cfg, int KMODE = kPlain>
__global__ void __launch_bounds__(kNumThreads, 1)
hgemm_bias_act_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                      const __grid_constant__ CUtensorMap tmap_c, int M, int N, int K, int group_m, int splits_arg,
                      int aux_arg, float* __restrict__ splitk_ws, unsigned* __restrict__ splitk_ctr,
                      __half* __restrict__ c_raw, uint64_t hint_a, uint64_t hint_b, BiasActArgs epi) {
  static_assert(bias_act<Cfg>(), "a BiasAct<> configuration");
  const Scales& scales = epi.scales;
#include "hgemm_tn_kernel_body.inc"
}

// The same with 1 x 128 scales on both operands (BlockScaled1D1D<>): the parameters of hgemm_tn_kernel, Block1D1DArgs
// last.
template <class Cfg, int KMODE = kPlain>
__global__ void __launch_bounds__(kNumThreads, 1)
hgemm_block_1d1d_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                        const __grid_constant__ CUtensorMap tmap_c, int M, int N, int K, int group_m, int splits_arg,
                        int aux_arg, float* __restrict__ splitk_ws, unsigned* __restrict__ splitk_ctr,
                        __half* __restrict__ c_raw, uint64_t hint_a, uint64_t hint_b, Block1D1DArgs epi) {
  static_assert(block_1d1d<Cfg>(), "a BlockScaled1D1D<> configuration");
  const Scales& scales = epi.scales;
#include "hgemm_tn_kernel_body.inc"
}

// The same adding into an fp32 C (AccumF32<>): the parameters of hgemm_tn_kernel, AccumArgs (the wrapped kernel's
// EpiArgs and the fp32 C) last. tmap_c and c_raw are not written.
template <class Cfg, int KMODE = kPlain>
__global__ void __launch_bounds__(kNumThreads, 1)
hgemm_accum_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   const __grid_constant__ CUtensorMap tmap_c, int M, int N, int K, int group_m, int splits_arg,
                   int aux_arg, float* __restrict__ splitk_ws, unsigned* __restrict__ splitk_ctr,
                   __half* __restrict__ c_raw, uint64_t hint_a, uint64_t hint_b, typename Cfg::EpiArgs epi) {
  static_assert(accum_f32<Cfg>(), "an AccumF32<> configuration");
  const Scales& scales = scales_of(epi);
#include "hgemm_tn_kernel_body.inc"
}

// The same with the SwiGLU epilogue (Gated<>): the parameters of hgemm_tn_kernel, GatedArgs (y's map, read in place as
// tmap_c is) last; tmap_c is h's map, written only when epi.store_h is set. Plain schedule only.
template <class Cfg, int KMODE = kPlain>
__global__ void __launch_bounds__(kNumThreads, 1)
hgemm_gated_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   const __grid_constant__ CUtensorMap tmap_c, int M, int N, int K, int group_m, int splits_arg,
                   int aux_arg, float* __restrict__ splitk_ws, unsigned* __restrict__ splitk_ctr,
                   __half* __restrict__ c_raw, uint64_t hint_a, uint64_t hint_b, const __grid_constant__ GatedArgs epi) {
  static_assert(is_gated<Cfg>() && KMODE == kPlain, "a Gated<> configuration, plain schedule");
  const Scales scales{nullptr, nullptr};   // 16-bit operands: no scales
#include "hgemm_tn_kernel_body.inc"
}

// The same over contiguous row groups (Gated<Grouped<>>): the parameters of hgemm_tn_kernel with Grouped<>'s meaning
// (splits_arg G, splitk_ctr the offsets, c_raw h), GroupedGatedArgs (y's map and y itself) last.
template <class Cfg, int KMODE = kPlain>
__global__ void __launch_bounds__(kNumThreads, 1)
hgemm_grouped_gated_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                           const __grid_constant__ CUtensorMap tmap_c, int M, int N, int K, int group_m,
                           int splits_arg, int aux_arg, float* __restrict__ splitk_ws,
                           unsigned* __restrict__ splitk_ctr, __half* __restrict__ c_raw, uint64_t hint_a,
                           uint64_t hint_b, const __grid_constant__ GroupedGatedArgs epi) {
  static_assert(is_gated<Cfg>() && grouped<Cfg>() && KMODE == kPlain, "a Gated<Grouped<>> configuration, plain schedule");
  const Scales scales{nullptr, nullptr};   // 16-bit operands: no scales
#include "hgemm_tn_kernel_body.inc"
}

// The kernel of (Cfg, KMODE).
template <class Cfg, int KMODE>
constexpr auto kernel_of() {
  if constexpr (is_gated<Cfg>() && grouped<Cfg>()) return &hgemm_grouped_gated_kernel<Cfg, KMODE>;
  else if constexpr (is_gated<Cfg>()) return &hgemm_gated_kernel<Cfg, KMODE>;
  else if constexpr (accum_f32<Cfg>()) return &hgemm_accum_kernel<Cfg, KMODE>;
  else if constexpr (bias_act<Cfg>()) return &hgemm_bias_act_kernel<Cfg, KMODE>;
  else if constexpr (block_1d1d<Cfg>()) return &hgemm_block_1d1d_kernel<Cfg, KMODE>;
  else return &hgemm_tn_kernel<Cfg, KMODE>;
}

}  // namespace b200
