// H100 (sm_90a) HGEMM:  C[M,N] (fp16) = A[M,K] (fp16, K-contiguous) * Bt[N,K]^T (fp16, K-contiguous)
// with fp32 (F32F16F16F32) or fp16 (F16F16F16F16) accumulation in registers.
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

#include "hgemm_schedule.cuh"
#include "ptx_sm90.cuh"
#include "wgmma_sm90.cuh"


namespace b200 {

constexpr int kBlockK = 64;          // 64 fp16 = 128 B = one swizzle row
constexpr int kWgmmaK = 16;          // K per wgmma.mma_async (16-bit operands)
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

#ifndef B200_HGEMM_NO_K_DECOMP
#define B200_HGEMM_NO_K_DECOMP 0     // experiment: kernels without split-K / stream-K code
#endif

template <int BN_, int STAGES_, int CTA_GROUP_, bool ACC_F32_, int CLUSTER_M_ = 1, int CLUSTER_N_ = 1, int M_REP_ = 1, bool BF16_ = false>
struct Config {
  static constexpr int BN = BN_;               // tile N (= wgmma N)
  static constexpr int CTA_GROUP = CTA_GROUP_; // 1: one CTA per 128-row tile; 2: a pair of CTAs sharing the B tile
  static constexpr bool ACC_F32 = ACC_F32_;
  // bf16 operands and bf16 output instead of fp16 (README.md:73 "denser configurations" territory): same pipeline, the
  // wgmma type and the epilogue's convert differ. bf16 products accumulate in fp32 only.
  static constexpr bool BF16 = BF16_;
  static_assert(!BF16_ || ACC_F32_, "bf16 operands accumulate in fp32");
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
  static constexpr bool SPLIT_K = !B200_HGEMM_NO_K_DECOMP && CTA_GROUP_ * CLUSTER_M_ * CLUSTER_N_ == 1 && BN_ >= 64 && M_REP_ == 1;
  static constexpr bool STREAM_K = !B200_HGEMM_NO_K_DECOMP && CLUSTER_M_ * CLUSTER_N_ == 1 && BN_ >= 64 && M_REP_ == 1;
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

// registers -> swizzled staging buffer -> TMA store of one EPI_ROWS x EPI_N chunk of this warp
template <class Cfg, class Reg, int NR>
__device__ __forceinline__ void epilogue_store_chunk(const Reg (&d)[NR], int chunk, uint32_t epi_buf, int lane,
                                                     const CUtensorMap* tmap_c, int col0, int row0, int M, int N) {
  using namespace ptx;
  constexpr int EN = Cfg::EPI_N;
  constexpr int PER_CHUNK = EN / 4;   // packed pairs of one chunk per thread
  // the previous store from this warp's staging buffer must have finished reading it
  if (lane == 0) tma_store_wait_read<0>();
  __syncwarp();
#pragma unroll
  for (int q = 0; q < PER_CHUNK; ++q) {
    uint32_t off = uint32_t(frag_row(lane, q) * (EN * 2) + frag_col(lane, q) * 2);
    // 128-byte rows use the 128B swizzle (16-byte chunk ^= row % 8), 64-byte rows the 64B one (chunk ^= (row / 2) % 4)
    off ^= (EN == 64 ? ((off >> 7) & 7u) : ((off >> 7) & 3u)) << 4;
    st_shared_b32(epi_buf + off, acc_packed<Cfg>(d, chunk * PER_CHUNK + q));
  }
  fence_proxy_async_smem();
  __syncwarp();
  if (lane == 0) {
    if (row0 < M && col0 < N)   // rows/cols past the edge are clipped by the tensor map
      tma_store_2d(tmap_c, epi_buf, col0, row0);
    tma_store_commit();
  }
}

// Split-K epilogue (CTA_GROUP == 1, one (tile, split) unit per CTA, all units resident at once).
//   phase 1  every split writes its 128 x BN fp32 partial tile to the workspace slot (tile, split);
//   barrier  a per-tile arrival counter in global memory (release/acquire at gpu scope);
//   phase 2  split s sums a contiguous 1/splits slice of the tile's rows over ALL partials in the fixed
//            order s' = 0..splits-1 (deterministic), rounds once to fp16 and stores to C.
// The last split to finish phase 2 zeroes both counters, so the next launch on the stream starts clean.
template <class Cfg, class Reg, int NR>
__device__ __forceinline__ void splitk_epilogue(const Reg (&d)[NR], int e, int row_base, int lane, int tile, int split,
                                                int splits, int m_base, int n0, int M, int N, float* __restrict__ ws,
                                                unsigned* __restrict__ ctr, __half* __restrict__ C,
                                                uint32_t red_smem, uint32_t red_bar) {
  using namespace ptx;
  constexpr int BN = Cfg::BN;
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
                                                      uint32_t part_smem, __half* __restrict__ C) {
  using namespace ptx;
  constexpr int BN = Cfg::BN;
  constexpr int V = BN / 4;
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
// accumulator in fp32 in that fixed order; fp16 accumulators are widened, summed and rounded once. The flags are
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

template <class Cfg, int KMODE = kPlain>
__global__ void __launch_bounds__(kNumThreads, 1)
hgemm_tn_kernel(const __grid_constant__ CUtensorMap tmap_a,   // A  [M,K]  box {64, A_BOX_ROWS}
                const __grid_constant__ CUtensorMap tmap_b,   // Bt [N,K]  box {64, B_BOX_ROWS}
                const __grid_constant__ CUtensorMap tmap_c,   // C  [M,N]  box {EPI_N, EPI_ROWS}
                int M, int N, int K, int group_m,
                int splits_arg,                   // split-K factor (modes kWorkspaceSplitK / kClusterSplitK: one unit per CTA)
                int sk_tiles_arg,                 // mode kStreamK: the first sk_tiles tiles are cut along K across all workers
                float* __restrict__ splitk_ws,    // [units][128][BN] fp32 partial tiles (workspace split-K) / stream-K slots
                unsigned* __restrict__ splitk_ctr,   // [2][kMaxSplitTiles] split-K arrive / done counters, then the
                                                     // stream-K flags; all zero between launches
                __half* __restrict__ c_raw,       // C base pointer, used by the split-K reductions' direct stores
                uint64_t hint_a, uint64_t hint_b  /* L2 eviction priority of the A / B loads (ptx::kL2Evict*) */) {
  constexpr int BN = Cfg::BN;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int EM = Cfg::MCAST_M;
  constexpr int CN = Cfg::CLUSTER_N;
  constexpr int MR = Cfg::M_REP;
  constexpr bool kSplit = (KMODE == kWorkspaceSplitK || KMODE == kClusterSplitK);
  static_assert(!kSplit || Cfg::SPLIT_K, "this configuration has no split-K epilogues");
  static_assert(KMODE != kStreamK || Cfg::STREAM_K, "this configuration has no stream-K epilogues");
  static_assert(!kSplit || (kBlockM + 32) * BN * 4 <= STAGES * Cfg::STAGE_BYTES, "split-K partials must fit the pipeline smem");
  // the schedule parameters a mode does not use are constants for it
  const int splits = kSplit ? splits_arg : 1;
  const int sk_tiles = (KMODE == kStreamK) ? sk_tiles_arg : 0;
  using namespace ptx;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_a = smem_base;
  const uint32_t smem_b = smem_a + STAGES * Cfg::A_STAGE_BYTES;
  const uint32_t smem_epi = smem_b + STAGES * Cfg::B_STAGE_BYTES;
  const uint32_t smem_bar = smem_epi + Cfg::EPI_BYTES;
  const uint32_t bar_full = smem_bar;                        // [STAGES]
  const uint32_t bar_empty = bar_full + 8 * STAGES;          // [STAGES]
  const uint32_t bar_splitk = bar_empty + 8 * STAGES;        // split-K: bulk loads of the partial slices

  const int warp = __shfl_sync(0xffffffffu, int(threadIdx.x) >> 5, 0);
  const int lane = threadIdx.x & 31;
  // Position inside the cluster: rank = mi + MCAST_M * cn (a cluster split-K launch of a plain config also has
  // ranks, but does not use them here).
  const uint32_t cluster_rank = (Cfg::CLUSTER_CTAS > 1) ? cluster_ctarank() : 0u;
  const int mi = int(cluster_rank) % EM;
  const int cn = int(cluster_rank) / EM;

  // The schedule is over cluster blocks of (MCAST_M x CTA_M) x (CN x BN); a plain config has 1 x 1 blocks.
  const int num_m_blocks = (M + Cfg::CTA_M * EM - 1) / (Cfg::CTA_M * EM);
  const int num_n_blocks = (N + BN * CN - 1) / (BN * CN);
  const int num_tiles = num_m_blocks * num_n_blocks;
  const int num_k_blocks = (K + kBlockK - 1) / kBlockK;
  const int num_workers = gridDim.x / Cfg::CLUSTER_CTAS;   // clusters (or single CTAs)
  const int worker = blockIdx.x / Cfg::CLUSTER_CTAS;
  // A work unit is (tile, k-block range), see hgemm_schedule.cuh. splits == 1: whole tiles walked persistently
  // (after the worker's stream-K slice, if any). splits > 1: the host launches exactly one CTA per (tile, split)
  // unit, so the sibling splits of a tile run concurrently.

  // ------------------------------------------------------------------ one-time setup
  // A stage of CTA X is refilled only after every CTA that X's loads land in (its cluster row and column) has
  // released it: one arrive per consumer warp of each of those CTAs.
  constexpr int kReleaseTargets = EM + CN - 1;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(bar_full + 8 * s, 1);                                  // the producer's arrive.expect_tx
      mbar_init(bar_empty + 8 * s, 8 * kReleaseTargets);
    }
    mbar_init(bar_splitk, 1);
    fence_mbar_init();
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_c);
  }
  if constexpr (Cfg::CLUSTER_CTAS > 1) cluster_sync_all(); else __syncthreads();

  // Programmatic dependent launch (the host sets cudaLaunchAttributeProgrammaticStreamSerialization): this grid may have
  // been started while the previous kernel of the stream was still running, so that everything above — barrier
  // initialisation, descriptor prefetch, the set-up barrier — overlaps that kernel's tail instead of following it.
  // Nothing above touches global memory; everything below may, so every thread first waits until the prerequisite
  // grids have completed and their writes are visible (a no-op for an ordinary launch). The next kernel of the
  // stream may in turn begin ITS prologue as soon as SMs free up.
  grid_dependency_launch_dependents();
  grid_dependency_wait();

  // ------------------------------------------------------------------ roles
  if (warp < kEpiWarp0) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      // ===== TMA producer: the warp walks the schedule, one elected lane issues =====
      // multicast masks: my A slice goes to the CTAs of my cluster row (same mi), my B slice to those of my
      // cluster column (same cn)
      uint16_t mask_a = 0, mask_b = 0;
#pragma unroll
      for (int j = 0; j < CN; ++j) mask_a |= uint16_t(1u << (mi + EM * j));
#pragma unroll
      for (int i = 0; i < EM; ++i) mask_b |= uint16_t(1u << (i + EM * cn));
      const uint32_t a_slice = uint32_t(cn) * (Cfg::A_BOX_ROWS * kBlockK * 2);
      const uint32_t b_slice = uint32_t(mi) * (Cfg::B_BOX_ROWS * kBlockK * 2);
      int stage = 0; uint32_t phase = 0;
      WorkIter work(worker, num_workers, num_tiles, num_k_blocks, splits, sk_tiles);
      WorkUnit u;
      while (work.next(u)) {
        const TileCoord tc = tile_coord(u.tile, num_m_blocks, num_n_blocks, group_m);
        const int m0 = (tc.m_blk * EM + mi) * Cfg::CTA_M + cn * Cfg::A_BOX_ROWS;
        const int n0 = (tc.n_blk * CN + cn) * BN + mi * Cfg::B_BOX_ROWS;
        for (int kb = u.kb0; kb < u.kb1; ++kb) {
          mbar_wait(bar_empty + 8 * stage, phase ^ 1);
          if (elect_one()) {
            const uint32_t full = bar_full + 8 * stage;
            mbar_arrive_expect_tx(full, Cfg::STAGE_BYTES);   // the whole stage lands here, from this CTA and its peers
            const uint32_t dst_a = smem_a + stage * Cfg::A_STAGE_BYTES + a_slice;
            const uint32_t dst_b = smem_b + stage * Cfg::B_STAGE_BYTES + b_slice;
            if constexpr (CN > 1) tma_load_2d_mcast_hint(dst_a, &tmap_a, full, kb * kBlockK, m0, mask_a, hint_a);
            else tma_load_2d_hint(dst_a, &tmap_a, full, kb * kBlockK, m0, hint_a);
            if constexpr (EM > 1) tma_load_2d_mcast_hint(dst_b, &tmap_b, full, kb * kBlockK, n0, mask_b, hint_b);
            else tma_load_2d_hint(dst_b, &tmap_b, full, kb * kBlockK, n0, hint_b);
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    // every warpgroup ends inside its own branch: these warps run with the reduced register budget from here on
    __syncwarp();
    if constexpr (KMODE == kClusterSplitK) {
      cluster_sync_all();   // the consumers' two cluster barriers around the split-K reduction
      cluster_sync_all();
    } else if constexpr (Cfg::CLUSTER_CTAS > 1) {
      cluster_sync_all();   // no CTA of a cluster leaves while a peer may still multicast into it or arrive on its barriers
    }
  } else {
    setmaxnreg_inc<kConsumerRegs>();
    // ===== consumers: warpgroup wg owns rows [wg * 64 * MR, (wg + 1) * 64 * MR) of the CTA's tile =====
    using W = Wgmma<BN, Cfg::ACC_F32, Cfg::BF16>;
    using Reg = typename W::Reg;
    constexpr int NR = W::kRegs;
    const int wg = warp / 4 - 1;
    const int wq = warp % 4;                       // warp inside the warpgroup: rows [16 wq, 16 wq + 16) of a 64-row block
    const int ew = warp - kEpiWarp0;               // 0..7
    const int t = int(threadIdx.x) - 128;          // 0..255
    const uint32_t epi_buf = smem_epi + uint32_t(ew) * (Cfg::EPI_ROWS * 64 * 2);
    [[maybe_unused]] int ck_m_base = 0, ck_n0 = 0, ck_split = 0;   // cluster split-K: where this CTA's unit lives
    Reg acc[MR][NR];
#pragma unroll
    for (int r = 0; r < MR; ++r)
#pragma unroll
      for (int i = 0; i < NR; ++i) acc[r][i] = Reg(0);
    // lanes 0 .. kReleaseTargets-1 each release a stage at one CTA: first my cluster column (including myself),
    // then the rest of my cluster row
    uint32_t empty_target = bar_empty;
    if constexpr (kReleaseTargets > 1) {
      uint32_t rank = cluster_rank;
      if (lane < EM) rank = uint32_t(lane + EM * cn);
      else if (lane < kReleaseTargets) { const int j = lane - EM; rank = uint32_t(mi + EM * (j < cn ? j : j + 1)); }
      empty_target = mapa(bar_empty, rank);
    }
    auto release = [&](int s) {
      __syncwarp();
      if constexpr (kReleaseTargets > 1) {
        if (lane < kReleaseTargets) mbar_arrive_cluster(empty_target + 8 * s);
      } else {
        if (lane == 0) mbar_arrive(bar_empty + 8 * s);
      }
    };
    int stage = 0; uint32_t phase = 0;
    WorkIter work(worker, num_workers, num_tiles, num_k_blocks, splits, sk_tiles);
    WorkUnit u;
    while (work.next(u)) {
      // ---- main loop: one wgmma group per k-block, the previous one retired before its stage is released
      int prev = -1;
      for (int kb = u.kb0; kb < u.kb1; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase);
        const uint64_t da = make_smem_desc(smem_a + stage * Cfg::A_STAGE_BYTES + uint32_t(wg * MR) * (64 * kBlockK * 2));
        const uint64_t db = make_smem_desc(smem_b + stage * Cfg::B_STAGE_BYTES);
#pragma unroll
        for (int r = 0; r < MR; ++r) reg_fence(acc[r]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kWgmmaK; ++k) {
#pragma unroll
          for (int r = 0; r < MR; ++r)
            W::mma(da + uint64_t(r * ((64 * kBlockK * 2) >> 4) + 2 * k), db + uint64_t(2 * k), acc[r],
                   (kb > u.kb0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        // One group stays in flight while the next stage is awaited. The stream-K kernels carry the owner and contributor
        // epilogues as well and spill under the 168-register launch bound; a spilled accumulator of an in-flight group
        // would be read before the wgmma wrote it, so there every group is retired before anything else runs.
        if constexpr (KMODE == kStreamK) wgmma_wait<0>();
        else wgmma_wait<1>();
#pragma unroll
        for (int r = 0; r < MR; ++r) reg_fence(acc[r]);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int r = 0; r < MR; ++r) reg_fence(acc[r]);
      release(prev);

      // ---- epilogue of the unit
      const int tile = u.tile;
      const TileCoord tc = tile_coord(tile, num_m_blocks, num_n_blocks, group_m);
      const int m_cta = (tc.m_blk * EM + mi) * Cfg::CTA_M;
      const int n0 = (tc.n_blk * CN + cn) * BN;
      [[maybe_unused]] uint4* ws4 = reinterpret_cast<uint4*>(splitk_ws);
      [[maybe_unused]] unsigned* sk_flags = splitk_ctr + 2 * kMaxSplitTiles;
      if constexpr (KMODE == kStreamK) {
        const int slot = worker * Cfg::CLUSTER_CTAS + int(cluster_rank);
        if (u.kb0 > 0) {   // a later part of a tile's k-range, handed to the tile's owner
          streamk_contribute<Cfg>(acc[0], t, ew, lane, ws4, sk_flags, slot);
          continue;
        }
        if (u.kb1 < num_k_blocks) {   // the head of a tile, which owns it: add the rest of its k-range
          const int n = streamk_contributors(worker, num_workers, sk_tiles * num_k_blocks, tile, num_k_blocks);
          streamk_own<Cfg>(acc[0], t, ew, lane, ws4, sk_flags, slot + Cfg::CLUSTER_CTAS, Cfg::CLUSTER_CTAS, n);
        }
      }
      if constexpr (KMODE == kClusterSplitK) {
        // the partial tile goes where the operands were: both warpgroups must be done reading them
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
        cluster_splitk_park<Cfg>(acc[0], wg * 64 + wq * 16, lane, smem_a);
        ck_m_base = m_cta; ck_n0 = n0; ck_split = worker - tile * splits;   // the reduction runs after the cluster barrier below
      } else if constexpr (KMODE == kWorkspaceSplitK) {
        splitk_epilogue<Cfg>(acc[0], t, wg * 64 + wq * 16, lane, tile, worker - tile * splits, splits, m_cta, n0, M, N,
                             splitk_ws, splitk_ctr, c_raw, smem_a, bar_splitk);
      } else {
#pragma unroll
        for (int r = 0; r < MR; ++r) {
          const int row0 = m_cta + (wg * MR + r) * 64 + wq * 16;
#pragma unroll
          for (int j = 0; j < Cfg::EPI_CHUNKS; ++j)
            epilogue_store_chunk<Cfg>(acc[r], j, epi_buf, lane, &tmap_c, n0 + j * Cfg::EPI_N, row0, M, N);
        }
      }
    }
    // smem may be released once the bulk stores have READ it; their global writes complete with the grid
    if (lane == 0) tma_store_wait_read<0>();
    __syncwarp();
    if constexpr (KMODE == kClusterSplitK) {
      cluster_sync_all();   // every split's partial tile is parked in its CTA's shared memory
      cluster_splitk_reduce<Cfg>(t, ck_split, splits, ck_m_base, ck_n0, M, N, smem_a, c_raw);
      __syncwarp();
      cluster_sync_all();   // no CTA leaves (and frees its smem) while a peer may still be reading it
    } else if constexpr (Cfg::CLUSTER_CTAS > 1) {
      cluster_sync_all();   // no CTA of a cluster leaves while a peer may still multicast into it or arrive on its barriers
    }
  }
}

}  // namespace b200
