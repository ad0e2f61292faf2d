// The family of kernel configurations compiled into libb200_hgemm.so and referenced by the
// generated per-shape translation units (kernels/b200_*/<M>_<N>_<K>.cu).
//   X(id, BN, STAGES, CTA_GROUP, CLUSTER_M, CLUSTER_N, M_REP)
// STAGES is the requested ring depth; Config caps it at what fits the 227 KB of shared memory next to the 16 KB
// epilogue staging area (every CTA of a pair holds the whole B tile, so pairs with BN >= 128 run shallower rings).
// CTA_GROUP = 2: two CTAs of a cluster on adjacent 128-row tiles that multicast their shared B tile.
// M_REP = 2: 256 rows per CTA (two wgmmas per k-step sharing the B tile): config 26 is a 512 x 128 tile per CTA pair,
// 27 / 28 two such pairs sharing B / A by multicast. Register accumulators limit these to BN = 128.
// 29 / 30: four CTA pairs in a 2 x 2 multicast cluster (8 CTAs: both operands fetched from L2 once per two pairs).
// CLUSTER_M x CLUSTER_N > 1: TMA-multicast clusters of groups (single CTAs or CTA pairs): A shared along N, B along M.
#pragma once
#include "hgemm_host.cuh"

#define B200_HGEMM_CONFIGS(X) \
  X(0, 256, 4, 1, 1, 1, 1)       \
  X(1, 128, 6, 1, 1, 1, 1)       \
  X(2, 64, 8, 1, 1, 1, 1)        \
  X(3, 256, 6, 2, 1, 1, 1)       \
  X(4, 128, 8, 2, 1, 1, 1)       \
  X(5, 192, 4, 1, 1, 1, 1)       \
  X(6, 192, 6, 2, 1, 1, 1)       \
  X(7, 64, 8, 1, 1, 2, 1)        \
  X(8, 64, 8, 1, 1, 4, 1)        \
  X(9, 64, 8, 1, 2, 2, 1)        \
  X(10, 128, 6, 1, 1, 2, 1)      \
  X(11, 128, 6, 1, 2, 2, 1)      \
  X(12, 32, 9, 1, 1, 1, 1)       \
  X(13, 32, 9, 1, 1, 4, 1)       \
  X(14, 32, 9, 1, 1, 8, 1)       \
  X(15, 64, 8, 1, 2, 1, 1)       \
  X(16, 64, 8, 1, 4, 1, 1)       \
  X(17, 128, 6, 1, 2, 1, 1)      \
  X(18, 256, 4, 1, 1, 2, 1)      \
  X(19, 256, 4, 1, 2, 1, 1)      \
  X(20, 256, 6, 2, 1, 2, 1)      \
  X(21, 256, 6, 2, 2, 1, 1)      \
  X(22, 128, 8, 2, 1, 2, 1)      \
  X(23, 128, 8, 2, 2, 1, 1)      \
  X(24, 192, 6, 2, 1, 2, 1)      \
  X(25, 192, 6, 2, 2, 1, 1)     \
  X(26, 128, 4, 2, 1, 1, 2)      \
  X(27, 128, 4, 2, 2, 1, 2)      \
  X(28, 128, 4, 2, 1, 2, 2)      \
  X(29, 256, 6, 2, 2, 2, 1)      \
  X(30, 128, 8, 2, 2, 2, 1)

namespace b200 {
constexpr int kNumConfigs = 31;
}
