// Work decomposition of the persistent HGEMM kernel: which (tile, k-range) units a worker (a CTA, a CTA pair or a
// cluster) runs, and in which order. Plain C++ compiled for both sides, so that the host (launcher, tests through
// b200_hgemm_schedule_units) and the three device roles (producer, MMA issuer, epilogue) walk the very same code.
//
// Three modes:
//   data-parallel   every worker takes whole tiles worker, worker + W, ... (W workers);
//   split-K         the host launches one worker per (tile, split); the worker runs that single unit;
//   stream-K        the first `sk_tiles` tiles are cut along K into W equal slices of k-block iterations, one per
//                   worker, so a tile count that does not fill the last wave still occupies every SM; the remaining
//                   tiles are data-parallel. A slice crosses tile boundaries, so a worker runs (in this order)
//                   the tail of one tile, whole tiles, the head of another tile, then its data-parallel tiles.
//                   A unit that starts at k-block 0 OWNS its tile: it adds the partial sums of the units holding the
//                   rest of the tile's k-range (they belong to the next workers, always as their FIRST unit, so they
//                   never wait on anybody) and writes C. See streamk_* in hgemm_sm90.cuh.
#pragma once
#include <cuda_runtime.h>

namespace b200 {

struct TileCoord { int m_blk, n_blk; };

// Grouped rasterisation: walk `group_m` row-blocks down before stepping one column-block right,
// so a wave of CTAs shares a compact set of A/B panels in L2.
__host__ __device__ __forceinline__ TileCoord tile_coord(int t, int num_m_blocks, int num_n_blocks, int group_m) {
  const int tiles_per_group = group_m * num_n_blocks;
  const int group = t / tiles_per_group;
  const int first_m = group * group_m;
  const int rest = num_m_blocks - first_m;
  const int gsz = group_m < rest ? group_m : rest;
  const int in_group = t - group * tiles_per_group;
  TileCoord c;
  c.m_blk = first_m + in_group % gsz;
  c.n_blk = in_group / gsz;
  // serpentine: odd groups sweep N backwards, so the B panels touched last by one group are still in L2 for the next
  if (group & 1) c.n_blk = num_n_blocks - 1 - c.n_blk;
  return c;
}

struct WorkUnit {
  int tile;        // index into the rasterised tile order
  int kb0, kb1;    // k-blocks [kb0, kb1) of that tile
};

// Stream-K slice of worker w: k-block iterations [begin, begin + count) of the sk_tiles * nkb in the stream-K region.
__host__ __device__ __forceinline__ int streamk_slice_begin(int w, int num_workers, int sk_iters) {
  const int base = sk_iters / num_workers, rem = sk_iters - base * num_workers;
  return w * base + (w < rem ? w : rem);
}

struct WorkIter {
  int it, end;         // remaining stream-K (or split-K) slice, in k-block iterations over the whole region
  int dp_tile;         // next data-parallel tile
  int nkb, num_tiles, num_workers;

  // splits > 1: one unit per worker (num_workers == num_tiles * splits). sk_tiles > 0: stream-K over tiles [0, sk_tiles).
  __host__ __device__ WorkIter(int worker, int num_workers_, int num_tiles_, int nkb_, int splits, int sk_tiles)
      : nkb(nkb_), num_tiles(num_tiles_), num_workers(num_workers_) {
    if (splits > 1) {
      const int t = worker / splits, s = worker - t * splits;
      const int per = (nkb + splits - 1) / splits;
      const int k0 = s * per, k1 = (k0 + per < nkb) ? k0 + per : nkb;
      it = t * nkb + k0;
      end = (t < num_tiles && k0 < k1) ? t * nkb + k1 : it;
      dp_tile = num_tiles;
    } else {
      const int sk_iters = sk_tiles * nkb;
      it = streamk_slice_begin(worker, num_workers, sk_iters);
      end = streamk_slice_begin(worker + 1, num_workers, sk_iters);
      dp_tile = sk_tiles + worker;
    }
  }

  // after next(): does this worker have another unit to run?
  __host__ __device__ __forceinline__ bool has_more() const { return it < end || dp_tile < num_tiles; }

  __host__ __device__ __forceinline__ bool next(WorkUnit& u) {
    if (it < end) {
      u.tile = it / nkb;
      u.kb0 = it - u.tile * nkb;
      const int left = end - it, room = nkb - u.kb0;
      u.kb1 = u.kb0 + (left < room ? left : room);
      it += u.kb1 - u.kb0;
      return true;
    }
    if (dp_tile < num_tiles) {
      u.tile = dp_tile;
      u.kb0 = 0;
      u.kb1 = nkb;
      dp_tile += num_workers;
      return true;
    }
    return false;
  }
};

// Batched launches (C[b] = A[b] Bt[b]^T for b < num_batches, plain schedule): one flat list of tiles, batch 0's first,
// each batch's own tiles in the grouped rasterisation of tile_coord. With per-batch row counts (`counts`, the masked
// form) batch b holds only the cluster blocks that start below clamp(counts[b], 0, M), so the list holds only tiles
// with work in them and the persistent workers stay balanced. Every role builds its own cursor, sums the list
// (total()), and then locates its tiles, whose indices only increase, so the cursor only moves forward: no shared
// memory and no bound on the batch count. The host walks the same code over a host copy of the counts.
struct BatchTile {
  int batch;
  int rows;        // valid rows of the batch: stores of boxes that start at or past them are skipped
  TileCoord tc;    // cluster block inside the batch
};

struct BatchCursor {
  const int* counts;   // valid rows per batch, clamped to [0, M]; null: every batch has M
  int num_batches, M, block_rows, n_blocks, group_m;
  int batch, first, m_blocks;   // the current batch: its tiles are [first, first + m_blocks * n_blocks)

  __host__ __device__ BatchCursor(const int* counts_, int num_batches_, int M_, int block_rows_, int n_blocks_,
                                  int group_m_)
      : counts(counts_), num_batches(num_batches_), M(M_), block_rows(block_rows_), n_blocks(n_blocks_),
        group_m(group_m_), batch(0), first(0), m_blocks(blocks_of(0)) {}

  // The longest list of a launch of Cfg over num_batches matrices of M x N (host side: it bounds the workers): the
  // dense one. 64-bit for M and N up to INT_MAX; a matrix's count is capped at 2^31 first (the launch refuses more than
  // INT_MAX tiles anyway), so that the product with num_batches cannot overflow.
  template <class Cfg>
  static constexpr long long max_tiles(int num_batches, int M, int N) {
    const long long per_matrix = ((M - 1LL + Cfg::TILE_M * Cfg::CLUSTER_M) / (Cfg::TILE_M * Cfg::CLUSTER_M)) *
                                 ((N - 1LL + Cfg::BN * Cfg::CLUSTER_N) / (Cfg::BN * Cfg::CLUSTER_N));
    return num_batches * (per_matrix < 0x80000000LL ? per_matrix : 0x80000000LL);
  }

  __host__ __device__ __forceinline__ int rows_of(int b) const {
    if (!counts) return M;
    const int r = counts[b];
    return r < 0 ? 0 : r < M ? r : M;
  }
  __host__ __device__ __forceinline__ int blocks_of(int b) const {
    return b < num_batches ? (rows_of(b) + block_rows - 1) / block_rows : 0;
  }
  // the length of the list
  __host__ __device__ __forceinline__ int total() const {
    if (!counts) return num_batches * m_blocks * n_blocks;
    int blocks = 0;
    for (int b = 0; b < num_batches; ++b) blocks += blocks_of(b);
    return blocks * n_blocks;
  }
  // tile t < total() of the list; t must not be smaller than at the previous call
  __host__ __device__ __forceinline__ BatchTile locate(int t) {
    if (!counts) {   // every batch has the same tiles
      const int per = m_blocks * n_blocks;
      batch = t / per;
      first = batch * per;
    } else {
      while (t >= first + m_blocks * n_blocks) {
        first += m_blocks * n_blocks;
        m_blocks = blocks_of(++batch);
      }
    }
    BatchTile r;
    r.batch = batch;
    r.rows = rows_of(batch);
    r.tc = tile_coord(t - first, m_blocks, n_blocks, group_m);
    return r;
  }
};

// Grouped launches (the contiguous MoE layout: C[start_g : end_g] = A[start_g : end_g] Bt[g]^T for g < num_groups,
// plain schedule): group g owns rows [start_g, end_g) of A and C, with start_0 = 0, start_g = end_{g-1} and
// end_g = clamp(offs[g], start_g, T), so decreasing, negative or too-large offsets give empty or shortened groups and
// no group reaches past T. The list is BatchCursor's, over the cluster blocks of each group's own rows: group g holds
// ceil((end_g - start_g) / block_rows) * n_blocks tiles in tile_coord's rasterisation. The same constructor and
// interface, so the kernel walks either cursor with the same code; locate() returns the group as `batch` and its row
// count as `rows`, and leaves the group's first row in `start`.
struct GroupCursor {
  const int* offs;   // cumulative ends of the groups (torch._grouped_mm's offs)
  int num_groups, T, block_rows, n_blocks, group_m;
  int group, first, m_blocks, start, end;   // the current group: rows [start, end), tiles [first, first + m_blocks * n_blocks)

  __host__ __device__ GroupCursor(const int* offs_, int num_groups_, int T_, int block_rows_, int n_blocks_,
                                  int group_m_)
      : offs(offs_), num_groups(num_groups_), T(T_), block_rows(block_rows_), n_blocks(n_blocks_), group_m(group_m_),
        group(0), first(0), start(0) {
    end = end_of(0, 0);
    m_blocks = (end - start + block_rows - 1) / block_rows;
  }

  // The longest list of a launch of Cfg over T rows in num_groups groups and N columns (host side: it bounds the
  // workers; the real list is only known on the device): every group adds at most one partial cluster row block to
  // the ceil(T / block_rows) of the rows themselves.
  template <class Cfg>
  static constexpr long long max_tiles(int num_groups, int T, int N) {
    return (((long long)T + Cfg::TILE_M * Cfg::CLUSTER_M - 1) / (Cfg::TILE_M * Cfg::CLUSTER_M) + num_groups) *
           (((long long)N + Cfg::BN * Cfg::CLUSTER_N - 1) / (Cfg::BN * Cfg::CLUSTER_N));
  }

  __host__ __device__ __forceinline__ int end_of(int g, int s) const {
    if (g >= num_groups) return s;
    const int e = offs[g];
    return e < s ? s : e < T ? e : T;
  }
  // the length of the list
  __host__ __device__ __forceinline__ int total() const {
    int blocks = 0, s = 0;
    for (int g = 0; g < num_groups; ++g) {
      const int e = end_of(g, s);
      blocks += (e - s + block_rows - 1) / block_rows;
      s = e;
    }
    return blocks * n_blocks;
  }
  // tile t < total() of the list; t must not be smaller than at the previous call
  __host__ __device__ __forceinline__ BatchTile locate(int t) {
    while (t >= first + m_blocks * n_blocks) {
      first += m_blocks * n_blocks;
      start = end;
      end = end_of(++group, start);
      m_blocks = (end - start + block_rows - 1) / block_rows;
    }
    BatchTile r;
    r.batch = group;
    r.rows = end - start;
    r.tc = tile_coord(t - first, m_blocks, n_blocks, group_m);
    return r;
  }
};

// K-grouped launches (the weight gradient of the grouped product: C[g] = A[start_g : end_g]^T B[start_g : end_g] for
// g < num_groups, plain schedule): the reduction runs over the group's own rows of A [T, M] and B [T, N], with the
// groups of GroupCursor (end_g = clamp(offs[g], start_g, T)). The output is one M x N matrix per group, so the list is
// BatchCursor's dense one over num_groups matrices; what differs per tile is its k-range: ceil((end_g - start_g) / 64)
// k-blocks of 64 rows from start_g on (none for an empty group). unit() gives a work unit that k-range: the producer,
// the consumers and the host's schedule view all bound a unit through it. locate() returns the group as `batch` and M
// as `rows`, and leaves the group's rows in [start, end).
struct GroupKCursor {
  static constexpr int kRowsPerKBlock = 64;   // kBlockK of the 16-bit kernels
  const int* offs;   // cumulative ends of the groups (torch._grouped_mm's offs)
  int num_groups, M, T, block_rows, n_blocks, group_m, m_blocks;
  int group, start, end;   // the current group: rows [start, end) of A and B

  __host__ __device__ GroupKCursor(const int* offs_, int num_groups_, int M_, int T_, int block_rows_, int n_blocks_,
                                   int group_m_)
      : offs(offs_), num_groups(num_groups_), M(M_), T(T_), block_rows(block_rows_), n_blocks(n_blocks_),
        group_m(group_m_), m_blocks((M_ + block_rows_ - 1) / block_rows_), group(0), start(0) {
    end = end_of(0, 0);
  }

  // The length of the list of a launch of Cfg over num_groups matrices of M x N: BatchCursor's dense list.
  template <class Cfg>
  static constexpr long long max_tiles(int num_groups, int M, int N) {
    return BatchCursor::max_tiles<Cfg>(num_groups, M, N);
  }

  __host__ __device__ __forceinline__ int end_of(int g, int s) const {
    if (g >= num_groups) return s;
    const int e = offs[g];
    return e < s ? s : e < T ? e : T;
  }
  __host__ __device__ __forceinline__ int total() const { return num_groups * m_blocks * n_blocks; }
  // tile t < total() of the list; t must not be smaller than at the previous call
  __host__ __device__ __forceinline__ BatchTile locate(int t) {
    const int per = m_blocks * n_blocks;
    const int g = t / per;
    while (group < g) {
      start = end;
      end = end_of(++group, start);
    }
    BatchTile r;
    r.batch = g;
    r.rows = M;
    r.tc = tile_coord(t - g * per, m_blocks, n_blocks, group_m);
    return r;
  }
  // the k-blocks of the current group
  __host__ __device__ __forceinline__ int k_blocks() const { return (end - start + kRowsPerKBlock - 1) / kRowsPerKBlock; }
  // the tile of unit u (from WorkIter's plain schedule), with u's k-range set to the tile's group: [0, k_blocks())
  __host__ __device__ __forceinline__ BatchTile unit(WorkUnit& u) {
    const BatchTile r = locate(u.tile);
    u.kb0 = 0;
    u.kb1 = k_blocks();
    return r;
  }
};

// What the kernels of the other variants hold in place of a BatchCursor: nothing.
struct NoBatches {
  __host__ __device__ NoBatches(const int*, int, int, int, int, int) {}
  __host__ __device__ int total() const { return 0; }
  __host__ __device__ BatchTile locate(int) { return BatchTile{}; }
};

// Owner side of a stream-K tile: the unit (tile, 0, kb1 < nkb) of worker w is completed by the first units of
// workers w+1 .. w+n. Returns n.
__host__ __device__ __forceinline__ int streamk_contributors(int w, int num_workers, int sk_iters, int tile, int nkb) {
  const int tile_end = (tile + 1) * nkb;
  int n = 0;
  while (w + n + 1 < num_workers && streamk_slice_begin(w + n + 1, num_workers, sk_iters) < tile_end) ++n;
  return n;
}

}  // namespace b200
