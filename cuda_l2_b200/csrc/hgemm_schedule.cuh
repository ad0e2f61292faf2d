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

// Owner side of a stream-K tile: the unit (tile, 0, kb1 < nkb) of worker w is completed by the first units of
// workers w+1 .. w+n. Returns n.
__host__ __device__ __forceinline__ int streamk_contributors(int w, int num_workers, int sk_iters, int tile, int nkb) {
  const int tile_end = (tile + 1) * nkb;
  int n = 0;
  while (w + n + 1 < num_workers && streamk_slice_begin(w + n + 1, num_workers, sk_iters) < tile_end) ++n;
  return n;
}

}  // namespace b200
