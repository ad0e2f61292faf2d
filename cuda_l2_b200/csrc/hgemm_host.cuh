// Host side of the H100 HGEMM: tensor-map construction (cached), one-time kernel attribute setup,
// and the cluster launch. Shared by the C-ABI library (b200_hgemm_capi.cu) and by the per-shape
// translation units under kernels/b200_*/ that the reference-style JIT harness compiles.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <algorithm>
#include <deque>
#include <mutex>

#include "hgemm_sm90.cuh"

namespace b200 {
namespace host {

enum Status : int {
  kOk = 0,
  kBadShape = -1,        // M, N or K <= 0
  kBadAlignment = -2,    // pointers must be 16-byte aligned, K % 8 == 0 and N % 8 == 0 (TMA strides)
  kNoDriver = -3,        // cuTensorMapEncodeTiled could not be resolved
  kEncodeFailed = -4,
  kNullPointer = -5,
  kBadConfig = -6,
  kNotHopper = -7,
  kNoScratch = -8,       // internal: no split-K scratch for this (device, stream) and none can be allocated now (stream capture)
  kBadFp8K = -9,         // e4m3 operands: K % 16 == 0 (16-byte TMA strides at one byte per element)
  kBadScaleLd = -10,     // block scales: the row stride of A's scales must be >= M and a multiple of 4
  kNoNNLibrary = -11,    // row-major B: libb200_nn.so, next to libb200_hgemm.so, is missing or does not load
  kBadActivation = -12,  // bias + activation epilogue: the activation code is not one of Activation's
  kBadScaleLdB = -13,    // 1 x 128 scales of Bt (BlockScaled1D1D<>): their row stride must be >= N and a multiple of 4
  // > 0: a cudaError_t from the launch
};

inline const char* status_string(int s) {
  switch (s) {
    case kOk: return "ok";
    case kBadShape: return "M, N and K must be positive";
    case kBadAlignment: return "operands must be 16-byte aligned with K % 8 == 0 and N % 8 == 0";
    case kNoDriver: return "cuTensorMapEncodeTiled unavailable (driver too old?)";
    case kEncodeFailed: return "cuTensorMapEncodeTiled failed";
    case kNullPointer: return "null operand pointer";
    case kBadConfig: return "unknown kernel configuration id";
    case kNotHopper: return "device is not compute capability 9.0 (sm_90a build)";
    case kNoScratch: return "split-K scratch unavailable (allocate it outside stream capture with b200_hgemm_prewarm)";
    case kBadFp8K: return "e4m3 operands need K % 16 == 0 (16-byte row strides at one byte per element)";
    case kBadScaleLd: return "block scales need ld_a >= M and ld_a % 4 == 0 (16-byte aligned k-block rows of A's scales)";
    case kNoNNLibrary: return "row-major B needs libb200_nn.so next to libb200_hgemm.so (missing, or it does not load)";
    case kBadActivation: return "unknown activation code (0 none, 1 relu, 2 gelu_tanh)";
    case kBadScaleLdB: return "1 x 128 scales of Bt need ld_b >= N and ld_b % 4 == 0 (16-byte aligned k-block rows)";
    default: return s > 0 ? cudaGetErrorString(static_cast<cudaError_t>(s)) : "unknown error";
  }
}

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// Element type of a tensor map. e4m3 is encoded as UINT8: TMA only moves the bytes, wgmma interprets them.
enum class Elem : int { kF16 = 0, kBF16 = 1, kE4M3 = 2 };
constexpr int elem_bytes(Elem e) { return e == Elem::kE4M3 ? 1 : 2; }

// The data-type variants of the kernel family. Everything the host does differently per variant (which kernels it
// instantiates, the argument rules, the tuned-table entry) reads the variant's row of kGemmTypes.
enum class GemmType : int { kF16Acc32, kF16Acc16, kBF16, kE4M3F16, kE4M3BF16, kE4M3F16Block, kE4M3BF16Block,
                            kE4M3F16Block1D1D, kE4M3BF16Block1D1D };
struct GemmTypeTraits {
  Elem operand, output;
  bool acc_f32;       // fp32 accumulation (fp16 otherwise); the dispatcher reads that accumulator's tuned entry ...
  int table_k_div;    // ... at K / table_k_div: the 16-bit problem that moves as many bytes per k-block
  bool scaled;        // takes fp32 scales in device memory (per tensor or rowwise, see Scales) ...
  bool block = false; // ... or block scales (BlockScaled<> kernels, a library of their own) ...
  bool block_1d1d = false;   // ... with 1 x 128 scales on Bt too (BlockScaled1D1D<> kernels, another library)
  // the Config<> flags: BF16 names the output type, E4M3 the operand type
  constexpr bool bf16() const { return output == Elem::kBF16; }
  constexpr bool e4m3() const { return operand == Elem::kE4M3; }
};
constexpr GemmTypeTraits kGemmTypes[] = {
    {Elem::kF16, Elem::kF16, true, 1, false},      // kF16Acc32
    {Elem::kF16, Elem::kF16, false, 1, false},     // kF16Acc16
    {Elem::kBF16, Elem::kBF16, true, 1, false},    // kBF16
    {Elem::kE4M3, Elem::kF16, true, 2, true},      // kE4M3F16
    {Elem::kE4M3, Elem::kBF16, true, 2, true},     // kE4M3BF16
    {Elem::kE4M3, Elem::kF16, true, 2, true, true},    // kE4M3F16Block
    {Elem::kE4M3, Elem::kBF16, true, 2, true, true},   // kE4M3BF16Block
    {Elem::kE4M3, Elem::kF16, true, 2, true, true, true},    // kE4M3F16Block1D1D
    {Elem::kE4M3, Elem::kBF16, true, 2, true, true, true},   // kE4M3BF16Block1D1D
};
constexpr const GemmTypeTraits& traits(GemmType t) { return kGemmTypes[int(t)]; }

// The variant whose Config<> flags Cfg carries (a Config that names none does not compile: the index runs past the rows).
template <class Cfg>
constexpr GemmType gemm_type(int t = 0) {
  const GemmTypeTraits& x = kGemmTypes[t];
  return x.acc_f32 == Cfg::ACC_F32 && x.bf16() == Cfg::BF16 && x.e4m3() == Cfg::E4M3 && x.block == block_scaled<Cfg>() &&
                 x.block_1d1d == block_1d1d<Cfg>()
             ? GemmType(t) : gemm_type<Cfg>(t + 1);
}

// Row-major matrix [rows, cols] (cols contiguous) -> 2-D tiled map, box = {box_cols columns, box_rows}, swizzled over the
// box's inner extent in bytes (128 or 64). Out-of-bounds elements read as zero / are not written. batches > 0: a
// contiguous batch of such matrices [batches, rows, cols] -> 3-D map {cols, rows, batches}, box depth 1, so that the
// bounds of each matrix hold for every box (batches == 1 is still a 3-D map: the batched kernels issue 3-D copies).
inline int encode_2d(CUtensorMap* map, const void* ptr, int rows, int cols, int box_rows, int box_cols = kBlockK,
                     Elem elem = Elem::kF16, int batches = 0) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return kNoDriver;
  const cuuint32_t rank = batches > 0 ? 3 : 2;
  cuuint64_t dims[3] = {cuuint64_t(cols), cuuint64_t(rows), cuuint64_t(batches)};
  cuuint64_t strides[2] = {cuuint64_t(cols) * elem_bytes(elem), cuuint64_t(rows) * cuuint64_t(cols) * elem_bytes(elem)};
  cuuint32_t box[3] = {cuuint32_t(box_cols), cuuint32_t(box_rows), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  // the swizzle span equals the box's inner extent: 64 fp16 or 128 e4m3 = 128 B, 32 fp16 = 64 B
  const CUtensorMapSwizzle swz = box_cols * elem_bytes(elem) == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  // experiment hook: B200_HGEMM_L2_PROMOTION = 0 (none) | 1 (64 B) | 2 (128 B) | 3 (256 B, the default)
  static const CUtensorMapL2promotion promo = [] {
    const char* e = std::getenv("B200_HGEMM_L2_PROMOTION");
    const int v = (e && e[0] >= '0' && e[0] <= '3') ? e[0] - '0' : 3;
    return v == 0 ? CU_TENSOR_MAP_L2_PROMOTION_NONE : v == 1 ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B
         : v == 2 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B : CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
  }();
  const CUtensorMapDataType dt = elem == Elem::kE4M3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                               : elem == Elem::kBF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUresult r = fn(map, dt, rank, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? kOk : kEncodeFailed;
}

// Small direct-mapped cache of encoded maps: benchmark loops re-present the same few pointers
// (the caching allocator recycles them), and an encode costs about a microsecond of host time. The key carries the
// element type: an e4m3 and an fp16 map of the same pointer and dimensions differ; and the batch count (0: a 2-D map),
// so one cache serves both ranks.
struct MapKey {
  const void* ptr; int rows, cols, box_rows, box_cols; Elem elem; int batches;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && rows == o.rows && cols == o.cols && box_rows == o.box_rows && box_cols == o.box_cols &&
           elem == o.elem && batches == o.batches;
  }
};
struct MapCache {
  static constexpr int kSlots = 64;
  MapKey keys[kSlots];
  CUtensorMap maps[kSlots];
  bool valid[kSlots];
  MapCache() { std::memset(valid, 0, sizeof(valid)); }
  // Copies the map out: two operands of one call may share a slot, so a pointer into the cache would alias.
  int get(const void* ptr, int rows, int cols, int box_rows, CUtensorMap* out, int box_cols = kBlockK, Elem elem = Elem::kF16,
          int batches = 0) {
    MapKey k{ptr, rows, cols, box_rows, box_cols, elem, batches};
    uint64_t h = (reinterpret_cast<uint64_t>(ptr) >> 8) * 0x9E3779B97F4A7C15ull;
    h ^= uint64_t(uint32_t(rows)) * 0xC2B2AE3D27D4EB4Full + uint64_t(uint32_t(cols)) * 0x165667B19E3779F9ull +
         uint64_t(box_rows) * 131u + uint64_t(box_cols) + uint64_t(uint32_t(batches)) * 0x27D4EB2F165667C5ull;
    int slot = int((h >> 32) % kSlots);
    if (!(valid[slot] && keys[slot] == k)) {
      int st = encode_2d(&maps[slot], ptr, rows, cols, box_rows, box_cols, elem, batches);
      if (st != kOk) { valid[slot] = false; return st; }
      keys[slot] = k;
      valid[slot] = true;
    }
    std::memcpy(out, &maps[slot], sizeof(CUtensorMap));
    return kOk;
  }
};
inline MapCache& map_cache() {
  static thread_local MapCache c;
  return c;
}

struct DeviceInfo { int dev; int num_sms; int cc_major; };
inline const DeviceInfo& device_info() {
  // per-device, resolved once (the harness pins one device per process)
  static thread_local int cached_dev = -1;
  static thread_local DeviceInfo info{-1, 0, 0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev != cached_dev) {
    // The tensor-map encoder is a driver call and needs the device's primary context current on this thread. A thread
    // whose first CUDA work is a call of this library (an autograd worker running a backward) has none yet:
    // cudaSetDevice makes it current (CUDA 12), and is legal during a stream capture.
    cudaSetDevice(dev);
    cudaDeviceGetAttribute(&info.num_sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&info.cc_major, cudaDevAttrComputeCapabilityMajor, dev);
    info.dev = dev;
    cached_dev = dev;
  }
  return info;
}

// The operands of a launch besides A, Bt and C. Each configuration reads only those of its kind, and `{}` is a plain
// 16-bit launch. Host code only: the kernels take their own argument types (Cfg::EpiArgs), which epilogue() builds.
struct EpiOperands {
  Scales scales{nullptr, nullptr};   // scaled variants: per-tensor or rowwise scales, or block scales (device memory)
  int ld_a = 0;                      // block scales: the row stride of scales.a
  int ld_b = 0;                      // BlockScaled1D1D<>: the row stride of Bt's 1 x 128 scales (scales.b)
  const void* bias = nullptr;        // BiasAct<>: the bias (null, or N values of the output type) ...
  int act = kActNone;                // ... and the activation code
  void* y = nullptr;                 // Gated<>: y [rows, N / 2], 16-byte aligned
};

// The argument rules of a variant, checked before anything touches the device. TMA wants 16-byte row strides: A / Bt
// rows hold K operand elements (K % 8 == 0 at two bytes, K % 16 == 0 at one byte), C rows N 16-bit elements. The scales
// (`op.scales`) of a scaled variant are fp32 values in device memory: 4-byte aligned per tensor, 16-byte aligned vectors
// (M and N values) rowwise, where the split-K reductions read the column scales as float4. Block scales: `a` 16-byte
// aligned (one bulk copy per k-block) with `op.ld_a` >= M and ld_a % 4 == 0, `b` 4-byte aligned (1 x 128 scales of Bt:
// 16-byte aligned, one bulk copy per k-block too; validate_epilogue() checks their ld_b). Tile-list launches
// (launch_list): batches >= 1 matrices, a tile list of at most INT_MAX `tiles`, and its device array `list` (a batched
// launch's optional row counts) 4-byte aligned. Grouped launches (validate_grouped) pass their offsets as `list`.
inline int validate(GemmType type, const void* A, const void* Bt, const void* C, const EpiOperands& op, int M, int N,
                    int K, int batches = 1, long long tiles = 1, const int* list = nullptr) {
  const GemmTypeTraits& t = traits(type);
  const Scales& scales = op.scales;
  const int ld_a = op.ld_a;
  if (!A || !Bt || !C || (t.scaled && (!scales.a || !scales.b))) return kNullPointer;
  if (M <= 0 || N <= 0 || K <= 0 || batches < 1 || tiles > 0x7fffffffLL) return kBadShape;
  if (reinterpret_cast<uintptr_t>(list) & 3) return kBadAlignment;
  if (K % (16 / elem_bytes(t.operand))) return t.e4m3() ? kBadFp8K : kBadAlignment;
  if (N % 8) return kBadAlignment;
  if ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(Bt) | reinterpret_cast<uintptr_t>(C)) & 15)
    return kBadAlignment;
  if (t.block) {
    if ((reinterpret_cast<uintptr_t>(scales.a) & 15) || (reinterpret_cast<uintptr_t>(scales.b) & (t.block_1d1d ? 15 : 3)))
      return kBadAlignment;
    if (ld_a < M || ld_a % 4) return kBadScaleLd;
    return kOk;
  }
  if (t.scaled && ((reinterpret_cast<uintptr_t>(scales.a) | reinterpret_cast<uintptr_t>(scales.b)) & (scales.rowwise ? 15 : 3)))
    return kBadAlignment;
  return kOk;
}

// The argument rules of the bias + activation epilogue (BiasAct<>), after validate()'s: a known activation code, and a
// bias that is null or 16-byte aligned (the split-K reductions read it 8 bytes at a time, at every fourth column).
inline int validate_bias_act(const void* bias, int act) {
  if (act < 0 || act >= kNumActivations) return kBadActivation;
  if (reinterpret_cast<uintptr_t>(bias) & 15) return kBadAlignment;
  return kOk;
}

// Split-K / stream-K scratch: fp32 partial tiles + arrival counters, one per (device, stream), allocated on first use
// (or ahead of time by b200_hgemm_prewarm — required before a CUDA-graph capture, where cudaMalloc is illegal) and kept
// until b200_hgemm_release(). Process-wide and mutex-protected: any host thread that launches on a (device, stream)
// finds the same scratch, and the pool grows with the number of streams instead of silently running out. Counters are
// zero between launches (the kernel resets them), so consecutive launches on a stream need no host-side clearing.
// Launches that share a scratch must be ordered by their stream — which they are, being on the same stream.
struct SplitKScratch {
  int dev = -1; cudaStream_t stream = nullptr; float* ws = nullptr; unsigned* ctr = nullptr;
};
constexpr size_t kSplitKWsBytes = size_t(kMaxStreamKSlots) * kBlockM * 256 * sizeof(float);   // 160 units of 128x256 fp32
// split-K arrive/done counters, then one stream-K flag per (CTA slot, epilogue warp)
constexpr size_t kSplitKCtrBytes = (2 * kMaxSplitTiles + kMaxStreamKSlots * kStreamKFlagsPerSlot) * sizeof(unsigned);
struct ScratchPool {
  std::mutex mu;
  std::deque<SplitKScratch> entries;   // deque: growing never moves an entry another thread holds a pointer to
};
inline ScratchPool& scratch_pool() {
  static ScratchPool pool;
  return pool;
}
inline int splitk_scratch(int dev, cudaStream_t stream, SplitKScratch** out) {
  ScratchPool& pool = scratch_pool();
  std::lock_guard<std::mutex> lock(pool.mu);
  for (auto& e : pool.entries)
    if (e.ws && e.dev == dev && e.stream == stream) { *out = &e; return kOk; }
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(stream, &cap) != cudaSuccess) { cudaGetLastError(); return kNoScratch; }
  if (cap != cudaStreamCaptureStatusNone) return kNoScratch;   // cudaMalloc would invalidate the capture
  SplitKScratch e;
  cudaError_t err = cudaMalloc(&e.ws, kSplitKWsBytes);
  if (err != cudaSuccess) return int(err);
  err = cudaMalloc(&e.ctr, kSplitKCtrBytes);
  if (err != cudaSuccess) { cudaFree(e.ws); return int(err); }
  err = cudaMemsetAsync(e.ctr, 0, kSplitKCtrBytes, stream);
  if (err != cudaSuccess) { cudaFree(e.ws); cudaFree(e.ctr); return int(err); }
  e.dev = dev; e.stream = stream;
  SplitKScratch* slot = nullptr;
  for (auto& old : pool.entries) if (!old.ws) { slot = &old; break; }   // reuse a released entry
  if (slot) *slot = e; else { pool.entries.push_back(e); slot = &pool.entries.back(); }
  *out = slot;
  return kOk;
}
// Where a launch finds the scratch of (device, stream): this library's pool (splitk_scratch), or, for the row-major B
// kernels of libb200_nn.so, the pool of libb200_hgemm.so, handed over with each call, so that b200_hgemm_prewarm and
// b200_hgemm_release serve both libraries and a process holds one pool.
using ScratchFn = int (*)(int dev, cudaStream_t stream, SplitKScratch** out);

// Frees every scratch allocation of this process (all devices). The caller guarantees that no launch of this
// library is in flight or issued concurrently.
inline void release_scratch() {
  ScratchPool& pool = scratch_pool();
  std::lock_guard<std::mutex> lock(pool.mu);
  int cur = 0;
  cudaGetDevice(&cur);
  for (auto& e : pool.entries) {
    if (!e.ws) continue;
    cudaSetDevice(e.dev);
    cudaDeviceSynchronize();
    cudaFree(e.ws); cudaFree(e.ctr);
    e = SplitKScratch{};
  }
  cudaSetDevice(cur);
}

// `splits` codes with a special meaning (besides > 1: workspace split-K, -2/-4/-8: cluster split-K)
constexpr int kStreamKTail = 100;           // stream-K over the tiles of the partial last wave
constexpr int kStreamKTailPlusWave = 101;   // ... plus one full wave, so that every worker's slice is longer than a tile
constexpr int kMinStreamKSlice = 4;         // k-blocks; shorter slices are all pipeline fill and fix-up

// What a `splits` code asks for: a K-mode and its factor, which is the split count (workspace split-K), the cluster
// size (cluster split-K) or the code itself (stream-K: kStreamKTail or kStreamKTailPlusWave). 1, 0 and -1 ask for none.
struct KRequest { KMode mode; int factor; };
constexpr KRequest decode_splits(int splits) {
  return (splits == kStreamKTail || splits == kStreamKTailPlusWave) ? KRequest{kStreamK, splits}
         : splits > 1                                               ? KRequest{kWorkspaceSplitK, splits}
         : splits < -1                                              ? KRequest{kClusterSplitK, -splits}
                                                                    : KRequest{kPlain, 1};
}

// Does the call site have this configuration's kernel for this mode? MODES: bit mask of the K-modes it compiles. The
// K-decompositions are wired for single CTAs and CTA pairs without multicast, BN >= 64, 128 rows per CTA (split-K:
// single CTAs only); the plain schedule is always available.
template <class Cfg, unsigned MODES>
constexpr bool has_mode(KMode m) {
  return ((MODES >> m) & 1u) && (m == kPlain || (m == kStreamK ? Cfg::STREAM_K : Cfg::SPLIT_K));
}

// What a launch will run: its K-mode, how many workers (CTAs, CTA pairs or clusters), how K is divided.
struct Plan {
  KMode mode;
  int num_tiles, nkb;
  int workers;          // grid = workers * (CTAs per worker); split-K: one CTA per (tile, split)
  int splits;           // > 1: split-K, one worker per (tile, split)
  int cluster_reduce;   // != 0: the splits of a tile form a cluster of this many CTAs and reduce through DSMEM
  int sk_tiles;         // > 0: stream-K over the first sk_tiles tiles
};

// The one place that turns a `splits` request into a schedule. Pure host code: the device comes in as `max_workers`
// (SMs, or max_ctas, over the CTAs per worker) and `resident_clusters()`, the number of clusters of this configuration
// the device holds at once — an occupancy query, called only when that number bounds the workers. A request the call
// site or the configuration cannot run, or that the problem cannot use, runs plain; a factor is clamped to what fits.
template <class Cfg, unsigned MODES = 0xFu, class ResidentClusters>
Plan plan(int M, int N, int K, int splits, int max_workers, ResidentClusters&& resident_clusters) {
  KRequest req = decode_splits(splits);
  // A per-shape translation unit with a stream-K code compiles the stream-K kernel, but its launches run the plain
  // schedule: without the workspace split-K kernel, every code > 1 has always run plain there. Running stream-K in
  // those units changes their results' summation order and their timings, and is left to a change of its own.
  const bool per_shape_stream_k = req.mode == kStreamK && !((MODES >> kWorkspaceSplitK) & 1u);
  if (!has_mode<Cfg, MODES>(req.mode) || per_shape_stream_k) req = KRequest{kPlain, 1};
  Plan p{};
  const int num_m_blocks = (M + Cfg::TILE_M * Cfg::CLUSTER_M - 1) / (Cfg::TILE_M * Cfg::CLUSTER_M);
  const int num_n_blocks = (N + Cfg::BN * Cfg::CLUSTER_N - 1) / (Cfg::BN * Cfg::CLUSTER_N);
  p.num_tiles = num_m_blocks * num_n_blocks;
  p.nkb = (K + Cfg::BLOCK_K - 1) / Cfg::BLOCK_K;
  p.splits = 1;
  // Clusters must fit inside a GPC, so fewer than SMs / cluster size may be resident at once. Larger clusters are
  // always sized to what fits; CTA pairs only for stream-K, whose owners wait for contributors that must therefore be
  // running (for the plain schedule a pair that starts late is merely late).
  if (Cfg::CLUSTER_CTAS > 2 || (Cfg::CLUSTER_CTAS == 2 && req.mode == kStreamK))
    max_workers = std::min(max_workers, resident_clusters());
  p.workers = std::max(max_workers, 1);
  if (req.mode == kClusterSplitK) {
    int cs = req.factor;
    if (cs == 2 || cs == 4 || cs == 8) {
      // every CTA of the cluster must own at least one k-block: halve the cluster until no k-range is empty
      while (cs > 1 && (cs - 1) * ((p.nkb + cs - 1) / cs) >= p.nkb) cs /= 2;
      if (cs > 1) {
        p.mode = kClusterSplitK;
        p.splits = p.cluster_reduce = cs;
        p.workers = p.num_tiles * cs;   // one cluster per tile, one CTA per k-range
        return p;
      }
    }
  } else if (req.mode == kWorkspaceSplitK && p.num_tiles <= kMaxSplitTiles) {
    // units must fit the SMs (one CTA per unit), every split must own at least one k-block, and the partial tiles
    // must fit the workspace; <= 32: the slices of all partials must fit the pipeline smem
    int s = std::min(req.factor, std::min(p.workers / p.num_tiles, std::min(p.nkb, 32)));
    while (s > 1 && (s - 1) * ((p.nkb + s - 1) / s) >= p.nkb) --s;   // no empty split
    while (s > 1 && size_t(p.num_tiles) * s * kBlockM * Cfg::BN * sizeof(float) > kSplitKWsBytes) --s;
    if (s > 1) {
      p.mode = kWorkspaceSplitK;
      p.splits = s;
      p.workers = p.num_tiles * s;      // exactly one CTA per (tile, split) unit
      return p;
    }
  } else if (req.mode == kStreamK && p.num_tiles % p.workers != 0 && p.workers * Cfg::CTA_GROUP <= kMaxStreamKSlots) {
    int sk = p.num_tiles % p.workers;
    if (req.factor == kStreamKTailPlusWave && p.num_tiles > p.workers) sk += p.workers;
    if (sk * p.nkb / p.workers >= kMinStreamKSlice) {
      p.mode = kStreamK;
      p.sk_tiles = sk;
      return p;
    }
  }
  p.workers = std::min(p.workers, p.num_tiles);
  return p;
}

// The same launch on the plain schedule, when a workspace split-K or stream-K plan cannot run (no scratch, or the
// device refuses the co-resident grid). It keeps the plan's worker bound: CTA pairs planned for stream-K stay within
// the resident clusters.
inline Plan undivided(Plan p) {
  p.mode = kPlain;
  p.splits = 1;
  p.cluster_reduce = 0;
  p.sk_tiles = 0;
  p.workers = std::min(p.workers, p.num_tiles);
  return p;
}

inline bool cache_hints_enabled() {
  static const bool on = [] { const char* e = std::getenv("B200_HGEMM_NO_CACHE_HINTS"); return !(e && e[0] == '1'); }();
  return on;
}

// How many clusters of this configuration the device holds at once (asked once per device).
template <class Cfg>
int max_resident_clusters(const DeviceInfo& di) {
  static thread_local int max_clusters = 0, max_clusters_dev = -1;
  if (max_clusters_dev != di.dev) {
    cudaLaunchConfig_t probe{};
    probe.gridDim = dim3(unsigned(di.num_sms / Cfg::CLUSTER_CTAS * Cfg::CLUSTER_CTAS), 1, 1);
    probe.blockDim = dim3(Cfg::NUM_THREADS, 1, 1);
    probe.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cudaLaunchAttribute pa[1];
    pa[0].id = cudaLaunchAttributeClusterDimension;
    pa[0].val.clusterDim.x = Cfg::CLUSTER_CTAS; pa[0].val.clusterDim.y = 1; pa[0].val.clusterDim.z = 1;
    probe.attrs = pa; probe.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kernel_of<Cfg, kPlain>(), &probe) != cudaSuccess || n < 1) {
      cudaGetLastError();
      n = std::max(1, di.num_sms / Cfg::CLUSTER_CTAS * 7 / 8);
    }
    max_clusters = n; max_clusters_dev = di.dev;
  }
  return max_clusters;
}

// B200_HGEMM_NO_COOPERATIVE=1 launches the co-resident K-modes as ordinary grids (developer A/B of the launch cost).
inline bool cooperative_enabled() {
  static const bool on = [] { const char* e = std::getenv("B200_HGEMM_NO_COOPERATIVE"); return !(e && e[0] == '1'); }();
  return on;
}

// B200_HGEMM_NO_PDL=1 launches without programmatic stream serialisation (developer A/B).
inline bool pdl_enabled() {
  static const bool on = [] { const char* e = std::getenv("B200_HGEMM_NO_PDL"); return !(e && e[0] == '1'); }();
  return on;
}

// The launch of a configuration: the maps, the plan, and the kernel's arguments, its last one (Cfg::EpiArgs) built by
// epilogue().
template <class Cfg>
struct LaunchArgs {
  CUtensorMap ma, mb, mc;
  int M, N, K, group_m;
  Plan plan;
  float* ws; unsigned* ctr; __half* c;
  uint64_t hint_a, hint_b;
  int ld_a;             // block scales: the row stride of scales.a (the kernel's aux_arg)
  int batches;          // batched kernels: the batch count ...
  const int* masked_m;  // ... and the row counts per batch (null: dense); grouped kernels: G and the offsets
  cudaStream_t stream;
  typename Cfg::EpiArgs epi;
};

// The argument rules of Cfg's epilogue operands around `base(C)`, the launch's own rules (validate or validate_list), in
// this order: Gated<>'s y (non-null, then 16-byte aligned with N % 128 == 0: whole gate / up pairs), where a null h (C)
// is checked as y; the base rules; BiasAct<>'s bias and activation code (validate_bias_act); BlockScaled1D1D<>'s ld_b.
template <class Cfg, class BaseRules>
int validate_epilogue(const EpiOperands& op, const void* C, int N, BaseRules&& base) {
  if constexpr (is_gated<Cfg>()) {
    if (!op.y) return kNullPointer;
    if (!C) C = op.y;
    if ((reinterpret_cast<uintptr_t>(op.y) & 15) || N % 128) return kBadAlignment;
  }
  if (const int st = base(C)) return st;
  if constexpr (bias_act<Cfg>()) return validate_bias_act(op.bias, op.act);
  if constexpr (block_1d1d<Cfg>()) {
    if (op.ld_b < N || op.ld_b % 4) return kBadScaleLdB;
  }
  return kOk;
}

// C's map ([rows, N], `depth` matrices: 0 is a 2-D map), C itself and the kernel's last argument, after
// validate_epilogue(): the scales, BiasAct<>'s BiasActArgs, BlockScaled1D1D<>'s Block1D1DArgs, AccumF32<>'s AccumArgs
// (the wrapped kernel's argument and C, which is fp32), Gated<>'s GatedArgs (y's map, and whether h is stored: C is h,
// and when it is null y stands in for it, whose map is then never written) or Gated<Grouped<>>'s GroupedGatedArgs
// (GatedArgs and y).
template <class Cfg>
int epilogue(const EpiOperands& op, void* C, int rows, int N, int depth, MapCache& cache, LaunchArgs<Cfg>& a) {
  constexpr Elem output = traits(gemm_type<Cfg>()).output;
  if constexpr (is_gated<Cfg>()) {
    const bool store_h = C != nullptr;
    a.c = static_cast<__half*>(store_h ? C : op.y);
    // h's map (y's when h is not stored) and y's, both in 64-column store boxes
    int st = cache.get(a.c, rows, store_h ? N : N / 2, Cfg::EPI_ROWS, &a.mc, Cfg::EPI_N, output);
    if (st != kOk || (st = cache.get(op.y, rows, N / 2, Cfg::EPI_ROWS, &a.epi.y_map, Cfg::EPI_N, output)) != kOk)
      return st;
    a.epi.store_h = store_h ? 1 : 0;
    if constexpr (grouped<Cfg>()) a.epi.y = static_cast<__half*>(op.y);
    return kOk;
  } else {
    a.c = static_cast<__half*>(C);
    if constexpr (accum_f32<Cfg>() && block_1d1d<Cfg>())
      a.epi = {Block1D1DArgs{op.scales, op.ld_b}, static_cast<float*>(C)};
    else if constexpr (accum_f32<Cfg>()) a.epi = {op.scales, static_cast<float*>(C)};
    else if constexpr (bias_act<Cfg>()) a.epi = BiasActArgs{op.scales, op.bias, op.act};
    else if constexpr (block_1d1d<Cfg>()) a.epi = Block1D1DArgs{op.scales, op.ld_b};
    else a.epi = op.scales;
    return cache.get(C, rows, N, Cfg::EPI_ROWS, &a.mc, Cfg::EPI_N, output, depth);
  }
}

// One (configuration, K-mode) instance of the kernel: opt into its dynamic shared memory once, then launch.
// Function attributes are per device AND per copy of the kernel: when two shared objects instantiate this template
// (libb200_hgemm.so and a JIT-built hgemm_lib.so in one process), a function-local static may be merged across
// them (STB_GNU_UNIQUE) while each object still launches its own kernel copy. Key on both.
template <class Cfg, int KMODE>
int launch_mode(const DeviceInfo& di, const LaunchArgs<Cfg>& a) {
  static thread_local int attr_dev = -1;
  static thread_local const void* attr_fn = nullptr;
  constexpr auto kernel = kernel_of<Cfg, KMODE>();
  const void* this_fn = reinterpret_cast<const void*>(kernel);
  if (attr_dev != di.dev || attr_fn != this_fn) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return int(e);
    attr_dev = di.dev;
    attr_fn = this_fn;
  }
  constexpr bool kSplit = (KMODE == kWorkspaceSplitK || KMODE == kClusterSplitK);
  const int cluster = (KMODE == kClusterSplitK) ? a.plan.cluster_reduce : Cfg::CLUSTER_CTAS;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(unsigned(a.plan.workers * (kSplit ? 1 : Cfg::CLUSTER_CTAS)), 1, 1);   // split-K: one CTA per (tile, split)
  cfg.blockDim = dim3(Cfg::NUM_THREADS, 1, 1);
  cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
  cfg.stream = a.stream;
  cudaLaunchAttribute attr[3];
  unsigned na = 0;
  if (cluster > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = unsigned(cluster);
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  // Workspace split-K and stream-K CTAs wait for sibling CTAs of the same grid (arrival counters / flags in global
  // memory), so the whole grid must be resident at once. A cooperative launch makes that the driver's guarantee: the
  // grid starts only when all of it fits (other kernels holding SMs delay it instead of starving half of it into
  // the watchdog), and a grid that can never fit is refused with cudaErrorCooperativeLaunchTooLarge, which launch()
  // turns into the undivided schedule. (Cluster split-K needs nothing: a cluster is co-scheduled by the hardware.)
  const bool coop = (KMODE == kWorkspaceSplitK || KMODE == kStreamK) && cooperative_enabled();
  if (coop) {
    attr[na].id = cudaLaunchAttributeCooperative;
    attr[na].val.cooperative = 1;
    ++na;
  }
  // programmatic dependent launch: this kernel's prologue may overlap the tail of the stream's previous kernel; the
  // kernel itself waits (griddepcontrol.wait) before its first global-memory access. Back-to-back GEMMs lose the
  // 2-3 us of launch + set-up between them; a caller that synchronises after every call sees no difference.
  // Together with the cooperative attribute only where the driver accepts the pair (B200_HGEMM_COOP_PDL=1 to try:
  // the first refusal switches it off for the process).
  static bool coop_pdl_ok = [] { const char* e = std::getenv("B200_HGEMM_COOP_PDL"); return e && e[0] == '1'; }();
  const bool pdl = pdl_enabled() && (!coop || coop_pdl_ok);
  if (pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  const int aux = block_scaled<Cfg>() ? a.ld_a : a.plan.sk_tiles;   // the kernel's aux_arg
  // batched kernels (plain only) take the batch count as splits_arg and the row counts as splitk_ctr; grouped and
  // K-grouped kernels the group count and the offsets
  constexpr bool kTileList = batched<Cfg>() || grouped<Cfg>() || k_grouped<Cfg>();
  const int splits_arg = kTileList ? a.batches : a.plan.splits;
  unsigned* ctr = kTileList ? reinterpret_cast<unsigned*>(const_cast<int*>(a.masked_m)) : a.ctr;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, a.ma, a.mb, a.mc, a.M, a.N, a.K, a.group_m, splits_arg, aux, a.ws,
                                     ctr, a.c, a.hint_a, a.hint_b, a.epi);
  if (e != cudaSuccess && coop && pdl && e != cudaErrorCooperativeLaunchTooLarge) {
    cudaGetLastError();
    coop_pdl_ok = false;               // the pair of attributes is not accepted here: cooperative only, from now on
    cfg.numAttrs = na - 1;
    e = cudaLaunchKernelEx(&cfg, kernel, a.ma, a.mb, a.mc, a.M, a.N, a.K, a.group_m, splits_arg, aux, a.ws, ctr, a.c,
                           a.hint_a, a.hint_b, a.epi);
  }
  return e == cudaSuccess ? kOk : int(e);
}

// The rasterisation width (tile_coord's group_m) of a launch that passes group_m <= 0.
template <class Cfg>
constexpr int default_group_m() { return Cfg::CTA_GROUP == 2 ? 8 : 16; }

// group_m <= 0 selects the default rasterisation width. max_ctas <= 0 means "all SMs". `splits`: 1 none, > 1 workspace
// split-K, -2/-4/-8 cluster split-K, kStreamKTail / kStreamKTailPlusWave stream-K, as plan() grants it. MODES: bit
// mask of the K-modes this call site may need (a per-shape translation unit names its one mode and so compiles two
// kernels instead of four; the plain mode is always available as fallback). `op`: the operands the configuration's
// epilogue reads (EpiOperands; validate_epilogue gives their rules): the scales of a scaled variant, the row stride of
// block scales (`ld_a`) and of BlockScaled1D1D<>'s 1 x 128 scales of Bt (`ld_b`), BiasAct<>'s bias and activation code,
// and Gated<>'s y [M, N / 2], for which C is h [M, N] (null: not stored). RowMajorB<> configurations read `Bt` as
// B [K, N] row-major. `scratch`: where the workspace of split-K and stream-K comes from.
template <class Cfg, unsigned MODES = 0xFu>
int launch(const void* A, const void* Bt, void* C, int M, int N, int K, cudaStream_t stream, int group_m = 0,
           int max_ctas = 0, int splits = 1, const EpiOperands& op = {}, ScratchFn scratch = splitk_scratch) {
  constexpr GemmType kType = gemm_type<Cfg>();
  int st = validate_epilogue<Cfg>(op, C, N, [&](const void* c) { return validate(kType, A, Bt, c, op, M, N, K); });
  if (st != kOk) return st;
  const DeviceInfo& di = device_info();
  if (di.cc_major != 9) return kNotHopper;

  LaunchArgs<Cfg> a{};
  MapCache& cache = map_cache();
  const Elem operand = traits(kType).operand;
  if ((st = cache.get(A, M, K, Cfg::A_BOX_ROWS, &a.ma, Cfg::BLOCK_K, operand)) != kOk) return st;
  if constexpr (row_major_b<Cfg>()) {   // B [K, N]: boxes of 64 columns (one atom column) by this CTA's K slice
    if ((st = cache.get(Bt, K, N, Cfg::B_K_ROWS, &a.mb, 64, operand)) != kOk) return st;
  } else {
    if ((st = cache.get(Bt, N, K, Cfg::B_BOX_ROWS, &a.mb, Cfg::BLOCK_K, operand)) != kOk) return st;
  }
  if ((st = epilogue<Cfg>(op, C, M, N, 0, cache, a)) != kOk) return st;

  const int max_workers = (max_ctas > 0 ? max_ctas : di.num_sms) / Cfg::CLUSTER_CTAS;
  a.plan = plan<Cfg, MODES>(M, N, K, splits, max_workers, [&] { return max_resident_clusters<Cfg>(di); });
  if (a.plan.mode == kWorkspaceSplitK || a.plan.mode == kStreamK) {
    SplitKScratch* sk = nullptr;
    if (scratch(di.dev, stream, &sk) == kOk) {
      a.ws = sk->ws; a.ctr = sk->ctr;
    } else {
      cudaGetLastError();   // no scratch (allocation failed, or first use inside a stream capture): run undivided
      a.plan = undivided(a.plan);
    }
  }
  a.M = M; a.N = N; a.K = K;
  a.group_m = group_m > 0 ? group_m : default_group_m<Cfg>();
  a.ld_a = op.ld_a;
  a.stream = stream;
  // L2 eviction priorities: when one operand is streamed (about) once while the other is re-read by every tile row
  // or column and is small enough to live in L2, keep the small one and let the streamed one go first.
  a.hint_a = ptx::kL2EvictNormal; a.hint_b = ptx::kL2EvictNormal;
  if (cache_hints_enabled()) {
    const size_t a_bytes = size_t(M) * K * Cfg::OP_BYTES, b_bytes = size_t(N) * K * Cfg::OP_BYTES;
    const int n_tiles = (N + Cfg::BN - 1) / Cfg::BN, m_tiles = (M + Cfg::TILE_M - 1) / Cfg::TILE_M;
    constexpr size_t kL2Keep = size_t(20) << 20, kStream = size_t(40) << 20;   // against the 50 MB L2
    if (a_bytes >= kStream && b_bytes <= kL2Keep && n_tiles <= 4) { a.hint_a = ptx::kL2EvictFirst; a.hint_b = ptx::kL2EvictLast; }
    else if (b_bytes >= kStream && a_bytes <= kL2Keep && m_tiles <= 4) { a.hint_b = ptx::kL2EvictFirst; a.hint_a = ptx::kL2EvictLast; }
  }
  // a co-resident mode the device cannot hold (refused before anything ran) falls back to the undivided schedule
  auto or_undivided = [&](int err) {
    if (err != int(cudaErrorCooperativeLaunchTooLarge) && err != int(cudaErrorLaunchOutOfResources)) return err;
    cudaGetLastError();
    a.plan = undivided(a.plan);
    return launch_mode<Cfg, kPlain>(di, a);
  };
  // plan() only picks a mode for which has_mode holds; the `if constexpr` keeps the others from being instantiated
  switch (a.plan.mode) {
    case kStreamK:
      if constexpr (has_mode<Cfg, MODES>(kStreamK)) return or_undivided(launch_mode<Cfg, kStreamK>(di, a));
      break;
    case kClusterSplitK:
      if constexpr (has_mode<Cfg, MODES>(kClusterSplitK)) return launch_mode<Cfg, kClusterSplitK>(di, a);
      break;
    case kWorkspaceSplitK:
      if constexpr (has_mode<Cfg, MODES>(kWorkspaceSplitK)) return or_undivided(launch_mode<Cfg, kWorkspaceSplitK>(di, a));
      break;
    case kPlain:
      break;
  }
  return launch_mode<Cfg, kPlain>(di, a);
}

// The schedule of a tile-list launch: plain (there is no other for these kernels, so a launch needs no scratch and is
// always safe to capture in a graph), workers bounded by the cursor's longest list, `max_tiles`. The kernel's list may
// be shorter (row counts, group offsets), and the workers without a tile leave at once.
template <class Cfg, class ResidentClusters>
Plan list_plan(long long max_tiles, int K, int max_workers, ResidentClusters&& resident_clusters) {
  Plan p{};
  p.mode = kPlain;
  p.splits = 1;
  p.num_tiles = int(max_tiles);   // validate() bounds it
  p.nkb = (K + Cfg::BLOCK_K - 1) / Cfg::BLOCK_K;
  if (Cfg::CLUSTER_CTAS > 2) max_workers = std::min(max_workers, resident_clusters());
  p.workers = std::min(std::max(max_workers, 1), p.num_tiles);
  return p;
}

// The argument rules of a grouped launch: those of a 2-D [T, K] x [N, K] call (T == 0 is an empty problem and valid),
// G >= 1 groups whose offsets (G int32 values, device memory) are non-null and 4-byte aligned, and a worst-case tile
// list (`worst_tiles`, GroupCursor::max_tiles) of at most INT_MAX tiles. Block-scaled e4m3: the block-scale rules with
// M = T (at least one row: ld_a >= max(T, 1)).
inline int validate_grouped(GemmType type, const void* A, const void* Bt, const void* C, const int* offs, int groups,
                            int T, int N, int K, long long worst_tiles, const EpiOperands& op = {}) {
  if (!A || !Bt || !C || !offs) return kNullPointer;
  if (T < 0 || groups < 1) return kBadShape;
  return validate(type, A, Bt, C, op, T > 0 ? T : 1, N, K, 1, worst_tiles, offs);
}

// The argument rules of a K-grouped launch (GroupedK<>): A [T, M], B [T, N] and C [G, M, N] with 16-byte rows (M % 8 and
// N % 8: validate's rule for K and N, with M in K's place), G >= 1 groups whose offsets are non-null and 4-byte aligned,
// T >= 0 (an empty reduction), and a tile list (`tiles`, the dense G x M x N one) of at most INT_MAX tiles. With T == 0
// neither operand is read, and A and B may be null (torch's pointer for a tensor without elements).
inline int validate_k_grouped(GemmType type, const void* A, const void* B, const void* C, const int* offs, int groups,
                              int T, int M, int N, long long tiles) {
  if (!C || !offs || (T != 0 && (!A || !B))) return kNullPointer;
  if (T < 0 || groups < 1) return kBadShape;
  if (T == 0) A = B = C;   // not read
  return validate(type, A, B, C, {}, M, N, M, 1, tiles, offs);
}

// The argument rules of a tile-list launch of Cfg's kind, with launch_list's arguments.
template <class Cfg>
int validate_list(GemmType type, const void* A, const void* Bt, const void* C, const int* list, int count, int rows,
                  int N, int K, long long tiles, const EpiOperands& op) {
  return k_grouped<Cfg>() ? validate_k_grouped(type, A, Bt, C, list, count, K, rows, N, tiles)
         : grouped<Cfg>() ? validate_grouped(type, A, Bt, C, list, count, rows, N, K, tiles, op)
                          : validate(type, A, Bt, C, op, rows, N, K, count, tiles, list);
}

// One launch of a Batched<>, Grouped<> or GroupedK<> configuration, which walks the flat tile list of its Cfg::Cursor over
// `count` matrices or groups. No L2 eviction hints: which operand is re-read depends on the batch or group as much as
// on the shapes. rows == 0 launches nothing.
//   Batched<>: C[b] = A[b] Bt[b]^T for b < count, A [count, rows, K], Bt [count, N, K], C [count, rows, N], all
//   contiguous; `list` (device memory, optional): only rows [0, clamp(list[b], 0, rows)) of C[b] are computed, and no
//   16-row store box starting at or past that count is written.
//   Grouped<>: C[start_g : end_g] = A[start_g : end_g] Bt[g]^T for g < count, A [rows, K], Bt [count, N, K],
//   C [rows, N], contiguous; `list` (device memory, read by the kernel only): the cumulative group ends,
//   end_g = clamp(list[g], start_g, rows) with start_0 = 0 and start_g = end_{g-1}. Every row of C below
//   end_{count-1} is written once, by its own group; no other is written.
//   Grouped<BlockScaled<>> (e4m3 operands): the same, with the block scales of the 2-D call over M = rows
//   (`op.scales.a`, `op.ld_a`) and one [ceil(N/128), ceil(K/128)] matrix of Bt's scales per group (`op.scales.b`).
//   Batched<BlockScaled<>> (e4m3 operands): the batched product, with one [ceil(K/128), ld_a] block of A's scales per
//   matrix, stacked (value (b, m, kb) at scales.a[(b * ceil(K/128) + kb) * ld_a + m]), and one [ceil(N/128),
//   ceil(K/128)] matrix of Bt's scales per batch (`op.scales.b`).
//   Grouped<RowMajorB<>>: Grouped<>'s product with `Bt` read as B [count, K, N] row-major: C[start_g : end_g] =
//   A[start_g : end_g] B[g].
//   GroupedK<> (`rows` is M, `K` is T): C[g] = A[start_g : end_g]^T B[start_g : end_g] for g < count, A [T, M] and
//   `Bt` as B [T, N] row-major, C [count, M, N], the groups as for Grouped<>. Every matrix of C is written, an empty
//   group's with +0.0; T == 0 zero-fills C on the stream and launches nothing (a map needs at least one row).
//   Gated<Grouped<>>: Grouped<>'s product h = C [rows, N] (null: not stored) with the SwiGLU epilogue, y [rows, N / 2]
//   (`op.y`, 16-byte aligned, N % 128 == 0): the rows of y below the last group's end are written, each by its own
//   group.
template <class Cfg>
int launch_list(const void* A, const void* Bt, void* C, const int* list, int count, int rows, int N, int K,
                cudaStream_t stream, int group_m = 0, int max_ctas = 0, const EpiOperands& op = {}) {
  static_assert(batched<Cfg>() || grouped<Cfg>() || k_grouped<Cfg>(), "a Batched<>, Grouped<> or GroupedK<> configuration");
  constexpr GemmType kType = gemm_type<Cfg>();
  const long long tiles = Cfg::Cursor::template max_tiles<Cfg>(count, rows, N);
  int st = validate_epilogue<Cfg>(
      op, C, N, [&](const void* c) { return validate_list<Cfg>(kType, A, Bt, c, list, count, rows, N, K, tiles, op); });
  if (st != kOk || rows == 0) return st;
  const Elem elem = traits(kType).operand, output = traits(kType).output;
  if constexpr (k_grouped<Cfg>()) {
    if (K == 0) {   // no row to reduce over: every matrix of C is zero (AccumF32<>: C stays as it is)
      if constexpr (accum_f32<Cfg>()) return kOk;
      const cudaError_t e = cudaMemsetAsync(C, 0, size_t(count) * size_t(rows) * size_t(N) * elem_bytes(output),
                                            stream);
      return e == cudaSuccess ? kOk : int(e);
    }
  }
  const DeviceInfo& di = device_info();
  if (di.cc_major != 9) return kNotHopper;

  LaunchArgs<Cfg> a{};
  MapCache& cache = map_cache();
  if constexpr (k_grouped<Cfg>()) {
    // A [T, M] and B [T, N] in boxes of 64 columns (one atom column) by this CTA's K slice
    if ((st = cache.get(A, K, rows, Cfg::A_K_ROWS, &a.ma, 64, elem)) != kOk) return st;
    if ((st = cache.get(Bt, K, N, Cfg::B_K_ROWS, &a.mb, 64, elem)) != kOk) return st;
  } else {
    // Bt is one N x K matrix per batch or group (row-major B: one K x N matrix per group, in atom-column boxes); A is
    // one matrix per batch (a 3-D map, so that TMA clips each box at its own matrix's edge), or the rows of all groups
    if ((st = cache.get(A, rows, K, Cfg::A_BOX_ROWS, &a.ma, Cfg::BLOCK_K, elem, batched<Cfg>() ? count : 0)) != kOk)
      return st;
    if constexpr (row_major_b<Cfg>()) {
      if ((st = cache.get(Bt, K, N, Cfg::B_K_ROWS, &a.mb, 64, elem, count)) != kOk) return st;
    } else {
      if ((st = cache.get(Bt, N, K, Cfg::B_BOX_ROWS, &a.mb, Cfg::BLOCK_K, elem, count)) != kOk) return st;
    }
  }
  // C: one M x N matrix per group (K-grouped) or per batch, as A, or the rows of all groups
  if ((st = epilogue<Cfg>(op, C, rows, N, k_grouped<Cfg>() || batched<Cfg>() ? count : 0, cache, a)) != kOk) return st;
  const int max_workers = (max_ctas > 0 ? max_ctas : di.num_sms) / Cfg::CLUSTER_CTAS;
  a.plan = list_plan<Cfg>(tiles, K, max_workers, [&] { return max_resident_clusters<Cfg>(di); });
  a.M = rows; a.N = N; a.K = K;
  a.group_m = group_m > 0 ? group_m : default_group_m<Cfg>();
  a.hint_a = ptx::kL2EvictNormal; a.hint_b = ptx::kL2EvictNormal;
  a.ld_a = op.ld_a;
  a.batches = count;
  a.masked_m = list;
  a.stream = stream;
  return launch_mode<Cfg, kPlain>(di, a);
}

}  // namespace host
}  // namespace b200
