/* hgemm_oracle.c — CPU restatement of the HGEMM hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Nothing under cuda_l2_b200/, kernels/, pybind/ or the harness scripts may call into this file;
 * it exists so that tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg have an
 * independent statement of what the GPU path must produce.
 *
 * What it restates (paths relative to the CUDA-L2 reference checkout):
 *   - the GEMM contract of every cuda_l2_<dev>_<acc> kernel: fp16 x fp16 products, fp32 accumulation,
 *     ONE round-to-nearest-even conversion to fp16 at the end
 *       kernels/a100_F32F16F16F32/4096_4096_4096.cu:139-144 (cute::gemm into float acc, then convert)
 *       cublas/fp32/hgemm_cublas.cu:43-52 (alpha = 1, beta = 0, CUBLAS_COMPUTE_32F)
 *   - the fp16-accumulate variant
 *       kernels/a100_F16F16F16F16/8192_8192_8192.cu:185 (SM80_16x8x16_F16F16F16F16_TN atom),
 *       cublas/fp16/hgemm_cublas.cu:43-52 (CUBLAS_COMPUTE_16F)
 *   - the operand layout: B is consumed K-major ("b_col_major"), tools/utils.py:110-115
 *   - the ground truth and pass rule of the reference's only correctness test
 *       zero_one_correctness_check.py:87-92 (fp32 matmul on the CPU, .half(), mask |truth| > 2047)
 *       zero_one_correctness_check.py:169-172, 263-268 (max |out - truth| over unmasked == 0)
 *
 * Pinning: the reference stores no golden vectors; its contract is procedural (0/1 inputs, exact
 * match on integers < 2048). On that domain every summation order gives the same bits, so this
 * restatement is pinned by tests/golden/ (vectors generated with the reference's own truth
 * expression, torch.matmul in fp32 on the CPU — see tests/golden/make_golden.py). Outside that domain
 * (non-integer inputs, fp16 accumulation order inside the tensor core) parity is UNPINNED: the
 * reference does not define it, and tests use a stated tolerance there.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ---- IEEE binary16 <-> binary32, bit-exact, no ISA extensions required ---------------------- */
static inline float h2f(uint16_t h) {
  const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1fu;
  uint32_t man = h & 0x3ffu;
  uint32_t bits;
  if (exp == 0) {
    if (man == 0) {
      bits = sign;
    } else { /* subnormal: normalise */
      int e = -1;
      do { man <<= 1; ++e; } while (!(man & 0x400u));
      man &= 0x3ffu;
      bits = sign | ((uint32_t)(127 - 15 - e) << 23) | (man << 13);
    }
  } else if (exp == 31) {
    bits = sign | 0x7f800000u | (man << 13);
  } else {
    bits = sign | ((exp + 127 - 15) << 23) | (man << 13);
  }
  float f;
  memcpy(&f, &bits, 4);
  return f;
}

/* round-to-nearest-even, overflow to inf, NaN preserved (quiet) — what cvt.rn.f16.f32 does */
static inline uint16_t f2h(float f) {
  uint32_t x;
  memcpy(&x, &f, 4);
  const uint16_t sign = (uint16_t)((x >> 16) & 0x8000u);
  x &= 0x7fffffffu;
  if (x >= 0x7f800000u) return (uint16_t)(sign | (x > 0x7f800000u ? 0x7e00u : 0x7c00u));
  if (x >= 0x477ff000u) return (uint16_t)(sign | 0x7c00u);         /* >= 65520 rounds to inf */
  if (x < 0x33000001u) return sign;                                 /* <= 2^-25 rounds to zero */
  int32_t exp = (int32_t)(x >> 23) - 127;
  uint32_t man = (x & 0x7fffffu) | 0x800000u;
  uint32_t shift, half_bits;
  if (exp < -14) { /* subnormal result */
    shift = (uint32_t)(13 + (-14 - exp));
    half_bits = 0;
  } else {
    shift = 13;
    half_bits = (uint32_t)(exp + 15) << 10;
    man &= 0x7fffffu;
  }
  uint32_t q = man >> shift;
  const uint32_t rem = man & ((1u << shift) - 1u);
  const uint32_t halfway = 1u << (shift - 1);
  if (rem > halfway || (rem == halfway && (q & 1u))) ++q;           /* may carry into the exponent */
  return (uint16_t)(sign | (half_bits + q));
}

uint16_t oracle_f32_to_f16(float f) { return f2h(f); }
float oracle_f16_to_f32(uint16_t h) { return h2f(h); }

/* ---- layout helper: tools/utils.py:110-115 as_col_major — B[K,N] row-major -> Bt[N,K] -------- */
void oracle_as_col_major(const uint16_t* B, uint16_t* Bt, int K, int N) {
  for (int k = 0; k < K; ++k)
    for (int n = 0; n < N; ++n) Bt[(size_t)n * K + k] = B[(size_t)k * N + n];
}

/* ---- F32F16F16F32: canonical statement — one fp32 accumulator, k ascending, one RN at the end - */
void oracle_hgemm_f32acc(const uint16_t* A, const uint16_t* Bt, uint16_t* C, int M, int N, int K) {
  float* a = (float*)malloc((size_t)K * sizeof(float));
  float* b = (float*)malloc((size_t)N * K * sizeof(float));
  for (size_t i = 0; i < (size_t)N * K; ++i) b[i] = h2f(Bt[i]);
  for (int m = 0; m < M; ++m) {
    for (int k = 0; k < K; ++k) a[k] = h2f(A[(size_t)m * K + k]);
    for (int n = 0; n < N; ++n) {
      const float* bn = b + (size_t)n * K;
      float acc = 0.0f;
      for (int k = 0; k < K; ++k) acc += a[k] * bn[k];  /* fp16*fp16 is exact in fp32; the add rounds */
      C[(size_t)m * N + n] = f2h(acc);
    }
  }
  free(a);
  free(b);
}

/* Same contract, throughput-oriented (8 interleaved partial sums, OpenMP over rows). Identical bits
 * to the canonical form whenever all partial sums are exactly representable (the 0/1 domain);
 * otherwise it is another legal fp32 summation order. Used for larger cases and CPU timing. */
void oracle_hgemm_f32acc_fast(const uint16_t* A, const uint16_t* Bt, uint16_t* C, int M, int N, int K) {
  float* a = (float*)malloc((size_t)M * K * sizeof(float));
  float* b = (float*)malloc((size_t)N * K * sizeof(float));
  for (size_t i = 0; i < (size_t)M * K; ++i) a[i] = h2f(A[i]);
  for (size_t i = 0; i < (size_t)N * K; ++i) b[i] = h2f(Bt[i]);
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m) {
    const float* am = a + (size_t)m * K;
    for (int n = 0; n < N; ++n) {
      const float* bn = b + (size_t)n * K;
      float p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      int k = 0;
      for (; k + 8 <= K; k += 8)
        for (int u = 0; u < 8; ++u) p[u] += am[k + u] * bn[k + u];
      float acc = ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
      for (; k < K; ++k) acc += am[k] * bn[k];
      C[(size_t)m * N + n] = f2h(acc);
    }
  }
  free(a);
  free(b);
}

/* ---- F16F16F16F16: the accumulator is re-rounded to fp16 after every `chunk` products ----------
 * (chunk = 16 models one m16n8k16 / wgmma K=16 step: products summed wide, accumulator stored in
 * fp16). The hardware's exact internal order is not specified by the reference or by NVIDIA; on
 * the 0/1 domain with |sum| < 2048 every order is exact. */
void oracle_hgemm_f16acc(const uint16_t* A, const uint16_t* Bt, uint16_t* C, int M, int N, int K, int chunk) {
  if (chunk <= 0) chunk = 16;
  float* a = (float*)malloc((size_t)K * sizeof(float));
  float* b = (float*)malloc((size_t)N * K * sizeof(float));
  for (size_t i = 0; i < (size_t)N * K; ++i) b[i] = h2f(Bt[i]);
  for (int m = 0; m < M; ++m) {
    for (int k = 0; k < K; ++k) a[k] = h2f(A[(size_t)m * K + k]);
    for (int n = 0; n < N; ++n) {
      const float* bn = b + (size_t)n * K;
      uint16_t acc = 0;
      for (int k0 = 0; k0 < K; k0 += chunk) {
        const int k1 = k0 + chunk < K ? k0 + chunk : K;
        float s = 0.0f;
        for (int k = k0; k < k1; ++k) s += a[k] * bn[k];
        acc = f2h(h2f(acc) + s);
      }
      C[(size_t)m * N + n] = acc;
    }
  }
  free(a);
  free(b);
}

/* ---- bf16 variant (an extension of this repository: the reference ships no bf16 kernel, README.md:73 lists
 * further data types as future work). Same contract as F32F16F16F32 with bfloat16 operands and output:
 * exact bf16 x bf16 products (8 x 8 significant bits), fp32 accumulation, ONE round-to-nearest-even
 * conversion to bf16 — what torch.matmul(a.float(), b.float()).bfloat16() computes, which is the expression
 * tests/golden/make_golden.py uses to pin it (0/1 operands, K <= 256 so that every sum is a bf16 integer).
 * PARITY UNPINNED by the reference (it defines no bf16 result); pinned against that torch expression. */
static inline float bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
/* round-to-nearest-even on the upper 16 bits, NaN kept quiet — cvt.rn.bf16.f32 */
static inline uint16_t f2bf(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x0040u);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
uint16_t oracle_f32_to_bf16(float f) { return f2bf(f); }
float oracle_bf16_to_f32(uint16_t h) { return bf2f(h); }

void oracle_bgemm_f32acc(const uint16_t* A, const uint16_t* Bt, uint16_t* C, int M, int N, int K) {
  float* a = (float*)malloc((size_t)M * K * sizeof(float));
  float* b = (float*)malloc((size_t)N * K * sizeof(float));
  for (size_t i = 0; i < (size_t)M * K; ++i) a[i] = bf2f(A[i]);
  for (size_t i = 0; i < (size_t)N * K; ++i) b[i] = bf2f(Bt[i]);
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m) {
    const float* am = a + (size_t)m * K;
    for (int n = 0; n < N; ++n) {
      const float* bn = b + (size_t)n * K;
      float acc = 0.0f;
      for (int k = 0; k < K; ++k) acc += am[k] * bn[k];   /* one fp32 accumulator, k ascending */
      C[(size_t)m * N + n] = f2bf(acc);
    }
  }
  free(a);
  free(b);
}

/* ---- the reference's pass rule (zero_one_correctness_check.py:92,169-172): ---------------------
 * diff = |out - truth| in fp16 arithmetic (torch subtracts the two half tensors), entries with
 * |truth| > 2047 are ignored, result = max diff. Returns that max as float; *n_masked and *n_nonfinite
 * report how many entries were masked / were NaN or Inf in `out`. */
float oracle_zero_one_max_diff(const uint16_t* out, const uint16_t* truth, size_t n, size_t* n_masked,
                               size_t* n_nonfinite) {
  float worst = 0.0f;
  size_t masked = 0, bad = 0;
  for (size_t i = 0; i < n; ++i) {
    const float t = h2f(truth[i]);
    const float o = h2f(out[i]);
    if (!isfinite(o)) ++bad;
    if (fabsf(t) > 2047.0f) { ++masked; continue; }
    float d = h2f(f2h(o - t));   /* half - half, rounded to half like torch.abs(out - truth) */
    d = fabsf(d);
    if (d > worst || d != d) worst = d;
  }
  if (n_masked) *n_masked = masked;
  if (n_nonfinite) *n_nonfinite = bad;
  return worst;
}

/* ---- deterministic 0/1 operand generator (splitmix64), mirrors the reference's choice of density:
 * zero_one_correctness_check.py:65-73 — uniform over {0,1} when max(m,n,k) <= 8192, else over {0,0,1}. */
static inline uint64_t splitmix64(uint64_t* s) {
  uint64_t z = (*s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
void oracle_fill_zero_one(uint16_t* dst, size_t n, int levels /* 2 or 3 */, uint64_t seed) {
  uint64_t s = seed;
  for (size_t i = 0; i < n; ++i) {
    const uint64_t r = splitmix64(&s) % (uint64_t)levels;
    dst[i] = (r == (uint64_t)(levels - 1)) ? 0x3c00u : 0u;   /* 1.0h or 0.0h */
  }
}
