/* fp8_oracle.c — CPU restatement of the FP8 (e4m3) GEMM.  TEST INFRASTRUCTURE ONLY.
 *
 * An extension of this repository (the reference has no fp8 path). It includes hgemm_oracle.c so that the output
 * roundings are the same bit-exact binary16 / bfloat16 conversions the 16-bit oracle uses; it is compiled into its own
 * library (oracle/fp8.py), and hgemm_oracle.c is not changed by it.
 *
 * float8_e4m3fn operands (OCP FP8 E4M3: 1 sign, 4 exponent bits with bias 7, 3 mantissa bits, no infinities, 0x7F /
 * 0xFF are NaN, largest finite value 448), per-tensor fp32 scales, fp16 or bf16 output:
 *     C = RN_out( fp32( sum_k a*b ) * fp32(sa * sb) )
 * Every e4m3 x e4m3 product is exact in fp32 (4 x 4 significant bits); the sum is the canonical one fp32 accumulator,
 * k ascending; the scale product is rounded to fp32 once, multiplies the finished sum once (rounded to fp32), and one
 * RN-even conversion to the output type follows. Pinned against torch's expression
 * ((a.float() @ bt.float().t()) * (sa * sb)).to(out_dtype) by tests/golden/fp8_cases.npz. */
#include "hgemm_oracle.c"

static inline float e4m3_to_f32(uint8_t v) {
  const uint32_t exp = (v >> 3) & 0xfu, man = v & 0x7u;
  float f;
  if ((v & 0x7fu) == 0x7fu) return NAN;
  if (exp == 0) f = ldexpf((float)man, -9);                 /* subnormal: man * 2^(1 - 7 - 3) */
  else f = ldexpf((float)(8u + man), (int)exp - 10);        /* (1 + man / 8) * 2^(exp - 7) */
  return (v & 0x80u) ? -f : f;
}

/* round-to-nearest-even for |f| <= 448 (and up to the rounding boundary 464, which rounds to 448); larger magnitudes
 * and NaN give NaN, as torch's float8_e4m3fn cast does. */
static inline uint8_t f32_to_e4m3(float f) {
  const uint8_t sign = signbit(f) ? 0x80u : 0u;
  const float x = fabsf(f);
  if (!(x < 464.0f)) return (uint8_t)(sign | 0x7fu);
  if (x >= 448.0f) return (uint8_t)(sign | 0x7eu);
  /* the finite codes 0x00..0x7E decode to increasing values: find lo with e4m3(lo) <= x < e4m3(lo + 1) */
  uint8_t lo = 0, hi = 0x7e;
  while (hi - lo > 1) {
    const uint8_t mid = (uint8_t)((lo + hi) / 2);
    if (e4m3_to_f32(mid) <= x) lo = mid; else hi = mid;
  }
  if (e4m3_to_f32(hi) <= x) lo = hi;
  if (lo == 0x7e) return (uint8_t)(sign | lo);
  const float below = x - e4m3_to_f32(lo), above = e4m3_to_f32((uint8_t)(lo + 1)) - x;   /* both exact */
  const uint8_t q = (below < above || (below == above && !(lo & 1u))) ? lo : (uint8_t)(lo + 1);
  return (uint8_t)(sign | q);
}

float oracle_e4m3_to_f32(uint8_t v) { return e4m3_to_f32(v); }
uint8_t oracle_f32_to_e4m3(float f) { return f32_to_e4m3(f); }

void oracle_fp8gemm_f32acc(const uint8_t* A, const uint8_t* Bt, float scale_a, float scale_b, uint16_t* C, int M,
                           int N, int K, int out_bf16) {
  float* a = (float*)malloc((size_t)M * K * sizeof(float));
  float* b = (float*)malloc((size_t)N * K * sizeof(float));
  for (size_t i = 0; i < (size_t)M * K; ++i) a[i] = e4m3_to_f32(A[i]);
  for (size_t i = 0; i < (size_t)N * K; ++i) b[i] = e4m3_to_f32(Bt[i]);
  volatile float s_rounded = scale_a * scale_b;   /* fp32(sa * sb), kept apart from the product below */
  const float s = s_rounded;
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m) {
    const float* am = a + (size_t)m * K;
    for (int n = 0; n < N; ++n) {
      const float* bn = b + (size_t)n * K;
      float acc = 0.0f;
      for (int k = 0; k < K; ++k) acc += am[k] * bn[k];   /* one fp32 accumulator, k ascending */
      const float y = acc * s;
      C[(size_t)m * N + n] = out_bf16 ? f2bf(y) : f2h(y);
    }
  }
  free(a);
  free(b);
}
