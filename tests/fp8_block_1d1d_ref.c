/* fp8_block_1d1d_ref.c — CPU reference of the block-scaled FP8 (e4m3) GEMM with 1 x 128 scales on both operands
 * (cuda_l2_b200/csrc/b200_fp8_block_1d1d.h).  TEST INFRASTRUCTURE ONLY.
 *
 * fp8_block_ref.c's contract with only the index of sb changed: for every output element and k-block kb (128 k, the last
 * one ragged): p = the fp32 sum of the block's products, k ascending; s = fp32(sa(m, kb) * sb(n, kb)), both M-major
 * (value (m, kb) at sa[kb * ld_a + m], (n, kb) at sb[kb * ld_b + n]); acc = fp32(p * s) on a split's first k-block,
 * acc = fmaf(p, s, acc) on every later one. With splits > 1 the k-blocks are divided as the kernel's cluster split-K
 * divides them (ceil(nkb / splits) per split) and the splits' results are summed in order from +0. Compiled with
 * -ffp-contract=off so that no other multiply-add is fused. */
#include "../oracle/fp8_oracle.c"

void ref_fp8gemm_f32acc_block_1d1d(const uint8_t* A, const uint8_t* Bt, const float* sa, int ld_a, const float* sb,
                                   int ld_b, uint16_t* C, int M, int N, int K, int out_bf16, int splits) {
  const int nkb = (K + 127) / 128;
  float* a = (float*)malloc((size_t)M * K * sizeof(float));
  float* b = (float*)malloc((size_t)N * K * sizeof(float));
  for (size_t i = 0; i < (size_t)M * K; ++i) a[i] = e4m3_to_f32(A[i]);
  for (size_t i = 0; i < (size_t)N * K; ++i) b[i] = e4m3_to_f32(Bt[i]);
  const int per = (nkb + splits - 1) / splits;
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m) {
    const float* am = a + (size_t)m * K;
    for (int n = 0; n < N; ++n) {
      const float* bn = b + (size_t)n * K;
      float total = 0.0f;
      for (int sp = 0; sp < splits; ++sp) {
        const int kb0 = sp * per, kb1 = kb0 + per < nkb ? kb0 + per : nkb;
        float acc = 0.0f;
        for (int kb = kb0; kb < kb1; ++kb) {
          float p = 0.0f;
          const int k1 = (kb + 1) * 128 < K ? (kb + 1) * 128 : K;
          for (int k = kb * 128; k < k1; ++k) p += am[k] * bn[k];
          const float s = sa[(size_t)kb * ld_a + m] * sb[(size_t)kb * ld_b + n];
          acc = kb == kb0 ? p * s : fmaf(p, s, acc);
        }
        if (splits == 1) total = acc;
        else if (kb0 < kb1) total += acc;
      }
      C[(size_t)m * N + n] = out_bf16 ? f2bf(total) : f2h(total);
    }
  }
  free(a);
  free(b);
}
