"""CPU restatement of the FP8 (e4m3) GEMM with rowwise scales — TEST INFRASTRUCTURE, never the product.

    C[m,n] = RN_out( fp32( fp32(acc[m,n] * scale_b[n]) * scale_a[m] ) ),   acc[m,n] = sum_k A[m,k] * Bt[n,k]

The operands are decoded through the e4m3 codec of ``oracle.fp8`` (a 256-entry table); every e4m3 x e4m3 product is
exact in fp32, and ``acc`` is the canonical one fp32 accumulator, k ascending, as in ``oracle/fp8_oracle.c``. numpy's
float32 products round once each (IEEE round-to-nearest-even); the output roundings are numpy's float32 -> float16
cast and ``oracle.f32_to_bf16_bits``, both RN-even. Pinned against torch's CPU expression
``(((a.float() @ bt.float().t()) * sb[None, :]) * sa[:, None]).to(out_dtype)`` by ``tests/golden/fp8_rowwise_cases.npz``
(``tests/golden/make_fp8_rowwise_golden.py``).
"""
from __future__ import annotations

import numpy as np

import oracle
from oracle import fp8 as fp8_oracle

_E4M3 = None


def e4m3_values(codes: np.ndarray) -> np.ndarray:
    global _E4M3
    if _E4M3 is None:
        _E4M3 = fp8_oracle.e4m3_to_f32(np.arange(256, dtype=np.uint8))
    return _E4M3[np.asarray(codes, dtype=np.uint8)]


def fp8gemm_f32acc_rowwise(a_codes: np.ndarray, bt_codes: np.ndarray, scale_a, scale_b, out_bf16: bool) -> np.ndarray:
    """``a_codes`` [M,K], ``bt_codes`` [N,K]: uint8 float8_e4m3fn codes; ``scale_a`` M and ``scale_b`` N fp32 values.
    Returns the uint16 bits of C [M,N], fp16 or bf16."""
    (m, k), (n, k2) = a_codes.shape, bt_codes.shape
    assert k == k2 and a_codes.dtype == np.uint8 and bt_codes.dtype == np.uint8
    sa = np.asarray(scale_a, dtype=np.float32).reshape(-1)
    sb = np.asarray(scale_b, dtype=np.float32).reshape(-1)
    assert sa.size == m and sb.size == n
    a, b = e4m3_values(a_codes), e4m3_values(bt_codes)
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    if np.all(a64 == np.rint(a64)) and np.all(b64 == np.rint(b64)) and (np.abs(a64) @ np.abs(b64).T).max() < 2.0 ** 24:
        # integer operands whose partial sums all stay below 2^24: every fp32 partial sum is exact, so the canonical
        # accumulator equals the exact sum, whatever the order
        acc = (a64 @ b64.T).astype(np.float32)
    else:
        acc = np.zeros((m, n), dtype=np.float32)
        for kk in range(k):                               # one fp32 accumulator per element, k ascending
            acc += a[:, kk, None] * b[None, :, kk]
    y = (acc * sb[None, :]) * sa[:, None]                 # two fp32 products, column scale first
    return oracle.f32_to_bf16_bits(y) if out_bf16 else y.astype(np.float16).view(np.uint16)
