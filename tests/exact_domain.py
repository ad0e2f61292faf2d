"""Exactly summable, full-range operands for bit-exact GEMM tests — TEST INFRASTRUCTURE.

Every operand is ``A[m,k] = i * 2^r_m`` and ``Bt[n,k] = j * 2^c_n`` with small signed integers i, j, so every product of
row m and column n, and every partial sum of them in any order and any division of K, is an integer multiple of
``2^(r_m + c_n)``. The generators bound ``sum_k |i * j|`` per element, so those multiples stay exact in the kernel's
accumulator and the true output is ONE rounding of the exact (float64) product:

* fp16 / bf16 operands, fp32 accumulation: ``sum_k |i * j| < EXACT_SUM_BOUND = 2^24``. Measured on an H100 80GB HBM3
  (700 W power limit): the wgmma fp32 sums were exact up to this bound in every configuration and K-mode. A unit
  product next to a 2^23 one survived in the same k16 step, the next k-block and the last split
  (test_gpu_exact_range.py::test_fp32_accumulation_is_exact_to_2_24), and planted sums up to 2^24 - 1 came out exact.
  2^24 is what an fp32 accumulator can hold in any order; beyond it the sum itself has to round.
* fp16 operands, fp16 accumulation: ``sum_k |i * j| < 2048`` (the non-saturating domain of the oracle's fp16 model),
  scaled by powers of two across the normal fp16 range.
* e4m3 operands: small integers with ``sum_k |i * j| <= E4M3_SUM_BOUND = 2047`` (the FP8 tensor core's running sum keeps
  fewer bits than fp32; see test_gpu_fp8.py). The full output range is reached through the scales instead: odd integer
  multipliers Q < 4096 times powers of two, per tensor, per row / column or per block, chosen so that the scaled values
  stay exact in fp32 too.

Where the output must round is steered by PROBE rows: every ``PROBE_EVERY``-th row of A is zero except three weights
at fixed k positions (two adjacent, one in the last k-block, so the sum crosses a k16 step, k-blocks and any split), and
Bt holds, at those positions of each column, the digits of a planted integer target. A probe row times column n is then
exactly ``sign_m * target[n] * 2^(r_m + c_n)``. The targets are the rounding cases (exact ties at every number of
dropped bits, rounding up and down, near misses), the row and column exponents move them through the subnormal, normal
and overflowing ranges of the output type. The remaining rows are random integers over the whole k range.

Kept out of the domain, because they exercise the tensor core rather than the kernel's code: subnormal operands,
fp32-subnormal accumulators (bf16 subnormal outputs) and fp16-accumulator overflow.
"""
from __future__ import annotations

import numpy as np

EXACT_SUM_BOUND = 2 ** 24          # fp16 / bf16 operands, fp32 accumulation (measured, module docstring)
FP16_ACC_SUM_BOUND = 2048          # fp16 accumulation: every partial sum an fp16 integer
E4M3_SUM_BOUND = 2047              # e4m3 operands: what test_gpu_fp8.py asserts of its data
PROBE_EVERY = 5

# Significand bits (with the hidden bit) and exponent limits of the output / operand types.
FORMATS = {"fp16": dict(p=11, emin=-14, emax=15), "bf16": dict(p=8, emin=-126, emax=127)}

# Row / column exponents. fp16: operands stay normal (>= 2^-14) and finite; r + c reaches -28 (subnormal outputs) and
# +5 (overflow). bf16: r + c reaches 104, where a target just under 2^24 rounds past the largest bf16 to inf, and
# stays >= -110, far above the fp32 subnormals; every partial sum stays below 2^24 * 2^104 (finite in fp32).
ROW_EXP = {"fp16": (-14, -13, -9, -5, -2, 0, 2), "bf16": (-60, -31, -7, 0, 17, 41, 60)}
COL_EXP = {"fp16": (-14, -10, -6, -1, 0, 3), "bf16": (-50, -19, 0, 9, 28, 44)}
# fp16 accumulation: 2047 * 2^(r + c) stays below 65504 and 2^(r + c) >= 2^-14
ROW_EXP_ACC16, COL_EXP_ACC16 = (-7, -4, -1, 0, 2), (-7, -3, 0, 2)


def probe_positions(k: int) -> tuple[int, int, int]:
    """The k positions of the probe weights (lowest weight first): the last k-block, and two adjacent ones a third in."""
    p = k // 3
    return k - 5, p + 1, p


def _weights(kind: str) -> tuple[int, int, int]:
    # the digit ranges these weights need keep every digit an exactly representable integer of the operand type
    return {"fp16": (1, 2 ** 8, 2 ** 13), "bf16": (1, 2 ** 8, 2 ** 16), "e4m3": (1, 16, 256)}[kind]


def _digits(kind: str, s: int) -> tuple[int, int, int]:
    """Digits d0, d1, d2 with d0 + w1 d1 + w2 d2 = |s|, each representable in the operand type (fp16: d2 <= 2047,
    bf16: all <= 255, e4m3: d0, d1 <= 15, d2 <= 7)."""
    w = _weights(kind)
    s = abs(int(s))
    d2 = s // w[2]
    rest = s - d2 * w[2]
    d1, d0 = rest // w[1], rest % w[1]
    assert d0 + w[1] * d1 + w[2] * d2 == s
    lim = {"fp16": (255, 31, 2047), "bf16": (255, 255, 255), "e4m3": (15, 15, 7)}[kind]
    assert all(0 <= d <= l for d, l in zip((d0, d1, d2), lim)), (kind, s)
    return d0, d1, d2


def rounding_targets(kind: str) -> list[int]:
    """Integers whose rounding to ``kind`` (fp16 / bf16) drops 1 to 13 bits: an exact tie that rounds up (odd kept
    significand), one that rounds down (even), and one just off a tie, for each number of dropped bits; then the
    overflow edges (fp16: 65504, 65519, 65520 = the tie that goes to inf, 65535; bf16: the largest bf16 and the tie,
    just below it and 2^24 - 1 at 2^104, i.e. at and past the largest bf16)."""
    p = FORMATS[kind]["p"]
    out = []
    for d in range(1, 14):
        top = 1 << (p - 1)                      # kept significands of p bits: [2^(p-1), 2^p)
        for kept, rem in ((top + 5, 1 << (d - 1)), (top + 6, 1 << (d - 1)), (top + 9, (1 << (d - 1)) + (d > 1))):
            out.append((kept << d) | rem)
    if kind == "fp16":
        out += [65504, 65519, 65520, 65535]
    else:
        out += [2 ** 24 - 2 ** 16, 2 ** 24 - 2 ** 15 - 1, 2 ** 24 - 2 ** 15, 2 ** 24 - 1]
    assert all(0 < t < EXACT_SUM_BOUND for t in out)
    return out


def _cycle(values, idx):
    return np.asarray(values)[np.asarray(idx) % len(values)]


class Operands:
    """A[M,K], Bt[N,K] as exact float64 values, plus what they were built from (tests and fixtures checks)."""

    def __init__(self, a, bt, row_exp, col_exp, probe_rows, targets):
        self.a, self.bt = a, bt
        self.row_exp, self.col_exp = row_exp, col_exp
        self.probe_rows, self.targets = probe_rows, targets

    def exact(self) -> np.ndarray:
        """The exact product A @ Bt^T (float64 is exact here: every partial sum has fewer than 53 bits)."""
        return self.a @ self.bt.T

    def sum_bound(self) -> float:
        """max over elements of sum_k |i * j|: the integer magnitudes, the exponents divided out."""
        ia = np.abs(self.a) / np.exp2(self.row_exp)[:, None]
        jb = np.abs(self.bt) / np.exp2(self.col_exp)[:, None]
        return float((ia @ jb.T).max())


def operands16(m: int, n: int, k: int, kind: str, seed: int, acc16: bool = False) -> Operands:
    """Full-range operands for the 16-bit kernels: ``kind`` "fp16" or "bf16" (the operand and output type). ``acc16``:
    the fp16-accumulation domain instead (random +-1 / 0 data, at most 2047 nonzero products per element, no probe
    rows, exponents that keep every partial sum a normal fp16 value)."""
    assert k >= 16 and (kind == "fp16" or not acc16)
    rng = np.random.default_rng(seed)
    rows, cols = np.arange(m), np.arange(n)
    if acc16:
        r, c = _cycle(ROW_EXP_ACC16, rows * 3), _cycle(COL_EXP_ACC16, cols)
        ia = rng.integers(-1, 2, size=(m, k))
        keep = np.argsort(rng.random((m, k)), axis=1) < min(k, FP16_ACC_SUM_BOUND - 1)   # <= 2047 nonzeros per row
        ia = ia * keep
        jb = rng.integers(-1, 2, size=(n, k))
        ops = Operands(ia * np.exp2(r)[:, None], jb * np.exp2(c)[:, None], r, c, np.array([], dtype=int), [])
        assert ops.sum_bound() < FP16_ACC_SUM_BOUND
        return ops
    targets = rounding_targets(kind)
    nt = len(targets)
    probe = rows[rows % PROBE_EVERY == 2]
    # probe rows: exponent and sign cycle independently; column n: target n % nt, exponent (n // nt) % len(COL_EXP)
    r = _cycle(ROW_EXP[kind], rows * 3)
    r[probe] = _cycle(ROW_EXP[kind], np.arange(len(probe)))
    sign = np.where((np.arange(len(probe)) // len(ROW_EXP[kind])) % 2 == 0, 1, -1)
    c = _cycle(COL_EXP[kind], cols // nt)
    pos = probe_positions(k)
    # random rows: sum_k |i j| <= k * lim_a * lim_b < 2^24, the digits of Bt at the probe positions meet zeros in them
    lim_b = 63 if kind == "fp16" else 31
    lim_a = int(min(2047 if kind == "fp16" else 255, (EXACT_SUM_BOUND - 1) // (k * lim_b)))
    ia = rng.integers(-lim_a, lim_a + 1, size=(m, k))
    jb = rng.integers(-lim_b, lim_b + 1, size=(n, k))
    ia[:, list(pos)] = 0
    ia[probe] = 0
    for w, p in zip(_weights(kind), pos):
        ia[probe, p] = w * sign
    for col in cols:
        t = targets[col % nt]
        jb[col, list(pos)] = _digits(kind, t)
    ops = Operands(ia * np.exp2(r)[:, None], jb * np.exp2(c)[:, None], r, c, probe,
                   [targets[col % nt] for col in cols])
    assert ops.sum_bound() < EXACT_SUM_BOUND
    return ops


# ------------------------------------------------------------------------------------------------------------- e4m3
# Scale multipliers, odd, per output type. A target 2^(d-1) times Q keeps Q's bits shifted: with Q of 12 bits (fp16
# out) or 9 bits (bf16 out) it is an exact tie after dropping d bits, rounding up when Q's second-lowest bit is set
# (4095, 511) and down when it is not (4093, 509). fp16: 2^8 * 4095 / 2^4 = 65520, the tie that goes to inf. bf16:
# 2041 * 513 * 2^108 lies between the largest bf16 and the largest fp32, so it rounds to inf (per tensor only).
E4M3_Q = {"fp16": (4095, 4093), "bf16": (511, 509)}
E4M3_TARGETS = tuple([1 << d for d in range(11)] + [3, 5, 7, 99, 1000, 1365, 2041, 2047])


def operands_e4m3(m: int, n: int, k: int, seed: int):
    """e4m3 operands as small integers (float64 values, every one exactly an e4m3 value), with probe rows planting
    E4M3_TARGETS; at most 2000 nonzeros per random row of A, so every sum_k |i j| <= 2047 at any K."""
    rng = np.random.default_rng(seed)
    rows, cols = np.arange(m), np.arange(n)
    probe = rows[rows % PROBE_EVERY == 2]
    pos = probe_positions(k)
    ia = rng.integers(-1, 2, size=(m, k))
    ia *= np.argsort(rng.random((m, k)), axis=1) < min(k, 2000)
    ia[:, list(pos)] = 0
    ia[probe] = 0
    sign = np.where(np.arange(len(probe)) % 2 == 0, 1, -1)
    for w, p in zip(_weights("e4m3"), pos):
        ia[probe, p] = w * sign
    jb = rng.integers(-1, 2, size=(n, k))
    nt = len(E4M3_TARGETS)
    for col in cols:
        jb[col, list(pos)] = _digits("e4m3", E4M3_TARGETS[col % nt])
    a, bt = ia.astype(np.float64), jb.astype(np.float64)
    assert (np.abs(a) @ np.abs(bt).T).max() <= E4M3_SUM_BOUND
    return a, bt


# Exponents of the e4m3 scales: per row of A (rowwise and block scales), per column or 128-column block (of Bt). Row
# exponent 104 (block scales: 103, their k-block exponent adds one) takes the largest targets past the largest bf16 while
# every fp32 value stays finite: 2047 * 4095 * 2^105 < 2^128.
E4M3_ROW_EXP = (-30, -22, -12, -4, 0, 3, 104)
E4M3_COL_EXP = (-2, 0, 1)


def e4m3_tensor_scales(out: str) -> list[tuple[float, float]]:
    """Per-tensor (scale_a, scale_b) pairs, both multipliers each. fp16 out: one pair reaching overflow (a target 2^8
    lands on 65520) with rounding below it, one the subnormals. bf16 out: one taking 2041 past the largest bf16, and
    plain rounding."""
    q0, q1 = E4M3_Q[out]
    if out == "fp16":
        return [(q0 * 2.0 ** -4, 1.0), (q1 * 2.0 ** -5, 0.5), (q0 * 2.0 ** -29, 0.5), (q1 * 2.0 ** -30, 1.0)]
    return [(513 * 2.0 ** 108, 1.0), (q0 * 2.0 ** -40, 0.25), (q1 * 2.0 ** -20, 1.0)]


def e4m3_row_q(m: int, out: str) -> np.ndarray:
    return _cycle(E4M3_Q[out], np.arange(m) // 2)


def e4m3_rowwise_scales(m: int, n: int, out: str, block: bool = False) -> tuple[np.ndarray, np.ndarray]:
    """scale_a [M] = Q_m 2^r_m, scale_b [N] = 2^c_n (fp32 values): every output fp32(fp32(acc sb) sa) is exact."""
    r = _cycle(E4M3_ROW_EXP, np.arange(m) // 4)
    sa = e4m3_row_q(m, out) * np.exp2(np.minimum(r, 103) if block else r)
    sb = np.exp2(_cycle(E4M3_COL_EXP, np.arange(n) // 3))
    return sa.astype(np.float32), sb.astype(np.float32)


def e4m3_block_scales(m: int, n: int, k: int, out: str) -> tuple[np.ndarray, np.ndarray]:
    """scale_a [M, nkb] = Q_m 2^r_m, scale_b [ceil(N/128), nkb] = 2^(c_b + t_kb) with t_kb in {0, 1} varying along K
    (0 on the probe positions' k-blocks), so a scale read for the wrong k-block, 32 k-blocks off included, changes the
    result. Every promotion
    fmaf(p, s, acc) is exact: sum |p| * Q * 2 < 2^24."""
    nkb, nb = -(-k // 128), -(-n // 128)
    sa, _ = e4m3_rowwise_scales(m, 1, out, block=True)
    kb = np.arange(nkb)
    t = (kb % 32 + kb // 32) % 2                      # differs from t 32 k-blocks earlier (one sb load per 32)
    t[[p // 128 for p in probe_positions(k)]] = 0
    sb = np.exp2(_cycle(E4M3_COL_EXP, np.arange(nb))[:, None] + t[None, :])
    assert E4M3_SUM_BOUND * max(E4M3_Q[out]) * 2 < 2 ** 24
    return np.repeat(sa[:, None], nkb, axis=1).astype(np.float32), sb.astype(np.float32)


def e4m3_1d1d_kb_bits(k: int) -> tuple[np.ndarray, np.ndarray]:
    """The k-block exponents (u, t) of e4m3_block_1d1d_scales: u (A's) only on even k-blocks, t (Bt's) only on odd ones,
    so u + t <= 1; each an aperiodic-looking pattern of the k-block pair index j = kb // 2 (u: j % 7 in {0, 1, 3}, t:
    j % 5 in {0, 2}), so that no shift by 1..9 or 32 k-blocks maps either pattern, or their sum, onto itself; 0 on the
    probe positions' k-blocks."""
    kb = np.arange(-(-k // 128))
    j = kb // 2
    u = ((kb % 2 == 0) & np.isin(j % 7, (0, 1, 3))).astype(np.int64)
    t = ((kb % 2 == 1) & np.isin(j % 5, (0, 2))).astype(np.int64)
    probe = [p // 128 for p in probe_positions(k)]
    u[probe] = t[probe] = 0
    return u, t


def e4m3_block_1d1d_scales(m: int, n: int, k: int, out: str) -> tuple[np.ndarray, np.ndarray]:
    """Scales of the GEMM with 1 x 128 scales on both operands: scale_a [M, nkb] = Q_m 2^(r_m + u_kb) and scale_b
    [N, nkb] = 2^(c_n + t_kb), fp32 values (e4m3_1d1d_kb_bits for u, t). c_n cycles E4M3_COL_EXP column by column, so
    adjacent columns differ and so do columns 8 apart (8 % 3 != 0): a swapped column pair, or a column read from another
    pair group, changes the result. A scale of either operand read for another k-block changes it too. Every promotion
    fmaf(p, fp32(sa sb), acc) is exact: u and t never meet, so sum |p| * Q * 2^(u + t) <= 2047 * Q * 2 < 2^24."""
    u, t = e4m3_1d1d_kb_bits(k)
    assert (u + t).max(initial=0) <= 1
    assert E4M3_SUM_BOUND * max(E4M3_Q[out]) * 2 < 2 ** 24
    r = np.minimum(_cycle(E4M3_ROW_EXP, np.arange(m) // 4), 103)      # 2047 * 4095 * 2^(103 + 1 + 1) < 2^128
    sa = e4m3_row_q(m, out)[:, None] * np.exp2(r[:, None] + u[None, :])
    sb = np.exp2(_cycle(E4M3_COL_EXP, np.arange(n))[:, None] + t[None, :])
    assert np.array_equal(sa.astype(np.float32).astype(np.float64), sa)
    return sa.astype(np.float32), sb.astype(np.float32)


def exact_1d1d(a: np.ndarray, bt: np.ndarray, sa: np.ndarray, sb: np.ndarray) -> np.ndarray:
    """The exact float64 output of the 1 x 128 x 1 x 128 contract: sum over k-blocks of (A_kb Bt_kb^T) sa[:, kb] sb[:, kb]
    (every term and partial sum an integer multiple of a power of two below 2^53 units, so float64 is exact)."""
    y = np.zeros((a.shape[0], bt.shape[0]))
    for kb in range(sa.shape[1]):
        part = a[:, kb * 128:(kb + 1) * 128] @ bt[:, kb * 128:(kb + 1) * 128].T
        y += part * sa[:, kb:kb + 1].astype(np.float64) * sb[None, :, kb].astype(np.float64)
    return y


# ------------------------------------------------------------------------------------------------ the reference
def round_fp16_bits(x: np.ndarray) -> np.ndarray:
    """float64 -> fp16 bits, one round to nearest even (numpy's cast rounds the double directly)."""
    return np.asarray(x, dtype=np.float64).astype(np.float16).view(np.uint16)


def round_bf16_bits(x: np.ndarray) -> np.ndarray:
    """float64 -> bf16 bits, one round to nearest even. The values of this domain are exact in fp32 (asserted), so
    going through fp32 first rounds nothing."""
    import oracle
    x32 = np.asarray(x, dtype=np.float64).astype(np.float32)
    fin = np.isfinite(x)
    assert np.array_equal(x32[fin].astype(np.float64), np.asarray(x)[fin]), "not exact in fp32"
    return oracle.f32_to_bf16_bits(x32)


def reference16(ops: Operands, kind: str) -> np.ndarray:
    """Bits of the true output: the exact product, rounded once to fp16 / bf16."""
    y = ops.exact()
    return round_fp16_bits(y) if kind == "fp16" else round_bf16_bits(y)


# ------------------------------------------------------------------------------------------ what a fixture holds
def classify(exact: np.ndarray, kind: str, unit: np.ndarray) -> dict:
    """Masks over the exact (pre-rounding) values of an output of type ``kind``, ``unit`` being each element's integer
    unit 2^(r_m + c_n) (e4m3: the power-of-two part of its scales): ``tie_up[d]`` / ``tie_down[d]`` (an exact tie of a
    finite result after dropping d bits of its integer, rounding away from / toward zero), ``rounds`` (inexact),
    ``subnormal`` (fp16 result below 2^-14, nonzero), ``inf`` (a finite value that rounds to +-inf), ``max_finite``
    (rounds to +-the largest finite value)."""
    f = FORMATS[kind]
    exact = np.asarray(exact, dtype=np.float64)
    x = np.abs(exact)
    nz = x > 0
    e = np.maximum(np.frexp(x)[1] - 1, f["emin"])      # subnormals share the smallest normal exponent's ulp
    ulp = np.exp2((e - (f["p"] - 1)).astype(np.float64))
    q = x / ulp                                        # exact: ulp is a power of two
    frac = q - np.floor(q)
    bits = round_fp16_bits(exact) if kind == "fp16" else round_bf16_bits(exact)
    rounded = (bits.view(np.float16).astype(np.float64) if kind == "fp16"
               else (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64))
    out = {"inf": np.isfinite(exact) & np.isinf(rounded), "rounds": nz & (frac != 0)}
    tie = nz & (frac == 0.5) & ~out["inf"]
    drop = np.rint(np.log2(ulp / np.broadcast_to(unit, x.shape))).astype(int)
    odd = (np.floor(q) % 2) == 1
    out["tie_up"] = {d: tie & odd & (drop == d) for d in range(1, 14)}
    out["tie_down"] = {d: tie & ~odd & (drop == d) for d in range(1, 14)}
    out["subnormal"] = nz & (x < 2.0 ** f["emin"]) & (kind == "fp16")
    top = 65504.0 if kind == "fp16" else float(np.float32(2.0 ** 128 - 2.0 ** 120))
    out["max_finite"] = np.abs(rounded) == top
    return out
