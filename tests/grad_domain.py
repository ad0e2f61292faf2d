"""Exactly summable operands for the three products of a linear layer's training step — TEST INFRASTRUCTURE.

A linear layer y = x W^T has three products, and a 16-bit training step runs all three on the GEMM kernels: y, the input
gradient dX = dY W and the weight gradient dW = dY^T X. The operands here make each of them ONE rounding of an exact
float64 value, so that all three can be checked bit for bit:

    A[m,k]  = i * 2^r_m                 (x, or the GEMM's A)
    Bt[n,k] = j * 2^c_n                 (W, K-major)
    dY[m,n] = h * 2^(q - r_m - c_n)

with small signed integers i, j, h. Then

    y[m,n]  = 2^(r_m + c_n) * sum_k i j
    dX[m,k] = 2^(q - r_m)   * sum_n h j
    dW[n,k] = 2^(q - c_n)   * sum_m h i

Each product has one exponent per output element, constant along its reduction, so every partial sum in any order and
any division of the reduction is an integer multiple of it. The integer limits keep sum_k |i j|, sum_n |h j| and
sum_m |h i| below exact_domain.EXACT_SUM_BOUND (2^24, what the fp32 accumulator holds exactly); the generator asserts
all three. The exponents move the outputs across the whole range of the type: with them, y, dX and dW each hold values
that round up, round down and tie, and in fp16 subnormal values, values that round to zero and values that overflow to
inf (tests/test_grad_exact_cpu.py checks the fixtures for all of this).

Every operand value is exact and either zero or a normal number of the operand type: an element of dY whose exponent
q - r_m - c_n would leave the normal range is zero. Each integer row carries its own limit (the full one, 1/16 of it or
1/256 of it, cycling), so small sums meet the smallest exponents (subnormal and zero outputs) and large ones the
largest (overflow).

``bias=True`` narrows the row exponents to two values one apart. Then the bias gradient, torch's fp32 column sum of dY
(``dZ.sum(0, dtype=torch.float32)``), is exact too: sum_m |h| 2^(r_max - r_m) < 2^24 in units of 2^(q - r_max - c_n).
The bias itself is b_n 2^(r_min + c_n) with |b_n| below the sum bound's slack, so the fused epilogue's fp32 sum
z = A Bt^T + bias is exact before its one rounding.
"""
from __future__ import annotations

import math

import numpy as np

import exact_domain as ed

BOUND = ed.EXACT_SUM_BOUND
LIM_BITS = 8                       # |integer| <= 255: exact in fp16 and bf16
# Normal range of the operand types (smallest and largest exponent of a normal number)
NORMAL = {"fp16": (-14, 15), "bf16": (-126, 127)}
# Row exponents r_m, column exponents c_n and q. fp16: r + c spans -28..13, so y reaches subnormal and zero outputs
# (small sums at 2^-28) and overflow (large sums at 2^13); dX's exponent q - r spans -19..2 and dW's q - c -18..2, so
# small sums of either are subnormal and large ones overflow. About half of dY is then zero (exponent out of range).
# bf16: the outputs span about 2^-110..2^140 without fp32 subnormals; bf16 has no subnormal outputs here.
ROW_EXP = {"fp16": (-14, -10, -6, -2, 3, 7), "bf16": (-60, -30, -7, 0, 20, 60)}
COL_EXP = {"fp16": (-14, -9, -4, 1, 6), "bf16": (-50, -20, 0, 10, 45)}
Q = {"fp16": -12, "bf16": 10}
# bias=True: two row exponents one apart (the fp32 column sum of dY stays exact)
ROW_EXP_BIAS = {"fp16": (-2, -1), "bf16": (0, 1)}
ROW_SHIFTS = (0, 4, 8)             # an integer row's limit is the full one >> shift, cycling


class GradOperands:
    """a [M,K], bt [N,K], dy [M,N] (and bias [N] or None) in the operand dtype, every value exact, with the exponents
    r [M], c [N] and q, and the integer limits (li, lj, lh)."""

    def __init__(self, a, bt, dy, bias, r, c, q, limits):
        self.a, self.bt, self.dy, self.bias = a, bt, dy, bias
        self.r, self.c, self.q, self.limits = r, c, q, limits


def limits(m: int, n: int, k: int, bias: bool = False) -> tuple[int, int, int]:
    """(li, lj, lh), the largest |i|, |j|, |h|: K li lj, N lh lj and M lh li stay below 2^24 (2^23 with a bias, whose
    sums carry one more factor of 2 and the bias term), balanced in log space and capped at 2^LIM_BITS - 1."""
    bound = BOUND // 4 if bias else BOUND
    x, y, z = (math.log2((bound - 1) / max(d, 1)) for d in (k, n, m))   # li lj, lh lj, lh li  <= 2^x, 2^y, 2^z
    cap = 2 ** LIM_BITS - 1
    li, lj, lh = (max(1, min(cap, int(2 ** ((u + v - w) / 2)))) for u, v, w in ((x, z, y), (x, y, z), (y, z, x)))
    assert k * li * lj < bound and n * lh * lj < bound and m * lh * li < bound, (m, n, k, li, lj, lh)
    return li, lj, lh


def _cycle(torch, values, idx):
    return torch.tensor(values, dtype=torch.int64, device=idx.device)[idx % len(values)]


def _ints(torch, rows: int, cols: int, lim: int, gen, device):
    """[rows, cols] int32 uniform in [-lim_row, lim_row], lim_row = lim >> ROW_SHIFTS[row % 3] (at least 1)."""
    x = torch.randint(-lim, lim + 1, (rows, cols), generator=gen, device=device, dtype=torch.int32)
    shift = _cycle(torch, ROW_SHIFTS, torch.arange(rows, device=device)).to(torch.int32)
    x = torch.div(x, (1 << shift)[:, None], rounding_mode="trunc")
    return x


def operands(torch, m: int, n: int, k: int, kind: str, seed: int, bias: bool = False, device="cuda") -> GradOperands:
    """The operands of one training step on the exact gradient domain (module docstring), generated on ``device`` with
    a torch generator seeded with ``seed``. ``kind``: "fp16" or "bf16". Every bound is asserted."""
    dtype = torch.float16 if kind == "fp16" else torch.bfloat16
    gen = torch.Generator(device=device).manual_seed(seed)
    li, lj, lh = limits(m, n, k, bias)
    rows, cols = torch.arange(m, device=device), torch.arange(n, device=device)
    r = _cycle(torch, ROW_EXP_BIAS[kind] if bias else ROW_EXP[kind], rows * 5 // 3)
    c = _cycle(torch, COL_EXP[kind], cols)
    q = Q[kind]
    ia, jb = _ints(torch, m, k, li, gen, device), _ints(torch, n, k, lj, gen, device)
    # dY's integers: the row limits cycle along n, so that each column of dW and each row of dX mixes them
    h = _ints(torch, n, m, lh, gen, device).t()
    e = q - r[:, None] - c[None, :]
    lo, hi = NORMAL[kind]
    h = h * ((e >= lo) & (e + LIM_BITS <= hi))            # zero where h 2^e could leave the normal range
    for x, lim in ((ia, li), (jb, lj), (h, lh)):
        assert int(x.abs().max()) <= lim
    # the three sums, per element, are bounded through the limits (K li lj, N lh lj, M lh li; limits() asserts them)
    lo_op = NORMAL[kind][0]
    assert int(r.min()) >= lo_op and int(c.min()) >= lo_op
    assert int(r.max()) + LIM_BITS <= NORMAL[kind][1] and int(c.max()) + LIM_BITS <= NORMAL[kind][1]
    a = _scale(torch, ia, r[:, None], dtype)
    bt = _scale(torch, jb, c[:, None], dtype)
    dy = _scale(torch, h, e, dtype)
    b = None
    if bias:
        # b_n 2^eb_n, eb_n = r_min + c_n raised to the smallest normal exponent: z in units of 2^(r_min + c_n) is at
        # most 2 K li lj + |b_n| 2^(eb_n - r_min - c_n) < 2^23 + 2^22
        lb = 2 ** LIM_BITS - 1
        bi = torch.randint(-lb, lb + 1, (n,), generator=gen, device=device, dtype=torch.int32)
        eb = (int(r.min()) + c).clamp(min=lo)
        assert lb * 2 ** int((eb - int(r.min()) - c).max()) < BOUND // 4
        b = _scale(torch, bi, eb, dtype)
        # the column sum of dY in units of 2^(q - r_max - c_n): M lh 2^(r_max - r_min) < 2^24
        assert m * lh * 2 ** (int(r.max()) - int(r.min())) < BOUND
    return GradOperands(a, bt, dy, b, r, c, q, (li, lj, lh))


def _scale(torch, ints, exp, dtype):
    """ints * 2^exp in ``dtype``, exactly (asserted: the value survives the cast)."""
    v = ints.to(torch.float64) * torch.exp2(exp.to(torch.float64))
    out = v.to(dtype)
    assert torch.equal(out.to(torch.float64), v), "operand not exact in its type"
    return out


# ------------------------------------------------------------------------------------------------- the reference
def exact(torch, ops: GradOperands, activation: str = "none"):
    """float64 (y, dX, dW, dbias) of one step with output gradient dY, before rounding: y = act(A Bt^T (+ bias)),
    dZ = dY, or for relu dY where the ROUNDED output is > 0 (a positive z that rounds to zero has no gradient, as in the
    operator, whose mask is read from its output) and 0 elsewhere; dX = dZ Bt, dW = dZ^T A, dbias = the column sum of
    dZ (None without a bias). Exact zeros are +0.0, as in an accumulator that starts at +0.0."""
    assert activation in ("none", "relu")
    a, bt, dz = ops.a.to(torch.float64), ops.bt.to(torch.float64), ops.dy.to(torch.float64)
    y = a @ bt.T
    if ops.bias is not None:
        y += ops.bias.to(torch.float64)
    if activation == "relu":
        y = torch.relu(y)
        dz = dz * (y.to(torch.float32).to(ops.a.dtype) > 0)
    db = dz.sum(0).add_(0.0) if ops.bias is not None else None
    return y.add_(0.0), (dz @ bt).add_(0.0), (dz.T @ a).add_(0.0), db


# --------------------------------------------------------------------------------------- what a fixture holds
def classify(x: np.ndarray, kind: str) -> dict:
    """Counts over the exact values ``x`` (float64, every one exact in fp32) of an output of type ``kind``: ``up`` /
    ``down`` (rounded away from / toward zero, not a tie), ``tie`` (exactly halfway), ``subnormal`` (fp16: nonzero
    below 2^-14), ``zero`` (nonzero, rounds to zero) and ``inf`` (finite, rounds to inf)."""
    x = np.asarray(x, dtype=np.float64)
    bits = ed.round_fp16_bits(x) if kind == "fp16" else ed.round_bf16_bits(x)
    got = (bits.view(np.float16).astype(np.float64) if kind == "fp16"
           else (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64))
    fin = np.isfinite(got)
    ax, ag = np.abs(x), np.abs(got)
    p, emin = ed.FORMATS[kind]["p"], ed.FORMATS[kind]["emin"]
    e = np.maximum(np.frexp(ax)[1] - 1, emin)
    frac = ax / np.exp2((e - (p - 1)).astype(np.float64))
    frac = frac - np.floor(frac)
    tie = (ax > 0) & (frac == 0.5) & fin
    return {"up": int((fin & (ag > ax) & ~tie).sum()), "down": int((fin & (ag < ax) & ~tie).sum()),
            "tie": int(tie.sum()), "subnormal": int(((ax > 0) & (ax < 2.0 ** -14)).sum()) if kind == "fp16" else 0,
            "zero": int(((ax > 0) & (ag == 0)).sum()), "inf": int(((~fin) & np.isfinite(x)).sum())}
