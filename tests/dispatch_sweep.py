"""Operands, reference and shape lists for sweeping the DISPATCHED calls bit-exactly — TEST INFRASTRUCTURE.

The operands are those of ``exact_domain.py`` (``A[m,k] = i * 2^r_m``, ``Bt[n,k] = j * 2^c_n``, probe rows planting
the rounding targets), generated with torch so that they can be built on the GPU at any grid size (16384^3 included),
seeded per shape. Their true product is one rounding of the exact float64 product; :func:`reference_blocks` computes
it on the operands' device in float64, one block of rows at a time, applies the scales in float64, asserts that the
result is exact in fp32 and rounds it once to fp16 / bf16. Every value is an integer multiple of a power of two below
2^53, so the summation order of the float64 GEMM cannot matter. :func:`numpy_rows` recomputes a few rows of it in numpy
with exact_domain's rounding.

The shape lists are shared by test_dispatch_sweep_cpu.py (coverage of the dispatcher's choices, without a GPU) and
test_gpu_dispatch_sweep.py (the results):

* :func:`grid_shapes`: the tuned grid, every shape the benchmark times;
* :func:`offgrid_shapes`: a seeded sample per leg (small and odd M, ragged N and K, neighbours of grid values and of
  the points where the nearest grid value changes, and shapes whose borrowed entry ``usable()`` rejects), at most
  ``OFFGRID_MAX_FLOP`` each;
* :func:`tile_list_cases`: batched and grouped problems shaped like bmm and MoE layers.

The row-major B (NN) and bias + activation legs (NN_LEGS, EPI_LEGS) and :func:`grouped_bwd_cases` (the MoE expert
backward) are shared the same way by test_dispatch_sweep_late_cpu.py and test_gpu_dispatch_sweep_late.py. The bias legs'
reference keeps the exact domain: :func:`epi_bias` draws biases exact in the output type, :func:`epilogue_blocks` adds
them to the exact product in one fp32 addition, and gelu_tanh is held to epilogue_ref's allowance (:func:`gelu_ok`).
"""
from __future__ import annotations

import functools
import math
import random
import re
from pathlib import Path

import numpy as np

import exact_domain as ed

REPO = Path(__file__).resolve().parent.parent
GRID = (64, 128, 256, 512, 1024, 2048, 4096, 8192, 12288, 16384)
NUM_SMS = 132
OFFGRID_MAX_FLOP = 2 ** 36
E4M3_NNZ = 2000                 # nonzeros per random row of an e4m3 A (exact_domain.operands_e4m3)

# The legs of the sweep: operand kind, output kind, accumulator, scale granularity, the table's K divisor.
LEGS = {
    "fp16": dict(operand="fp16", out="fp16", acc="fp32", scales=None, k_div=1, k_align=8),
    "fp16acc16": dict(operand="fp16", out="fp16", acc="fp16", scales=None, k_div=1, k_align=8),
    "bf16": dict(operand="bf16", out="bf16", acc="fp32", scales=None, k_div=1, k_align=8),
    "e4m3_tensor_fp16": dict(operand="e4m3", out="fp16", acc="fp32", scales="tensor", k_div=2, k_align=16),
    "e4m3_rowwise_bf16": dict(operand="e4m3", out="bf16", acc="fp32", scales="rowwise", k_div=2, k_align=16),
    "e4m3_block_fp16": dict(operand="e4m3", out="fp16", acc="fp32", scales="block", k_div=2, k_align=16),
    "e4m3_block_bf16": dict(operand="e4m3", out="bf16", acc="fp32", scales="block", k_div=2, k_align=16),
}
# block scales: the grid with one output type, the off-grid sample with the other
LEG_LISTS = {leg: ("grid", "offgrid") for leg in LEGS}
LEG_LISTS["e4m3_block_fp16"] = ("grid",)
LEG_LISTS["e4m3_block_bf16"] = ("offgrid",)
TILE_LIST_VARIANTS = {"fp16": 0, "fp16acc16": 1, "bf16": 2}      # include/b200_batched.h's `variant`

# The legs of the row-major B (NN) and bias + activation libraries (test_gpu_dispatch_sweep_late.py), kept apart from
# LEGS so that the legs above, their lists and their seeds stay as they are. Same fields as LEGS.
NN_LEGS = {
    "nn_fp16": dict(operand="fp16", out="fp16", acc="fp32", scales=None, k_div=1, k_align=8),
    "nn_fp16acc16": dict(operand="fp16", out="fp16", acc="fp16", scales=None, k_div=1, k_align=8),
    "nn_bf16": dict(operand="bf16", out="bf16", acc="fp32", scales=None, k_div=1, k_align=8),
}
EPI_LEGS = {
    "epi_fp16": dict(operand="fp16", out="fp16", acc="fp32", scales=None, k_div=1, k_align=8),
    "epi_bf16": dict(operand="bf16", out="bf16", acc="fp32", scales=None, k_div=1, k_align=8),
    "epi_e4m3_tensor_fp16": dict(operand="e4m3", out="fp16", acc="fp32", scales="tensor", k_div=2, k_align=16),
    "epi_e4m3_rowwise_bf16": dict(operand="e4m3", out="bf16", acc="fp32", scales="rowwise", k_div=2, k_align=16),
}
LATE_LEGS = {**NN_LEGS, **EPI_LEGS}
LATE_LEG_LISTS = {"nn_fp16": ("grid", "offgrid"), "nn_bf16": ("grid",), "nn_fp16acc16": ("offgrid",),
                  "epi_fp16": ("grid",), "epi_e4m3_tensor_fp16": ("grid",), "epi_bf16": ("offgrid",),
                  "epi_e4m3_rowwise_bf16": ("offgrid",)}
EPI_VARIANTS = {"epi_fp16": 0, "epi_bf16": 2, "epi_e4m3_tensor_fp16": 3, "epi_e4m3_rowwise_bf16": 4}   # b200_epilogue.h
ACTIVATIONS = ("none", "relu", "gelu_tanh")

# The legs of the GEMM with 1 x 128 scales on both operands (the weight gradient of blockwise FP8 training,
# test_gpu_fp8_train_exact.py), kept apart like NN_LEGS: one output type on the grid, the other off it. Same fields.
TRAIN_LEGS = {
    "e4m3_1d1d_fp16": dict(operand="e4m3", out="fp16", acc="fp32", scales="block_1d1d", k_div=2, k_align=16),
    "e4m3_1d1d_bf16": dict(operand="e4m3", out="bf16", acc="fp32", scales="block_1d1d", k_div=2, k_align=16),
}
TRAIN_LEG_LISTS = {"e4m3_1d1d_fp16": ("grid",), "e4m3_1d1d_bf16": ("offgrid",)}
# weight-gradient samples dW [out_features, in_features] = dY^T X over T tokens: K = dual_ld_t(T), T off 128 and 16
DW_FEATURES = ((4096, 4096), (11008, 4096), (4096, 11008), (14336, 4096), (768, 3072), (1024, 4096))
DW_TOKENS = (300, 4104, 16400, 65550)


def leg_spec(leg: str) -> dict:
    """The fields of ``leg``, a key of LEGS, LATE_LEGS or TRAIN_LEGS."""
    return LEGS[leg] if leg in LEGS else LATE_LEGS[leg] if leg in LATE_LEGS else TRAIN_LEGS[leg]


def shape_seed(*dims) -> int:
    return int(sum((2 * i + 1) * 7919 ** i * d for i, d in enumerate(dims)) % (2 ** 31 - 1))


# ------------------------------------------------------------------------------------------------- the tuned table
@functools.lru_cache(maxsize=None)
def tuned_table() -> dict:
    """(M, N, K) -> ((cfg, group_m, splits) with fp32 accumulation, the same with fp16 accumulation), as
    hgemm_tuned_table.inc lists them (splits 0 read as 1, like the dispatcher)."""
    text = (REPO / "cuda_l2_b200" / "csrc" / "hgemm_tuned_table.inc").read_text()
    out = {}
    for row in re.findall(r"\{\s*(-?\d+(?:\s*,\s*-?\d+){8})\s*\}", text):
        m, n, k, c32, g32, s32, c16, g16, s16 = (int(x) for x in row.split(","))
        if m > 0:
            out[(m, n, k)] = ((c32, g32, s32 or 1), (c16, g16, s16 or 1))
    return out


def nearest_grid_value(d: int) -> int:
    """hgemm_dispatch.cuh's nearest_grid_value: the grid value closest to d on a log scale, the smaller one on a tie."""
    best, best_ratio = GRID[0], 1e30
    for g in GRID:
        r = d / g if d > g else g / d
        if r < best_ratio:
            best, best_ratio = g, r
    return best


def usable(cfg: dict, m: int, n: int) -> bool:
    """hgemm_dispatch.cuh's usable() in Python integers (no overflow at any size)."""
    return (-(-m // 128) >= cfg["cta_group"] * cfg["cluster_m"] * cfg["m_rep"]
            and -(-n // cfg["bn"]) >= cfg["cluster_n"])


def tier(configs: list, acc: str, m: int, n: int, k: int, k_div: int = 1) -> tuple[str, tuple | None]:
    """Which rule of dispatch::select decides (M, N, K): "exact" (the tuned entry), "nearest" (the entry of the nearest
    grid shape) or "heuristic", and the entry's (cfg, group_m, splits) for the first two."""
    col = 0 if acc == "fp32" else 1
    kk = max(k // k_div, 1)
    table = tuned_table()
    for name, key in (("exact", (m, n, kk)),
                      ("nearest", (nearest_grid_value(m), nearest_grid_value(n), nearest_grid_value(kk)))):
        e = table.get(key)
        if e is not None and 0 <= e[col][0] < len(configs) and usable(configs[e[col][0]], m, n):
            return name, e[col]
    return "heuristic", None


def choice(leg: str, m: int, n: int, k: int) -> tuple[int, int, int]:
    """(cfg, group_m, splits) the dispatched call of ``leg`` uses for (M, N, K)."""
    from cuda_l2_b200 import capi
    spec = leg_spec(leg)
    if spec["scales"] == "block_1d1d":
        return capi.fp8_blockwise_1d1d_select(m, n, k)
    if spec["scales"] == "block":
        return capi.fp8_blockwise_select(m, n, k)
    if spec["scales"]:
        return capi.fp8_select(m, n, k)
    return capi.select(spec["acc"], m, n, k)


def plan(leg: str, cfg: int, m: int, n: int, k: int, splits: int) -> tuple[str, int]:
    """(K-mode, sk_tiles) of the launcher's plan at 132 SMs (b200_hgemm_schedule_units; e4m3: the same k-blocks as a
    16-bit problem of K / 2)."""
    import ctypes

    from cuda_l2_b200 import capi
    lib = capi.hgemm_lib()
    nw, sk, mode = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    buf, contrib = (ctypes.c_int * 3)(), (ctypes.c_int * 1)()
    kk = max(k // leg_spec(leg)["k_div"], 1)
    st = lib.b200_hgemm_schedule_units(cfg, m, n, kk, splits, NUM_SMS, 0, buf, 0, ctypes.byref(nw), ctypes.byref(sk),
                                       ctypes.byref(mode), contrib)
    assert st >= 0, (leg, cfg, m, n, k, splits, st)
    return capi.KMODES[mode.value], sk.value


def l2_hint(cfg: dict, m: int, n: int, k: int, op_bytes: int) -> bool:
    """Whether host::launch gives the two operands different L2 eviction priorities (hgemm_host.cuh): one operand
    streamed (>= 40 MiB) while the other (<= 20 MiB) is re-read by at most four tile columns / rows."""
    a_bytes, b_bytes = m * k * op_bytes, n * k * op_bytes
    n_tiles, m_tiles = -(-n // cfg["bn"]), -(-m // (128 * cfg["m_rep"] * cfg["cta_group"]))
    keep, stream = 20 << 20, 40 << 20
    return (a_bytes >= stream and b_bytes <= keep and n_tiles <= 4) or (b_bytes >= stream and a_bytes <= keep and m_tiles <= 4)


def nn_sibling(configs: list, cid: int) -> int:
    """hgemm_configs.cuh's nn::sibling: the configuration itself if it has a row-major B kernel (BN % 64 == 0), else the
    BN = 64 one with the same CTA group, cluster_m and M_REP and the widest cluster_n up to its own."""
    c = configs[cid]
    if c["bn"] % 64 == 0:
        return cid
    cands = [d for d in configs if d["bn"] == 64 and d["cta_group"] == c["cta_group"] and d["cluster_m"] == c["cluster_m"]
             and d["m_rep"] == c["m_rep"] and d["cluster_n"] <= c["cluster_n"]]
    return max(cands, key=lambda d: d["cluster_n"])["id"]


def nn_choice(leg: str, m: int, n: int, k: int) -> tuple[int, int, int, int]:
    """hgemm_dispatch.cuh's select_rowmajor in Python: (cfg, group_m, splits) the dispatched NN call of ``leg`` runs,
    and the TN configuration it was mapped from. A mapped BN = 32 choice loses its split code."""
    from cuda_l2_b200 import capi
    tn, gm, sp = capi.select(NN_LEGS[leg]["acc"], m, n, k)
    cfg = nn_sibling(capi.configs(), tn)
    return cfg, gm, sp if cfg == tn else 1, tn


def epi_choice(leg: str, m: int, n: int, k: int) -> tuple[int, int, int]:
    """(cfg, group_m, splits) the dispatched bias + activation call of ``leg`` uses."""
    from cuda_l2_b200 import capi
    return capi.epilogue_select(EPI_VARIANTS[leg], m, n, k)


def epi_activation(leg: str, m: int, n: int, k: int) -> str:
    """The activation an epilogue leg runs at (M, N, K): a seeded draw per shape and leg."""
    return ACTIVATIONS[random.Random(shape_seed(m, n, k, len(leg), *map(ord, leg))).randrange(3)]


# ------------------------------------------------------------------------------------------------- shape lists
def grid_shapes() -> list[tuple[int, int, int]]:
    from cuda_l2_b200 import farm
    return farm.grid_shapes()


def _flip_points() -> list[int]:
    """Where nearest_grid_value changes: the geometric means of neighbouring grid values."""
    return [int(math.sqrt(a * b)) for a, b in zip(GRID, GRID[1:])]


def _round_up(x: int, a: int) -> int:
    return max(a, -(-x // a) * a)


@functools.lru_cache(maxsize=None)
def offgrid_shapes(leg: str) -> list[tuple[int, int, int]]:
    """A seeded off-grid sample for ``leg`` (a few hundred shapes): M = 1..16, odd M, ragged N (multiples of 8) and K
    (multiples of the leg's 16-byte K rule), neighbours g +- 8 / g +- 64 of grid values and of the points where the
    nearest grid value flips, and shapes that the heuristic decides because usable() rejects the borrowed entry. Every
    shape does at most OFFGRID_MAX_FLOP. ``leg``: a key of LEGS or of LATE_LEGS (seeded by its name either way)."""
    spec = leg_spec(leg)
    ka = spec["k_align"]
    rng = random.Random(shape_seed(len(leg), *map(ord, leg)))
    grid = set(grid_shapes())

    def dim(lo=1, hi=16384):
        return int(round(math.exp(rng.uniform(math.log(lo), math.log(hi)))))

    def fit(m, n, k):
        n, k = _round_up(n, 8), _round_up(max(k, 16), ka)      # K >= 16: distinct probe positions
        while 2 * m * n * k > OFFGRID_MAX_FLOP:          # shrink the largest of N and K, then M
            if max(n, k) > 256:
                if n >= k:
                    n = _round_up(n // 2, 8)
                else:
                    k = _round_up(max(k // 2, 16), ka)
            else:
                m = max(1, m // 2)
        return (m, n, k)

    out = []
    for m in range(1, 17):                                            # tiny M
        out.append(fit(m, dim(8, 16384), dim(ka, 16384)))
    for _ in range(40):                                               # odd M, ragged N and K
        out.append(fit(dim(17, 16384) | 1, 8 * dim(1, 2048) + 8 * (rng.random() < 0.5), ka * dim(1, 1024)))
    near = [g + d for g in GRID for d in (-64, -8, 8, 64) if g + d > 0] + \
           [p + d for p in _flip_points() for d in (-8, 0, 8)]
    for _ in range(120):                                              # neighbours of grid values and flip points
        m, n, k = (rng.choice(near) if rng.random() < 0.7 else rng.choice(GRID) for _ in range(3))
        out.append(fit(m, n, k))
    for _ in range(60):                                               # anywhere
        out.append(fit(dim(), dim(8), dim(ka)))
    # shapes where the borrowed entry is not usable: draw until enough of them are decided by the heuristic
    from cuda_l2_b200 import capi
    configs = capi.configs()
    heur = 0
    while heur < 40:
        s = fit(dim(1, 4096), dim(8, 16384), dim(ka, 16384))
        if tier(configs, spec["acc"], *s, k_div=spec["k_div"])[0] == "heuristic":
            out.append(s)
            heur += 1
    if spec["k_div"] == 2:
        # the e4m3 table lookup is at K / 2, so grid K never reaches the entries at K = 12288 and 16384: their
        # configurations, where no shorter entry names them, at twice their K
        table = tuned_table()
        short = {e[0][0] for (m, n, k), e in table.items() if k <= 8192}
        for (m, n, k), e in sorted(table.items()):
            if k > 8192 and e[0][0] not in short and 4 * m * n * k <= OFFGRID_MAX_FLOP:
                out.append((m, n, 2 * k))
                short.add(e[0][0])
    seen, uniq = set(), []
    for s in out:
        if s not in seen and s not in grid:
            seen.add(s)
            uniq.append(s)
    return uniq


def leg_shapes(leg: str) -> list[tuple[int, int, int]]:
    shapes = []
    lists = LEG_LISTS if leg in LEG_LISTS else LATE_LEG_LISTS if leg in LATE_LEG_LISTS else TRAIN_LEG_LISTS
    for name in lists[leg]:
        shapes += grid_shapes() if name == "grid" else offgrid_shapes(leg)
    return shapes


def dw_shapes() -> list[tuple[int, int, int]]:
    """(M, N, K) of the weight-gradient samples: M = out_features, N = in_features, K = dual_ld_t(T), the token count
    padded to 16 as the dual quantisers pad the transposed copies (the last 128-token block partial)."""
    from cuda_l2_b200 import capi
    return [(m, n, capi.dual_ld_t(t)) for m, n in DW_FEATURES for t in DW_TOKENS]


@functools.lru_cache(maxsize=None)
def tile_list_cases() -> list[dict]:
    """Batched problems (bmm-like, dense or with row counts including 0, full and ragged) and grouped problems (MoE
    prefill: G up to 256 experts, skewed group sizes with empty groups, the last group ending before T or at it), a
    few hundred to tens of thousands of rows each. Dicts: kind "batched" (b, m, n, k, counts or None) or "grouped"
    (g, t, n, k, offs)."""
    rng = random.Random(20261016)
    cases = []
    for i in range(24):
        b = rng.choice((1, 2, 3, 4, 8, 16, 32, 64))
        m = rng.choice((64, 100, 128, 200, 256, 384, 500, 1000, 1024, 2048))
        m = min(m, max(16, 40000 // b))
        n = rng.choice((64, 128, 136, 256, 512, 1024, 1536, 4096))
        k = rng.choice((64, 128, 256, 512, 1024, 2048, 4096))
        while 2 * b * m * n * k > 2 ** 37:
            k = max(64, k // 2) if k > 64 else k
            n = max(64, n // 2)
        counts = None
        if i % 2:
            counts = [rng.choice((0, m, rng.randrange(0, m + 1), rng.randrange(1, 17), m + 5)) for _ in range(b)]
        cases.append(dict(kind="batched", b=b, m=m, n=n, k=k, counts=counts))
    for i in range(24):
        g = rng.choice((1, 2, 4, 8, 16, 32, 64, 128, 256))
        t = rng.choice((300, 1000, 2048, 4000, 8192, 16000, 30000))
        n = rng.choice((64, 128, 256, 512, 1024, 2048, 2816))
        k = rng.choice((128, 256, 512, 1024, 2048, 4096))
        while 2 * t * n * k > 2 ** 37:
            n = max(64, n // 2)
            k = max(64, k // 2)
        # skewed sizes: a Zipf-like weight per group, some groups empty
        w = [0.0 if rng.random() < 0.2 else 1.0 / (1 + rng.randrange(g)) ** 1.2 for _ in range(g)]
        if not any(w):
            w[0] = 1.0
        used = t if i % 3 else t - rng.randrange(1, t // 4 + 2)      # one in three ends before T
        sizes = [int(used * x / sum(w)) for x in w]
        sizes[max(range(g), key=lambda j: w[j])] += used - sum(sizes)
        offs = list(np.cumsum(sizes).astype(int))
        cases.append(dict(kind="grouped", g=g, t=t, n=n, k=k, offs=[int(x) for x in offs]))
    return cases


GROUPED_BWD_VARIANTS = {"fp16": 0, "bf16": 2}       # csrc/b200_grouped_bwd.h's `variant`
GROUPED_BWD_OUT_MAX = 2 ** 28                        # elements of the weight gradient, G * M * N


@functools.lru_cache(maxsize=None)
def grouped_bwd_cases() -> list[dict]:
    """MoE-shaped backward problems of an expert layer x [T, d_in] -> y [T, d_out] with G experts: the input gradient
    dX [T, d_in] = dY [T, d_out] @ W[g] (the grouped NN call, N = d_in, K = d_out) and the weight gradient
    dW[g] = dY[s:e]^T X[s:e] [d_out, d_in] (the K-grouped call, M = d_out, N = d_in). Hidden sizes 1024..7168 and
    expert widths 1408 / 2816 in either role, G in {1, 8, 64, 256}, T up to 64k, at most 2^37 FLOP (tile_list_cases'
    cap) and GROUPED_BWD_OUT_MAX weight-gradient elements. Skewed group sizes with empty groups, one-row groups, starts
    off every multiple of 8, the last end before T in one case of three; then T == 0 and an all-empty histogram.
    Dicts: g, t, d_in, d_out, offs."""
    rng = random.Random(20261017)
    hidden, expert = (1024, 2048, 2560, 4096, 5120, 7168), (1408, 2816)
    cases = []
    for i in range(28):
        g = (1, 8, 64, 256)[i % 4]
        t = rng.choice((256, 1000, 2048, 4000, 8192, 16000, 30000, 65536))
        h, e = rng.choice(hidden), rng.choice(expert)
        d_in, d_out = (h, e) if i % 2 else (e, h)
        if i == 0:
            t, d_in, d_out = 65536, 1024, 1024                       # the longest T, at the FLOP cap
        while 2 * t * d_in * d_out > 2 ** 37 or g * d_in * d_out > GROUPED_BWD_OUT_MAX:
            if t > 2048 and 2 * t * d_in * d_out > 2 ** 37:
                t //= 2
            elif d_in >= d_out:
                d_in = _round_up(d_in // 2, 8)
            else:
                d_out = _round_up(d_out // 2, 8)
        w = [0.0 if rng.random() < 0.2 else 1.0 / (1 + rng.randrange(g)) ** 1.2 for _ in range(g)]
        if not any(w):
            w[0] = 1.0
        used = t if i % 3 else t - rng.randrange(1, t // 4 + 2)       # one in three ends before T
        sizes = [int(used * x / sum(w)) for x in w]
        big = max(range(g), key=lambda j: w[j])
        sizes[big] += used - sum(sizes)
        j = (big + 1) % g
        if g > 1 and sizes[big] + sizes[j] >= 2:                      # a one-row group, the total kept
            sizes[big] += sizes[j] - 1
            sizes[j] = 1
        offs = [int(x) for x in np.cumsum(sizes)]
        cases.append(dict(g=g, t=t, d_in=d_in, d_out=d_out, offs=offs))
    cases.append(dict(g=8, t=0, d_in=1408, d_out=1024, offs=[0] * 8))           # T == 0 (weight gradient only)
    cases.append(dict(g=64, t=1000, d_in=1024, d_out=1408, offs=[0] * 64))      # every group empty
    return cases


# ------------------------------------------------------------------------------------------------- operands (torch)
class TorchOperands:
    """A [M,K] and Bt [N,K] in the operand dtype (every value exact), the exponents and the probe rows."""

    def __init__(self, a, bt, row_exp, col_exp, probe_rows):
        self.a, self.bt, self.row_exp, self.col_exp, self.probe_rows = a, bt, row_exp, col_exp, probe_rows


def _cycle(torch, values, idx):
    return torch.tensor(values, dtype=torch.int64, device=idx.device)[idx % len(values)]


def _digits_table(torch, kind: str, targets, device):
    return torch.tensor([ed._digits(kind, t) for t in targets], dtype=torch.int32, device=device)


def _strided_keep(torch, m: int, k: int, nnz: int, gen, device):
    """[M,K] bool: at most ``nnz`` kept positions per row, every ``ceil(K / nnz)``-th from a random offset, so that every
    k-block of 64 keeps some."""
    s = -(-k // nnz)
    off = torch.randint(0, s, (m, 1), generator=gen, device=device)
    return (torch.arange(k, device=device)[None, :] + off) % s == 0


def operands16(torch, m: int, n: int, k: int, kind: str, seed: int, acc16: bool = False, device="cuda"):
    """exact_domain.operands16 on ``device``: the same exponents, probe rows, targets, digits and bounds; the random
    integers come from a torch generator seeded with ``seed``, and the fp16-accumulation rows keep at most 2047
    nonzeros spread over every k-block. Each bound is asserted from the integers."""
    assert k >= 16 and (kind == "fp16" or not acc16)
    dtype = torch.float16 if kind == "fp16" else torch.bfloat16
    gen = torch.Generator(device=device).manual_seed(seed)
    rows, cols = torch.arange(m, device=device), torch.arange(n, device=device)
    if acc16:
        r, c = _cycle(torch, ed.ROW_EXP_ACC16, rows * 3), _cycle(torch, ed.COL_EXP_ACC16, cols)
        ia = torch.randint(-1, 2, (m, k), generator=gen, device=device, dtype=torch.int16)
        ia *= _strided_keep(torch, m, k, ed.FP16_ACC_SUM_BOUND - 1, gen, device)
        jb = torch.randint(-1, 2, (n, k), generator=gen, device=device, dtype=torch.int16)
        # sum_k |i j| <= nonzeros of the row of A (|j| <= 1)
        assert int((ia != 0).sum(1).max()) < ed.FP16_ACC_SUM_BOUND and int(jb.abs().max()) <= 1
        probe = rows[:0]
    else:
        targets = ed.rounding_targets(kind)
        nt = len(targets)
        probe = rows[rows % ed.PROBE_EVERY == 2]
        nrow = len(ed.ROW_EXP[kind])
        r = _cycle(torch, ed.ROW_EXP[kind], rows * 3)
        r[probe] = _cycle(torch, ed.ROW_EXP[kind], torch.arange(len(probe), device=device))
        sign = torch.where((torch.arange(len(probe), device=device) // nrow) % 2 == 0, 1, -1).to(torch.int32)
        c = _cycle(torch, ed.COL_EXP[kind], cols // nt)
        pos = list(ed.probe_positions(k))
        lim_b = 63 if kind == "fp16" else 31
        lim_a = int(min(2047 if kind == "fp16" else 255, (ed.EXACT_SUM_BOUND - 1) // (k * lim_b)))
        ia = torch.randint(-lim_a, lim_a + 1, (m, k), generator=gen, device=device, dtype=torch.int32)  # bf16 weight 2^16
        jb = torch.randint(-lim_b, lim_b + 1, (n, k), generator=gen, device=device, dtype=torch.int16)
        ia[:, pos] = 0
        # random rows: sum_k |i j| <= K lim_a lim_b (the digits at the probe positions meet zeros in them)
        assert k * lim_a * lim_b < ed.EXACT_SUM_BOUND
        assert int(ia.abs().max()) <= lim_a and int(jb.abs().max()) <= lim_b
        ia[probe] = 0
        for w, p in zip(ed._weights(kind), pos):
            ia[probe, p] = (w * sign).to(torch.int32)
        jb[:, pos] = _digits_table(torch, kind, targets, device)[cols % nt].to(torch.int16)
        # probe rows: three nonzeros, at the probe positions; their sum is the column's target, below 2^24
        if len(probe):
            assert int((ia[probe] != 0).sum(1).max()) == 3
        assert max(targets) < ed.EXACT_SUM_BOUND
    a = ia.to(torch.float32).mul_(torch.exp2(r.to(torch.float32))[:, None]).to(dtype)
    bt = jb.to(torch.float32).mul_(torch.exp2(c.to(torch.float32))[:, None]).to(dtype)
    return TorchOperands(a, bt, r, c, probe)


def operands_e4m3(torch, m: int, n: int, k: int, seed: int, device="cuda"):
    """exact_domain.operands_e4m3 on ``device``: at most E4M3_NNZ nonzeros +-1 per random row of A, spread over every
    k-block, probe rows planting E4M3_TARGETS; sum_k |i j| <= 2047, asserted from the integers."""
    gen = torch.Generator(device=device).manual_seed(seed)
    rows, cols = torch.arange(m, device=device), torch.arange(n, device=device)
    probe = rows[rows % ed.PROBE_EVERY == 2]
    pos = list(ed.probe_positions(k))
    ia = torch.randint(-1, 2, (m, k), generator=gen, device=device, dtype=torch.int16)
    ia *= _strided_keep(torch, m, k, E4M3_NNZ, gen, device)
    ia[:, pos] = 0
    assert int((ia != 0).sum(1).max()) <= E4M3_NNZ
    ia[probe] = 0
    sign = torch.where(torch.arange(len(probe), device=device) % 2 == 0, 1, -1).to(torch.int16)
    for w, p in zip(ed._weights("e4m3"), pos):
        ia[probe, p] = (w * sign).to(torch.int16)
    jb = torch.randint(-1, 2, (n, k), generator=gen, device=device, dtype=torch.int16)
    nt = len(ed.E4M3_TARGETS)
    jb[:, pos] = _digits_table(torch, "e4m3", ed.E4M3_TARGETS, device)[cols % nt].to(torch.int16)
    assert max(ed.E4M3_TARGETS) <= ed.E4M3_SUM_BOUND and E4M3_NNZ <= ed.E4M3_SUM_BOUND
    e4 = torch.float8_e4m3fn
    return TorchOperands(ia.to(torch.float32).to(e4), jb.to(torch.float32).to(e4), None, None, probe)


def e4m3_scales(torch, granularity: str, m: int, n: int, k: int, out: str, seed: int, device="cuda"):
    """(scale_a, scale_b) fp32 tensors as the kernel reads them (block: scale_a M-major with ld_a = M rounded up to 4;
    block_1d1d: scale_b N-major the same way), and their float64 values as numpy arrays (tensor: scalars; rowwise: [M],
    [N]; block: [M, nkb], [ceil(N/128), nkb]; block_1d1d: [M, nkb], [N, nkb])."""
    if granularity == "tensor":
        pairs = ed.e4m3_tensor_scales(out)
        sa, sb = pairs[seed % len(pairs)]
        dev = [torch.tensor([v], dtype=torch.float32, device=device) for v in (sa, sb)]
        return dev[0], dev[1], np.float64(np.float32(sa)), np.float64(np.float32(sb))
    if granularity == "rowwise":
        sa, sb = ed.e4m3_rowwise_scales(m, n, out)
        return (torch.from_numpy(sa).reshape(m, 1).to(device), torch.from_numpy(sb).reshape(1, n).to(device),
                sa.astype(np.float64), sb.astype(np.float64))
    if granularity == "block_1d1d":
        sa, sb = ed.e4m3_block_1d1d_scales(m, n, k, out)
        return (m_major(torch, sa, device), m_major(torch, sb, device), sa.astype(np.float64),
                sb.astype(np.float64))
    sa, sb = ed.e4m3_block_scales(m, n, k, out)
    return m_major(torch, sa, device), torch.from_numpy(sb).to(device), sa.astype(np.float64), sb.astype(np.float64)


def m_major(torch, s: np.ndarray, device="cuda", ld: int | None = None):
    """The (1, ld)-strided view [R, nkb] of scales ``s`` [R, nkb] that the block-scaled kernels read in place, ld = ``ld``
    or R rounded up to 4, NaN in the padding rows."""
    r, nkb = s.shape
    ld = ld or -(-r // 4) * 4
    buf = torch.full((nkb, ld), float("nan"), dtype=torch.float32, device=device)
    buf[:, :r] = torch.from_numpy(np.ascontiguousarray(s, dtype=np.float32)).t().to(device)
    return buf[:, :r].t()


# ------------------------------------------------------------------------------------------------- the reference
def round_to(torch, y, out: str):
    """float64 values -> int16 bits of fp16 / bf16: exact in fp32 (asserted; per-tensor e4m3 scales may take a value
    past the largest fp32, which goes to inf there as in the kernel's fp32 product), then one rounding."""
    y32 = y.to(torch.float32)
    fin = torch.isfinite(y32)
    assert torch.equal(y32[fin].to(torch.float64), y[fin]), "not exact in fp32"
    return y32.to(torch.float16 if out == "fp16" else torch.bfloat16).view(torch.int16)


def _block_factors(s, k: int):
    """Per-element factors [*, K] of scales ``s`` [*, nkb], one per 128 k."""
    return s.repeat_interleave(128, dim=1)[:, :k]


def reference_blocks(torch, ops, out: str, scales=None, granularity=None, rows_per_block=None):
    """Yield (lo, hi, bits) for row blocks of the true output: int16 bits [hi - lo, N]. ``scales``: the float64 numpy
    values of e4m3_scales for ``granularity``. The product is a float64 GEMM on the operands' device."""
    for lo, hi, y in exact_blocks(torch, ops, scales, granularity, rows_per_block):
        yield lo, hi, round_to(torch, y, out)


def exact_blocks(torch, ops, scales=None, granularity=None, rows_per_block=None):
    """Yield (lo, hi, y) for row blocks of the exact scaled product, float64 [hi - lo, N] (reference_blocks before its
    one rounding)."""
    a, bt = ops.a, ops.bt
    (m, k), n = a.shape, bt.shape[0]
    dev = a.device
    b64 = bt.to(torch.float64)
    sa = sb = None
    if granularity in ("block", "block_1d1d"):
        sa = torch.from_numpy(scales[0]).to(dev)
        sb = torch.from_numpy(scales[1]).to(dev)
        if granularity == "block":
            b64 *= _block_factors(sb, k).repeat_interleave(128, dim=0)[:n]
        else:                                                   # one scale per row of Bt and 128 k
            for n0 in range(0, n, 4096):
                b64[n0:n0 + 4096] *= _block_factors(sb[n0:n0 + 4096], k)
    elif granularity == "rowwise":
        sa, sb = torch.from_numpy(scales[0]).to(dev), torch.from_numpy(scales[1]).to(dev)
    rb = rows_per_block or max(16, (1 << 26) // max(n, k))
    for lo in range(0, m, rb):
        hi = min(m, lo + rb)
        a64 = a[lo:hi].to(torch.float64)
        if granularity in ("block", "block_1d1d"):
            a64 *= _block_factors(sa[lo:hi], k)
        y = a64 @ b64.T
        del a64
        if granularity == "tensor":
            y *= float(np.float32(np.float32(scales[0]) * np.float32(scales[1])))
        elif granularity == "rowwise":
            y *= sb[None, :]
            y *= sa[lo:hi, None]
        yield lo, hi, y


def numpy_rows(torch, ops, rows, cols, out: str, scales=None, granularity=None) -> np.ndarray:
    """uint16 bits of the true output at ``rows`` x ``cols``, recomputed in numpy float64 from the operands and rounded
    by exact_domain (round_fp16_bits / round_bf16_bits)."""
    k = ops.a.shape[1]
    ri, ci = torch.as_tensor(rows, device=ops.a.device), torch.as_tensor(cols, device=ops.a.device)
    a = ops.a[ri].to(torch.float32).cpu().numpy().astype(np.float64)
    b = ops.bt[ci].to(torch.float32).cpu().numpy().astype(np.float64)
    rows, cols = np.asarray(rows), np.asarray(cols)
    if granularity == "block":
        sa, sb = scales
        a = a * np.repeat(sa[rows], 128, axis=1)[:, :k]
        b = b * np.repeat(sb[cols // 128], 128, axis=1)[:, :k]
    elif granularity == "block_1d1d":
        sa, sb = scales
        a = a * np.repeat(sa[rows], 128, axis=1)[:, :k]
        b = b * np.repeat(sb[cols], 128, axis=1)[:, :k]
    y = a @ b.T
    if granularity == "tensor":
        y = y * np.float64(np.float32(np.float32(scales[0]) * np.float32(scales[1])))
    elif granularity == "rowwise":
        y = y * scales[1][cols][None, :] * scales[0][rows][:, None]
    with np.errstate(over="ignore"):
        if out == "fp16":
            return ed.round_fp16_bits(y)
        big = np.abs(y) > np.finfo(np.float32).max          # past fp32: inf, as in round_to
        return ed.round_bf16_bits(np.where(big, np.copysign(np.inf, y), y))


def sample_rows(m: int, probe_rows, seed: int) -> list[int]:
    """About eight rows: three probe rows, four seeded random rows, the last row."""
    rng = random.Random(seed)
    probe = [int(x) for x in probe_rows[:: max(1, len(probe_rows) // 3)][:3]] if len(probe_rows) else []
    rows = set(probe) | {rng.randrange(m) for _ in range(4)} | {m - 1}
    return sorted(rows)


def sample_cols(n: int, seed: int, limit: int = 1024) -> list[int]:
    """Every column when N <= limit, else a seeded ``limit`` of them with the first and the last."""
    if n <= limit:
        return list(range(n))
    rng = random.Random(seed)
    return sorted(set(rng.sample(range(n), limit - 2)) | {0, n - 1})


# ------------------------------------------------------------------------------------------------- bias + activation
BIAS_NEG_ZERO, BIAS_POS_ZERO = 0.25, 0.05     # fractions of the columns whose bias is -0.0 / +0.0
GELU_ABS = 2.0 ** -22                          # epilogue_ref.GELU_ABS
_OUT_DTYPE = {"fp16": "float16", "bf16": "bfloat16"}


def _median(values) -> int:
    return sorted(values)[len(values) // 2]


def _sum_log2(spec: dict, k: int) -> float:
    """log2 of the spread of a random row's sum_k i j (operands16 / operands_e4m3): sqrt(K) lim_a lim_b / 3 for the
    uniform 16-bit integers, sqrt(4/9 nonzeros) for the e4m3 +-1 / 0 ones."""
    if spec["operand"] == "e4m3":
        return 0.5 * math.log2(4 / 9 * min(k, E4M3_NNZ))
    lim_b = 63 if spec["operand"] == "fp16" else 31
    lim_a = min(2047 if spec["operand"] == "fp16" else 255, (ed.EXACT_SUM_BOUND - 1) // (k * lim_b))
    return math.log2(math.sqrt(k) * lim_a * lim_b / 3)


def epi_bias(torch, leg: str, ops, scales, n: int, k: int, seed: int, device="cuda"):
    """The bias [N] of an epilogue leg, in the output type, every value exact there: a quarter of the columns -0.0 (z is
    the product itself, so the probe rows' planted rounding targets still round), a few +0.0, the rest +-q 2^e with a
    significand q of the output's width and an exponent within a few binades of what the column's product reaches at a
    typical row (the column exponent of operands16, or the e4m3 scales, at the median row exponent), so that
    z = s + bias takes the bias's sign on the rows of smaller exponent and the product's on the others."""
    spec = EPI_LEGS[leg]
    out = spec["out"]
    p, emin, emax = (11, -24, 15) if out == "fp16" else (8, -133, 127)
    if spec["operand"] != "e4m3":
        col = ops.col_exp.to(torch.float64) + _median(ed.ROW_EXP[spec["operand"]])
    elif spec["scales"] == "tensor":
        col = torch.full((n,), math.log2(float(np.float32(scales[0]) * np.float32(scales[1]))), dtype=torch.float64,
                         device=device)
    else:
        q = _median(ed.E4M3_Q[out])
        col = torch.log2(torch.from_numpy(scales[1]).to(device)) + math.log2(q) + _median(ed.E4M3_ROW_EXP)
    gen = torch.Generator(device=device).manual_seed(seed)
    u = torch.rand((n,), generator=gen, device=device, dtype=torch.float64)
    q = torch.randint(1 << (p - 1), 1 << p, (n,), generator=gen, device=device).to(torch.float64)
    sign = torch.randint(0, 2, (n,), generator=gen, device=device).to(torch.float64) * 2 - 1
    jitter = torch.randint(-3, 3, (n,), generator=gen, device=device).to(torch.float64)
    e = (torch.round(col + _sum_log2(spec, k)) + jitter - (p - 1)).clamp(emin, emax - (p - 1))
    val = sign * q * torch.exp2(e)
    val[u < BIAS_NEG_ZERO + BIAS_POS_ZERO] = 0.0
    val[u < BIAS_NEG_ZERO] = -0.0
    bias = val.to(getattr(torch, _OUT_DTYPE[out]))
    assert torch.equal(bias.to(torch.float64), val), "bias not exact in the output type"
    return bias


def epilogue_blocks(torch, ops, bias, scales=None, granularity=None, rows_per_block=None):
    """Yield (lo, hi, z) for row blocks of the fused call's pre-activation, fp32 [hi - lo, N]: the exact scaled product s
    (exact_blocks; asserted exact in fp32, per-tensor e4m3 scales may take it past the largest fp32, to inf as in the
    kernel) plus the bias, one IEEE fp32 addition on the operands' device."""
    b32 = bias.to(torch.float32)
    for lo, hi, y in exact_blocks(torch, ops, scales, granularity, rows_per_block):
        s = y.to(torch.float32)
        fin = torch.isfinite(s)
        assert torch.equal(s[fin].to(torch.float64), y[fin]), "not exact in fp32"
        del y, fin
        yield lo, hi, s.add_(b32[None, :])


def activated_bits(torch, z, activation: str, out: str):
    """int16 bits of none / relu of fp32 z, rounded once to ``out``: relu is z > 0 ? z : +0.0."""
    if activation == "relu":
        z = torch.where(z > 0, z, torch.zeros_like(z))
    else:
        assert activation == "none", activation
    return z.to(getattr(torch, _OUT_DTYPE[out])).view(torch.int16)


def _ulp_at(torch, x, out: str):
    """epilogue_ref.ulp_at on the device."""
    p, emin = (11, -14) if out == "fp16" else (8, -126)
    ax = x.abs()
    e = torch.where(ax > 0, torch.clamp(torch.frexp(ax).exponent.to(torch.float64) - 1, min=emin),
                    torch.full_like(ax, emin))
    return torch.exp2(e - (p - 1))


def gelu_ok(torch, got_bits, z, out: str):
    """Where a gelu_tanh output is what epilogue_ref.gelu_excess allows (within one unit in the last place of the
    float64 tanh form, plus |z| GELU_ABS), on the device; an output equal to the float64 form rounded (infinities) or
    NaN where it is NaN passes too. Bool [like z]."""
    z64 = z.to(torch.float64)
    want = 0.5 * z64 * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (z64 + 0.044715 * z64 ** 3)))
    dt = getattr(torch, _OUT_DTYPE[out])
    got = got_bits.view(dt).to(torch.float64)
    excess = (got - want).abs() - (_ulp_at(torch, want, out) + z64.abs() * GELU_ABS)
    return (excess <= 0) | (got == want.to(torch.float32).to(dt).to(torch.float64)) | (got.isnan() & want.isnan())


def epilogue_numpy_rows(torch, ops, rows, cols, bias, activation: str, out: str, scales=None, granularity=None):
    """epilogue_ref on ``rows`` x ``cols``, in numpy from the operands: (fp32 z, output bits or None for gelu_tanh)."""
    import epilogue_ref
    ri, ci = torch.as_tensor(rows, device=ops.a.device), torch.as_tensor(cols, device=ops.a.device)
    a = ops.a[ri].to(torch.float32).cpu().numpy().astype(np.float64)
    b = ops.bt[ci].to(torch.float32).cpu().numpy().astype(np.float64)
    b32 = bias[ci].to(torch.float32).cpu().numpy()
    sa = sb = None
    if granularity == "tensor":
        sa, sb = np.float32(scales[0]), np.float32(scales[1])
    elif granularity == "rowwise":
        sa, sb = scales[0][np.asarray(rows)], scales[1][np.asarray(cols)]
    rowwise = granularity == "rowwise"
    with np.errstate(over="ignore", invalid="ignore"):
        z = epilogue_ref.pre_activation(a, b, b32, sa, sb, rowwise)
        bits = None if activation == "gelu_tanh" else epilogue_ref.reference(a, b, b32, activation, out, sa, sb, rowwise)
    return z, bits


# ------------------------------------------------------------------------------------------------- grouped backward
def grouped_nn_operands(torch, t: int, g: int, n: int, k: int, kind: str, seed: int, device="cuda"):
    """a [T, K] and b [G, K, N] row-major of the grouped NN call: operands16(T, G N, K), b[g] = bt[g]^T."""
    ops = operands16(torch, t, g * n, k, kind, seed, device=device)
    return ops.a, ops.bt.view(g, n, k).transpose(1, 2).contiguous()


def wgrad_operands(torch, t: int, m: int, n: int, kind: str, seed: int, device="cuda"):
    """a [T, M] and b [T, N] of the K-grouped call: operands16(M, N, T) transposed, so that each row and column exponent
    is constant along the reduction axis T. A group's sum over rows [s, e) of T is then a subset of an exactly summable
    row sum, and exact too. T == 0: empty operands."""
    dtype = torch.float16 if kind == "fp16" else torch.bfloat16
    if t == 0:
        return torch.empty((0, m), dtype=dtype, device=device), torch.empty((0, n), dtype=dtype, device=device)
    ops = operands16(torch, m, n, t, kind, seed, device=device)
    return ops.a.t().contiguous(), ops.bt.t().contiguous()


def grouped_nn_reference(torch, a, b, s: int, e: int, g: int, out: str):
    """int16 bits of group g's rows [s, e) of the grouped NN product, rounded once."""
    return round_to(torch, a[s:e].to(torch.float64) @ b[g].to(torch.float64), out)


def wgrad_reference(torch, a, b, s: int, e: int, out: str):
    """int16 bits of one group's weight gradient a[s:e]^T b[s:e] [M, N], rounded once (+0.0 for an empty group). A sum
    of zero products is +0.0, as in an accumulator that starts at +0.0: a one-row group's float64 product of 0 and a
    negative value is -0.0, so the zeros are normalised (y + 0.0)."""
    return round_to(torch, (a[s:e].to(torch.float64).T @ b[s:e].to(torch.float64)).add_(0.0), out)
