"""Steady-state schedules, every K-mode and the full output range of the 16-bit and e4m3 kernels on the H100, bit-exact
against a plain reference on the exactly summable domain of ``exact_domain.py``.

* Steady state: every configuration of bf16, e4m3 (per-tensor and rowwise scales, fp16 and bf16 out) and block-scaled
  e4m3 (its eligible configurations) on a ragged problem, with ``max_ctas`` limiting the launch to one worker, which runs
  every tile, the ring wraps, and (block scales) each unit spans more than 32 k-blocks.
* K-modes: workspace split-K (factors 4, 16 and 64, as granted), cluster split-K -2/-4/-8 and stream-K 100/101 on every
  configuration that carries the kernel, for fp16 (fp32 and fp16 accumulation) and bf16. The e4m3 ones are the K_MODES
  of test_gpu_fp8.py.
* Output rounding: exact ties rounding both ways after dropping 1 to 13 bits, fp16 subnormal results, 65504 / just
  under 65520 / exactly 65520 (to inf) and their negatives, bf16 values past the largest finite bf16; every rounding
  site (TMA-store epilogue, split-K and cluster reductions, the stream-K owner) sees them.
* Non-finite operands in every K-mode: a NaN in A in a late split's k-range makes its row NaN; Infs in Bt give +-inf
  against products of one sign and NaN against mixed signs or a zero; every other element stays exact.
  float8_e4m3fn has no Inf, so e4m3 takes the NaN case only.

Each case's schedule is checked without a GPU by test_exact_range_cpu.py.
"""
import functools

import numpy as np
import pytest
import torch

import exact_domain as ed
from cuda_l2_b200 import capi
from fp8_block_ref import fp8gemm_f32acc_block
from fp8_rowwise_ref import fp8gemm_f32acc_rowwise
from oracle import fp8 as fp8_oracle

pytestmark = pytest.mark.gpu

E4 = torch.float8_e4m3fn
BLOCK_ELIGIBLE = (1, 2, 4, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 22, 23, 30)
VARIANTS16 = ("fp16", "fp16acc16", "bf16")      # fp16 with fp32 / fp16 accumulation, bf16 (fp32 accumulation)

# Steady state: (M, N) off every tile multiple; K gives 16 k-blocks per tile (34 with block scales, > 32), so every
# worker's k-blocks wrap the ring (at most 9 stages) many times over.
STEADY_MN = (600, 392)
STEADY_K = {"16": 1000, "e4m3": 2000, "block": 4288}

# K-modes, K of the 16-bit problem (e4m3: twice that, the same k-blocks): split-K shapes have few tiles, the stream-K
# shape leaves a partial wave at 132 SMs.
SPLIT_SHAPE, STREAMK_SHAPE = (520, 392, 2048), (1160, 1000, 2048)
SPLIT_CONFIGS, STREAMK_CONFIGS = (0, 1, 2, 5), (0, 1, 2, 3, 4, 5, 6)
KMODE_CASES = (
    [(cfg, *SPLIT_SHAPE, sp, "split-k") for cfg in SPLIT_CONFIGS for sp in (4, 16, 64)]
    + [(cfg, *SPLIT_SHAPE, sp, "cluster-split-k") for cfg in SPLIT_CONFIGS for sp in (-2, -4, -8)]
    + [(cfg, *STREAMK_SHAPE, sp, "stream-k") for cfg in STREAMK_CONFIGS for sp in (100, 101)]
)
# non-finite operands: one configuration per K-mode
NONFINITE_CASES = [(1, *SPLIT_SHAPE, 1, "plain"), (1, *SPLIT_SHAPE, 4, "split-k"), (2, *SPLIT_SHAPE, -4, "cluster-split-k"),
                   (0, *STREAMK_SHAPE, 100, "stream-k")]


def cluster_ctas(cfg: int) -> int:
    c = capi.configs()[cfg]
    return c["cta_group"] * c["cluster_m"] * c["cluster_n"]


def steady_max_ctas(cfg: int) -> int:
    """One worker (a CTA, CTA pair or cluster), which runs every tile of the problem."""
    return cluster_ctas(cfg)


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def dev(x: np.ndarray, dtype) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(dtype).cuda()


def bits(c: torch.Tensor) -> np.ndarray:
    return c.view(torch.int16).cpu().numpy().view(np.uint16)


def out_dtype(kind: str):
    return torch.bfloat16 if kind == "bf16" else torch.float16


# ------------------------------------------------------------------------------------------------- 16-bit kernels
@functools.lru_cache(maxsize=None)
def case16(variant: str, m: int, n: int, k: int):
    """Device operands and the reference bits of one 16-bit variant on an (M, N, K) problem (built once per test run)."""
    kind = "bf16" if variant == "bf16" else "fp16"
    ops = ed.operands16(m, n, k, kind, seed=m + 3 * n + 7 * k, acc16=variant == "fp16acc16")
    with np.errstate(over="ignore"):
        want = ed.reference16(ops, kind)
    return dev(ops.a, out_dtype(kind)), dev(ops.bt, out_dtype(kind)), want


def run16(variant, a, bt, **kw) -> np.ndarray:
    c = torch.full((a.shape[0], bt.shape[0]), float("nan"), dtype=a.dtype, device="cuda")
    capi.gemm_kmajor(a, bt, c, "fp16" if variant == "fp16acc16" else "fp32", **kw)
    torch.cuda.synchronize()
    return bits(c)


def test_fp32_accumulation_is_exact_to_2_24():
    """The bound the domain rests on. S = 2^23 + h + 1, h half an output ulp at 2^23 (fp16: 2^12, bf16: 2^15), rounds up
    only if the unit product survives next to the 2^23 one; it sits in the same k16 step, the next k-block or the last
    split. Plain, split-K, cluster split-K and stream-K; both signs."""
    m, n, k = 120, 64, 4096
    for kind in ("fp16", "bf16"):
        lo, hi = (6, 6) if kind == "fp16" else (8, 7)
        e = -14 if kind == "fp16" else 0                            # fp16: every operand normal, C near 2^-5
        a, bt = np.zeros((m, k)), np.zeros((n, k))
        a[:, 0], bt[:, 0] = 2.0 ** 12, 2.0 ** 11                    # 2^23
        a[:, 100], bt[:, 100] = 2.0 ** lo, 2.0 ** hi                # h
        for r, pos in enumerate((1, 70, k - 3)):
            a[r::3, pos] = 1.0
            bt[:, pos] = 1.0
        a[1::2] *= -1
        a, bt = a * 2.0 ** e, bt * 2.0 ** e
        exact = a @ bt.T
        assert np.array_equal(np.abs(exact), np.full((m, n), (2 ** 23 + 2 ** (lo + hi) + 1) * 2.0 ** (2 * e)))
        want = ed.round_fp16_bits(exact) if kind == "fp16" else ed.round_bf16_bits(exact)
        da, dbt = dev(a, out_dtype(kind)), dev(bt, out_dtype(kind))
        for cfg, splits in ((1, 1), (1, 8), (1, -4), (0, 100)):
            got = run16(kind, da, dbt, config_id=cfg, splits=splits)
            assert np.array_equal(got, want), (kind, cfg, splits)


@pytest.mark.parametrize("variant", VARIANTS16)
def test_16bit_every_configuration_steady_state(variant):
    m, n = STEADY_MN
    a, bt, want = case16(variant, m, n, STEADY_K["16"])
    for cfg in capi.configs():
        got = run16(variant, a, bt, config_id=cfg["id"], max_ctas=steady_max_ctas(cfg["id"]))
        assert np.array_equal(got, want), (variant, cfg)


@pytest.mark.parametrize("cfg,m,n,k,splits,mode", KMODE_CASES)
def test_16bit_every_k_mode_full_range(cfg, m, n, k, splits, mode):
    assert capi.schedule(cfg, m, n, k, splits)["mode"] == mode
    for variant in VARIANTS16:
        a, bt, want = case16(variant, m, n, k)
        assert np.array_equal(run16(variant, a, bt, config_id=cfg, splits=splits), want), (variant, cfg, splits)


# ------------------------------------------------------------------------------------------------- e4m3 kernels
@functools.lru_cache(maxsize=None)
def case8(m: int, n: int, k: int):
    a, bt = ed.operands_e4m3(m, n, k, seed=m + 5 * n + 3 * k)
    da, dbt = dev(a, E4), dev(bt, E4)
    return da, dbt, da.cpu().view(torch.uint8).numpy(), dbt.cpu().view(torch.uint8).numpy()


def run8(a, bt, sa, sb, out, **kw) -> np.ndarray:
    c = torch.full((a.shape[0], bt.shape[0]), float("nan"), dtype=out, device="cuda")
    capi.fp8_gemm(a, bt, c, sa, sb, **kw)
    torch.cuda.synchronize()
    return bits(c)


def tensor_scale_refs(m, n, k):
    """[(out dtype, (sa, sb) device tensors, reference bits)] for the per-tensor pairs of exact_domain."""
    _, _, ca, cb = case8(m, n, k)
    out = []
    for kind in ("fp16", "bf16"):
        for pair in ed.e4m3_tensor_scales(kind):
            sa, sb = (torch.tensor([v], dtype=torch.float32, device="cuda") for v in pair)
            out.append((out_dtype(kind), sa, sb, fp8_oracle.fp8gemm_f32acc(ca, cb, pair[0], pair[1], kind == "bf16")))
    return out


def rowwise_refs(m, n, k):
    _, _, ca, cb = case8(m, n, k)
    out = []
    for kind in ("fp16", "bf16"):
        sa, sb = ed.e4m3_rowwise_scales(m, n, kind)
        dsa, dsb = torch.from_numpy(sa).reshape(m, 1).cuda(), torch.from_numpy(sb).reshape(1, n).cuda()
        with np.errstate(over="ignore"):
            out.append((out_dtype(kind), dsa, dsb, fp8gemm_f32acc_rowwise(ca, cb, sa, sb, kind == "bf16")))
    return out


@functools.lru_cache(maxsize=None)
def e4m3_refs(m, n, k):
    return {"tensor": tensor_scale_refs(m, n, k), "rowwise": rowwise_refs(m, n, k)}


@pytest.mark.parametrize("granularity", ["tensor", "rowwise"])
def test_e4m3_every_configuration_steady_state(granularity):
    m, n = STEADY_MN
    k = STEADY_K["e4m3"]
    a, bt, _, _ = case8(m, n, k)
    refs = e4m3_refs(m, n, k)[granularity]
    for cfg in capi.configs():
        for i, (out, sa, sb, want) in enumerate(refs):
            if granularity == "tensor" and i % 2 != cfg["id"] % 2:
                continue                               # each configuration: one fp16 and one bf16 pair, alternating
            got = run8(a, bt, sa, sb, out, config_id=cfg["id"], max_ctas=steady_max_ctas(cfg["id"]))
            assert np.array_equal(got, want), (granularity, cfg, out, i)


def block_case(m, n, k, kind):
    a, bt, ca, cb = case8(m, n, k)
    sa, sb = ed.e4m3_block_scales(m, n, k, kind)
    nkb, ld = sa.shape[1], -(-m // 4) * 4
    buf = torch.full((nkb, ld), float("nan"), dtype=torch.float32, device="cuda")
    buf[:, :m] = torch.from_numpy(sa).t().cuda()
    return a, bt, ca, cb, sa, sb, buf[:, :m].t(), torch.from_numpy(sb).cuda()


def test_e4m3_block_scaled_every_eligible_configuration_steady_state():
    m, n = STEADY_MN
    k = STEADY_K["block"]
    for kind in ("fp16", "bf16"):
        a, bt, ca, cb, sa, sb, dsa, dsb = block_case(m, n, k, kind)
        want = fp8gemm_f32acc_block(ca, cb, sa, sb, kind == "bf16")
        for cfg in BLOCK_ELIGIBLE:
            got = run8(a, bt, dsa, dsb, out_dtype(kind), config_id=cfg, max_ctas=steady_max_ctas(cfg))
            assert np.array_equal(got, want), (cfg, kind)


@pytest.mark.parametrize("cfg", [1, 2])
@pytest.mark.parametrize("splits", [-2, -4, -8])
def test_e4m3_block_scaled_cluster_split_k_full_range(cfg, splits):
    m, n, k = SPLIT_SHAPE[0], SPLIT_SHAPE[1], 2 * 4288
    assert capi.schedule(cfg, m, n, k // 2, splits)["mode"] == "cluster-split-k"
    for kind in ("fp16", "bf16"):
        a, bt, ca, cb, sa, sb, dsa, dsb = block_case(m, n, k, kind)
        want = fp8gemm_f32acc_block(ca, cb, sa, sb, kind == "bf16", -splits)
        got = run8(a, bt, dsa, dsb, out_dtype(kind), config_id=cfg, splits=splits)
        assert np.array_equal(got, want), (cfg, splits, kind)


# ----------------------------------------------------------------------------------------------- non-finite inputs
def nonfinite_positions(k):
    """k of the NaN in A (inside the last split's range for any split count), and of the two Infs in Bt (early, late)."""
    return k - 40, 24, k - 200


def check_nonfinite(got_bits, expect, kind):
    """NaN where ``expect`` is NaN, the same signed inf where it is inf, the one rounding of ``expect`` elsewhere."""
    got = (got_bits.view(np.float16) if kind == "fp16" else (got_bits.astype(np.uint32) << 16).view(np.float32)).astype(np.float64)
    nan, inf = np.isnan(expect), np.isinf(expect)
    assert np.isnan(got[nan]).all()
    assert np.array_equal(got[inf], expect[inf])
    fin = ~nan & ~inf
    want = ed.round_fp16_bits(expect[fin]) if kind == "fp16" else ed.round_bf16_bits(expect[fin])
    assert np.array_equal(got_bits[fin], want)


@pytest.mark.parametrize("cfg,m,n,k,splits,mode", NONFINITE_CASES)
def test_nonfinite_operands_propagate_in_every_k_mode(cfg, m, n, k, splits, mode):
    assert capi.schedule(cfg, m, n, k, splits)["mode"] == mode
    kn, ka, kb = nonfinite_positions(k)
    row_nan, col_inf = 7, 13
    for variant in VARIANTS16:
        kind = "bf16" if variant == "bf16" else "fp16"
        ops = ed.operands16(m, n, k, kind, seed=11 + k, acc16=variant == "fp16acc16")
        a, bt = ops.a.copy(), ops.bt.copy()
        a[row_nan, kn] = np.nan
        bt[col_inf, ka] = bt[col_inf, kb] = np.inf
        fa, fbt = np.nan_to_num(a, nan=0.0), np.nan_to_num(bt, posinf=0.0)
        with np.errstate(invalid="ignore", over="ignore"):
            expect = fa @ fbt.T
            expect[:, col_inf] += a[:, ka] * np.inf + a[:, kb] * np.inf     # IEEE: one sign -> inf, mixed or 0 -> NaN
            expect[row_nan, :] = np.nan
        col = expect[:, col_inf]
        assert (col == np.inf).any() and (col == -np.inf).any() and np.isnan(col).sum() > 1
        got = run16(variant, dev(a, out_dtype(kind)), dev(bt, out_dtype(kind)), config_id=cfg, splits=splits)
        with np.errstate(over="ignore"):
            check_nonfinite(got, expect, kind)
    # e4m3 (no Inf encoding): the NaN row, per-tensor scales
    a8, bt8 = ed.operands_e4m3(m, n, 2 * k, seed=13 + k)
    a8[row_nan, 2 * k - 40] = np.nan
    da, dbt = dev(a8, E4), dev(bt8, E4)
    expect = np.nan_to_num(a8, nan=0.0) @ bt8.T
    expect[row_nan, :] = np.nan
    for kind, (sa_v, sb_v) in (("fp16", ed.e4m3_tensor_scales("fp16")[0]), ("bf16", ed.e4m3_tensor_scales("bf16")[1])):
        sa, sb = (torch.tensor([v], dtype=torch.float32, device="cuda") for v in (sa_v, sb_v))
        got = run8(da, dbt, sa, sb, out_dtype(kind), config_id=cfg, splits=splits)
        with np.errstate(over="ignore"):
            check_nonfinite(got, expect * np.float64(np.float32(sa_v) * np.float32(sb_v)), kind)
