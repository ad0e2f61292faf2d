"""CPU companion of test_gpu_exact_range.py (and of the e4m3 K_MODES of test_gpu_fp8.py): the GPU cases are not vacuous.

* Every steady-state case runs the plain schedule with some worker on two or more tiles, at least one worker's k-blocks
  wrapping the ring, M and N off the tile, and (block scales) every unit longer than 32 k-blocks.
* Every K-mode case is planned in the K-mode it names, on a ragged problem.
* The operands are exactly representable, keep the sum bounds, and the fixtures contain what the tests claim: exact ties
  rounding both ways at 1 to 13 dropped bits, fp16 subnormal results, the fp16 overflow edges, values rounding to inf.
* The numpy reference agrees with an independent torch expression (float64 matmul, then .half() / .bfloat16()).
"""
import numpy as np
import pytest
import torch

import exact_domain as ed
import test_gpu_exact_range as g
from cuda_l2_b200 import capi
from test_gpu_fp8 import K_MODES


@pytest.fixture(scope="module", autouse=True)
def _libs(built_libs):
    return built_libs


def steady_cases():
    """(variant, config, M, N, K of the 16-bit schedule, max_ctas) of every steady-state launch."""
    m, n = g.STEADY_MN
    out = []
    for cfg in range(31):
        out += [(v, cfg, m, n, g.STEADY_K["16"], g.steady_max_ctas(cfg)) for v in g.VARIANTS16]
        out += [("e4m3", cfg, m, n, g.STEADY_K["e4m3"] // 2, g.steady_max_ctas(cfg))]
    out += [("block", cfg, m, n, g.STEADY_K["block"] // 2, g.steady_max_ctas(cfg)) for cfg in g.BLOCK_ELIGIBLE]
    return out


def test_steady_state_cases_run_several_tiles_per_worker_and_wrap_the_ring():
    configs = capi.configs()
    for variant, cfg, m, n, k, max_ctas in steady_cases():
        c = configs[cfg]
        s = capi.schedule(cfg, m, n, k, 1, num_sms=max_ctas)
        case = (variant, cfg, m, n, k, max_ctas)
        assert s["mode"] == "plain" and s["workers"] == 1, case
        assert max(len(u) for u in s["units"]) >= 2, case
        assert max(sum(kb1 - kb0 for _, kb0, kb1, _ in u) for u in s["units"]) > c["stages"], case
        assert m % (128 * c["m_rep"]) and n % c["bn"], case
        if variant == "block":
            assert min(kb1 - kb0 for u in s["units"] for _, kb0, kb1, _ in u) > 32, case


def test_k_mode_cases_are_planned_as_named():
    for cfg, m, n, k, splits, mode in g.KMODE_CASES + g.NONFINITE_CASES:
        assert capi.schedule(cfg, m, n, k, splits)["mode"] == mode, (cfg, splits)
        assert m % 128 and n % capi.configs()[cfg]["bn"], (cfg, m, n)
    for cfg, m, n, k, splits, mode in K_MODES:          # e4m3: the 16-bit schedule at K / 2 has the same k-blocks
        assert capi.schedule(cfg, m, n, k // 2, splits)["mode"] == mode, (cfg, splits)
    # every configuration that carries a mode is covered
    configs = capi.configs()
    split_cfgs = {c["id"] for c in configs if c["cta_group"] == 1 and c["cluster_m"] * c["cluster_n"] == 1 and c["bn"] >= 64
                  and c["m_rep"] == 1}
    stream_cfgs = {c["id"] for c in configs if c["cluster_m"] * c["cluster_n"] == 1 and c["bn"] >= 64 and c["m_rep"] == 1}
    for mode, want in (("split-k", split_cfgs), ("cluster-split-k", split_cfgs), ("stream-k", stream_cfgs)):
        for cases in (g.KMODE_CASES, K_MODES):
            assert {c[0] for c in cases if c[5] == mode} == want, mode
    assert {c[4] for c in g.KMODE_CASES if c[5] == "split-k"} == {4, 16, 64}
    assert {c[4] for c in g.KMODE_CASES if c[5] == "cluster-split-k"} == {-2, -4, -8}
    assert {c[4] for c in g.KMODE_CASES if c[5] == "stream-k"} == {100, 101}


def unit16(ops):
    return np.exp2(ops.row_exp[:, None] + ops.col_exp[None, :])


def shapes16():
    return [(*g.STEADY_MN, g.STEADY_K["16"]), g.SPLIT_SHAPE, g.STREAMK_SHAPE]


@pytest.mark.parametrize("kind", ["fp16", "bf16"])
def test_16bit_fixtures_hold_every_rounding_case(kind):
    for m, n, k in shapes16():
        ops = ed.operands16(m, n, k, kind, seed=m + 3 * n + 7 * k)
        assert ops.sum_bound() < ed.EXACT_SUM_BOUND
        for x in (ops.a, ops.bt):                      # exactly representable, no subnormal operands
            if kind == "fp16":
                assert np.array_equal(x.astype(np.float16).astype(np.float64), x)
                assert (np.abs(x[x != 0]) >= 2.0 ** -14).all() and np.isfinite(x.astype(np.float16)).all()
            else:
                back = (ed.round_bf16_bits(x).astype(np.uint32) << 16).view(np.float32).astype(np.float64)
                assert np.array_equal(back, x) and (np.abs(x[x != 0]) >= 2.0 ** -126).all()
        y = ops.exact()
        with np.errstate(over="ignore"):
            c = ed.classify(y, kind, unit16(ops))
        for d in range(1, 14):
            assert c["tie_up"][d].any() and c["tie_down"][d].any(), (kind, (m, n, k), d)
        assert c["inf"].any() and c["max_finite"].any()
        if kind == "fp16":
            assert (c["subnormal"] & c["rounds"]).any()
            for v in (65504.0, 65520.0):
                assert (y == v).any() and (y == -v).any(), v
            assert ((np.abs(y) > 65504) & (np.abs(y) < 65520)).any()
            assert np.isinf(y[np.abs(y) == 65520].astype(np.float16)).all()
        else:
            top = 2.0 ** 128 - 2.0 ** 120
            assert ((np.abs(y) > top) & np.isfinite(y.astype(np.float32))).any()
            assert np.abs(y[y != 0]).min() >= 2.0 ** -126        # no fp32-subnormal sums


def test_fp16_accumulation_fixtures_stay_non_saturating():
    for m, n, k in shapes16():
        ops = ed.operands16(m, n, k, "fp16", seed=m + 3 * n + 7 * k, acc16=True)
        assert ops.sum_bound() < ed.FP16_ACC_SUM_BOUND
        y = np.abs(ops.exact())
        assert (y[y != 0] >= 2.0 ** -14).all() and (ops.sum_bound() * unit16(ops) <= 65504).all()
        assert np.array_equal(y.astype(np.float16).astype(np.float64), y)


def e4m3_exact(a, bt, granularity, out, k):
    """[(exact pre-rounding values, integer units)] of the e4m3 fixtures of test_gpu_exact_range at one shape."""
    m, n = a.shape[0], bt.shape[0]
    s = a @ bt.T
    if granularity == "tensor":
        pairs = ed.e4m3_tensor_scales(out)
        qs = (*ed.E4M3_Q[out], *ed.E4M3_Q[out]) if out == "fp16" else (513, *ed.E4M3_Q[out])
        # past the largest fp32 (2047 * 513 * 2^108) the kernel's fp32 product is already inf
        fp32 = lambda y: np.where(np.abs(y) >= 2.0 ** 128 - 2.0 ** 103, np.sign(y) * np.inf, y)
        return [(fp32(s * (sa * sb)), np.full((m, n), sa * sb / q)) for (sa, sb), q in zip(pairs, qs)]
    q = ed.e4m3_row_q(m, out)
    if granularity == "rowwise":
        sa, sb = ed.e4m3_rowwise_scales(m, n, out)
        return [((s * sb[None, :].astype(np.float64)) * sa[:, None], (sa / q)[:, None] * sb[None, :])]
    sa, sb = ed.e4m3_block_scales(m, n, k, out)
    y = np.zeros((m, n))
    for kb in range(sa.shape[1]):
        part = a[:, kb * 128:(kb + 1) * 128] @ bt[:, kb * 128:(kb + 1) * 128].T
        y += part * sa[:, kb:kb + 1] * np.repeat(sb[:, kb], 128)[None, :n]
    return [(y, (sa[:, 0] / q)[:, None] * np.ones((1, n)))]


@pytest.mark.parametrize("granularity", ["tensor", "rowwise", "block"])
def test_e4m3_fixtures_reach_the_full_output_range(granularity):
    m, n = g.STEADY_MN
    k = g.STEADY_K["block" if granularity == "block" else "e4m3"]
    a, bt = ed.operands_e4m3(m, n, k, seed=m + 5 * n + 3 * k)
    codes = torch.from_numpy(np.concatenate([a, bt]).astype(np.float32)).to(torch.float8_e4m3fn)
    assert np.array_equal(codes.float().numpy().astype(np.float64), np.concatenate([a, bt]))
    assert (np.abs(a) @ np.abs(bt).T).max() <= ed.E4M3_SUM_BOUND
    for out in ("fp16", "bf16"):
        seen = {"tie_up": False, "tie_down": False, "inf": False, "subnormal": False}
        for y, unit in e4m3_exact(a, bt, granularity, out, k):
            assert np.array_equal(y.astype(np.float32).astype(np.float64), y)       # exact in fp32 as well
            with np.errstate(over="ignore"):
                c = ed.classify(y, out, unit)
            seen["tie_up"] |= any(v.any() for v in c["tie_up"].values())
            seen["tie_down"] |= any(v.any() for v in c["tie_down"].values())
            seen["inf"] |= bool(c["inf"].any())
            seen["subnormal"] |= bool((c["subnormal"] & c["rounds"]).any())
        if out == "bf16":
            seen["subnormal"] = True                    # no bf16 subnormals in the domain
            seen["inf"] |= granularity != "tensor"      # bf16 inf: the per-tensor pair (rowwise / block stay finite)
        assert all(seen.values()), (granularity, out, seen)


@pytest.mark.parametrize("kind", ["fp16", "bf16"])
def test_reference_matches_torch_on_the_fixtures(kind):
    m, n, k = g.SPLIT_SHAPE
    ops = ed.operands16(m, n, k, kind, seed=m + 3 * n + 7 * k)
    with np.errstate(over="ignore"):
        want = ed.reference16(ops, kind)
    y = torch.from_numpy(ops.a) @ torch.from_numpy(ops.bt).t()
    t = y.half() if kind == "fp16" else y.bfloat16()
    assert np.array_equal(t.view(torch.int16).numpy().view(np.uint16), want)
