"""scale_cases.py without a GPU: each case really crosses its boundary where it says, the routing histograms keep their
guarantees, the operand domains keep exact_domain.py's bounds, the banded float64 reference equals a numpy product
rounded once, and the memory each case budgets is what it allocates."""
import numpy as np
import pytest
import torch

import exact_domain as ed
import scale_cases as sc
from cuda_l2_b200 import capi

REDUCTIONS = {"fp16": sc.TN[2], "fp16acc16": sc.TN[2], "bf16": sc.TN[2], "tall": sc.TALL[2],
              "nn_long": sc.NN_LONG[2], "wgrad": sc.WGRAD["t"], "wgrad_long": max(sc.WGRAD_LONG_SIZES)}


@pytest.mark.parametrize("name", sorted(sc.CASES))
def test_case_crosses_its_boundaries_where_it_says(name):
    case = sc.CASES[name]
    size = case.size()
    for boundary, index in case.crossings:
        assert size > boundary, (name, size, boundary)
        assert case.crossing_index(boundary) == index, (name, boundary)
    first = case.crossings[0][0]
    assert (size - first) / size >= 0.25, (name, size)            # a large share of the tensor lies past it
    assert case.memory_bytes() < 14 * 10 ** 9, name


def test_memory_need_is_what_the_gpu_test_allocates():
    for case in sc.CASES.values():
        for dtype in (torch.float16, torch.bfloat16):
            d = sc.allocate(case, dtype, device="meta")
            allocated = sum(t.untyped_storage().nbytes() for k, t in d.items()
                            if k.endswith(":buf") or k not in case.outputs)
            assert allocated == case.tensor_bytes(), case.name
            assert {k for k in d if ":" not in k} == {t.name for t in case.tensors}
            for out in case.outputs:
                assert d[out].shape == case.tensor(out).shape


def test_routing_histogram_guarantees():
    cross = sc.HISTOGRAMS["grouped"]["cross_rows"]
    sizes = sc.histogram("grouped")
    assert len(sizes) == sc.NUM_EXPERTS and sizes.sum() == sc.T_GROUPED and (sizes >= 0).all()
    r = sc.histogram_report(sizes, cross)
    assert 0 in r["empty"] and sc.NUM_EXPERTS - 1 in r["empty"] and len(r["empty"]) >= 16
    assert r["one_row"] >= 5
    assert r["largest"] >= sc.BIG_GROUP
    assert r["res4"] == set(range(4)) and r["res128"] == set(range(128))
    for row, c in zip(cross, r["crossings"]):
        assert c["start"] <= row < c["start"] + c["size"] and c["size"] < 128, c   # its tile straddles the group end
        assert c["before"] == 0 and c["after"] == 0, c
        assert c["start"] % 128 != 0 or (c["start"] + c["size"]) % 128 != 0
    # the same seed gives the same histogram
    assert np.array_equal(sizes, sc.histogram("grouped"))


def test_other_histograms():
    w = sc.histogram("wgrad")
    assert w.sum() == sc.WGRAD["t"] and len(w) == sc.NUM_EXPERTS
    assert w[113] > 0 and w[227] > 0 and w[114] == 0 and w[228] == 0 and w[0] == 0 and w[-1] == 0
    assert max(w) * sc.sum_bound(sc.DOMAINS["wgrad"], 1) < ed.EXACT_SUM_BOUND
    f = sc.histogram("fp8_experts")
    assert f.sum() == sc.FP8_EXPERTS["t"] and f[117] > 0 and f[234] > 0
    s = np.asarray(sc.WGRAD_LONG_SIZES)
    ends = np.cumsum(s)
    assert s.max() >= 131072 and 0 in s and 1 in s and ends[-1] == sc.T_GROUPED
    g = int(np.searchsorted(ends, 174648, side="right"))
    assert ends[g] - s[g] < 174648 < ends[g] - 1                     # dY's crossing row inside a group, not at an edge
    for seed in range(3):                                           # other seeds keep the guarantees too
        r = sc.histogram_report(sc.routing_histogram(sc.T_GROUPED, seed, cross_rows=(100000,)), (100000,))
        assert r["res128"] == set(range(128)) and r["largest"] >= sc.BIG_GROUP


@pytest.mark.parametrize("kind", sorted(sc.DOMAINS))
def test_domains_keep_the_exact_bounds(kind):
    dom = sc.DOMAINS[kind]
    if kind == "e4m3":
        assert dom["a"][:2] == (-1, 1) and dom["b"] == (-1, 1)    # |i j| <= 1: the sum is the nonzero count
        p = dom["a"][2]
        k = sc.FP8_EXPERTS["k"]
        mean, sd = k * p, (k * p * (1 - p)) ** 0.5
        assert mean + 10 * sd < ed.E4M3_SUM_BOUND                  # and the GPU test asserts the count per row
        assert sc.TN[2] <= ed.E4M3_SUM_BOUND                       # the 2-D case: K itself is below the bound
        return
    if kind == "nn_long":
        p = dom["a"][2]
        k = sc.NN_LONG[2]
        assert k < ed.EXACT_SUM_BOUND and k * p + 10 * (k * p) ** 0.5 < 65504   # the GPU test asserts the row sums
        return
    assert sc.sum_bound(dom, REDUCTIONS[kind]) < sc.exact_bound(kind)
    if kind.startswith("bf16"):
        assert max(map(abs, dom["a"])) <= 256 and max(map(abs, dom["b"])) <= 256   # integers exact in bf16


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float8_e4m3fn])
def test_fill_ints_stays_in_its_range(dtype):
    x = torch.empty((300, 200), dtype=dtype)
    sc.fill_ints_(x, (-7, 7) if dtype != torch.float8_e4m3fn else (-1, 1, 0.2), sc.generator(1, "cpu"), band=7000)
    v = x.float()
    assert v.eq(v.round()).all()
    lim = 7 if dtype != torch.float8_e4m3fn else 1
    assert v.abs().max() <= lim and len(v.unique()) == 2 * lim + 1
    if dtype == torch.float8_e4m3fn:
        share = float(v.ne(0).float().mean())
        assert 0.1 < share < 0.17                                   # p = 0.2 of the 2/3 nonzero draws
    s = sc.pow2_scales_(torch.empty(1000), sc.generator(2, "cpu"))
    assert set(s.tolist()) == {0.5, 1.0, 2.0}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_banded_reference_equals_numpy_rounded_once(dtype, monkeypatch):
    rng = np.random.default_rng(3)
    m, n, k = 37, 24, 200
    a = rng.integers(-31, 32, size=(m, k)).astype(np.float64)
    b = rng.integers(-31, 32, size=(k, n)).astype(np.float64)
    a[:, :20] *= 2.0 ** -4                                          # values that need the fraction bits too
    want = ed.round_fp16_bits(a @ b) if dtype == torch.float16 else ed.round_bf16_bits(a @ b)
    monkeypatch.setattr(sc, "BAND_BYTES", 8 * 24 * 5)               # 5-row bands, 5-long reduction chunks
    ta, tb = torch.from_numpy(a).to(dtype), torch.from_numpy(b).to(dtype)
    assert torch.equal(ta.double(), torch.from_numpy(a)) and torch.equal(tb.double(), torch.from_numpy(b))
    ref = lambda r0, r1: sc.matmul64(ta[r0:r1], tb, sc.BAND_BYTES)
    bits = torch.cat([sc.round_bits(ref(r0, min(m, r0 + 5)), dtype) for r0 in range(0, m, 5)])
    assert np.array_equal(bits.numpy().view(np.uint16), want)
    out = bits.view(dtype).clone()
    assert sc.first_mismatch(out, ref) is None
    out.view(torch.int16)[23, 5] ^= 1
    msg = sc.first_mismatch(out, ref, base=2 ** 31 - 100)
    assert msg is not None and f"element {2 ** 31 - 100 + 23 * n + 5} (+{23 * n + 5 - 100} from 2^31)" in msg


def test_guard_bands_catch_writes_past_either_end():
    buf, c = sc.guarded((30, 16), torch.bfloat16, "cpu")
    c.zero_()
    assert sc.guards_intact(buf) and torch.isnan(buf[:10]).all()
    buf[buf.numel() - 1] = 0
    assert not sc.guards_intact(buf)


def test_masked_counts_take_every_kind_past_the_crossing():
    b, m = sc.CASES["batched"].tensor("a").shape[:2]
    counts = sc.masked_counts(b, m, seed=5)
    past = counts[42:]
    assert {0, 1, m, m + 37, -5} <= set(past) and any(1 < c < m for c in past)


def test_pinned_configurations_run_their_k_modes(built_libs):
    import test_gpu_scale as t
    m, n, k = sc.TN
    for cfg, splits, mode in t.TN_PINNED:
        assert capi.schedule(cfg, m, n, k, splits)["mode"] == mode, (cfg, splits)
    cfgs = capi.configs()
    assert cfgs[t.TN_PINNED[0][0]]["cta_group"] == 2
    assert cfgs[t.TN_PINNED[1][0]]["cluster_m"] * cfgs[t.TN_PINNED[1][0]]["cluster_n"] > 1
    m, n, k = sc.NN_LONG
    for cfg, splits, mode in t.NN_LONG_PINNED:
        assert cfgs[cfg]["bn"] % 64 == 0                            # the NN kernels run the configuration itself
        assert capi.schedule(cfg, m, n, k, splits)["mode"] == mode, (cfg, splits)
    assert k // 64 > 4096                                           # k-blocks per tile
