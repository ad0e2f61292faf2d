"""Parity of the CUDA path (through the C ABI) with the oracle — the tests proper, run on the H100.

Bars: BIT-EXACT against the oracle / golden truth on the reference's test domain (0/1 operands, entries with
|truth| <= 2047; reference zero_one_correctness_check.py:92,169-172); on N(0,1) operands — where the reference
pins nothing — within  |err| <= 2^-10 |truth| + 2^-10 * sqrt(K) * 0.05 + 1e-3  for fp32 accumulation (one fp16
rounding plus summation-order noise); for fp16 accumulation the running sum is re-rounded to fp16 about K/16 times,
so the bound is a random walk of half-ulps at the running magnitude: 2^-11 * sqrt(K/16) * 2 * (|truth| + sqrt(K)) + 1e-3.
"""
import numpy as np
import pytest
import torch

import oracle
from cuda_l2_b200 import capi
from cuda_l2_b200.harness import correctness as zc
from cuda_l2_b200.harness.common import Padding

pytestmark = pytest.mark.gpu
ACCS = ("fp32", "fp16")


def dev(x: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def run(a: torch.Tensor, bt: torch.Tensor, acc: str, cfg=None, **kw) -> torch.Tensor:
    """a [M,K], bt [N,K] (K-major B) device tensors -> C [M,N] through libb200_hgemm.so."""
    m, n = a.shape[0], bt.shape[0]
    c = torch.full((m, n), float("nan"), dtype=torch.half, device="cuda")
    b_col_major = bt.reshape(bt.shape[1], bt.shape[0])     # labelled [K,N], storage [N,K] (as_col_major's output)
    if cfg is None:
        capi.hgemm(a, b_col_major, c, acc)
    else:
        capi.hgemm_config(a, b_col_major, c, cfg, acc, **kw)
    torch.cuda.synchronize()
    return c


@pytest.fixture(scope="module", autouse=True)
def _need_h100(built_libs):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert torch.cuda.get_device_capability() == (9, 0), "these kernels are sm_90a only"
    before = capi.launch_count()
    yield
    assert capi.launch_count() > before, "no kernel of libb200_hgemm.so was launched"


@pytest.mark.parametrize("acc", ACCS)
def test_golden_zero_one_vectors_bit_exact(zero_one_cases, acc):
    for c in zero_one_cases:
        if c["k"] % 8 or c["n"] % 8:
            continue
        got = run(dev(c["a"]), dev(c["b"].T), acc).cpu().numpy()
        truth = c["truth"]
        keep = np.abs(truth.astype(np.float32)) <= 2047
        assert np.array_equal(got[keep], truth[keep]), (acc, c["m"], c["n"], c["k"])
        d, _, n_bad = oracle.zero_one_max_diff(got, truth)
        assert d == 0.0 and n_bad == 0
        if acc == "fp32":      # fp32 accumulation is exact far beyond the mask: every entry must agree
            assert np.array_equal(got.view(np.uint16), truth.view(np.uint16))


@pytest.mark.parametrize("acc", ACCS)
def test_every_configuration_matches_the_oracle(acc):
    shapes = [(128, 64, 64), (256, 256, 64), (200, 328, 72), (512, 768, 512), (1000, 1000, 1000), (64, 4096, 64)]
    for cfg in capi.configs():
        for (m, n, k) in shapes:
            a = oracle.fill_zero_one((m, k), 2, seed=m * 7 + cfg["id"])
            bt = oracle.fill_zero_one((n, k), 2, seed=n * 13 + k)
            want = oracle.hgemm_f32acc(a, bt, fast=True)
            got = run(dev(a), dev(bt), acc, cfg=cfg["id"]).cpu().numpy()
            assert np.array_equal(got.view(np.uint16), want.view(np.uint16)), (acc, cfg, m, n, k)


@pytest.mark.parametrize("acc", ACCS)
@pytest.mark.parametrize("group_m,max_ctas", [(1, 0), (3, 0), (64, 0), (0, 8), (0, 37)])
def test_schedule_knobs_do_not_change_results(acc, group_m, max_ctas):
    m, n, k = 1536, 1280, 256
    a, bt = oracle.fill_zero_one((m, k), 2, 1), oracle.fill_zero_one((n, k), 2, 2)
    want = oracle.hgemm_f32acc(a, bt, fast=True)
    for cfg in capi.configs():
        got = run(dev(a), dev(bt), acc, cfg=cfg["id"], group_m=group_m, max_ctas=max_ctas).cpu().numpy()
        assert np.array_equal(got, want), (cfg, group_m, max_ctas)


@pytest.mark.parametrize("acc", ACCS)
def test_split_k_is_exact_deterministic_and_self_resetting(acc):
    """Split-K (small M x N, long K): bit-exact on 0/1 operands for every split factor, identical bits run to
    run on N(0,1) operands (fixed summation order), and repeated launches work (the arrival counters reset)."""
    one_cta = [c["id"] for c in capi.configs() if c["cta_group"] == 1]
    for (m, n, k) in [(64, 64, 4096), (200, 328, 1096), (256, 512, 2048), (128, 64, 16384)]:
        a, bt = oracle.fill_zero_one((m, k), 3, 11), oracle.fill_zero_one((n, k), 3, 12)
        want = oracle.hgemm_f32acc(a, bt, fast=True)
        da, dbt = dev(a), dev(bt)
        for cfg in one_cta:
            for splits in (2, 3, 8, 17, 64, -2, -4, -8):
                for _ in range(2):
                    got = run(da, dbt, acc, cfg=cfg, splits=splits).cpu().numpy()
                    assert np.array_equal(got, want), (acc, cfg, splits, m, n, k)
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn((256, 8192), device="cuda", generator=g).half()
    bt = torch.randn((192, 8192), device="cuda", generator=g).half()
    for splits in (16, -4):
        first = run(a, bt, acc, cfg=one_cta[0], splits=splits)
        for _ in range(3):
            assert torch.equal(run(a, bt, acc, cfg=one_cta[0], splits=splits), first)
    # the dispatcher's own choice for a split-K-class problem agrees with the unsplit kernel on exact data
    a01, bt01 = oracle.fill_zero_one((64, 16384), 3, 1), oracle.fill_zero_one((64, 16384), 3, 2)
    assert capi.select(acc, 64, 64, 16384)[2] not in (0, 1)
    assert np.array_equal(run(dev(a01), dev(bt01), acc).cpu().numpy(), oracle.hgemm_f32acc(a01, bt01, fast=True))


@pytest.mark.parametrize("acc", ACCS)
def test_stream_k_is_exact_deterministic_and_self_resetting(acc):
    """Stream-K (tile counts that do not fill the last wave): bit-exact on 0/1 operands for single CTAs and CTA pairs,
    one and many contributors per tile, ragged edges; identical bits run to run on N(0,1) operands; repeated launches
    work (every flag is lowered by its reader); and the stream-K schedule really was in effect."""
    cfgs = capi.configs()
    plain = [c for c in cfgs if c["cluster_m"] * c["cluster_n"] == 1 and c["bn"] >= 64]
    # (shape, max_ctas): few tiles on all SMs (many contributors per tile), several waves + a tail on a few CTAs
    # (one or two contributors, stream-K followed by data-parallel tiles), ragged edges
    cases = [((512, 768, 4096), 0), ((1024, 1536, 1024), 20), ((1000, 1224, 2048), 28), ((384, 4096, 8192), 0),
             ((2048, 2048, 512), 36)]
    for (m, n, k), max_ctas in cases:
        a, bt = oracle.fill_zero_one((m, k), 3, 21), oracle.fill_zero_one((n, k), 3, 22)
        want = oracle.hgemm_f32acc(a, bt, fast=True)
        da, dbt = dev(a), dev(bt)
        for c in plain:
            if c["cta_group"] == 2 and m <= 128:
                continue
            for mode in (capi.STREAMK_TAIL, capi.STREAMK_TAIL_PLUS_WAVE):
                sched = capi.schedule(c["id"], m, n, k, mode, max_ctas or 132)
                for _ in range(2):
                    got = run(da, dbt, acc, cfg=c["id"], splits=mode, max_ctas=max_ctas).cpu().numpy()
                    assert np.array_equal(got, want), (acc, c, mode, m, n, k, max_ctas, sched["sk_tiles"])
    # the cases above are not vacuous: most (config, case) pairs do run a stream-K schedule
    active = sum(capi.schedule(c["id"], m, n, k, capi.STREAMK_TAIL, mc or 132)["sk_tiles"] > 0
                 for c in plain for (m, n, k), mc in cases)
    assert active >= len(plain) * len(cases) // 2
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randn((512, 8192), device="cuda", generator=g).half()
    bt = torch.randn((2048, 8192), device="cuda", generator=g).half()
    for cfg in (0, 3):
        first = run(a, bt, acc, cfg=cfg, splits=capi.STREAMK_TAIL)
        plain_c = run(a, bt, acc, cfg=cfg)
        for _ in range(3):
            assert torch.equal(run(a, bt, acc, cfg=cfg, splits=capi.STREAMK_TAIL), first)
        # a different summation grouping, not a different result. fp32 accumulation: within one fp16 ulp of the unsplit
        # kernel at these magnitudes (|c| < 512: ulp 0.25). fp16 accumulation: both runs re-round a running sum of
        # magnitude ~sqrt(K) = 90..400 to fp16 (ulp 0.06..0.25) some K/16 = 512 times, in different groupings — two
        # random walks of half-ulps; bound 8 = 32 ulps at 256..512
        err = (first.float() - plain_c.float()).abs()
        assert float(err.max()) <= (0.25 if acc == "fp32" else 8.0), float(err.max())


@pytest.mark.parametrize("acc", ACCS)
def test_randn_golden_within_stated_tolerance(randn_cases, acc):
    for c in randn_cases:
        got = run(dev(c["a"]), dev(c["b"].T), acc).cpu().numpy().astype(np.float32)
        truth = c["truth"].astype(np.float32)
        if acc == "fp32":
            tol = 2.0**-10 * np.abs(truth) + 2.0**-10 * np.sqrt(c["k"]) * 0.05 + 1e-3
        else:
            tol = 2.0**-11 * np.sqrt(max(c["k"] / 16.0, 1.0)) * 2.0 * (np.abs(truth) + np.sqrt(c["k"])) + 1e-3
        assert (np.abs(got - truth) <= tol).all(), (acc, c["m"], c["n"], c["k"], float(np.abs(got - truth).max()))


@pytest.mark.parametrize("acc", ACCS)
def test_guard_bands_untouched_and_c_fully_overwritten(acc):
    # the reference's OOB-write probe (zero_one_correctness_check.py:101-150) on ragged and tile-aligned shapes
    for (m, n, k) in [(200, 328, 72), (128, 256, 64), (1000, 1000, 1000), (64, 4096, 64)]:
        ga, gbt, gc = zc.GuardedOperand(m, k, "cuda"), zc.GuardedOperand(n, k, "cuda"), zc.GuardedOperand(m, n, "cuda")
        ga.view.copy_(dev(oracle.fill_zero_one((m, k), 2, 3)))
        gbt.view.copy_(dev(oracle.fill_zero_one((n, k), 2, 4)))
        gc.view.fill_(float("nan"))
        capi.hgemm(ga.view, gbt.view.reshape(k, n), gc.view, acc)
        torch.cuda.synchronize()
        assert ga.bands_intact() and gbt.bands_intact() and gc.bands_intact()
        assert not torch.isnan(gc.view).any()
        want = oracle.hgemm_f32acc(ga.view.cpu().numpy(), gbt.view.cpu().numpy(), fast=True)
        assert np.array_equal(gc.view.cpu().numpy(), want)


@pytest.mark.parametrize("acc,mnk", [("fp32", (4096, 4096, 4096)), ("fp16", (8192, 8192, 8192)),
                                     ("fp32", (2048, 11008, 4096)), ("fp32", (64, 4096, 64)), ("fp16", (64, 4096, 64))])
def test_baseline_configs_pass_the_reference_check_procedure(acc, mnk):
    """BASELINE.json configs at FULL size through the harness's own 0/1 procedure (CPU fp32 truth, mask, guard
    bands, == 0 rule), with the C-ABI call in the kernel slot."""
    name = f"cuda_l2_b200_{acc}"

    def kernel(a, b, b_col_major, c):
        capi.hgemm(a, b_col_major, c, acc)
    kernel.__name__ = name
    m, n, k = mnk
    res = zc.run_zero_one_check(kernel_funcs=[torch.matmul, kernel], kernel_under_test_name=name, m=m, n=n, k=k,
                                padding=Padding(), device="cuda", num_iterations=2, max_seconds=120,
                                generator=torch.Generator(device="cuda").manual_seed(0))
    assert res.success, res.message


@pytest.mark.parametrize("acc", ACCS)
def test_size_independent_properties_at_full_size(acc):
    """Properties that need no CPU reference, at 8192-class sizes: identity, exact power-of-two scaling,
    row-block decomposition, row-sum against a ones matrix."""
    n = k = 4096
    m = 8192
    g = torch.Generator(device="cuda").manual_seed(1)
    a = (torch.randint(0, 3, (m, k), device="cuda", generator=g) - 1).half()         # {-1, 0, 1}
    eye_t = torch.eye(n, dtype=torch.half, device="cuda")                              # Bt = I  -> C = A
    assert torch.equal(run(a, eye_t, acc), a)
    bt = (torch.randint(0, 3, (n, k), device="cuda", generator=g) - 1).half()
    c = run(a, bt, acc)
    assert torch.equal(run(a * 2, bt, acc), c * 2)                                     # scaling by 2 is exact
    assert torch.equal(run(a[1024:3072].contiguous(), bt, acc), c[1024:3072])          # rows are independent
    ones_t = torch.ones((64, k), dtype=torch.half, device="cuda")
    small = (torch.rand((m, k), device="cuda", generator=g) < 0.25).half()            # row sums ~1024 < 2048: exact
    rs = run(small, ones_t, acc)
    assert torch.equal(rs[:, 0].float(), small.float().sum(dim=1))
    assert torch.equal(rs, rs[:, :1].expand(-1, 64))


def test_host_buffer_entry_point_round_trips():
    # small: one copy in, one GEMM, one copy out; large: B first, then A / GEMM / C in four pipelined row blocks
    # (ragged M: the last block is shorter), from pinned and from pageable memory, twice (streams and events are reused)
    for (m, n, k), acc in (((512, 768, 256), "fp32"), ((4096, 2048, 1024), "fp32"), ((3000, 1224, 2048), "fp16")):
        a_np, bt_np = oracle.fill_zero_one((m, k), 3, 5), oracle.fill_zero_one((n, k), 3, 6)
        want = oracle.hgemm_f32acc(a_np, bt_np, fast=True)
        for pinned in (True, False):
            a, bt = torch.from_numpy(a_np.copy()), torch.from_numpy(bt_np.copy())
            c = torch.full((m, n), float("nan"), dtype=torch.half)
            if pinned:
                a, bt, c = a.pin_memory(), bt.pin_memory(), c.pin_memory()
            for _ in range(2):
                c.fill_(float("nan"))
                capi.hgemm_host(a, bt.reshape(k, n), c, acc)
                assert np.array_equal(c.numpy(), want), (m, n, k, acc, pinned)


def test_errors_are_loud():
    a = torch.zeros((64, 60), dtype=torch.half, device="cuda")       # K % 8 != 0
    with pytest.raises(capi.B200HgemmError):
        capi.hgemm(a, torch.zeros((60, 64), dtype=torch.half, device="cuda"),
                   torch.zeros((64, 64), dtype=torch.half, device="cuda"))
    with pytest.raises(capi.B200HgemmError):                           # shape mismatch
        capi.hgemm(torch.zeros((64, 64), dtype=torch.half, device="cuda"),
                   torch.zeros((32, 64), dtype=torch.half, device="cuda"),
                   torch.zeros((64, 64), dtype=torch.half, device="cuda"))
