"""Round-2 parity tests on the H100: the top of the shape grid at full size through the reference's procedure, the
fp16-accumulate path against the oracle's fp16 model, the bf16 variant, concurrent / captured split-K launches, and
the deployable operator."""
import numpy as np
import pytest
import torch

import oracle
from cuda_l2_b200 import capi, ops
from cuda_l2_b200.harness import correctness as zc
from cuda_l2_b200.harness.common import Padding

pytestmark = pytest.mark.gpu


def dev(x: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.fixture(scope="module", autouse=True)
def _need_h100(built_libs):
    assert torch.cuda.is_available() and torch.cuda.get_device_capability() == (9, 0)
    before = capi.launch_count()
    yield
    assert capi.launch_count() > before, "no kernel of libb200_hgemm.so was launched"


@pytest.mark.parametrize("acc,mnk", [("fp32", (16384, 16384, 16384)), ("fp32", (12288, 16384, 64)),
                                     ("fp16", (16384, 8192, 12288)), ("fp32", (64, 64, 16384))])
def test_top_of_the_grid_passes_the_reference_check_procedure(acc, mnk):
    """The 12288/16384 class at FULL size through the harness's 0/1 procedure — {0,0,1} operand density because
    max(M,N,K) > 8192 (zero_one_correctness_check.py:65-73), CPU fp32 truth, |truth| > 2047 masked, guard bands,
    == 0 rule — with the dispatcher's own choice for the shape (512-row pair tiles, L2 hints, split-K) in the kernel slot."""
    name = f"cuda_l2_b200_{acc}"

    def kernel(a, b, b_col_major, c):
        capi.hgemm(a, b_col_major, c, acc)
    kernel.__name__ = name
    m, n, k = mnk
    res = zc.run_zero_one_check(kernel_funcs=[torch.matmul, kernel], kernel_under_test_name=name, m=m, n=n, k=k,
                                padding=Padding(), device="cuda", num_iterations=1, max_seconds=300,
                                generator=torch.Generator(device="cuda").manual_seed(0))
    assert res.success, res.message


def test_wide_tiles_and_multicast_pairs_are_exact_on_their_own_shapes():
    """Configurations 20-30 (CTA pairs in multicast clusters, 512-row tiles) on shapes that give every CTA of the
    cluster real work, several waves and ragged edges: bit-exact against the oracle, both accumulators."""
    shapes = [(2048, 2048, 512), (1536, 1280, 2112), (1000, 1224, 2048), (4096, 1024, 1024)]
    wide = [c for c in capi.configs() if c["id"] >= 20]
    assert len(wide) >= 11
    for (m, n, k) in shapes:
        a, bt = oracle.fill_zero_one((m, k), 3, m + k), oracle.fill_zero_one((n, k), 3, n + 5 * k)
        want = oracle.hgemm_f32acc(a, bt, fast=True)
        da, dbt = dev(a), dev(bt)
        for cfg in wide:
            for acc in ("fp32", "fp16"):
                for gm in (0, 2):
                    c = torch.full((m, n), float("nan"), dtype=torch.half, device="cuda")
                    capi.hgemm_config(da, dbt.reshape(k, n), c, cfg["id"], acc, group_m=gm)
                    torch.cuda.synchronize()
                    assert np.array_equal(c.cpu().numpy(), want), (cfg, acc, gm, m, n, k)


def test_fp16_accumulation_matches_the_oracles_fp16_model_on_a_non_saturating_domain():
    """fp16-accumulate kernels against oracle.hgemm_f16acc (accumulator re-rounded to fp16 every 16 products) on signed
    small integers: every partial sum stays an integer below 2048, so the fp16 running sum is exact in ANY order and the
    model pins the result bit for bit (outside this domain the tensor core's internal order is unspecified)."""
    rng = np.random.default_rng(7)
    for (m, n, k) in [(256, 512, 4096), (200, 328, 1096), (1024, 1024, 2048), (64, 64, 16384)]:
        a = rng.integers(-3, 4, size=(m, k)).astype(np.float16)
        bt = rng.integers(-3, 4, size=(n, k)).astype(np.float16)
        want16 = oracle.hgemm_f16acc(a, bt, chunk=16)
        want32 = oracle.hgemm_f32acc(a, bt, fast=True)
        assert np.abs(want32.astype(np.float32)).max() < 2048 and np.array_equal(want16, want32)   # the domain is exact
        c = torch.full((m, n), float("nan"), dtype=torch.half, device="cuda")
        capi.hgemm(dev(a), dev(bt).reshape(k, n), c, "fp16")
        torch.cuda.synchronize()
        assert np.array_equal(c.cpu().numpy(), want16), (m, n, k)
    # and where fp16 accumulation does lose bits (0/1 operands, sums far above 2048) it must still sit inside the
    # model's envelope: exact fp32 sum +- one fp16 ulp per re-rounding step that can have happened at that magnitude
    m, n, k = 128, 256, 16384
    a, bt = oracle.fill_zero_one((m, k), 2, 3), oracle.fill_zero_one((n, k), 2, 4)
    exact = a.astype(np.float32) @ bt.astype(np.float32).T          # ~4096 +- 64: integers, exact in fp32
    c = torch.empty((m, n), dtype=torch.half, device="cuda")
    capi.hgemm(dev(a), dev(bt).reshape(k, n), c, "fp16")
    torch.cuda.synchronize()
    got = c.cpu().numpy().astype(np.float32)
    assert np.isfinite(got).all() and np.abs(got - exact).max() <= 4.0 * (k / 16) ** 0.5 * 4


def test_bf16_variant_matches_the_oracle(bf16_cases):
    """bf16 x bf16 -> fp32 accumulate -> bf16 (this repository's extension): bit-exact on the integer fixtures and for
    every configuration on 0/1 operands with K <= 256; within a bf16 ulp + summation noise on N(0,1) operands."""
    def run(a_bits, bt_bits, cfg=None):
        a = torch.from_numpy(a_bits.view(np.int16)).cuda().view(torch.bfloat16)
        bt = torch.from_numpy(np.ascontiguousarray(bt_bits).view(np.int16)).cuda().view(torch.bfloat16)
        c = torch.full((a.shape[0], bt.shape[0]), float("nan"), dtype=torch.bfloat16, device="cuda")
        capi.gemm_kmajor(a, bt, c, "fp32", config_id=cfg)
        torch.cuda.synchronize()
        return c.view(torch.int16).cpu().numpy().view(np.uint16)
    for c in bf16_cases:
        if c["k"] % 8 or c["n"] % 8:
            continue
        got = run(c["a"], np.ascontiguousarray(c["b"].T))
        if c["kind"] == "randn":
            g, t = oracle.bf16_bits_to_f32(got), oracle.bf16_bits_to_f32(c["truth"])
            assert (np.abs(g - t) <= 2.0**-7 * np.abs(t) + 1e-2).all(), (c["m"], c["n"], c["k"])
        else:
            assert np.array_equal(got, c["truth"]), (c["m"], c["n"], c["k"], c["kind"])
    rng = np.random.default_rng(1)
    for (m, n, k) in [(256, 256, 64), (200, 328, 72), (1000, 1000, 256), (512, 768, 192)]:
        a = oracle.f32_to_bf16_bits(rng.integers(0, 2, size=(m, k)).astype(np.float32))
        bt = oracle.f32_to_bf16_bits(rng.integers(0, 2, size=(n, k)).astype(np.float32))
        want = oracle.bgemm_f32acc(a, bt)
        for cfg in capi.configs():
            assert np.array_equal(run(a, bt, cfg["id"]), want), (cfg, m, n, k)
    # a split-K class problem (cluster reduction in fp32, one conversion to bf16): signed integers keep |c| <= 256
    a = oracle.f32_to_bf16_bits(rng.integers(-1, 2, size=(64, 4096)).astype(np.float32))
    bt = oracle.f32_to_bf16_bits(rng.integers(-1, 2, size=(128, 4096)).astype(np.float32))
    want = oracle.bgemm_f32acc(a, bt)
    assert np.abs(oracle.bf16_bits_to_f32(want)).max() <= 256
    assert np.array_equal(run(a, bt), want)


def test_split_k_launches_may_overlap_and_survive_graph_capture():
    """Workspace split-K waits for sibling CTAs of its own grid; it is launched cooperatively, so two such grids on
    different streams (each with its own scratch) cannot starve each other. Inside a CUDA-graph capture a first-use
    allocation is impossible: after prewarm the split-K kernel is captured, without it the undivided schedule is."""
    m, n, k = 128, 64, 16384
    a, bt = oracle.fill_zero_one((m, k), 3, 11), oracle.fill_zero_one((n, k), 3, 12)
    want = oracle.hgemm_f32acc(a, bt, fast=True)
    da, dbt = dev(a), dev(bt).reshape(k, n)
    cfg = next(c["id"] for c in capi.configs() if c["cta_group"] == 1 and c["bn"] == 64 and c["cluster_m"] * c["cluster_n"] == 1)
    streams = [torch.cuda.Stream() for _ in range(3)]
    outs = [torch.full((m, n), float("nan"), dtype=torch.half, device="cuda") for _ in streams]
    torch.cuda.synchronize()
    for _ in range(20):
        for s, c in zip(streams, outs):
            capi.hgemm_config(da, dbt, c, cfg, "fp32", splits=16, stream=s.cuda_stream)
    torch.cuda.synchronize()
    for c in outs:
        assert np.array_equal(c.cpu().numpy(), want)
    # graph capture on a fresh stream: no scratch yet -> undivided schedule captured, still exact
    for prewarm in (False, True):
        s = torch.cuda.Stream()
        c = torch.full((m, n), float("nan"), dtype=torch.half, device="cuda")
        if prewarm:
            capi.prewarm(s.cuda_stream)
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            capi.hgemm_config(da, dbt, c, cfg, "fp32", splits=16, stream=torch.cuda.current_stream().cuda_stream)
        for _ in range(3):
            c.fill_(float("nan"))
            g.replay()
            torch.cuda.synchronize()
            assert np.array_equal(c.cpu().numpy(), want), prewarm
    capi.release()
    c = torch.full((m, n), float("nan"), dtype=torch.half, device="cuda")
    capi.hgemm_config(da, dbt, c, cfg, "fp32", splits=16)          # scratch is re-allocated on demand after a release
    torch.cuda.synchronize()
    assert np.array_equal(c.cpu().numpy(), want)


def test_back_to_back_launches_with_dependent_data_are_ordered():
    """Programmatic dependent launch lets a GEMM's prologue overlap the previous kernel's tail; its loads must still
    see everything earlier kernels of the stream wrote. Chain: C1 = A B, C2 = C1 B2 (reads C1), repeated back to back
    with no host synchronisation, operands rewritten by torch kernels in between; compared with the oracle."""
    m, k, n = 512, 256, 256
    rng = np.random.default_rng(5)
    a = rng.integers(0, 2, size=(m, k)).astype(np.float16)
    bt = (rng.integers(0, 8, size=(n, k)) == 0).astype(np.float16)         # sparse 0/1: C1 entries ~32 < 2048
    b2t = (rng.integers(0, 8, size=(n, n)) == 0).astype(np.float16)
    c1_want = oracle.hgemm_f32acc(a, bt, fast=True)
    c2_want = oracle.hgemm_f32acc(c1_want, b2t, fast=True)
    assert np.abs(c2_want.astype(np.float32)).max() <= 2047
    da, dbt, db2t = dev(a), dev(bt).reshape(k, n), dev(b2t).reshape(n, n)
    c1 = torch.empty((m, n), dtype=torch.half, device="cuda")
    c2 = torch.empty((m, n), dtype=torch.half, device="cuda")
    for it in range(50):
        c1.fill_(float("nan")); c2.fill_(float("nan"))      # torch kernels between ours, same stream
        capi.hgemm(da, dbt, c1, "fp32")
        capi.hgemm(c1, db2t, c2, "fp32")
        capi.hgemm(da, dbt, c1, "fp16")                      # overwrites C1 right after the kernel that read it
    torch.cuda.synchronize()
    assert np.array_equal(c2.cpu().numpy(), c2_want) and np.array_equal(c1.cpu().numpy(), c1_want)


def test_operator_and_linear_drop_in():
    """torch.ops.cuda_l2_b200.hgemm and B200Linear: exact against the oracle on 0/1 data (nn.Linear weight layout IS the
    K-major operand), any leading dimensions, bias, bf16, module replacement against nn.Linear, autograd."""
    m, k, n = 300, 512, 1024
    a, w = oracle.fill_zero_one((m, k), 2, 1), oracle.fill_zero_one((n, k), 2, 2)
    want = oracle.hgemm_f32acc(a, w, fast=True)
    for acc in ("fp32", "fp16"):
        got = ops.hgemm(dev(a), dev(w), acc)
        assert np.array_equal(got.cpu().numpy(), want)
    lin = ops.B200Linear(k, n, bias=True, device="cuda")
    with torch.no_grad():
        lin.weight.copy_(dev(w)); lin.bias.copy_(torch.arange(n, device="cuda").remainder(5).half())
    x = dev(a).view(3, 100, k)
    with torch.no_grad():
        y = lin(x)
    assert y.shape == (3, 100, n)
    want_b = (want.astype(np.float32) + (np.arange(n) % 5).astype(np.float32)).astype(np.float16)
    assert np.array_equal(y.reshape(m, n).cpu().numpy(), want_b)
    # drop-in: a small MLP, every eligible nn.Linear replaced, outputs within fp16 rounding of torch's own
    torch.manual_seed(0)
    for dt in (torch.float16, torch.bfloat16):
        mlp = torch.nn.Sequential(torch.nn.Linear(512, 2048), torch.nn.GELU(), torch.nn.Linear(2048, 512)).to("cuda", dt)
        xin = torch.randn(4, 77, 512, device="cuda", dtype=dt)
        with torch.no_grad():
            ref = mlp(xin).float()
            assert ops.replace_linear_modules(mlp) == ["0", "2"]
            out = mlp(xin).float()
        tol = 2e-2 if dt == torch.float16 else 1.5e-1
        assert (out - ref).abs().max() <= tol * max(1.0, float(ref.abs().max())), float((out - ref).abs().max())
    # autograd through the op (fp32 reference with tolerance); explicit enable_grad: harness code run earlier in the same
    # session may have switched autograd off globally, as the reference's scripts do (benchmarking_utils.py:9)
    with torch.enable_grad():
        xa = torch.randn(64, 256, device="cuda", dtype=torch.half, requires_grad=True)
        wa = (torch.randn(128, 256, device="cuda", dtype=torch.half) * 0.1).requires_grad_()
        ops.hgemm(xa, wa).float().square().sum().backward()
        xr, wr = xa.detach().float().requires_grad_(), wa.detach().float().requires_grad_()
        (xr @ wr.t()).square().sum().backward()
    assert torch.allclose(xa.grad.float(), xr.grad, rtol=3e-2, atol=0.5)
    assert torch.allclose(wa.grad.float(), wr.grad, rtol=3e-2, atol=0.5)
    with pytest.raises(capi.B200HgemmError):
        ops.hgemm(xa.detach(), torch.zeros(128, 200, device="cuda", dtype=torch.half))
