"""Batched fp16 / bf16 GEMM on the H100 (libb200_batched.so).

The anchor: a batched launch runs the 2-D kernel's main loop unchanged, only the tensor maps gain a batch coordinate
and the schedule a batch index. So on N(0,1) data every matrix of a batched launch must be BIT-IDENTICAL to the 2-D
kernel (b200_hgemm_run_config / b200_bgemm_run_config) with the same configuration and group_m on that matrix's
operands: for all 31 configurations x 3 types, ragged M (a tile at the bottom of one matrix would read the next
matrix's rows through a 2-D map), different data per matrix, and a CTA cap that makes workers cross matrices. Then:
exactness against the C oracle, the masked form (rows below the count as the 2-D call computes them with NaN in the
padding rows of A; rows from round_up(count, 16) untouched; all counts zero writes nothing), counts written by a torch
kernel just before the launch and changed between CUDA-graph replays, guard bands, the operator against torch.bmm,
gradients, and B = 1 against the 2-D operator.

Tolerances against torch.bmm (an fp32 product of the same 16-bit operands): max |C - ref| / rms(ref) of at most
FP16_TOL for fp16 output with fp32 accumulation (the one output rounding: 2^-11 relative, on values up to about five
rms), BF16_TOL for bf16 output (2^-8 relative), FP16_ACC16_TOL with fp16 accumulation over K = 1024; gradients
GRAD_TOL, their output gradient having been rounded to the operand type first.
"""
import numpy as np
import pytest
import torch

import oracle
from cuda_l2_b200 import capi, ops

pytestmark = pytest.mark.gpu

NUM_CONFIGS = 31
VARIANTS = {0: (torch.float16, "fp32"), 1: (torch.float16, "fp16"), 2: (torch.bfloat16, "fp32")}
FP16_TOL, BF16_TOL, FP16_ACC16_TOL = 0.005, 0.03, 0.1
GRAD_TOL = {torch.float16: 0.01, torch.bfloat16: 0.05}   # the fp16 / bf16 output gradient is rounded once more
SENTINEL = 0x7BCD          # a finite fp16 / bf16 bit pattern no product here produces by accident


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def randn(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, device="cuda", generator=g).to(dtype)


def sentinel(shape, dtype):
    return torch.full(shape, SENTINEL, dtype=torch.int16, device="cuda").view(dtype)


def bits(x):
    return x.view(torch.int16)


def run_2d(a, bt, c, variant, config_id, group_m=0):
    dtype, acc = VARIANTS[variant]
    capi.gemm_kmajor(a, bt, c, acc, config_id=config_id, group_m=group_m, splits=1)


def cta_count(config_id):
    c = capi.configs()[config_id]
    return c["cta_group"] * c["cluster_m"] * c["cluster_n"]


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("config_id", range(NUM_CONFIGS))
def test_every_matrix_is_bit_identical_to_the_2d_kernel(config_id, variant):
    dtype, acc = VARIANTS[variant]
    bsz, m, n, k = 3, 700, 520, 136          # M is no multiple of any tile: the last tile of a matrix is ragged
    a = randn((bsz, m, k), dtype, 10 * config_id + variant)
    bt = randn((bsz, n, k), dtype, 10 * config_id + variant + 5)
    want = torch.empty((bsz, m, n), dtype=dtype, device="cuda")
    for i in range(bsz):
        run_2d(a[i], bt[i], want[i], variant, config_id)
    # workers cross matrices: all SMs, and a cap of two workers (each walks tiles of every matrix)
    for max_ctas in (0, 2 * cta_count(config_id)):
        c = sentinel((bsz, m, n), dtype)
        capi.gemm_batched(a, bt, c, acc, config_id=config_id, max_ctas=max_ctas)
        torch.cuda.synchronize()
        assert torch.equal(bits(c), bits(want)), (config_id, variant, max_ctas)


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_group_m_and_tiny_matrices_match_the_2d_kernel(variant):
    dtype, acc = VARIANTS[variant]
    for config_id in (0, 4, 9, 26, 30):
        for (bsz, m, n, k, gm) in ((5, 1, 8, 8, 0), (9, 37, 64, 64, 3), (4, 513, 264, 200, 1)):
            a, bt = randn((bsz, m, k), dtype, m + config_id), randn((bsz, n, k), dtype, n + config_id)
            want = torch.empty((bsz, m, n), dtype=dtype, device="cuda")
            for i in range(bsz):
                run_2d(a[i], bt[i], want[i], variant, config_id, gm)
            c = sentinel((bsz, m, n), dtype)
            capi.gemm_batched(a, bt, c, acc, config_id=config_id, group_m=gm, max_ctas=cta_count(config_id))
            torch.cuda.synchronize()
            assert torch.equal(bits(c), bits(want)), (config_id, bsz, m, n, k, gm)


def test_bit_exact_against_the_oracle():
    bsz, m, n, k = 4, 200, 328, 72
    rng = np.random.default_rng(7)
    a = [oracle.fill_zero_one((m, k), 2, seed=11 + i) for i in range(bsz)]
    bt = [oracle.fill_zero_one((n, k), 2, seed=31 + i) for i in range(bsz)]
    ta, tb = torch.from_numpy(np.stack(a)).cuda(), torch.from_numpy(np.stack(bt)).cuda()
    for variant, truth in ((0, lambda x, y: oracle.hgemm_f32acc(x, y, fast=True)), (1, oracle.hgemm_f16acc)):
        for config_id in (None, 1, 3, 11, 27):
            c = sentinel((bsz, m, n), torch.float16)
            capi.gemm_batched(ta, tb, c, VARIANTS[variant][1], config_id=config_id)
            torch.cuda.synchronize()
            got = c.cpu().numpy()
            for i in range(bsz):
                assert np.array_equal(got[i].view(np.uint16), truth(a[i], bt[i]).view(np.uint16)), (variant, config_id, i)
    # bf16 on small integers (|values| <= 3, K = 72): every sum is exact in fp32, and both sides round it once to bf16
    ab = [oracle.f32_to_bf16_bits(rng.integers(-3, 4, size=(m, k)).astype(np.float32)) for _ in range(bsz)]
    bb = [oracle.f32_to_bf16_bits(rng.integers(-3, 4, size=(n, k)).astype(np.float32)) for _ in range(bsz)]
    ta = torch.from_numpy(np.stack(ab).view(np.int16)).cuda().view(torch.bfloat16)
    tb = torch.from_numpy(np.stack(bb).view(np.int16)).cuda().view(torch.bfloat16)
    for config_id in (None, 0, 6, 29):
        c = sentinel((bsz, m, n), torch.bfloat16)
        capi.gemm_batched(ta, tb, c, "fp32", config_id=config_id)
        torch.cuda.synchronize()
        got = bits(c).cpu().numpy().view(np.uint16)
        for i in range(bsz):
            assert np.array_equal(got[i], oracle.bgemm_f32acc(ab[i], bb[i])), (config_id, i)


def masked_reference(a, bt, counts, variant, config_id):
    """Per matrix, the 2-D kernel on the rows below the count (None where there are none)."""
    out = []
    for i, cnt in enumerate(counts):
        r = min(max(cnt, 0), a.shape[1])
        if r == 0:
            out.append(None)
            continue
        c = torch.empty((r, bt.shape[1]), dtype=a.dtype, device="cuda")
        run_2d(a[i, :r].contiguous(), bt[i], c, variant, config_id)
        out.append(c)
    return out


def check_masked(c, ref, counts, m):
    for i, cnt in enumerate(counts):
        r = min(max(cnt, 0), m)
        if r:
            assert torch.equal(bits(c[i, :r]), bits(ref[i])), (i, cnt)
        untouched = bits(c[i, -(-r // 16) * 16:])
        assert bool((untouched == SENTINEL).all()), (i, cnt)


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_masked_rows_match_and_nothing_past_them_is_written(variant):
    dtype, acc = VARIANTS[variant]
    bsz, m, n, k = 8, 600, 264, 200
    counts = [0, 600, 777, -4, 1, 17, 256, 433]
    a = randn((bsz, m, k), dtype, 99 + variant)
    for i, cnt in enumerate(counts):
        a[i, max(cnt, 0):] = float("nan")       # padding rows: their values must not reach the rows below the count
    bt = randn((bsz, n, k), dtype, 199 + variant)
    mm = torch.tensor(counts, dtype=torch.int32, device="cuda")
    for config_id in range(NUM_CONFIGS):
        ref = masked_reference(a, bt, counts, variant, config_id)
        for max_ctas in (0, 2 * cta_count(config_id)):
            c = sentinel((bsz, m, n), dtype)
            capi.gemm_batched(a, bt, c, acc, masked_m=mm, config_id=config_id, max_ctas=max_ctas)
            torch.cuda.synchronize()
            check_masked(c, ref, counts, m)
    # the dispatched call and the operator take the same path
    c = sentinel((bsz, m, n), dtype)
    capi.gemm_batched(a, bt, c, acc, masked_m=mm)
    cid, gm = capi.batched_select(variant, bsz, m, n, k)
    ref = masked_reference(a, bt, counts, variant, cid)
    torch.cuda.synchronize()
    check_masked(c, ref, counts, m)
    y = ops.hgemm_batched(a, bt, acc, mm)
    for i, cnt in enumerate(counts):
        r = min(max(cnt, 0), m)
        if r:
            assert torch.equal(bits(y[i, :r]), bits(ref[i]))


def test_all_counts_zero_writes_nothing():
    before = capi.batched_launch_count()
    for config_id in range(NUM_CONFIGS):
        a, bt = randn((6, 300, 64), torch.float16, 1), randn((6, 128, 64), torch.float16, 2)
        c = sentinel((6, 300, 128), torch.float16)
        capi.gemm_batched(a, bt, c, "fp32", masked_m=torch.zeros(6, dtype=torch.int32, device="cuda"),
                          config_id=config_id)
        torch.cuda.synchronize()
        assert bool((bits(c) == SENTINEL).all()), config_id
    assert capi.batched_launch_count() - before == NUM_CONFIGS     # launched, and its kernel found no tile


def test_counts_written_by_a_kernel_just_before_the_launch():
    bsz, m, n, k = 16, 256, 256, 128
    a, bt = randn((bsz, m, k), torch.float16, 3), randn((bsz, n, k), torch.float16, 4)
    full = torch.empty((bsz, m, n), dtype=torch.float16, device="cuda")
    capi.gemm_batched(a, bt, full, "fp32", config_id=1)
    base = torch.arange(bsz, dtype=torch.int32, device="cuda") * 37
    mm = torch.empty(bsz, dtype=torch.int32, device="cuda")
    outs = []
    for it in range(40):
        # a torch kernel on the same stream writes the counts; the GEMM's prologue may overlap it, its reads may not
        torch.remainder(base * (it + 1) + 11 * it, m + 40, out=mm)
        c = sentinel((bsz, m, n), torch.float16)
        capi.gemm_batched(a, bt, c, "fp32", masked_m=mm, config_id=1, stream=torch.cuda.current_stream().cuda_stream)
        outs.append(c)
    torch.cuda.synchronize()
    for it, c in enumerate(outs):
        counts = [int(x) for x in ((np.arange(bsz) * 37) * (it + 1) + 11 * it) % (m + 40)]
        check_masked(c, [full[i, :min(cnt, m)] for i, cnt in enumerate(counts)], counts, m)


def test_cuda_graph_replays_read_the_current_counts():
    bsz, m, n, k = 8, 384, 512, 256
    a, bt = randn((bsz, m, k), torch.bfloat16, 5), randn((bsz, n, k), torch.bfloat16, 6)
    full = torch.empty((bsz, m, n), dtype=torch.bfloat16, device="cuda")
    capi.gemm_batched(a, bt, full, "fp32", config_id=4)
    mm = torch.full((bsz,), m, dtype=torch.int32, device="cuda")
    c = sentinel((bsz, m, n), torch.bfloat16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up outside the capture (attributes, tensor maps)
        capi.gemm_batched(a, bt, c, "fp32", masked_m=mm, config_id=4, stream=s.cuda_stream)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        capi.gemm_batched(a, bt, c, "fp32", masked_m=mm, config_id=4,
                          stream=torch.cuda.current_stream().cuda_stream)
    rng = np.random.default_rng(8)
    for _ in range(6):
        counts = [int(x) for x in rng.integers(-20, m + 50, size=bsz)]
        mm.copy_(torch.tensor(counts, dtype=torch.int32))
        c.copy_(sentinel((bsz, m, n), torch.bfloat16))
        g.replay()
        torch.cuda.synchronize()
        check_masked(c, [full[i, :min(max(cnt, 0), m)] for i, cnt in enumerate(counts)], counts, m)


def test_guard_bands_around_c():
    for variant, (dtype, acc) in VARIANTS.items():
        bsz, m, n, k = 3, 77, 72, 64
        a, bt = randn((bsz, m, k), dtype, 12), randn((bsz, n, k), dtype, 13)
        guard = 4096
        buf = sentinel((2 * guard + bsz * m * n,), dtype)
        c = buf[guard:guard + bsz * m * n].view(bsz, m, n)
        for config_id in (0, 3, 14, 26, 29):
            capi.gemm_batched(a, bt, c, acc, config_id=config_id)
            capi.gemm_batched(a, bt, c, acc, config_id=config_id,
                              masked_m=torch.tensor([5, 77, 100], dtype=torch.int32, device="cuda"))
        torch.cuda.synchronize()
        assert bool((bits(buf[:guard]) == SENTINEL).all()) and bool((bits(buf[guard + bsz * m * n:]) == SENTINEL).all())


@pytest.mark.parametrize("dtype,acc,tol", [(torch.float16, "fp32", FP16_TOL), (torch.float16, "fp16", FP16_ACC16_TOL),
                                           (torch.bfloat16, "fp32", BF16_TOL)])
def test_operator_against_torch_bmm(dtype, acc, tol):
    for (bsz, m, n, k) in ((8, 256, 512, 1024), (64, 1024, 128, 64), (5, 333, 200, 1024)):
        a, bt = randn((bsz, m, k), dtype, m), randn((bsz, n, k), dtype, n)
        ref = torch.bmm(a.float(), bt.float().transpose(1, 2))
        got = ops.hgemm_batched(a, bt, acc)
        assert got.shape == (bsz, m, n) and got.dtype == dtype
        err = float((got.float() - ref).abs().max() / ref.pow(2).mean().sqrt())
        assert err <= tol, (bsz, m, n, k, err)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_gradients_against_torch_bmm(dtype):
    bsz, m, n, k = 4, 64, 128, 96
    a = randn((bsz, m, k), dtype, 20).requires_grad_(True)
    bt = randn((bsz, n, k), dtype, 21).requires_grad_(True)
    w = randn((bsz, m, n), torch.float32, 22)
    (ops.hgemm_batched(a, bt).float() * w).sum().backward()
    a32, bt32 = a.detach().float().requires_grad_(True), bt.detach().float().requires_grad_(True)
    (torch.bmm(a32, bt32.transpose(1, 2)) * w).sum().backward()
    tol = GRAD_TOL[dtype]
    for got, ref in ((a.grad, a32.grad), (bt.grad, bt32.grad)):
        assert got.dtype == dtype and got.shape == ref.shape
        assert float((got.float() - ref).abs().max() / ref.pow(2).mean().sqrt()) <= tol
    # the masked form is inference only
    x = randn((bsz, m, k), dtype, 23).requires_grad_(True)
    y = ops.hgemm_batched(x, bt.detach(), "fp32", torch.full((bsz,), 10, dtype=torch.int32, device="cuda"))
    with pytest.raises(capi.B200HgemmError):
        y.sum().backward()


def test_single_matrix_against_the_2d_operator():
    for dtype, acc in VARIANTS.values():
        for (m, n, k) in ((4096, 4096, 4096), (200, 328, 72), (2048, 11008, 4096)):
            a, bt = randn((m, k), dtype, m + 1), randn((n, k), dtype, n + 1)
            got = ops.hgemm_batched(a[None], bt[None], acc)[0]
            # the 2-D kernel of the configuration the batched dispatcher picked, plain: the same bits
            cid, gm = capi.batched_select(capi.batched_variant(dtype, acc), 1, m, n, k)
            want = torch.empty((m, n), dtype=dtype, device="cuda")
            capi.gemm_kmajor(a, bt, want, acc, config_id=cid, group_m=gm, splits=1)
            torch.cuda.synchronize()
            assert torch.equal(bits(got), bits(want)), (dtype, acc, m, n, k)
            # the 2-D operator may divide K (split-K, stream-K): equal up to the summation order
            ref = ops.hgemm(a, bt, acc).float()
            tol = FP16_ACC16_TOL if acc == "fp16" else FP16_TOL if dtype == torch.float16 else BF16_TOL
            assert float((got.float() - ref).abs().max() / ref.pow(2).mean().sqrt()) <= tol


def test_empty_batches_launch_nothing():
    before = capi.batched_launch_count()
    a = torch.zeros((0, 16, 64), dtype=torch.float16, device="cuda")
    assert ops.hgemm_batched(a, torch.zeros((0, 32, 64), dtype=torch.float16, device="cuda")).shape == (0, 16, 32)
    a = torch.zeros((3, 0, 64), dtype=torch.bfloat16, device="cuda")
    assert ops.hgemm_batched(a, torch.zeros((3, 32, 64), dtype=torch.bfloat16, device="cuda")).shape == (3, 0, 32)
    assert capi.batched_launch_count() == before
