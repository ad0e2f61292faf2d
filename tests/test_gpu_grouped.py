"""Grouped fp16 / bf16 GEMM over contiguous row groups on the H100 (libb200_grouped.so).

The anchor: a grouped launch runs the 2-D kernel's main loop unchanged; only A's box starts at the group's first row,
Bt's map gains a group coordinate, and the store of a box that straddles a group's end is cut at that end. An output
row depends only on its own row of A, so on N(0,1) data every group's rows must be BIT-IDENTICAL to the 2-D kernel
(b200_hgemm_run_config / b200_bgemm_run_config) with the same configuration and group_m on that group's rows of A and
its Bt: for all 31 configurations x 3 types, on ragged offsets (empty groups, one-row groups, sizes that are no multiple
of 16, groups shorter and longer than a tile, rows past the last group), and with a CTA cap that makes workers cross
groups. Then: exactness against the C oracle, rows past the last group's end and guard bands around C untouched (also
for malformed offsets), offsets written by a torch kernel just before the launch and changed between CUDA-graph
replays, one launch per call, and the operator against torch._grouped_mm (bf16) and per-group fp32 torch.matmul.

Tolerances of the operator: max |C - ref| / rms(ref) of at most FP16_TOL for fp16 output with fp32 accumulation (the
one output rounding, 2^-11 relative, on values up to about five rms), BF16_TOL for bf16 output (2^-8 relative; against
torch._grouped_mm, whose own bf16 rounding may differ by one unit in the last place), FP16_ACC16_TOL with fp16
accumulation over K = 1024.
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
SENTINEL = 0x7BCD          # a finite fp16 / bf16 bit pattern no product here produces by accident
# group sizes: empty, one row, no multiple of 16, shorter and longer than every tile (up to 512 rows per pair block)
SIZES = [0, 1, 37, 300, 0, 17, 530, 1, 128, 0, 1100, 15]


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


def cumulative(sizes):
    return [int(x) for x in np.cumsum(sizes)]


def clamped_groups(offs, t):
    out, s = [], 0
    for o in offs:
        e = min(max(o, s), t)
        out.append((s, e))
        s = e
    return out


def offs_tensor(offs):
    return torch.tensor(offs, dtype=torch.int32, device="cuda")


def run_2d(a, bt, c, variant, config_id, group_m=0):
    capi.gemm_kmajor(a, bt, c, VARIANTS[variant][1], config_id=config_id, group_m=group_m, splits=1)


def reference(a, bt, offs, variant, config_id, group_m=0):
    """The 2-D kernel on each group's rows (sentinel elsewhere)."""
    t, n = a.shape[0], bt.shape[1]
    want = sentinel((t, n), a.dtype)
    for g, (s, e) in enumerate(clamped_groups(offs, t)):
        if e > s:
            c = torch.empty((e - s, n), dtype=a.dtype, device="cuda")
            run_2d(a[s:e].contiguous(), bt[g], c, variant, config_id, group_m)
            want[s:e] = c
    return want


def cta_count(config_id):
    c = capi.configs()[config_id]
    return c["cta_group"] * c["cluster_m"] * c["cluster_n"]


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("config_id", range(NUM_CONFIGS))
def test_every_group_is_bit_identical_to_the_2d_kernel(config_id, variant):
    dtype, acc = VARIANTS[variant]
    offs = cumulative(SIZES)
    t, n, k = offs[-1] + 29, 264, 136       # 29 rows past the last group; N ragged for every tile width
    a = randn((t, k), dtype, 10 * config_id + variant)
    bt = randn((len(SIZES), n, k), dtype, 10 * config_id + variant + 5)
    want = reference(a, bt, offs, variant, config_id)
    o = offs_tensor(offs)
    for max_ctas in (0, 2 * cta_count(config_id)):   # all SMs, and two workers that walk every group
        c = sentinel((t, n), dtype)
        capi.gemm_grouped(a, bt, c, o, acc, config_id=config_id, max_ctas=max_ctas)
        torch.cuda.synchronize()
        assert torch.equal(bits(c), bits(want)), (config_id, variant, max_ctas)


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_group_m_and_tiny_groups_match_the_2d_kernel(variant):
    dtype, acc = VARIANTS[variant]
    for config_id in (0, 4, 9, 12, 26, 30):
        for (sizes, n, k, gm) in (([1, 0, 1], 8, 8, 0), ([40, 3, 700, 64], 64, 64, 3), ([513, 257], 264, 200, 1)):
            offs = cumulative(sizes)
            t = offs[-1]
            a, bt = randn((t, k), dtype, t + config_id), randn((len(sizes), n, k), dtype, n + config_id)
            want = reference(a, bt, offs, variant, config_id, gm)
            c = sentinel((t, n), dtype)
            capi.gemm_grouped(a, bt, c, offs_tensor(offs), acc, config_id=config_id, group_m=gm,
                              max_ctas=cta_count(config_id))
            torch.cuda.synchronize()
            assert torch.equal(bits(c), bits(want)), (config_id, sizes, n, k, gm)


def test_bit_exact_against_the_oracle():
    sizes, n, k = [70, 0, 1, 129, 200], 328, 72
    offs = cumulative(sizes)
    t = offs[-1]
    a = oracle.fill_zero_one((t, k), 2, seed=11)
    bt = [oracle.fill_zero_one((n, k), 2, seed=31 + g) for g in range(len(sizes))]
    ta, tb, o = torch.from_numpy(a).cuda(), torch.from_numpy(np.stack(bt)).cuda(), offs_tensor(offs)
    groups = clamped_groups(offs, t)
    for variant, truth in ((0, lambda x, y: oracle.hgemm_f32acc(x, y, fast=True)), (1, oracle.hgemm_f16acc)):
        for config_id in (None, 1, 3, 11, 27):
            c = sentinel((t, n), torch.float16)
            capi.gemm_grouped(ta, tb, c, o, VARIANTS[variant][1], config_id=config_id)
            torch.cuda.synchronize()
            got = c.cpu().numpy()
            for g, (s, e) in enumerate(groups):
                if e > s:
                    assert np.array_equal(got[s:e].view(np.uint16), truth(a[s:e], bt[g]).view(np.uint16)), \
                        (variant, config_id, g)
    # bf16 on small integers (|values| <= 3, K = 72): every sum is exact in fp32, and both sides round it once to bf16
    rng = np.random.default_rng(7)
    ab = oracle.f32_to_bf16_bits(rng.integers(-3, 4, size=(t, k)).astype(np.float32))
    bb = [oracle.f32_to_bf16_bits(rng.integers(-3, 4, size=(n, k)).astype(np.float32)) for _ in sizes]
    ta = torch.from_numpy(ab.view(np.int16)).cuda().view(torch.bfloat16)
    tb = torch.from_numpy(np.stack(bb).view(np.int16)).cuda().view(torch.bfloat16)
    for config_id in (None, 0, 6, 29):
        c = sentinel((t, n), torch.bfloat16)
        capi.gemm_grouped(ta, tb, c, o, "fp32", config_id=config_id)
        torch.cuda.synchronize()
        got = bits(c).cpu().numpy().view(np.uint16)
        for g, (s, e) in enumerate(groups):
            if e > s:
                assert np.array_equal(got[s:e], oracle.bgemm_f32acc(ab[s:e], bb[g])), (config_id, g)


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_rows_past_the_last_group_and_guard_bands_are_untouched(variant):
    dtype, acc = VARIANTS[variant]
    t, n, k = 1000, 72, 64
    a = randn((t, k), dtype, 12 + variant)
    bt = randn((6, n, k), dtype, 13 + variant)
    guard = 4096
    cases = [
        [5, 77, 100, 100, 321, 600],          # offs[-1] < T: rows 600.. are no group's
        [300, 100, -5, 700, 5000, 900],      # decreasing, negative, past T: clamped
        [-1, -1, -1, -1, -1, -1],           # every group empty
        [0, 0, 0, 1, 999, 1000],             # the last group ends at T
    ]
    for offs in cases:
        o = offs_tensor(offs)
        for config_id in (0, 3, 12, 14, 26, 29):
            want = reference(a, bt, offs, variant, config_id)
            buf = sentinel((2 * guard + t * n,), dtype)
            c = buf[guard:guard + t * n].view(t, n)
            capi.gemm_grouped(a, bt, c, o, acc, config_id=config_id)
            torch.cuda.synchronize()
            assert torch.equal(bits(c), bits(want)), (offs, config_id)   # sentinel past the last group's end
            assert bool((bits(buf[:guard]) == SENTINEL).all()) and bool((bits(buf[guard + t * n:]) == SENTINEL).all())


def test_offsets_written_by_a_kernel_just_before_the_launch():
    g, t, n, k = 16, 2048, 256, 128
    a, bt = randn((t, k), torch.float16, 3), randn((g, n, k), torch.float16, 4)
    offs = torch.empty(g, dtype=torch.int32, device="cuda")
    steps = torch.arange(1, g + 1, dtype=torch.int32, device="cuda")
    outs = []
    for it in range(30):
        # a torch kernel on the same stream writes the offsets; the GEMM's prologue may overlap it, its reads may not
        torch.mul(steps, 7 * it + 3, out=offs)
        torch.remainder(offs, t + 100, out=offs)
        c = sentinel((t, n), torch.float16)
        capi.gemm_grouped(a, bt, c, offs, "fp32", config_id=1, stream=torch.cuda.current_stream().cuda_stream)
        outs.append(c)
    torch.cuda.synchronize()
    for it, c in enumerate(outs):
        host = [int(x) for x in (np.arange(1, g + 1) * (7 * it + 3)) % (t + 100)]
        assert torch.equal(bits(c), bits(reference(a, bt, host, 0, 1))), it


def test_cuda_graph_replays_read_the_current_offsets():
    g, t, n, k = 8, 1500, 512, 256
    a, bt = randn((t, k), torch.bfloat16, 5), randn((g, n, k), torch.bfloat16, 6)
    offs = offs_tensor(cumulative([t // g] * g))
    c = sentinel((t, n), torch.bfloat16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up outside the capture (attributes, tensor maps)
        capi.gemm_grouped(a, bt, c, offs, "fp32", config_id=4, stream=s.cuda_stream)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        capi.gemm_grouped(a, bt, c, offs, "fp32", config_id=4, stream=torch.cuda.current_stream().cuda_stream)
    rng = np.random.default_rng(8)
    for _ in range(6):
        host = cumulative(rng.integers(0, 2 * t // g, size=g))
        offs.copy_(torch.tensor(host, dtype=torch.int32))
        c.copy_(sentinel((t, n), torch.bfloat16))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(c), bits(reference(a, bt, host, 2, 4))), host


def test_one_launch_per_call_and_empty_problems_launch_nothing():
    before = capi.grouped_launch_count()
    a, bt = randn((500, 64), torch.float16, 1), randn((64, 128, 64), torch.float16, 2)
    offs = offs_tensor(cumulative([7] * 64))
    ops.hgemm_grouped(a, bt, offs)
    capi.gemm_grouped(a, bt, torch.empty((500, 128), dtype=torch.float16, device="cuda"), offs)
    torch.cuda.synchronize()
    assert capi.grouped_launch_count() - before == 2
    before = capi.grouped_launch_count()
    y = ops.hgemm_grouped(a[:0], bt, offs)                                            # T == 0
    assert y.shape == (0, 128)
    y = ops.hgemm_grouped(a, bt[:0], offs[:0])                                        # G == 0
    assert y.shape == (500, 128)
    assert capi.grouped_launch_count() == before


def operator_offsets(t, g, seed):
    rng = np.random.default_rng(seed)
    sizes = rng.multinomial(t, rng.dirichlet(np.ones(g)))
    sizes[rng.integers(0, g)] = 0
    return cumulative(sizes)


@pytest.mark.parametrize("dtype,acc,tol", [(torch.float16, "fp32", FP16_TOL), (torch.float16, "fp16", FP16_ACC16_TOL),
                                           (torch.bfloat16, "fp32", BF16_TOL)])
def test_operator_against_torch(dtype, acc, tol):
    for (g, t, n, k) in ((8, 2000, 512, 1024), (64, 4096, 128, 256), (5, 333, 200, 1024)):
        a, bt = randn((t, k), dtype, t), randn((g, n, k), dtype, n)
        offs = operator_offsets(t - 3, g, g + t)           # three rows past the last group: unspecified
        o = offs_tensor(offs)
        got = ops.hgemm_grouped(a, bt, o, acc)
        assert got.shape == (t, n) and got.dtype == dtype
        end = offs[-1]
        if dtype == torch.bfloat16:
            ref = torch._grouped_mm(a, bt.transpose(-2, -1), offs=o)[:end].float()
        else:
            ref = torch.cat([a[s:e].float() @ bt[i].float().t() for i, (s, e) in enumerate(clamped_groups(offs, t))])
        err = float((got[:end].float() - ref).abs().max() / ref.pow(2).mean().sqrt())
        assert err <= tol, (g, t, n, k, err)


def test_operator_has_no_gradient():
    a = randn((64, 32), torch.bfloat16, 20).requires_grad_(True)
    bt = randn((2, 16, 32), torch.bfloat16, 21)
    y = ops.hgemm_grouped(a, bt, offs_tensor([30, 64]))
    with pytest.raises(capi.B200HgemmError):
        y.float().sum().backward()
