"""Block-scaled FP8 grouped GEMM over contiguous row groups on the H100 (libb200_grouped_fp8.so).

The anchor: a grouped launch runs the 2-D block-scaled kernel's main loop and promotion; only A's box starts at the
group's first row, A's scales come from an aligned window around that row, Bt's map and scales gain a group
coordinate, and the store of a box that straddles a group's end is cut at that end. An output row depends only on its
own row of A and its own scales, so every group's rows must be BIT-IDENTICAL to b200_fp8gemm_blockwise_run_config with
the same configuration and group_m, run on that group's rows of A, its scale rows (copied into a fresh aligned buffer),
Bt[g] and scale_b[g]: for all 17 block-scaled configurations x 2 output types, on ragged offsets (empty and one-row
groups, starts that are no multiple of 4 or 16, groups shorter and longer than a tile, rows past the last group), K and
N off the 128 blocks, and with a CTA cap that makes workers cross groups. Then: exactness against the C reference on
small integers with power-of-two scales, ld_a > T and the quantiser's scale_a read in place, rows past the last group
and guard bands untouched (also for malformed offsets), offsets and scales written by a torch kernel just before the
launch and changed between CUDA-graph replays, one launch per call, the operator and module, and the dispatched call
over dispatch_sweep.py's MoE-shaped problems against the exact product.
"""
import numpy as np
import pytest
import torch

import dispatch_sweep as ds
import exact_domain as ed
from cuda_l2_b200 import capi, ops
from fp8_block_ref import fp8gemm_f32acc_block
from test_gpu_fp8 import small_ints

pytestmark = pytest.mark.gpu

E4 = torch.float8_e4m3fn
ELIGIBLE = (1, 2, 4, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 22, 23, 30)
OUT = (torch.float16, torch.bfloat16)
SENTINEL = 0x7BCD          # a finite fp16 / bf16 bit pattern no product here produces by accident
RANDOM_TOL = {torch.float16: 0.005, torch.bfloat16: 0.025}   # test_gpu_fp8_blockwise.py's, max |C - truth| / rms(truth)
# group sizes: empty, one row, starts at every residue mod 4 and off multiples of 16, shorter and longer than a tile
SIZES = [0, 1, 37, 300, 0, 17, 530, 1, 2, 129, 0, 700, 15, 3]


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


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


def sentinel(shape, dtype):
    return torch.full(shape, SENTINEL, dtype=torch.int16, device="cuda").view(dtype)


def bits(x):
    return x.view(torch.int16)


def m_major(sa, ld=None):
    """A fresh (1, ld_a)-strided copy of sa [M, nkb], ld_a = ld or M rounded up to 4 (NaN in the padding)."""
    m, kb = sa.shape
    ld = ld or -(-m // 4) * 4
    buf = torch.full((kb, ld), float("nan"), dtype=torch.float32, device=sa.device)
    buf[:, :m] = sa.t()
    return buf[:, :m].t()


def randn_problem(t, g, n, k, seed):
    """Quantised N(0,1) operands: a [T,K] with its M-major scales, bt [G,N,K] with scales [G, ceil(N/128), nkb]."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    a, sa = ops.quantize_e4m3_blockwise(torch.randn((t, k), device="cuda", generator=gen))
    bt, sb = ops.quantize_e4m3_block128x128(torch.randn((g, n, k), device="cuda", generator=gen))
    return a, sa, bt, sb


def reference(a, sa, bt, sb, offs, out_dtype, config_id, group_m=0):
    """The 2-D block-scaled kernel on each group's rows (sentinel elsewhere)."""
    t, n = a.shape[0], bt.shape[1]
    want = sentinel((t, n), out_dtype)
    for g, (s, e) in enumerate(clamped_groups(offs, t)):
        if e > s:
            c = torch.empty((e - s, n), dtype=out_dtype, device="cuda")
            capi.fp8_gemm(a[s:e].contiguous(), bt[g], c, m_major(sa[s:e]), sb[g].contiguous(), config_id=config_id,
                          group_m=group_m, splits=1)
            want[s:e] = c
    return want


def cta_count(config_id):
    c = capi.configs()[config_id]
    return c["cta_group"] * c["cluster_m"] * c["cluster_n"]


@pytest.mark.parametrize("out_dtype", OUT)
@pytest.mark.parametrize("config_id", ELIGIBLE)
def test_every_group_is_bit_identical_to_the_2d_kernel(config_id, out_dtype):
    offs = cumulative(SIZES)
    before = capi.fp8_grouped_launch_count()
    for t, n, k in ((offs[-1] + 29, 264, 400), (offs[-1], 392, 256)):   # K % 128 != 0 / N % 128 != 0; rows past the end
        a, sa, bt, sb = randn_problem(t, len(SIZES), n, k, 10 * config_id + n)
        want = reference(a, sa, bt, sb, offs, out_dtype, config_id)
        for max_ctas in (0, 2 * cta_count(config_id)):   # all SMs, and two workers that walk every group
            c = sentinel((t, n), out_dtype)
            capi.fp8_grouped_gemm(a, bt, c, sa, sb, offs_tensor(offs), config_id=config_id, max_ctas=max_ctas)
            torch.cuda.synchronize()
            assert torch.equal(bits(c), bits(want)), (config_id, out_dtype, t, n, k, max_ctas)
    assert capi.fp8_grouped_launch_count() - before == 4


def test_group_m_and_tiny_groups_match_the_2d_kernel():
    for config_id in (1, 4, 9, 12, 23, 30):
        for (sizes, n, k, gm) in (([1, 0, 1, 2], 8, 16, 0), ([41, 3, 700, 66], 64, 128, 3), ([513, 259], 264, 272, 1)):
            offs = cumulative(sizes)
            a, sa, bt, sb = randn_problem(offs[-1], len(sizes), n, k, n + config_id)
            for out_dtype in OUT:
                want = reference(a, sa, bt, sb, offs, out_dtype, config_id, gm)
                c = sentinel((offs[-1], n), out_dtype)
                capi.fp8_grouped_gemm(a, bt, c, sa, sb, offs_tensor(offs), config_id=config_id, group_m=gm,
                                      max_ctas=cta_count(config_id))
                torch.cuda.synchronize()
                assert torch.equal(bits(c), bits(want)), (config_id, sizes, n, k, gm, out_dtype)


def pow2_scales(t, g, n, k, seed):
    gen = torch.Generator().manual_seed(seed)
    nkb = -(-k // 128)
    sa = torch.pow(2.0, torch.randint(-3, 4, (t, nkb), generator=gen).float())
    sb = torch.pow(2.0, torch.randint(-3, 4, (g, -(-n // 128), nkb), generator=gen).float())
    return sa.cuda(), sb.cuda()


def codes(x):
    return x.cpu().view(torch.uint8).numpy()


def test_exact_against_the_reference_per_group():
    sizes, n, k = [70, 0, 1, 129, 3, 200], 328, 400
    offs = cumulative(sizes)
    t = offs[-1] + 5
    a = small_ints((t, k), 1, 11)
    bt = small_ints((len(sizes), n, k), 1, 12)
    sa, sb = pow2_scales(t, len(sizes), n, k, 13)
    for out_dtype in OUT:
        for config_id in (None, 2, 10, 22):
            c = sentinel((t, n), out_dtype)
            capi.fp8_grouped_gemm(a.cuda(), bt.cuda(), c, m_major(sa), sb, offs_tensor(offs), config_id=config_id)
            torch.cuda.synchronize()
            got = bits(c).cpu().numpy().view(np.uint16)
            for g, (s, e) in enumerate(clamped_groups(offs, t)):
                if e > s:
                    want = fp8gemm_f32acc_block(codes(a[s:e]), codes(bt[g]), sa[s:e].cpu().numpy(), sb[g].cpu().numpy(),
                                                out_dtype == torch.bfloat16)
                    assert np.array_equal(got[s:e], want), (out_dtype, config_id, g)
            assert bool((bits(c)[offs[-1]:] == SENTINEL).all())


def test_row_stride_larger_than_t_and_quantiser_scales_in_place():
    sizes, n, k = [5, 300, 0, 77, 130], 256, 528
    offs = cumulative(sizes)
    t = offs[-1]
    a, sa, bt, sb = randn_problem(t, len(sizes), n, k, 21)
    assert capi.blockwise_ld_a(sa) == -(-t // 4) * 4                      # read in place, as the quantiser returns it
    for out_dtype in OUT:
        want = reference(a, sa, bt, sb, offs, out_dtype, 4)
        for view in (sa, m_major(sa, t + 4 - t % 4 + 8), m_major(sa, 2048)):
            c = sentinel((t, n), out_dtype)
            capi.fp8_grouped_gemm(a, bt, c, view, sb, offs_tensor(offs), config_id=4)
            torch.cuda.synchronize()
            assert torch.equal(bits(c), bits(want)), (out_dtype, view.stride())


@pytest.mark.parametrize("out_dtype", OUT)
def test_rows_past_the_last_group_and_guard_bands_are_untouched(out_dtype):
    t, n, k = 1000, 72, 144
    a, sa, bt, sb = randn_problem(t, 6, n, k, 12)
    guard = 4096
    cases = [
        [5, 77, 100, 100, 321, 602],          # offs[-1] < T: rows 602.. are no group's
        [300, 101, -5, 703, 5000, 900],      # decreasing, negative, past T: clamped
        [-1, -1, -1, -1, -1, -1],           # every group empty
        [0, 0, 0, 1, 999, 1000],             # the last group ends at T
    ]
    for offs in cases:
        o = offs_tensor(offs)
        for config_id in (1, 4, 12, 14, 30):
            want = reference(a, sa, bt, sb, offs, out_dtype, config_id)
            buf = sentinel((2 * guard + t * n,), out_dtype)
            c = buf[guard:guard + t * n].view(t, n)
            capi.fp8_grouped_gemm(a, bt, c, sa, sb, o, config_id=config_id)
            torch.cuda.synchronize()
            assert torch.equal(bits(c), bits(want)), (offs, config_id)   # sentinel past the last group's end
            assert bool((bits(buf[:guard]) == SENTINEL).all()) and bool((bits(buf[guard + t * n:]) == SENTINEL).all())


def test_offsets_and_scales_written_by_a_kernel_just_before_the_launch():
    g, t, n, k = 16, 2048, 256, 384
    a, sa0, bt, sb0 = randn_problem(t, g, n, k, 3)
    sa, sb = sa0.clone(), sb0.clone()
    view = m_major(sa)
    offs = torch.empty(g, dtype=torch.int32, device="cuda")
    steps = torch.arange(1, g + 1, dtype=torch.int32, device="cuda")
    outs = []
    for it in range(12):
        # torch kernels on the same stream write the offsets and both scales; the GEMM's prologue may overlap them,
        # its reads may not
        torch.mul(steps, 7 * it + 3, out=offs)
        torch.remainder(offs, t + 100, out=offs)
        torch.mul(sa0, 1 + it % 3, out=view)
        torch.mul(sb0, 2.0 ** -(it % 4), out=sb)
        c = sentinel((t, n), torch.bfloat16)
        capi.fp8_grouped_gemm(a, bt, c, view, sb, offs, config_id=1, stream=torch.cuda.current_stream().cuda_stream)
        outs.append(c)
    torch.cuda.synchronize()
    for it, c in enumerate(outs):
        host = [int(x) for x in (np.arange(1, g + 1) * (7 * it + 3)) % (t + 100)]
        want = reference(a, sa0 * (1 + it % 3), bt, sb0 * 2.0 ** -(it % 4), host, torch.bfloat16, 1)
        assert torch.equal(bits(c), bits(want)), it


def test_cuda_graph_replays_read_the_current_offsets_and_scales():
    g, t, n, k = 8, 1500, 512, 256
    a, sa0, bt, sb0 = randn_problem(t, g, n, k, 5)
    view, sb = m_major(sa0), sb0.clone()
    offs = offs_tensor(cumulative([t // g] * g))
    c = sentinel((t, n), torch.float16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up outside the capture (attributes, tensor maps)
        capi.fp8_grouped_gemm(a, bt, c, view, sb, offs, config_id=4, stream=s.cuda_stream)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        capi.fp8_grouped_gemm(a, bt, c, view, sb, offs, config_id=4, stream=torch.cuda.current_stream().cuda_stream)
    rng = np.random.default_rng(8)
    for i in range(6):
        host = cumulative(rng.integers(0, 2 * t // g, size=g))
        offs.copy_(torch.tensor(host, dtype=torch.int32))
        view.copy_(sa0 * (i + 1))
        sb.copy_(sb0 * 2.0 ** -i)
        c.copy_(sentinel((t, n), torch.float16))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(c), bits(reference(a, sa0 * (i + 1), bt, sb0 * 2.0 ** -i, host, torch.float16, 4))), host


def test_one_launch_per_call_and_empty_problems_launch_nothing():
    a, sa, bt, sb = randn_problem(500, 64, 128, 128, 1)
    offs = offs_tensor(cumulative([7] * 64))
    before = capi.fp8_grouped_launch_count()
    ops.fp8_grouped_gemm(a, bt, sa, sb, offs)
    capi.fp8_grouped_gemm(a, bt, torch.empty((500, 128), dtype=torch.float16, device="cuda"), sa, sb, offs)
    torch.cuda.synchronize()
    assert capi.fp8_grouped_launch_count() - before == 2
    before = capi.fp8_grouped_launch_count()
    y = ops.fp8_grouped_gemm(a[:0], bt, sa[:0], sb, offs)                               # T == 0
    assert y.shape == (0, 128)
    y = ops.fp8_grouped_gemm(a, bt[:0], sa, sb[:0], offs[:0])                           # G == 0
    assert y.shape == (500, 128)
    assert capi.fp8_grouped_launch_count() == before


def test_operator_equals_the_2d_operator_per_group():
    sizes, n, k = [100, 0, 3, 517, 64, 1], 200, 1040
    offs = cumulative(sizes)
    t = offs[-1] + 3
    gen = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn((t, k), device="cuda", generator=gen)
    a, sa = ops.quantize_e4m3_blockwise(x)
    bt, sb = ops.quantize_e4m3_block128x128(torch.randn((len(sizes), n, k), device="cuda", generator=gen))
    for out_dtype in OUT:
        for scale_a in (sa, sa.contiguous()):                        # M-major in place, and a contiguous copy
            y = ops.fp8_grouped_gemm(a, bt, scale_a, sb, offs_tensor(offs), out_dtype)
            assert y.shape == (t, n) and y.dtype == out_dtype
            for g, (s, e) in enumerate(clamped_groups(offs, t)):
                if e > s:
                    want = ops.fp8_gemm(a[s:e], bt[g], sa[s:e], sb[g], out_dtype)
                    assert torch.equal(bits(y[s:e]), bits(want)), (out_dtype, g)


def dequantised_grouped(x_q, x_s, w_q, w_s, offs):
    t, k = x_q.shape
    n = w_q.shape[1]
    a64 = x_q.double() * x_s.double().repeat_interleave(128, dim=1)[:, :k]
    out = torch.zeros((t, n), dtype=torch.float64, device="cuda")
    for g, (s, e) in enumerate(clamped_groups(offs, t)):
        b64 = w_q[g].double() * w_s[g].double().repeat_interleave(128, dim=0)[:n].repeat_interleave(128, dim=1)[:, :k]
        out[s:e] = a64[s:e] @ b64.t()
    return out


@pytest.mark.parametrize("out_dtype", OUT)
def test_from_fp8_matches_the_dequantised_experts(out_dtype):
    g, n, k, t = 8, 1000, 1040, 3000                                # ragged in both block dimensions
    gen = torch.Generator(device="cuda").manual_seed(8)
    w_fp8, w_scale = ops.quantize_e4m3_block128x128(torch.randn((g, n, k), device="cuda", generator=gen))
    layer = ops.B200Fp8GroupedLinear.from_fp8(w_fp8, w_scale, out_dtype)
    offs = cumulative(np.random.default_rng(3).multinomial(t, np.ones(g) / g))
    x = torch.randn((t, k), device="cuda", dtype=torch.bfloat16, generator=gen)
    with torch.no_grad():
        y = layer(x, offs_tensor(offs))
    x_q, x_s = ops.quantize_e4m3_blockwise(x)
    ref = dequantised_grouped(x_q, x_s, w_fp8, w_scale, offs)
    assert y.shape == (t, n) and y.dtype == out_dtype
    err = float((y.double() - ref).abs().max() / ref.pow(2).mean().sqrt())
    assert err <= RANDOM_TOL[out_dtype], err


def test_module_forward_captures_in_a_graph():
    g, n, k, t = 4, 256, 512, 700
    gen = torch.Generator(device="cuda").manual_seed(2)
    layer = ops.B200Fp8GroupedLinear.from_weights(torch.randn((g, n, k), device="cuda", generator=gen).bfloat16())
    x = torch.randn((t, k), device="cuda", dtype=torch.bfloat16, generator=gen)
    offs = offs_tensor(cumulative([100, 0, 350, 250]))
    s = torch.cuda.Stream()
    with torch.no_grad():
        with torch.cuda.stream(s):
            layer(x, offs)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            y = layer(x, offs)
        for seed, ends in ((1, [10, 300, 301, 690]), (2, [0, 0, 699, 700])):
            x.copy_(torch.randn((t, k), device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed)))
            offs.copy_(torch.tensor(ends, dtype=torch.int32))
            graph.replay()
            torch.cuda.synchronize()
            ref = layer(x, offs)
            assert torch.equal(bits(y[:ends[-1]]), bits(ref[:ends[-1]])), seed


def test_operator_has_no_gradient():
    a, sa, bt, sb = randn_problem(64, 2, 16, 128, 20)
    sa = sa.clone().requires_grad_(True)
    y = ops.fp8_grouped_gemm(a, bt, sa, sb, offs_tensor([30, 64]))
    with pytest.raises(capi.B200HgemmError, match="inference only"):
        y.float().sum().backward()


# ------------------------------------------------------------------------------------------------- dispatched, exact
GUARD = 64
NAN = 0x7E55               # a NaN in fp16 and in bf16


def run_dispatched(i: int, case: dict):
    g, t, n, k, offs = case["g"], case["t"], case["n"], case["k"], case["offs"]
    out = ("bf16", "fp16")[i % 2]
    dtype = torch.bfloat16 if out == "bf16" else torch.float16
    seed = ds.shape_seed(g, t, n, k)
    opr = ds.operands_e4m3(torch, t, g * n, k, seed)
    a, bt = opr.a, opr.bt.view(g, n, k)
    sa_np, sb_np = ed.e4m3_block_scales(t, n, k, out)
    sb_np = np.stack([sb_np * np.float32(2.0 ** -(j % 2)) for j in range(g)])   # a wrong group's scales show
    sa, sb = m_major(torch.from_numpy(sa_np).cuda()), torch.from_numpy(sb_np).cuda()
    buf = torch.full((t * n + 2 * GUARD,), NAN, dtype=torch.int16, device="cuda")
    c = buf[GUARD:GUARD + t * n].view(dtype).view(t, n)
    capi.fp8_grouped_gemm(a, bt, c, sa, sb, offs_tensor(offs))
    got = c.view(torch.int16)
    errs = [] if bool((buf[:GUARD] == NAN).all()) and bool((buf[-GUARD:] == NAN).all()) else ["guard band written"]
    sa64 = torch.from_numpy(sa_np.astype(np.float64)).cuda().repeat_interleave(128, dim=1)[:, :k]
    for j, (s, e) in enumerate(clamped_groups(offs, t)):
        if e > s:
            b64 = bt[j].double() * torch.from_numpy(sb_np[j].astype(np.float64)).cuda() \
                .repeat_interleave(128, dim=1)[:, :k].repeat_interleave(128, dim=0)[:n]
            want = ds.round_to(torch, (a[s:e].double() * sa64[s:e]) @ b64.T, out)
            bad = int((got[s:e] != want).sum())
            if bad:
                errs.append(f"group {j} (rows {s}:{e}): {bad} mismatches")
    if not bool((got[offs[-1]:] == NAN).all()):
        errs.append(f"rows from the last end {offs[-1]} written")
    if not errs:
        return None
    return f"grouped fp8 {(g, t, n, k)} {out}: choice {capi.fp8_grouped_select(g, t, n, k)}: " + "; ".join(errs[:5])


def test_dispatched_call_over_the_grouped_problems_is_exact():
    failures = []
    cases = [c for c in ds.tile_list_cases() if c["kind"] == "grouped"]
    assert len(cases) == 24
    for i, case in enumerate(cases):
        if case["k"] % 16 == 0:
            r = run_dispatched(i, case)
            if r:
                failures.append(r)
    torch.cuda.synchronize()
    assert not failures, f"{len(failures)} problems fail:\n" + "\n".join(failures)
