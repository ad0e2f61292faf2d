"""Block-scaled FP8 batched GEMM with per-batch row counts on the H100 (libb200_batched_fp8.so), the MoE decode layout.

The anchor: a batched launch runs the 2-D block-scaled kernel's main loop and promotion; A's, Bt's and C's maps gain a
batch coordinate, A's scales and Bt's scales are read at the batch's own block, and the store is cut at the batch's
row count. An output row depends only on its own row of A and its own scales, so every matrix's computed rows must be
BIT-IDENTICAL to b200_fp8gemm_blockwise_run_config with the same configuration and group_m, run on that matrix's rows
of A, its scale rows (copied into a fresh aligned buffer), Bt[b] and scale_b[b]: for all 17 block-scaled
configurations x 2 output types, dense and with counts 0, 1, 15, 17, M, M + 5 and -3, with M % 4 != 0, K and N off
the 128 blocks, at all SMs and with a CTA cap that makes workers cross matrices. Then: NaN past the counts, rows from
round_up(count, 16) and guard bands untouched, exactness against the C reference on small integers with power-of-two
scales, ld_a > M and the quantiser's scale_a read in place, counts and scales written by a torch kernel just before
the launch and changed between CUDA-graph replays, one launch per call, the masked module form against the packed one,
and the dispatched call over dispatch_sweep.py's batched problems against the exact product.
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
COUNTS = [0, 1, 15, 17, None, "M+5", -3]   # None: M


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def counts_for(m):
    return [m if c is None else m + 5 if c == "M+5" else c for c in COUNTS]


def rows_of(counts, b, m):
    return [m] * b if counts is None else [min(max(c, 0), m) for c in counts]


def mask_tensor(counts):
    return None if counts is None else torch.tensor(counts, dtype=torch.int32, device="cuda")


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


def batched_m_major(sa, ld=None):
    """A fresh (nkb * ld_a, 1, ld_a)-strided copy of sa [B, M, nkb] (NaN in the padding)."""
    b, m, kb = sa.shape
    ld = ld or -(-m // 4) * 4
    buf = torch.full((b, kb, ld), float("nan"), dtype=torch.float32, device=sa.device)
    buf[:, :, :m] = sa.transpose(1, 2)
    return buf[:, :, :m].transpose(1, 2)


def randn_problem(b, m, n, k, seed):
    """Quantised N(0,1) operands: a [B,M,K] with its in-place scales, bt [B,N,K] with scales [B, ceil(N/128), nkb]."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    a, sa = ops.quantize_e4m3_blockwise(torch.randn((b, m, k), device="cuda", generator=gen))
    bt, sb = ops.quantize_e4m3_block128x128(torch.randn((b, n, k), device="cuda", generator=gen))
    return a, sa, bt, sb


def reference(a, sa, bt, sb, rows, out_dtype, config_id, group_m=0):
    """The 2-D block-scaled kernel on each matrix's first rows[b] rows (sentinel elsewhere)."""
    b, m, n = a.shape[0], a.shape[1], bt.shape[1]
    want = sentinel((b, m, n), out_dtype)
    for j, r in enumerate(rows):
        if r > 0:
            c = torch.empty((r, n), dtype=out_dtype, device="cuda")
            capi.fp8_gemm(a[j, :r].contiguous(), bt[j], c, m_major(sa[j, :r]), sb[j].contiguous(), config_id=config_id,
                          group_m=group_m, splits=1)
            want[j, :r] = c
    return want


def check(c, want, rows, what):
    """Rows below each count bit-equal; rows from round_up(count, 16) on keep the sentinel."""
    for j, r in enumerate(rows):
        assert torch.equal(bits(c[j, :r]), bits(want[j, :r])), (what, j, r)
        assert bool((bits(c[j, -(-r // 16) * 16:]) == SENTINEL).all()), (what, j, r)


def cta_count(config_id):
    c = capi.configs()[config_id]
    return c["cta_group"] * c["cluster_m"] * c["cluster_n"]


@pytest.mark.parametrize("out_dtype", OUT)
@pytest.mark.parametrize("config_id", ELIGIBLE)
def test_every_matrix_is_bit_identical_to_the_2d_kernel(config_id, out_dtype):
    before = capi.fp8_batched_launch_count()
    launches = 0
    for m, n, k in ((203, 264, 400), (90, 392, 256)):   # M % 4 != 0 / M % 16 != 0, K % 128 != 0 / N % 128 != 0
        a, sa, bt, sb = randn_problem(len(COUNTS), m, n, k, 10 * config_id + n)
        dense = reference(a, sa, bt, sb, [m] * len(COUNTS), out_dtype, config_id)
        for counts in (None, counts_for(m)):
            rows = rows_of(counts, len(COUNTS), m)
            want = reference(a, sa, bt, sb, rows, out_dtype, config_id)
            for j, r in enumerate(rows):   # the 2-D kernel on fewer rows gives those rows' bits
                assert torch.equal(bits(want[j, :r]), bits(dense[j, :r]))
            for max_ctas in (0, 2 * cta_count(config_id)):   # all SMs, and two workers that walk every matrix
                c = sentinel((len(COUNTS), m, n), out_dtype)
                capi.fp8_batched_gemm(a, bt, c, sa, sb, mask_tensor(counts), config_id=config_id, max_ctas=max_ctas)
                torch.cuda.synchronize()
                launches += 1
                check(c, want, rows, (config_id, out_dtype, m, n, k, counts, max_ctas))
    assert capi.fp8_batched_launch_count() - before == launches


def test_group_m_and_tiny_matrices_match_the_2d_kernel():
    for config_id in (1, 4, 9, 12, 23, 30):
        for (b, m, n, k, gm) in ((3, 1, 8, 16, 0), (4, 41, 64, 128, 3), (2, 513, 264, 272, 1)):
            a, sa, bt, sb = randn_problem(b, m, n, k, n + config_id)
            counts = [m, 0, m // 2, m + 1][:b]
            rows = rows_of(counts, b, m)
            for out_dtype in OUT:
                want = reference(a, sa, bt, sb, rows, out_dtype, config_id, gm)
                c = sentinel((b, m, n), out_dtype)
                capi.fp8_batched_gemm(a, bt, c, sa, sb, mask_tensor(counts), config_id=config_id, group_m=gm,
                                      max_ctas=cta_count(config_id))
                torch.cuda.synchronize()
                check(c, want, rows, (config_id, b, m, n, k, gm, out_dtype))


@pytest.mark.parametrize("out_dtype", OUT)
def test_nan_past_the_counts_stays_in_its_rows_and_guard_bands_are_untouched(out_dtype):
    b, m, n, k = 7, 150, 200, 400
    counts = counts_for(m)
    rows = rows_of(counts, b, m)
    a, sa, bt, sb = randn_problem(b, m, n, k, 31)
    a_nan, sa_nan = a.clone(), batched_m_major(sa)
    for j, r in enumerate(rows):   # rows at or past the count: NaN codes in A, NaN scales
        a_nan[j, r:].view(torch.uint8).fill_(0x7F)
        sa_nan[j, r:] = float("nan")
    guard = 4096
    for config_id in (1, 4, 12, 14, 30):
        want = reference(a, sa, bt, sb, rows, out_dtype, config_id)
        buf = sentinel((2 * guard + b * m * n,), out_dtype)
        c = buf[guard:guard + b * m * n].view(b, m, n)
        capi.fp8_batched_gemm(a_nan, bt, c, sa_nan, sb, mask_tensor(counts), config_id=config_id)
        torch.cuda.synchronize()
        check(c, want, rows, config_id)
        assert bool((bits(buf[:guard]) == SENTINEL).all()) and bool((bits(buf[guard + b * m * n:]) == SENTINEL).all())


def pow2_scales(b, m, n, k, seed):
    gen = torch.Generator().manual_seed(seed)
    nkb = -(-k // 128)
    sa = torch.pow(2.0, torch.randint(-3, 4, (b, m, nkb), generator=gen).float())
    sb = torch.pow(2.0, torch.randint(-3, 4, (b, -(-n // 128), nkb), generator=gen).float())
    return sa.cuda(), sb.cuda()


def codes(x):
    return x.cpu().view(torch.uint8).numpy()


def test_exact_against_the_reference_per_matrix():
    b, m, n, k = 4, 130, 328, 400
    counts = [70, 0, 130, 3]
    a = small_ints((b, m, k), 1, 11)
    bt = small_ints((b, n, k), 1, 12)
    sa, sb = pow2_scales(b, m, n, k, 13)
    for out_dtype in OUT:
        for config_id in (None, 2, 10, 22):
            c = sentinel((b, m, n), out_dtype)
            capi.fp8_batched_gemm(a.cuda(), bt.cuda(), c, batched_m_major(sa), sb, mask_tensor(counts),
                                  config_id=config_id)
            torch.cuda.synchronize()
            got = bits(c).cpu().numpy().view(np.uint16)
            for j, r in enumerate(counts):
                if r > 0:
                    want = fp8gemm_f32acc_block(codes(a[j, :r]), codes(bt[j]), sa[j, :r].cpu().numpy(),
                                                sb[j].cpu().numpy(), out_dtype == torch.bfloat16)
                    assert np.array_equal(got[j, :r], want), (out_dtype, config_id, j)
                assert bool((bits(c[j, -(-r // 16) * 16:]) == SENTINEL).all())


def test_row_stride_larger_than_m_and_quantiser_scales_in_place():
    b, m, n, k = 5, 77, 256, 528
    counts = [5, 77, 0, 40, 100]
    rows = rows_of(counts, b, m)
    a, sa, bt, sb = randn_problem(b, m, n, k, 21)
    assert capi.blockwise_ld_a(sa) == -(-m // 4) * 4               # read in place, as the quantiser returns it
    for out_dtype in OUT:
        want = reference(a, sa, bt, sb, rows, out_dtype, 4)
        for view in (sa, batched_m_major(sa, 96), batched_m_major(sa, 1024)):
            c = sentinel((b, m, n), out_dtype)
            capi.fp8_batched_gemm(a, bt, c, view, sb, mask_tensor(counts), config_id=4)
            torch.cuda.synchronize()
            check(c, want, rows, (out_dtype, view.stride()))


def test_counts_and_scales_written_by_a_kernel_just_before_the_launch():
    b, m, n, k = 16, 128, 256, 384
    a, sa0, bt, sb0 = randn_problem(b, m, n, k, 3)
    view, sb = batched_m_major(sa0), sb0.clone()
    counts = torch.empty(b, dtype=torch.int32, device="cuda")
    steps = torch.arange(1, b + 1, dtype=torch.int32, device="cuda")
    outs = []
    for it in range(12):
        # torch kernels on the same stream write the counts and both scales; the GEMM's prologue may overlap them,
        # its reads may not
        torch.mul(steps, 7 * it + 3, out=counts)
        torch.remainder(counts, m + 20, out=counts)
        torch.mul(sa0, 1 + it % 3, out=view)
        torch.mul(sb0, 2.0 ** -(it % 4), out=sb)
        c = sentinel((b, m, n), torch.bfloat16)
        capi.fp8_batched_gemm(a, bt, c, view, sb, counts, config_id=1, stream=torch.cuda.current_stream().cuda_stream)
        outs.append(c)
    torch.cuda.synchronize()
    for it, c in enumerate(outs):
        host = [int(x) for x in (np.arange(1, b + 1) * (7 * it + 3)) % (m + 20)]
        rows = rows_of(host, b, m)
        want = reference(a, sa0 * (1 + it % 3), bt, sb0 * 2.0 ** -(it % 4), rows, torch.bfloat16, 1)
        check(c, want, rows, it)


def test_cuda_graph_replays_read_the_current_counts_and_scales():
    b, m, n, k = 8, 200, 512, 256
    a, sa0, bt, sb0 = randn_problem(b, m, n, k, 5)
    sb = sb0.clone()
    sa = sa0.clone()   # the quantiser's layout, which the operator reads in place
    counts = mask_tensor([m] * b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up outside the capture (attributes, tensor maps)
        ops.fp8_batched_gemm(a, bt, sa, sb, torch.float16, counts)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = ops.fp8_batched_gemm(a, bt, sa, sb, torch.float16, counts)
    rng = np.random.default_rng(8)
    for i in range(6):
        host = [int(x) for x in rng.integers(-2, m + 10, size=b)]
        counts.copy_(torch.tensor(host, dtype=torch.int32))
        sa.copy_(sa0 * (i + 1))
        sb.copy_(sb0 * 2.0 ** -i)
        graph.replay()
        torch.cuda.synchronize()
        rows = rows_of(host, b, m)
        # the operator runs the dispatched configuration: the 2-D kernel with that configuration is the reference
        cfg, gm = capi.fp8_batched_select(b, m, n, k)
        want = reference(a, sa0 * (i + 1), bt, sb0 * 2.0 ** -i, rows, torch.float16, cfg, gm)
        for j, r in enumerate(rows):
            assert torch.equal(bits(y[j, :r]), bits(want[j, :r])), (host, j)


def test_masked_forward_captures_in_a_graph_and_reads_the_current_counts():
    g, m, n, k = 4, 96, 256, 512
    gen = torch.Generator(device="cuda").manual_seed(2)
    layer = ops.B200Fp8GroupedLinear.from_weights(torch.randn((g, n, k), device="cuda", generator=gen).bfloat16())
    x = torch.randn((g, m, k), device="cuda", dtype=torch.bfloat16, generator=gen)
    counts = mask_tensor([m] * g)
    s = torch.cuda.Stream()
    with torch.no_grad():
        with torch.cuda.stream(s):
            layer.forward_masked(x, counts)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            y = layer.forward_masked(x, counts)
        for seed, host in ((1, [10, 0, 96, 50]), (2, [0, 200, 1, -4])):
            x.copy_(torch.randn((g, m, k), device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed)))
            counts.copy_(torch.tensor(host, dtype=torch.int32))
            graph.replay()
            torch.cuda.synchronize()
            ref = layer.forward_masked(x, counts)
            torch.cuda.synchronize()
            for j, r in enumerate(rows_of(host, g, m)):
                assert torch.equal(bits(y[j, :r]), bits(ref[j, :r])), (seed, j)


def test_one_launch_per_call_and_empty_problems_launch_nothing():
    a, sa, bt, sb = randn_problem(6, 50, 128, 128, 1)
    counts = mask_tensor([7] * 6)
    before = capi.fp8_batched_launch_count()
    ops.fp8_batched_gemm(a, bt, sa, sb, torch.bfloat16, counts)
    ops.fp8_batched_gemm(a, bt, sa, sb, torch.float16)
    capi.fp8_batched_gemm(a, bt, torch.empty((6, 50, 128), dtype=torch.float16, device="cuda"), sa, sb, counts)
    torch.cuda.synchronize()
    assert capi.fp8_batched_launch_count() - before == 3
    before = capi.fp8_batched_launch_count()
    y = ops.fp8_batched_gemm(a[:, :0], bt, sa[:, :0], sb, torch.bfloat16, counts)          # M == 0
    assert y.shape == (6, 0, 128)
    y = ops.fp8_batched_gemm(a[:0], bt[:0], sa[:0], sb[:0], torch.bfloat16, counts[:0])   # B == 0
    assert y.shape == (0, 50, 128)
    assert capi.fp8_batched_launch_count() == before
    lib, blib = capi.batched_fp8_lib(), capi.batched_lib()
    p, s = a.data_ptr(), sa.data_ptr()
    for m in (0, -1):   # the C ABI: the status of the 16-bit batched call
        st = lib.b200_batched_fp8_gemm(p, p, p, s, 4, s, 0, None, 6, m, 128, 128, None)
        assert st == blib.b200_batched_gemm(0, p, p, p, None, 6, m, 128, 128, None) == -1
    assert capi.fp8_batched_launch_count() == before


def test_masked_forward_equals_the_packed_forward_row_for_row():
    g, m, n, k = 6, 160, 200, 1040
    gen = torch.Generator(device="cuda").manual_seed(9)
    layer = ops.B200Fp8GroupedLinear.from_weights(torch.randn((g, n, k), device="cuda", generator=gen).bfloat16())
    x = torch.randn((g, m, k), device="cuda", dtype=torch.bfloat16, generator=gen)
    host = [100, 0, 3, 160, 64, 1]
    xq, xs = ops.quantize_e4m3_blockwise(x)
    packed = torch.cat([x[j, :r] for j, r in enumerate(host)])
    pq, ps = ops.quantize_e4m3_blockwise(packed)
    offs = torch.tensor(np.cumsum(host).tolist(), dtype=torch.int32, device="cuda")
    for config_id in (1, 4, 12, 30):
        ym = sentinel((g, m, n), torch.bfloat16)
        capi.fp8_batched_gemm(xq, layer.weight_fp8, ym, xs, layer.weight_scale, mask_tensor(host), config_id=config_id)
        yp = torch.empty((packed.shape[0], n), dtype=torch.bfloat16, device="cuda")
        capi.fp8_grouped_gemm(pq, layer.weight_fp8, yp, ps, layer.weight_scale, offs, config_id=config_id)
        torch.cuda.synchronize()
        s = 0
        for j, r in enumerate(host):
            assert torch.equal(bits(ym[j, :r]), bits(yp[s:s + r])), (config_id, j)
            s += r
    with torch.no_grad():   # the module's two entry points, each with its dispatched configuration, agree closely
        ym, yp = layer.forward_masked(x, mask_tensor(host)), layer(packed, offs)
    s = 0
    for j, r in enumerate(host):
        assert torch.allclose(ym[j, :r].float(), yp[s:s + r].float(), rtol=0.02, atol=0.02), j
        s += r


def test_operator_has_no_gradient():
    a, sa, bt, sb = randn_problem(2, 64, 16, 128, 20)
    sa = sa.clone().requires_grad_(True)
    y = ops.fp8_batched_gemm(a, bt, sa, sb, torch.bfloat16, mask_tensor([30, 64]))
    with pytest.raises(capi.B200HgemmError, match="inference only"):
        y.float().sum().backward()


# ------------------------------------------------------------------------------------------------- dispatched, exact
GUARD = 64
NAN = 0x7E55               # a NaN in fp16 and in bf16


def run_dispatched(i: int, case: dict):
    b, m, n, k, counts = case["b"], case["m"], case["n"], case["k"], case["counts"]
    out = ("bf16", "fp16")[i % 2]
    dtype = torch.bfloat16 if out == "bf16" else torch.float16
    seed = ds.shape_seed(b, m, n, k)
    opr = ds.operands_e4m3(torch, b * m, b * n, k, seed)
    a, bt = opr.a.view(b, m, k), opr.bt.view(b, n, k)
    sa_np, sb_np = ed.e4m3_block_scales(m, n, k, out)
    # a wrong matrix's scales show: each matrix's scales are a power of two apart
    sa_all = np.stack([sa_np * np.float32(2.0 ** -(j % 3)) for j in range(b)])
    sb_all = np.stack([sb_np * np.float32(2.0 ** -(j % 2)) for j in range(b)])
    sa, sb = batched_m_major(torch.from_numpy(sa_all).cuda()), torch.from_numpy(sb_all).cuda()
    buf = torch.full((b * m * n + 2 * GUARD,), NAN, dtype=torch.int16, device="cuda")
    c = buf[GUARD:GUARD + b * m * n].view(dtype).view(b, m, n)
    capi.fp8_batched_gemm(a, bt, c, sa, sb, mask_tensor(counts))
    got = c.view(torch.int16)
    errs = [] if bool((buf[:GUARD] == NAN).all()) and bool((buf[-GUARD:] == NAN).all()) else ["guard band written"]
    for j, r in enumerate(rows_of(counts, b, m)):
        if r > 0:
            sa64 = torch.from_numpy(sa_all[j].astype(np.float64)).cuda().repeat_interleave(128, dim=1)[:, :k]
            b64 = bt[j].double() * torch.from_numpy(sb_all[j].astype(np.float64)).cuda() \
                .repeat_interleave(128, dim=1)[:, :k].repeat_interleave(128, dim=0)[:n]
            want = ds.round_to(torch, (a[j, :r].double() * sa64[:r]) @ b64.T, out)
            bad = int((got[j, :r] != want).sum())
            if bad:
                errs.append(f"matrix {j} (rows :{r}): {bad} mismatches")
        if not bool((got[j, -(-r // 16) * 16:] == NAN).all()):
            errs.append(f"matrix {j}: rows from round_up({r}, 16) written")
    if not errs:
        return None
    return f"batched fp8 {(b, m, n, k)} {out}: choice {capi.fp8_batched_select(b, m, n, k)}: " + "; ".join(errs[:5])


def test_dispatched_call_over_the_batched_problems_is_exact():
    failures = []
    cases = [c for c in ds.tile_list_cases() if c["kind"] == "batched"]
    assert len(cases) == 24
    for i, case in enumerate(cases):
        r = run_dispatched(i, case)
        if r:
            failures.append(r)
    torch.cuda.synchronize()
    assert not failures, f"{len(failures)} problems fail:\n" + "\n".join(failures)
