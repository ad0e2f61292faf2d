"""FP8 (e4m3) GEMM with rowwise scales on the H100: bit-exact against the CPU reference on small-integer operands (every
configuration, both output types, every K-mode, ragged shapes), scale vectors read at run time (stream order, graph
replay), guard bands, random data at production sizes, torch._scaled_mm with rowwise scales, and B200Fp8Linear with
granularity="rowwise".

Exactness. As for per-tensor scales (test_gpu_fp8.py): on small integers every partial sum is an integer the FP8 tensor
core holds exactly, so the kernel's fp32 sum is the reference's in every K-mode, and both then apply
fp32(fp32(acc * sb[n]) * sa[m]) and one rounding.

Epilogue order. On exact small-integer sums with non-power-of-two vectors (528x400x400, bf16 out),
torch._scaled_mm with rowwise scales matched fp32(fp32(acc * sb[n]) * sa[m]) on every element, while (acc * sa) * sb and
acc * fp32(sa * sb) each differed on 2 elements: torch's Hopper rowwise epilogue applies the column scale first, as here.

Tolerances, measured on an H100 80GB HBM3 (700 W power limit), two seeds per case. N(0,1) data quantised per row (amax /
448), the truth being the fp32 product of the quantised operands, scaled: err = max |C - truth| / rms(truth):
  4096^3            fp16 out 0.0228-0.0240   bf16 out 0.0315-0.0383
  2048x11008x4096   fp16 out 0.0246-0.0255   bf16 out 0.0333-0.0383
  16x4096x4096      fp16 out 0.0147-0.0154   bf16 out 0.0186-0.0232
RANDOM_TOL = 0.05 is the largest (0.0383) with margin. Against torch._scaled_mm rowwise (use_fast_accum=True, bf16 out)
the output was bit-identical at 2048x11008x4096 and 16x4096x4096; at 4096^3 85-89 of 16.7M elements differed, by at most
0.0156 x rms (one bf16 rounding): SCALED_MM_TOL = 0.03 there, identity at the other two shapes.
B200Fp8Linear(granularity="rowwise") against its fp16 / bf16 source (1024 -> 512): 0.152-0.170 measured (tensorwise
0.160-0.176), bound LINEAR_TOL = 0.25. With row norms spanning 2^12 the eight smallest rows' mean error of the tensorwise
layer was 1.07-1.14 times the rowwise one's (the largest rowwise per-row error 0.148-0.182): bounds 1.05 and 0.25.
"""
import numpy as np
import pytest
import torch

from cuda_l2_b200 import capi
from fp8_rowwise_ref import fp8gemm_f32acc_rowwise
from test_gpu_exact_range import case8, e4m3_refs, run8
from test_gpu_fp8 import K_MODES, small_ints

pytestmark = pytest.mark.gpu

E4 = torch.float8_e4m3fn
RANDOM_TOL = 0.05          # max |C - truth| / rms(truth) on N(0,1) data quantised per row
LINEAR_TOL = 0.25          # B200Fp8Linear(rowwise) against its fp16 source
SCALED_MM_TOL = 0.03       # max |C - torch._scaled_mm rowwise| / rms, bf16 out, where it was not bit-identical


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def vectors(m, n, seed, pow2=False):
    """Rowwise scales as the operator takes them: sa [M,1], sb [1,N], fp32 on the device."""
    g = torch.Generator().manual_seed(seed)
    if pow2:
        sa, sb = (torch.pow(2.0, torch.randint(-3, 4, (s,), generator=g).float()) for s in (m, n))
    else:
        sa, sb = (torch.rand(s, generator=g) * 2.9 + 0.1 for s in (m, n))
    return sa.reshape(m, 1).cuda(), sb.reshape(1, n).cuda()


def codes(t):
    return t.cpu().view(torch.uint8).numpy()


def bits(c):
    return c.view(torch.int16).cpu().numpy().view(np.uint16)


def want_bits(a, bt, sa, sb, out_dtype):
    assert float((a.float() @ bt.float().t()).abs().max()) <= 2047      # the exact domain
    return fp8gemm_f32acc_rowwise(codes(a), codes(bt), sa.cpu().numpy(), sb.cpu().numpy(), out_dtype == torch.bfloat16)


def run(a, bt, sa, sb, out_dtype, **kw):
    c = torch.full((a.shape[0], bt.shape[0]), float("nan"), dtype=out_dtype, device="cuda")
    capi.fp8_gemm(a.cuda(), bt.cuda(), c, sa, sb, **kw)
    torch.cuda.synchronize()
    return c


def test_every_configuration_both_outputs_bit_exact():
    m, n = 520, 392                                  # off tile multiples in M and N
    before = capi.launch_count()
    launches = 0
    for out_dtype, k in ((torch.float16, 400), (torch.bfloat16, 240)):   # K off the 128-element k-block
        a, bt = small_ints((m, k), 1, 31), small_ints((n, k), 1, 32)
        sa, sb = vectors(m, n, 33)                   # non-power-of-two values
        want = want_bits(a, bt, sa, sb, out_dtype)
        for cfg in capi.configs():
            got = bits(run(a, bt, sa, sb, out_dtype, config_id=cfg["id"]))
            launches += 1
            assert np.array_equal(got, want), (cfg, out_dtype)
    assert capi.launch_count() - before == launches


@pytest.mark.parametrize("cfg,m,n,k,splits,mode", K_MODES)
def test_every_k_mode_bit_exact(cfg, m, n, k, splits, mode):
    assert capi.schedule(cfg, m, n, k // 2, splits)["mode"] == mode
    a, bt = small_ints((m, k), 1, 40 + splits), small_ints((n, k), 1, 50 + splits)
    for out_dtype, pow2 in ((torch.float16, True), (torch.bfloat16, False)):
        sa, sb = vectors(m, n, 60 + splits, pow2)
        got = bits(run(a, bt, sa, sb, out_dtype, config_id=cfg, splits=splits))
        assert np.array_equal(got, want_bits(a, bt, sa, sb, out_dtype)), (cfg, splits, out_dtype)
    # the full output range (exact_domain.py): ties, subnormals and overflow reach every reduction site
    da, dbt, _, _ = case8(m, n, k)
    for out_dtype, sa, sb, want in e4m3_refs(m, n, k)["rowwise"]:
        assert np.array_equal(run8(da, dbt, sa, sb, out_dtype, config_id=cfg, splits=splits), want), (cfg, splits, out_dtype)


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("mnk", [(200, 328, 144), (1, 8, 16), (1, 4096, 1024), (129, 136, 272), (16, 4096, 1024),
                                 (1000, 1032, 1040)])
def test_dispatched_ragged_shapes_bit_exact(mnk, out_dtype):
    from cuda_l2_b200 import ops
    m, n, k = mnk
    a, bt = small_ints((m, k), 1, m + k), small_ints((n, k), 1, n + 3 * k)
    for pow2 in (True, False):
        sa, sb = vectors(m, n, m + n, pow2)
        assert np.array_equal(bits(run(a, bt, sa, sb, out_dtype)), want_bits(a, bt, sa, sb, out_dtype)), (mnk, pow2)
        y = ops.fp8_gemm(a.cuda(), bt.cuda(), sa, sb, out_dtype)           # the operator picks the same entry point
        assert np.array_equal(bits(y), want_bits(a, bt, sa, sb, out_dtype)), (mnk, pow2)


def test_scale_vectors_written_just_before_the_gemm_are_the_ones_used():
    from cuda_l2_b200 import ops
    m, n, k = 256, 256, 512
    a, bt = small_ints((m, k), 1, 5).cuda(), small_ints((n, k), 1, 6).cuda()
    sa, sb = vectors(m, n, 7)
    ops.fp8_gemm(a, bt, sa, sb, torch.float16)
    for seed in (8, 9, 10):
        new_a, new_b = vectors(m, n, seed)
        sa.copy_(new_a); sb.copy_(new_b)                  # torch kernels, same stream, right before the GEMM
        y = ops.fp8_gemm(a, bt, sa, sb, torch.float16)
        assert np.array_equal(bits(y), want_bits(a, bt, sa, sb, torch.float16)), seed


@pytest.mark.parametrize("prewarm", [True, False])
def test_graph_replay_reads_the_current_vectors(prewarm):
    from cuda_l2_b200 import ops
    m, n, k = 512, 512, 8192                                 # dispatched with a K-decomposition
    a, bt = small_ints((m, k), 1, 11).cuda(), small_ints((n, k), 1, 12).cuda()
    sa, sb = vectors(m, n, 13)
    s = torch.cuda.Stream()                                  # without prewarm: captured undivided
    if prewarm:
        capi.prewarm(s.cuda_stream)
        with torch.cuda.stream(s):
            ops.fp8_gemm(a, bt, sa, sb, torch.bfloat16)
        torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        y = ops.fp8_gemm(a, bt, sa, sb, torch.bfloat16)
    for seed in (14, 15, 16):
        new_a, new_b = vectors(m, n, seed, pow2=seed % 2 == 0)
        sa.copy_(new_a); sb.copy_(new_b)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(bits(y), want_bits(a, bt, sa, sb, torch.bfloat16)), seed


@pytest.mark.parametrize("cfg,splits", [(1, 1), (3, 1), (26, 1), (14, 1), (0, 1), (1, 4), (1, -4), (1, 100), (30, 1)])
def test_guard_bands(cfg, splits):
    m, n, k = 200, 328, 4096
    a, bt = small_ints((m, k), 1, 17).cuda(), small_ints((n, k), 1, 18).cuda()
    sa, sb = vectors(m, n, 19)
    pad = 4096
    buf = torch.full((m * n + 2 * pad,), -7.0, dtype=torch.float16, device="cuda")
    c = buf[pad:pad + m * n].view(m, n)
    c.fill_(float("nan"))
    capi.fp8_gemm(a, bt, c, sa, sb, config_id=cfg, splits=splits)
    torch.cuda.synchronize()
    assert np.array_equal(bits(c), want_bits(a, bt, sa, sb, torch.float16))
    assert bool((buf[:pad] == -7).all()) and bool((buf[pad + m * n:] == -7).all())


def rowwise_randn(shape, seed):
    from cuda_l2_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    return ops.quantize_e4m3_rowwise(torch.randn(shape, device="cuda", generator=g))


def fp32_truth(a, bt, sa, sb):
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return ((a.float() @ bt.float().t()) * sb) * sa
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("mnk", [(4096, 4096, 4096), (2048, 11008, 4096), (16, 4096, 4096)])
@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16])
def test_random_data_within_the_measured_tolerance(mnk, out_dtype):
    from cuda_l2_b200 import ops
    m, n, k = mnk
    a, sa = rowwise_randn((m, k), 1)
    bt, sb = rowwise_randn((n, k), 2)
    sb = sb.reshape(1, n)
    y = ops.fp8_gemm(a, bt, sa, sb, out_dtype).float()
    truth = fp32_truth(a, bt, sa, sb)
    err = float((y - truth).abs().max() / truth.pow(2).mean().sqrt())
    assert err <= RANDOM_TOL, (mnk, out_dtype, err)


@pytest.mark.parametrize("mnk,identical", [((4096, 4096, 4096), False), ((2048, 11008, 4096), True),
                                           ((16, 4096, 4096), True)])
def test_bf16_output_against_torch_scaled_mm_rowwise(mnk, identical):
    from cuda_l2_b200 import ops
    m, n, k = mnk
    a, sa = rowwise_randn((m, k), 3)
    bt, sb = rowwise_randn((n, k), 4)
    sb = sb.reshape(1, n)
    y = ops.fp8_gemm(a, bt, sa, sb, torch.bfloat16)
    ref = torch._scaled_mm(a, bt.t(), scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16, use_fast_accum=True)
    if identical:
        assert torch.equal(y, ref), mnk
    else:
        diff = float((y.float() - ref.float()).abs().max() / ref.float().pow(2).mean().sqrt())
        assert diff <= SCALED_MM_TOL, (mnk, diff)


def _linear_pair(out_dtype, seed):
    from torch import nn

    from cuda_l2_b200 import ops
    torch.manual_seed(seed)
    lin = nn.Linear(1024, 512, dtype=out_dtype, device="cuda")
    return lin, ops.B200Fp8Linear.from_linear(lin), ops.B200Fp8Linear.from_linear(lin, granularity="rowwise")


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16])
def test_rowwise_linear_agrees_with_its_source(out_dtype):
    lin, _, m = _linear_pair(out_dtype, 3)
    x = torch.randn(4, 33, 1024, dtype=out_dtype, device="cuda")
    with torch.no_grad():
        y, ref = m(x), lin(x)
    assert y.shape == ref.shape and y.dtype == out_dtype
    rel = float((y.float() - ref.float()).abs().max() / ref.float().pow(2).mean().sqrt())
    assert rel <= LINEAR_TOL, rel          # measured 0.152-0.170 (module docstring)


def row_errors(lin, m, x):
    """Per row: max |y - ref| / rms(ref row), against the source layer's output."""
    with torch.no_grad():
        y, ref = m(x).float(), lin(x).float()
    return (y - ref).abs().amax(dim=1) / ref.pow(2).mean(dim=1).sqrt()


OUTLIER_ROWWISE_MAX = 0.25  # largest per-row error of the rowwise layer on the outlier input (measured 0.148-0.182)
OUTLIER_RATIO = 1.05        # mean error of the 8 smallest rows, tensorwise over rowwise (measured 1.07-1.14)


def test_rowwise_linear_keeps_small_rows_accurate_next_to_an_outlier():
    lin, t, r = _linear_pair(torch.float16, 5)
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(64, 1024, device="cuda", generator=g)
    x *= torch.pow(2.0, torch.linspace(-6, 6, 64, device="cuda"))[:, None]   # row norms spanning 2^12
    x = x.half()
    e_t, e_r = row_errors(lin, t, x), row_errors(lin, r, x)
    assert float(e_r.max()) <= OUTLIER_ROWWISE_MAX, float(e_r.max())
    assert float(e_t[:8].mean() / e_r[:8].mean()) >= OUTLIER_RATIO, (float(e_t[:8].mean()), float(e_r[:8].mean()))


def test_rowwise_linear_captures_in_a_graph():
    lin, _, m = _linear_pair(torch.bfloat16, 7)
    x = torch.randn(128, 1024, dtype=torch.bfloat16, device="cuda")
    s = torch.cuda.Stream()
    capi.prewarm(s.cuda_stream)
    with torch.no_grad():
        with torch.cuda.stream(s):
            m(x)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            y = m(x)
        for seed in (1, 2):
            x.copy_(torch.randn(128, 1024, generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda"))
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(y, m(x))
