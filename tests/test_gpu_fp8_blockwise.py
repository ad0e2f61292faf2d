"""FP8 (e4m3) GEMM with block scales on the H100 (libb200_fp8block.so): bit-exact against the C reference on
small-integer operands with non-power-of-two scales (every eligible configuration, both output types, plain and cluster
split-K, ragged shapes, M = 1..16, ld_a > M, the strided scale_a view, a contiguous scale_a through the operator), scales
read at run time (stream order, graph replay), guard bands, random data at production sizes, the accuracy of the
per-k-block promotion at long K, torch._scaled_mm's blockwise mode, and B200Fp8Linear with granularity="blockwise".

Exactness. On small integers every k-block's wgmma sum p is an integer the FP8 tensor core holds exactly, so the kernel's
p is the reference's; s = fp32(sa * sb), fp32(p * s) on a unit's first k-block and fmaf(p, s, acc) after it are
correctly rounded fp32 operations on both sides, so with arbitrary fp32 scales the bits must agree. Cluster split-K sums
the splits' results in fixed order, which the reference restates for the same division of the k-blocks.

Tolerances, measured on an H100 80GB HBM3 (400 W power limit), two seeds per case. N(0,1) data quantised per 1 x 128
(a) and 128 x 128 (bt) block, the truth being the fp64 product of the dequantised operands:
err = max |C - truth| / rms(truth):
  4096^3            fp16 out 0.0023-0.0023   bf16 out 0.0159-0.0160
  2048x11008x4096   fp16 out 0.0024-0.0025   bf16 out 0.0159-0.0160
That is about the output rounding alone (per-tensor e4m3 reached 0.023 / 0.028-0.031 there, test_gpu_fp8.py): the
promotion takes the FP8 tensor core's reduced-precision running sum out of the error. RANDOM_TOL is the largest
figure with margin. Long K (512 x 512 x 16384, N(0,1) cast to e4m3, unit scales), rms(C - truth) / rms(truth):
block-scaled 0.000243, per-tensor 0.000877-0.000879 (max error 0.0019-0.0020 against 0.0058-0.0070).
torch._scaled_mm refused blockwise scales with the installed torch ("only supported for CUDA 12.9 and above"), so that
comparison skips with torch's message; SCALED_MM_TOL is the rowwise comparison's bound, for where it runs.
"""
import numpy as np
import pytest
import torch

from cuda_l2_b200 import capi
from fp8_block_ref import fp8gemm_f32acc_block
from test_gpu_fp8 import small_ints

pytestmark = pytest.mark.gpu

E4 = torch.float8_e4m3fn
ELIGIBLE = (1, 2, 4, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 22, 23, 30)
RANDOM_TOL = {torch.float16: 0.005, torch.bfloat16: 0.025}   # max |C - truth| / rms(truth); measured 0.0025 / 0.0160
SCALED_MM_TOL = 0.03     # max |C - torch._scaled_mm blockwise| / rms(ref), bf16 out
LINEAR_TOL = 0.25        # B200Fp8Linear(blockwise) against its fp16 / bf16 source, as for the other granularities
FROM_FP8_TOL = 0.05      # from_fp8 layer (bf16 GEMM output, then a bf16 bias add) against the fp64 product; measured 0.030


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def nkb(k):
    return -(-k // 128)


def block_scales(m, n, k, seed, pow2=False):
    """sa [M, nkb] (contiguous, as the reference takes it) and sb [ceil(N/128), nkb], fp32 on the device."""
    g = torch.Generator().manual_seed(seed)
    shapes = ((m, nkb(k)), (-(-n // 128), nkb(k)))
    if pow2:
        sa, sb = (torch.pow(2.0, torch.randint(-3, 4, s, generator=g).float()) for s in shapes)
    else:
        sa, sb = (torch.rand(s, generator=g) * 2.9 + 0.1 for s in shapes)
    return sa.cuda(), sb.cuda()


def m_major(sa, ld=None):
    """The (1, ld_a)-strided view of sa [M, nkb] the kernel reads in place, ld_a = ld or M rounded up to 4."""
    m, kb = sa.shape
    ld = ld or -(-m // 4) * 4
    buf = torch.full((kb, ld), float("nan"), dtype=torch.float32, device=sa.device)
    buf[:, :m] = sa.t()
    return buf[:, :m].t()


def codes(t):
    return t.cpu().view(torch.uint8).numpy()


def bits(c):
    return c.view(torch.int16).cpu().numpy().view(np.uint16)


def want_bits(a, bt, sa, sb, out_dtype, splits=1):
    assert float((a.float() @ bt.float().t()).abs().max()) <= 2047      # every k-block's sum exact in the tensor core
    return fp8gemm_f32acc_block(codes(a), codes(bt), sa.cpu().numpy(), sb.cpu().numpy(), out_dtype == torch.bfloat16,
                                splits)


def planned_splits(m, n, k, cfg=None, sp=None):
    """How many cluster split-K splits a launch runs (1: plain): the dispatcher's choice unless cfg / sp are given."""
    if cfg is None:
        cfg, _, sp = capi.fp8_blockwise_select(m, n, k)
    s = capi.schedule(cfg, m, n, k // 2, sp)          # the 16-bit schedule at K / 2 has the same k-blocks
    if s["mode"] != "cluster-split-k":
        return 1
    return sum(1 for units in s["units"] for unit in units if unit[0] == 0)


def run(a, bt, sa, sb, out_dtype, **kw):
    c = torch.full((a.shape[0], bt.shape[0]), float("nan"), dtype=out_dtype, device="cuda")
    capi.fp8_gemm(a.cuda(), bt.cuda(), c, sa, sb, **kw)
    torch.cuda.synchronize()
    return c


def test_every_eligible_configuration_both_outputs_bit_exact():
    m, n = 520, 392                                  # off tile multiples in M and N
    before = capi.fp8block_launch_count()
    launches = 0
    for out_dtype, k in ((torch.float16, 400), (torch.bfloat16, 240)):   # K off the 128-element k-block
        a, bt = small_ints((m, k), 1, 131), small_ints((n, k), 1, 132)
        sa, sb = block_scales(m, n, k, 133)          # non-power-of-two values
        want = want_bits(a, bt, sa, sb, out_dtype)
        for cfg in ELIGIBLE:
            got = bits(run(a, bt, m_major(sa), sb, out_dtype, config_id=cfg))
            launches += 1
            assert np.array_equal(got, want), (cfg, out_dtype)
    assert capi.fp8block_launch_count() - before == launches


def test_ineligible_configurations_are_rejected():
    m, n, k = 256, 256, 256
    a, bt = small_ints((m, k), 1, 1).cuda(), small_ints((n, k), 1, 2).cuda()
    sa, sb = block_scales(m, n, k, 3)
    c = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
    before = capi.fp8block_launch_count()
    for cfg in sorted(set(range(31)) - set(ELIGIBLE)):
        with pytest.raises(capi.B200HgemmError, match="status -6"):
            capi.fp8_gemm(a, bt, c, m_major(sa), sb, config_id=cfg)
    assert capi.fp8block_launch_count() == before


@pytest.mark.parametrize("cfg", [1, 2])
@pytest.mark.parametrize("splits", [-2, -4, -8])
def test_cluster_split_k_bit_exact(cfg, splits):
    m, n, k = 200, 328, 4096
    assert planned_splits(m, n, k, cfg, splits) == -splits
    a, bt = small_ints((m, k), 1, 40 - splits), small_ints((n, k), 1, 50 - splits)
    for out_dtype in (torch.float16, torch.bfloat16):
        sa, sb = block_scales(m, n, k, 60 - splits)
        got = bits(run(a, bt, m_major(sa), sb, out_dtype, config_id=cfg, splits=splits))
        assert np.array_equal(got, want_bits(a, bt, sa, sb, out_dtype, -splits)), (cfg, splits, out_dtype)


@pytest.mark.parametrize("splits", [4, 100, 101])
def test_workspace_split_k_and_stream_k_requests_run_plain(splits):
    m, n, k = 200, 328, 4096
    a, bt = small_ints((m, k), 1, 7), small_ints((n, k), 1, 8)
    sa, sb = block_scales(m, n, k, 9)
    got = bits(run(a, bt, m_major(sa), sb, torch.bfloat16, config_id=1, splits=splits))
    assert np.array_equal(got, want_bits(a, bt, sa, sb, torch.bfloat16)), splits


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("mnk", [(200, 328, 144), (1, 8, 16), (1, 4096, 1024), (129, 136, 272), (16, 4096, 1024),
                                 (1000, 1032, 1040), (3, 264, 400), (512, 512, 8192)])
def test_dispatched_ragged_shapes_bit_exact(mnk, out_dtype):
    from cuda_l2_b200 import ops
    m, n, k = mnk
    a, bt = small_ints((m, k), 1, m + k), small_ints((n, k), 1, n + 3 * k)
    sa, sb = block_scales(m, n, k, m + n)
    want = want_bits(a, bt, sa, sb, out_dtype, planned_splits(m, n, k))
    assert np.array_equal(bits(run(a, bt, m_major(sa), sb, out_dtype)), want), mnk
    y = ops.fp8_gemm(a.cuda(), bt.cuda(), sa, sb, out_dtype)          # contiguous [M, nkb] scale_a through the operator
    assert np.array_equal(bits(y), want), mnk


def test_every_m_from_1_to_16_bit_exact():
    n, k = 264, 400
    bt = small_ints((n, k), 1, 77)
    for m in range(1, 17):
        a = small_ints((m, k), 1, m)
        sa, sb = block_scales(m, n, k, 100 + m)
        for out_dtype in (torch.float16, torch.bfloat16):
            assert np.array_equal(bits(run(a, bt, m_major(sa), sb, out_dtype, config_id=12)),
                                  want_bits(a, bt, sa, sb, out_dtype)), (m, out_dtype)
            assert np.array_equal(bits(run(a, bt, m_major(sa), sb, out_dtype)),
                                  want_bits(a, bt, sa, sb, out_dtype, planned_splits(m, n, k))), m


@pytest.mark.parametrize("cfg", [1, 4, 30])
def test_row_stride_of_scale_a_larger_than_m(cfg):
    m, n, k = 300, 392, 528
    a, bt = small_ints((m, k), 1, 21), small_ints((n, k), 1, 22)
    sa, sb = block_scales(m, n, k, 23)
    for ld in (304, 512, 1000):
        view = m_major(sa, ld)                        # NaN in the padding: rows past M are read but never stored
        assert view.stride() == (1, ld)
        got = bits(run(a, bt, view, sb, torch.float16, config_id=cfg))
        assert np.array_equal(got, want_bits(a, bt, sa, sb, torch.float16)), (cfg, ld)


def test_scales_written_just_before_the_gemm_are_the_ones_used():
    from cuda_l2_b200 import ops
    m, n, k = 256, 256, 512
    a, bt = small_ints((m, k), 1, 5).cuda(), small_ints((n, k), 1, 6).cuda()
    sa, sb = block_scales(m, n, k, 7)
    view = m_major(sa)
    ops.fp8_gemm(a, bt, view, sb, torch.float16)
    for seed in (8, 9, 10):
        new_a, new_b = block_scales(m, n, k, seed)
        view.copy_(new_a); sb.copy_(new_b)                  # torch kernels, same stream, right before the GEMM
        y = ops.fp8_gemm(a, bt, view, sb, torch.float16)
        assert np.array_equal(bits(y), want_bits(a, bt, new_a, new_b, torch.float16)), seed


@pytest.mark.parametrize("mnk", [(512, 512, 8192), (256, 512, 1024)])
def test_graph_replay_reads_the_current_scales(mnk):
    from cuda_l2_b200 import ops
    m, n, k = mnk
    a, bt = small_ints((m, k), 1, 11).cuda(), small_ints((n, k), 1, 12).cuda()
    sa, sb = block_scales(m, n, k, 13)
    view = m_major(sa)
    splits = planned_splits(m, n, k)
    s = torch.cuda.Stream()                                  # no prewarm: the variant never needs scratch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        y = ops.fp8_gemm(a, bt, view, sb, torch.bfloat16)
    for seed in (14, 15, 16):
        new_a, new_b = block_scales(m, n, k, seed, pow2=seed % 2 == 0)
        view.copy_(new_a); sb.copy_(new_b)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(bits(y), want_bits(a, bt, new_a, new_b, torch.bfloat16, splits)), seed


@pytest.mark.parametrize("cfg,splits", [(1, 1), (2, 1), (4, 1), (12, 1), (14, 1), (30, 1), (1, -4), (2, -8)])
def test_guard_bands(cfg, splits):
    m, n, k = 200, 328, 4096
    a, bt = small_ints((m, k), 1, 17).cuda(), small_ints((n, k), 1, 18).cuda()
    sa, sb = block_scales(m, n, k, 19)
    pad = 4096
    buf = torch.full((m * n + 2 * pad,), -7.0, dtype=torch.float16, device="cuda")
    c = buf[pad:pad + m * n].view(m, n)
    c.fill_(float("nan"))
    capi.fp8_gemm(a, bt, c, m_major(sa), sb, config_id=cfg, splits=splits)
    torch.cuda.synchronize()
    assert np.array_equal(bits(c), want_bits(a, bt, sa, sb, torch.float16, max(1, -splits)))
    assert bool((buf[:pad] == -7).all()) and bool((buf[pad + m * n:] == -7).all())


def block_randn(m, n, k, seed):
    from cuda_l2_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, sa = ops.quantize_e4m3_blockwise(torch.randn((m, k), device="cuda", generator=g))
    bt, sb = ops.quantize_e4m3_block128x128(torch.randn((n, k), device="cuda", generator=g))
    return a, sa, bt, sb


def dequantised_product(a, sa, bt, sb):
    """fp64 product of the dequantised operands."""
    m, k = a.shape
    n = bt.shape[0]
    a64 = a.double() * sa.double().repeat_interleave(128, dim=1)[:, :k]
    b64 = bt.double() * sb.double().repeat_interleave(128, dim=0)[:n].repeat_interleave(128, dim=1)[:, :k]
    return a64 @ b64.t()


@pytest.mark.parametrize("mnk", [(4096, 4096, 4096), (2048, 11008, 4096)])
@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16])
def test_dispatched_path_within_tolerance_of_the_fp64_product(mnk, out_dtype):
    from cuda_l2_b200 import ops
    m, n, k = mnk
    a, sa, bt, sb = block_randn(m, n, k, 1)
    y = ops.fp8_gemm(a, bt, sa, sb, out_dtype).double()
    truth = dequantised_product(a, sa, bt, sb)
    err = float((y - truth).abs().max() / truth.pow(2).mean().sqrt())
    assert err <= RANDOM_TOL[out_dtype], (mnk, out_dtype, err)


def test_block_promotion_is_at_least_as_accurate_as_the_per_tensor_kernel_at_long_k():
    """K = 16384, N(0,1) data cast to e4m3 with unit scales: the per-tensor kernel sums all 16384 products in the FP8
    tensor core's reduced-precision accumulator, the block-scaled one 128 at a time and promotes each block in fp32."""
    from cuda_l2_b200 import ops
    m, n, k = 512, 512, 16384
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn((m, k), device="cuda", generator=g).to(E4)
    bt = torch.randn((n, k), device="cuda", generator=g).to(E4)
    one = torch.ones(1, device="cuda")
    truth = a.double() @ bt.double().t()
    rms = truth.pow(2).mean().sqrt()
    tensor = ops.fp8_gemm(a, bt, one, one, torch.float16).double()
    block = ops.fp8_gemm(a, bt, torch.ones((m, nkb(k)), device="cuda"), torch.ones((n // 128, nkb(k)), device="cuda"),
                         torch.float16).double()
    e_tensor = float((tensor - truth).pow(2).mean().sqrt() / rms)
    e_block = float((block - truth).pow(2).mean().sqrt() / rms)
    assert e_block <= e_tensor, (e_block, e_tensor)


@pytest.mark.parametrize("mnk", [(4096, 4096, 4096), (2048, 11008, 4096), (16, 4096, 4096)])
def test_bf16_output_against_torch_scaled_mm_blockwise(mnk):
    from cuda_l2_b200 import ops
    m, n, k = mnk
    a, sa, bt, sb = block_randn(m, n, k, 4)
    try:   # scale_a [M, nkb] with strides (1, M); scale_b [nkb, ceil(N/128)] for mat2 = bt.t()
        ref = torch._scaled_mm(a, bt.t(), scale_a=sa, scale_b=sb.t(), out_dtype=torch.bfloat16)
    except (RuntimeError, NotImplementedError, ValueError) as e:
        pytest.skip(f"torch._scaled_mm refuses blockwise scales here: {e}")
    y = ops.fp8_gemm(a, bt, sa, sb, torch.bfloat16)
    diff = float((y.float() - ref.float()).abs().max() / ref.float().pow(2).mean().sqrt())
    assert diff <= SCALED_MM_TOL, (mnk, diff)


def _linear_pair(out_dtype, seed, in_features=1024, out_features=512):
    from torch import nn

    from cuda_l2_b200 import ops
    torch.manual_seed(seed)
    lin = nn.Linear(in_features, out_features, dtype=out_dtype, device="cuda")
    return lin, ops.B200Fp8Linear.from_linear(lin, granularity="blockwise")


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16])
def test_blockwise_linear_agrees_with_its_source(out_dtype):
    lin, m = _linear_pair(out_dtype, 3)
    x = torch.randn(4, 33, 1024, dtype=out_dtype, device="cuda")
    with torch.no_grad():
        y, ref = m(x), lin(x)
    assert y.shape == ref.shape and y.dtype == out_dtype
    rel = float((y.float() - ref.float()).abs().max() / ref.float().pow(2).mean().sqrt())
    assert rel <= LINEAR_TOL, rel


def test_from_fp8_matches_the_dequantised_checkpoint():
    from cuda_l2_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(8)
    w = torch.randn((1000, 1040), device="cuda", generator=g)           # ragged in both block dimensions
    w_fp8, w_scale = ops.quantize_e4m3_block128x128(w)
    bias = torch.randn(1000, device="cuda", dtype=torch.bfloat16)
    layer = ops.B200Fp8Linear.from_fp8(w_fp8, w_scale, bias)
    x = torch.randn((3, 40, 1040), device="cuda", dtype=torch.bfloat16, generator=g)
    with torch.no_grad():
        y = layer(x)
    x_q, x_s = ops.quantize_e4m3_blockwise(x.reshape(-1, 1040))
    ref = dequantised_product(x_q, x_s, w_fp8, w_scale) + bias.double()
    assert y.shape == (3, 40, 1000) and y.dtype == torch.bfloat16
    err = float((y.reshape(-1, 1000).double() - ref).abs().max() / ref.pow(2).mean().sqrt())
    assert err <= FROM_FP8_TOL, err


def test_blockwise_linear_captures_in_a_graph():
    lin, m = _linear_pair(torch.bfloat16, 7)
    x = torch.randn(128, 1024, dtype=torch.bfloat16, device="cuda")
    s = torch.cuda.Stream()
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
