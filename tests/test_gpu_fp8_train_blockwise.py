"""Blockwise FP8 training of linear layers on the H100: the GEMM with 1 x 128 scales on both operands
(libb200_fp8block_1d1d.so), the dual-orientation block quantisers (libb200_quant_block_dual.so) and
fp8_linear(granularity="blockwise").

The 1D1D GEMM is checked three ways. With block-constant scales of Bt (sb[n, kb] = sb_block[n // 128, kb]) its contract
is libb200_fp8block.so's, so on any data, N(0,1) included, its bits must be that library's for the same configuration
and splits. With per-row scales it is bit-exact against tests/fp8_block_1d1d_ref.c on small integers, where every
k-block's tensor-core sum is exact (tests/test_gpu_fp8_blockwise.py's argument), and within the block-scaled tolerance
of the float64 product on N(0,1) data. The dispatched call is _run_config of _select's choice.
"""
import ctypes
import hashlib
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cuda_l2_b200 import capi, ops
from test_gpu_fp8 import small_ints

pytestmark = pytest.mark.gpu

E4 = torch.float8_e4m3fn
ELIGIBLE = (1, 2, 4, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 22, 23, 30)
SPLIT_K = (1, 2)                 # the configurations with cluster split-K kernels
ROWS = (1, 15, 16, 17, 127, 128, 129, 300, 4104)
COLS = (16, 136, 300, 4096, 11008)
RANDOM_TOL = {torch.float16: 0.005, torch.bfloat16: 0.025}   # as tests/test_gpu_fp8_blockwise.py
SCALED_MM_TOL = 0.03
LINEAR_TOL = 0.3                 # fp8_linear against the float64 product, as the rowwise recipe
LOSS_RATIO = 1.05                # final loss of the FP8-trained MLP over the bf16-trained one


@pytest.fixture(scope="module", autouse=True)
def _need_h100(built_libs):
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0) != (9, 0):
        pytest.skip("needs an H100")
    torch.cuda.set_device(0)


# ------------------------------------------------------------------------------------------------ helpers
_REF = Path(__file__).resolve().parent / "fp8_block_1d1d_ref.c"
_ref_lib = None


def _ref():
    """tests/fp8_block_1d1d_ref.c, built with gcc on first use into a per-user temporary directory."""
    global _ref_lib
    if _ref_lib is None:
        srcs = (_REF, _REF.parent.parent / "oracle" / "fp8_oracle.c", _REF.parent.parent / "oracle" / "hgemm_oracle.c")
        digest = hashlib.sha256(b"".join(p.read_bytes() for p in srcs)).hexdigest()[:16]
        out = Path(tempfile.gettempdir()) / f"cuda_l2_b200_ref_{os.getuid()}" / f"libfp8_block_1d1d_ref_{digest}.so"
        if not out.exists():
            out.parent.mkdir(parents=True, exist_ok=True)
            tmp = out.with_suffix(f".{os.getpid()}.tmp")
            subprocess.run([shutil.which("gcc"), "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o",
                            str(tmp), str(_REF), "-lm"], check=True)
            os.replace(tmp, out)
        _ref_lib = ctypes.CDLL(str(out))
        u8p, u16p, fp, i = (ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint16),
                            ctypes.POINTER(ctypes.c_float), ctypes.c_int)
        _ref_lib.ref_fp8gemm_f32acc_block_1d1d.argtypes = [u8p, u8p, fp, i, fp, i, u16p, i, i, i, i, i]
    return _ref_lib


def ref_1d1d(a, bt, sa, sb, out_dtype, splits=1):
    """The bits of C by the 1D1D contract: a [M,K], bt [N,K] e4m3; sa [M, nkb], sb [N, nkb] fp32."""
    (m, k), n = a.shape, bt.shape[0]
    u8p, u16p, fp = ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint16), ctypes.POINTER(ctypes.c_float)
    ac, bc = (np.ascontiguousarray(t.cpu().view(torch.uint8).numpy()) for t in (a, bt))
    sam, sbm = (np.ascontiguousarray(s.cpu().numpy().T.astype(np.float32)) for s in (sa, sb))
    c = np.empty((m, n), dtype=np.uint16)
    _ref().ref_fp8gemm_f32acc_block_1d1d(ac.ctypes.data_as(u8p), bc.ctypes.data_as(u8p), sam.ctypes.data_as(fp), m,
                                         sbm.ctypes.data_as(fp), n, c.ctypes.data_as(u16p), m, n, k,
                                         int(out_dtype == torch.bfloat16), splits)
    return c


def nkb(k):
    return -(-k // 128)


def m_major(s, ld=None):
    """The (1, ld)-strided view of s [M, nkb] the kernels read in place, ld = ld or M rounded up to 4 (NaN padding)."""
    m, kb = s.shape
    ld = ld or -(-m // 4) * 4
    buf = torch.full((kb, ld), float("nan"), dtype=torch.float32, device="cuda")
    buf[:, :m] = s.t()
    return buf[:, :m].t()


def bits(t):
    if t.dtype == E4:
        return t.view(torch.uint8)
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def run(a, bt, sa, sb, out_dtype, **kw):
    c = torch.full((a.shape[0], bt.shape[0]), float("nan"), dtype=out_dtype, device="cuda")
    capi.fp8_gemm(a, bt, c, sa, sb, **kw)
    return c


def rand_scales(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(shape, generator=g) * 2.9 + 0.1).cuda()


def randn_e4m3(m, n, k, seed):
    """N(0,1) operands quantised by the 1 x 128 kernel: a [M,K] with sa, bt [N,K] with per-row sb."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, sa = ops.quantize_e4m3_blockwise(torch.randn((m, k), device="cuda", generator=g))
    bt, sb = ops.quantize_e4m3_blockwise(torch.randn((n, k), device="cuda", generator=g))
    return a, sa, bt, sb


def plans(cfg):
    return [1] + ([-2, -4, -8] if cfg in SPLIT_K else [])


# ------------------------------------------------------------------------------------------------ the 1D1D GEMM
def test_block_constant_scales_give_the_128x128_kernels_bits():
    """Every eligible configuration, both output types, plain and (where it exists) every cluster split-K: with
    sb[n, kb] = sb_block[n // 128, kb], N(0,1) data, the bits of libb200_fp8block.so run the same way."""
    m, n, k = 333, 392, 1040
    a, sa, bt, _ = randn_e4m3(m, n, k, 1)
    sb_block = rand_scales((-(-n // 128), nkb(k)), 2)
    sb_rows = sb_block.repeat_interleave(128, 0)[:n]
    before = capi.fp8block_1d1d_launch_count()
    launches = 0
    for out_dtype in (torch.float16, torch.bfloat16):
        for cfg in ELIGIBLE:
            for splits in plans(cfg):
                want = run(a, bt, sa, sb_block, out_dtype, config_id=cfg, splits=splits)
                got = run(a, bt, sa, m_major(sb_rows), out_dtype, config_id=cfg, splits=splits)
                launches += 1
                torch.cuda.synchronize()
                assert torch.equal(bits(got), bits(want)), (cfg, splits, out_dtype)
    assert capi.fp8block_1d1d_launch_count() - before == launches


@pytest.mark.parametrize("mnk", [(520, 392, 400), (1, 136, 272), (200, 328, 4096), (129, 8, 16), (64, 1000, 1040)])
def test_per_row_scales_bit_exact_against_the_reference(mnk):
    """Small integers (exact k-block sums) with non-power-of-two per-row scales on both operands: N off BN and 128,
    K % 128 != 0, M = 1, every eligible configuration and cluster split-K, both output types."""
    m, n, k = mnk
    a, bt = small_ints((m, k), 1, m + k).cuda(), small_ints((n, k), 1, n + k).cuda()
    assert float((a.float() @ bt.float().t()).abs().max()) <= 2047
    sa, sb = rand_scales((m, nkb(k)), m), rand_scales((n, nkb(k)), n)
    for out_dtype in (torch.float16, torch.bfloat16):
        want = ref_1d1d(a, bt, sa, sb, out_dtype)
        for cfg in ELIGIBLE:
            got = run(a, bt, m_major(sa), m_major(sb), out_dtype, config_id=cfg, splits=1)
            assert np.array_equal(bits(got).cpu().numpy().view(np.uint16), want), (mnk, cfg, out_dtype)
        for cfg in SPLIT_K:
            for splits in (-2, -4, -8):
                plan = capi.schedule(cfg, m, n, k // 2, splits)
                s = sum(1 for units in plan["units"] for u in units if u[0] == 0) if plan["mode"] == "cluster-split-k" \
                    else 1
                got = run(a, bt, m_major(sa), m_major(sb), out_dtype, config_id=cfg, splits=splits)
                assert np.array_equal(bits(got).cpu().numpy().view(np.uint16), ref_1d1d(a, bt, sa, sb, out_dtype, s)), \
                    (mnk, cfg, splits)


@pytest.mark.parametrize("cfg", [1, 4, 12, 30])
def test_row_strides_of_both_scales_larger_than_the_rows(cfg):
    m, n, k = 300, 392, 528
    a, bt = small_ints((m, k), 1, 21).cuda(), small_ints((n, k), 1, 22).cuda()
    sa, sb = rand_scales((m, nkb(k)), 23), rand_scales((n, nkb(k)), 24)
    want = ref_1d1d(a, bt, sa, sb, torch.float16)
    for ld_a, ld_b in ((304, 392), (512, 396), (300 + 4, 1000)):
        va, vb = m_major(sa, ld_a), m_major(sb, ld_b)   # NaN past the rows: read, never stored
        assert vb.stride() == (1, ld_b)
        got = run(a, bt, va, vb, torch.float16, config_id=cfg)
        assert np.array_equal(bits(got).cpu().numpy().view(np.uint16), want), (cfg, ld_a, ld_b)


@pytest.mark.parametrize("mnk", [(512, 4096, 4096), (1024, 768, 8192), (136, 200, 16384), (3, 1024, 272)])
def test_dispatch_is_run_config_of_select(mnk):
    m, n, k = mnk
    a, sa, bt, sb = randn_e4m3(m, n, k, m + n)
    cfg, gm, sp = capi.fp8_blockwise_1d1d_select(m, n, k)
    assert (cfg, gm, sp) == capi.fp8_blockwise_select(m, n, k)
    for out_dtype in (torch.float16, torch.bfloat16):
        got = run(a, bt, sa, sb, out_dtype)
        want = run(a, bt, sa, sb, out_dtype, config_id=cfg, group_m=gm, splits=sp)
        assert torch.equal(bits(got), bits(want)), (mnk, out_dtype)
        truth = (a.double() * sa.double().repeat_interleave(128, 1)[:, :k]) @ \
                (bt.double() * sb.double().repeat_interleave(128, 1)[:, :k]).t()
        err = float((got.double() - truth).abs().max() / truth.pow(2).mean().sqrt())
        assert err <= RANDOM_TOL[out_dtype], (mnk, out_dtype, err)
    y = ops.fp8_gemm(a, bt, sa.contiguous(), sb.contiguous(), torch.bfloat16)   # contiguous scales through the operator
    assert torch.equal(bits(y), bits(run(a, bt, sa, sb, torch.bfloat16)))


def test_against_torch_scaled_mm_1x128_both_operands():
    m, n, k = 1024, 2048, 4096
    a, sa, bt, sb = randn_e4m3(m, n, k, 9)
    got = run(a, bt, sa, sb, torch.bfloat16)
    try:
        ref = torch._scaled_mm(a, bt.t(), scale_a=sa, scale_b=sb.t(), out_dtype=torch.bfloat16)
    except (RuntimeError, ValueError) as e:
        pytest.skip(f"torch._scaled_mm refuses 1 x 128 scales on both operands: {str(e).splitlines()[0]}")
    diff = float((got.float() - ref.float()).abs().max() / ref.float().pow(2).mean().sqrt())
    print(f"MEASURED 1D1D against torch._scaled_mm: {diff:.5f}")
    assert diff <= SCALED_MM_TOL


def test_bad_arguments_are_refused_before_a_launch():
    m, n, k = 64, 136, 256
    a, sa, bt, sb = randn_e4m3(m, n, k, 3)
    c = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
    lib = capi.fp8block_1d1d_lib()
    before = capi.fp8block_1d1d_launch_count()
    ld_a, ld_b = capi.blockwise_ld_a(sa), capi.blockwise_ld_a(sb)
    args = lambda ld_b=ld_b, sbp=sb.data_ptr(): (a.data_ptr(), bt.data_ptr(), c.data_ptr(), sa.data_ptr(), ld_a, sbp,
                                                 ld_b)
    assert lib.cuda_l2_b200_fp8block_1d1d_run(*args(ld_b=n - 4), 1, m, n, k, None) == -13
    assert lib.cuda_l2_b200_fp8block_1d1d_run(*args(ld_b=n + 2), 1, m, n, k, None) == -13
    assert lib.cuda_l2_b200_fp8block_1d1d_run(*args(sbp=sb.data_ptr() + 4), 1, m, n, k, None) == -2
    assert lib.cuda_l2_b200_fp8block_1d1d_run_config(3, 1, a.data_ptr(), bt.data_ptr(), c.data_ptr(), sa.data_ptr(),
                                                     ld_a, sb.data_ptr(), ld_b, m, n, k, 0, 0, 1, None) == -6
    assert capi.fp8block_1d1d_launch_count() == before


# ------------------------------------------------------------------------------------------------ the quantisers
def _activations(shape, dtype, seed):
    """Normal values whose magnitude varies by row and column over decades, plus an outlier per row."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g)
    x *= torch.exp(torch.empty((shape[0], 1), device="cuda").uniform_(-4, 4, generator=g))
    x *= torch.exp(torch.empty((1, shape[1]), device="cuda").uniform_(-2, 2, generator=g))
    x[torch.arange(shape[0], device="cuda"), (torch.arange(shape[0], device="cuda") * 7 + seed) % shape[1]] *= 8
    return x.to(dtype)


def _strides(t):
    """The strides of the dimensions that are stepped (a size-1 dimension's stride is arbitrary)."""
    return tuple(st for st, size in zip(t.stride(), t.shape) if size > 1)


def _same(got, want, what=""):
    for i, (g, w) in enumerate(zip(got, want)):
        assert (g.shape, g.dtype, _strides(g)) == (w.shape, w.dtype, _strides(w)), (what, i)
        if not torch.equal(bits(g), bits(w)):
            bad = (bits(g) != bits(w)).nonzero()[:5].tolist()
            raise AssertionError(f"{what} result {i}: {int((bits(g) != bits(w)).sum())} elements differ, first at {bad}")


def _both_same(x, what=""):
    before = capi.quant_block_dual_launch_count()
    got = ops.quantize_e4m3_blockwise_dual(x)
    _same(got, ops.quantize_e4m3_blockwise_dual_reference(x), f"1x128 {what}")
    q, s = ops.quantize_e4m3_blockwise(x)   # q and its scale equal the single-orientation kernel's
    _same(got[:2], (q, s), f"1x128 against the 1 x 128 kernel {what}")
    _same(ops.quantize_e4m3_block128x128_dual(x), ops.quantize_e4m3_block128x128_dual_reference(x), f"128x128 {what}")
    assert capi.quant_block_dual_launch_count() - before == 2


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("rows", ROWS)
def test_quantisers_against_the_compositions(dtype, rows):
    for cols in COLS:
        _both_same(_activations((rows, cols), dtype, seed=rows + cols), f"{rows}x{cols} {dtype}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_every_bit_pattern(dtype):
    v = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(dtype)
    finite = v[torch.isfinite(v)]
    finite = finite[torch.argsort(finite.float().abs(), stable=True)]
    g = torch.Generator(device="cuda").manual_seed(11)
    for i, x in enumerate((finite, finite[torch.randperm(finite.numel(), device="cuda", generator=g)],
                           v[torch.randperm(v.numel(), device="cuda", generator=g)])):
        x = torch.cat([x, torch.zeros(-x.numel() % 65536, dtype=dtype, device="cuda")]).view(256, 256)
        _both_same(x, f"patterns {i}")
        _both_same(x.t().contiguous(), f"patterns {i} transposed")
        _both_same(x.reshape(-1)[:300 * 200].view(300, 200), f"patterns {i} 300 x 200")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("rows", [17, 128, 300])
def test_zero_signed_zero_subnormal_inf_nan_rows_columns_and_tiles(dtype, rows):
    sub = torch.finfo(dtype).tiny / 8
    x = _activations((rows, 392), torch.float32, seed=rows).to(dtype)
    x[1], x[2], x[3] = 0.0, -0.0, sub
    x[4, ::2] = -sub
    x[5, 3], x[6, 9], x[7, 11] = float("inf"), float("-inf"), float("nan")
    x[:, 0], x[:, 1], x[:, 2] = 0.0, -0.0, sub
    x[10, 140], x[12, 141] = float("inf"), float("nan")
    x[:, 8] = 448.0
    x[:, 256:] = 0.0                              # a whole zero tile column
    if rows > 128:
        x[128:256, 128:256] = float("nan")        # a NaN tile
    _both_same(x, "special")
    q, s, q_t, s_t = ops.quantize_e4m3_blockwise_dual(x)
    ld_t = capi.dual_ld_t(rows)
    if ld_t > rows:   # the padding of the last row block: e4m3(0 / s), 0x00, and the NaN code where s is NaN
        pad = bits(q_t[:, rows:])
        nan_cols = torch.isnan(s_t[:, -1])
        assert (pad[nan_cols] == 0x7F).all() and (pad[~nan_cols] == 0).all()


def test_unaligned_inputs():
    base = _activations((300, 1040), torch.bfloat16, seed=5)
    flat = base.reshape(-1)[3:3 + 300 * 1024].view(300, 1024)
    assert flat.data_ptr() % 16 == 6
    _both_same(flat, "unaligned")
    _both_same(base[:, 1:1025], "strided")
    for dtype in (torch.float16, torch.bfloat16):
        _both_same(_activations((2000, 1040), dtype, seed=9).reshape(-1)[1:1 + 37 * 4100].view(37, 4100), "odd")


def test_cuda_graph_capture_and_replay():
    x = _activations((300, 1536), torch.bfloat16, seed=2)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        ops.quantize_e4m3_blockwise_dual(x)
        ops.quantize_e4m3_block128x128_dual(x)
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.quantize_e4m3_blockwise_dual(x)
        out_w = ops.quantize_e4m3_block128x128_dual(x)
    for seed in (7, 8):
        x.copy_(_activations(x.shape, torch.bfloat16, seed=seed))
        if seed == 8:
            x[:, 5] = float("nan")
        graph.replay()
        torch.cuda.synchronize()
        _same(out, ops.quantize_e4m3_blockwise_dual_reference(x), f"graph {seed}")
        _same(out_w, ops.quantize_e4m3_block128x128_dual_reference(x), f"graph 128x128 {seed}")


def test_concurrent_calls_on_two_streams():
    xs = [_activations((4104, 4096), torch.bfloat16, seed=20 + i) for i in range(2)]
    want = [ops.quantize_e4m3_blockwise_dual_reference(x) for x in xs]
    streams = [torch.cuda.Stream() for _ in xs]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    outs = [[], []]
    for _ in range(6):
        for i, (x, s) in enumerate(zip(xs, streams)):
            with torch.cuda.stream(s):
                outs[i].append(ops.quantize_e4m3_blockwise_dual(x))
    torch.cuda.synchronize()
    for i in range(2):
        for got in outs[i]:
            _same(got, want[i], f"stream {i}")


# ------------------------------------------------------------------------------------------------ fp8_linear
def _reference_step(x2, w, gy):
    """y, dX, dW of blockwise fp8_linear from the reference quantisers and fp8_gemm."""
    xq, xs, xqt, xst = ops.quantize_e4m3_blockwise_dual_reference(x2)
    wq, ws, wqt, wst = ops.quantize_e4m3_block128x128_dual_reference(w)
    gq, gs, gqt, gst = ops.quantize_e4m3_blockwise_dual_reference(gy)
    return (ops.fp8_gemm(xq, wq, xs, ws, x2.dtype), ops.fp8_gemm(gq, wqt, gs, wst, x2.dtype),
            ops.fp8_gemm(gqt, xqt, gst, xst, w.dtype))


def _counts():
    return (capi.quant_block_dual_launch_count(), capi.quant_launch_count(), capi.fp8block_launch_count(),
            capi.fp8block_1d1d_launch_count())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("lead", [(300,), (37,), (3, 45)])
@pytest.mark.parametrize("need", [(True, True), (True, False), (False, True), (False, False)])
def test_fp8_linear_is_the_chain_of_reference_quantisers_and_fp8_gemm(dtype, lead, need):
    n, k = 272, 1040
    x = _activations((lead[0] * (lead[1] if len(lead) > 1 else 1), k), dtype, seed=3).view(*lead, k)
    w = (_activations((n, k), torch.float32, seed=4) / 64).to(dtype)
    gy = _activations((x.numel() // k, n), dtype, seed=5)
    want_y, want_dx, want_dw = _reference_step(x.reshape(-1, k), w, gy)
    x.requires_grad_(need[0])
    w.requires_grad_(need[1])
    before = _counts()
    y = ops.fp8_linear(x, w, granularity="blockwise")
    assert y.shape == (*lead, n)
    assert torch.equal(bits(y.detach().reshape(-1, n)), bits(want_y))
    if any(need):
        y.backward(gy.view(*lead, n))
    dual, quant, block, one_d = (a - b for a, b in zip(_counts(), before))
    if need[0]:
        assert torch.equal(bits(x.grad.reshape(-1, k)), bits(want_dx)) and x.grad.dtype == dtype
    if need[1]:
        assert torch.equal(bits(w.grad), bits(want_dw)) and w.grad.dtype == dtype
    # dual launches: x and dY for dW, W for dX; single 1 x 128 launches: x without dW, dY for dX without dW
    assert dual == 2 * need[1] + need[0], need
    assert quant == (0 if need[1] else 1) + (1 if need[0] and not need[1] else 0), need
    assert (block, one_d) == (1 + need[0], int(need[1])), need


def test_zero_tokens_launch_nothing():
    w = torch.randn((64, 128), device="cuda", dtype=torch.bfloat16).requires_grad_()
    x = torch.empty((0, 128), device="cuda", dtype=torch.bfloat16).requires_grad_()
    before = _counts()
    y = ops.fp8_linear(x, w, "blockwise")
    y.sum().backward()
    assert _counts() == before
    assert y.shape == (0, 64) and x.grad.shape == (0, 128) and not w.grad.view(torch.int16).any()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_eval_mode_is_b200_fp8_linear_blockwise(dtype):
    lin = torch.nn.Linear(1040, 528, device="cuda", dtype=dtype)
    train = ops.B200Fp8TrainLinear.from_linear(lin, granularity="blockwise")
    infer = ops.B200Fp8Linear.from_linear(lin, granularity="blockwise")
    x = _activations((300, 1040), dtype, seed=6).view(3, 100, 1040)
    want = infer(x)
    train.eval()
    with torch.no_grad():
        assert torch.equal(bits(train(x)), bits(want))
    assert torch.equal(bits(train(x).detach()), bits(want))   # with the gradient's copies prepared, the same bits


def _rel(got, truth):
    return float((got.double() - truth).abs().max() / truth.pow(2).mean().sqrt())


def test_outlier_tokens_blockwise_weight_gradient_is_no_worse_than_rowwise():
    """T = 16384 tokens with a few outliers (x 1000) in x and dY: the errors of y, dX and dW against the float64 product
    of the 16-bit operands (max |error| / rms, which the outlier rows dominate for y and dX), blockwise against
    rowwise; dW within the random-data bound."""
    t, n, k = 16384, 1024, 1024
    g = torch.Generator(device="cuda").manual_seed(12)
    x = torch.randn((t, k), device="cuda", generator=g)
    gy = torch.randn((t, n), device="cuda", generator=g)
    x[[17, 5000, 9001]] *= 1000
    gy[[40, 12000]] *= 1000
    x, gy = x.bfloat16(), gy.bfloat16()
    w = (torch.randn((n, k), device="cuda", generator=g) / 32).bfloat16()
    xd, wd, gd = x.double(), w.double(), gy.double()
    truth = {"y": xd @ wd.t(), "dx": gd @ wd, "dw": gd.t() @ xd}
    errs = {}
    for gran in ("rowwise", "blockwise"):
        xx, ww = x.clone().requires_grad_(), w.clone().requires_grad_()
        y = ops.fp8_linear(xx, ww, gran)
        y.backward(gy)
        errs[gran] = {"y": _rel(y.detach(), truth["y"]), "dx": _rel(xx.grad, truth["dx"]),
                      "dw": _rel(ww.grad, truth["dw"])}
    print(f"MEASURED outlier tokens: {errs}")
    for name in ("y", "dx", "dw"):
        assert errs["blockwise"][name] <= errs["rowwise"][name], (name, errs)
    assert errs["blockwise"]["dw"] <= LINEAR_TOL, errs


def test_training_step_captured_in_a_cuda_graph():
    layer = ops.B200Fp8TrainLinear(1024, 768, device="cuda", granularity="blockwise")
    x = _activations((500, 1024), torch.bfloat16, seed=7).requires_grad_()
    gy = _activations((500, 768), torch.bfloat16, seed=8)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for _ in range(2):
            layer.zero_grad(set_to_none=True)
            x.grad = None
            layer(x).backward(gy)
    torch.cuda.current_stream().wait_stream(stream)
    layer.zero_grad(set_to_none=True)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = layer(x)
        y.backward(gy)
    for seed in (9, 10):
        with torch.no_grad():
            x.copy_(_activations(x.shape, torch.bfloat16, seed=seed))
            gy.copy_(_activations(gy.shape, torch.bfloat16, seed=seed + 1))
            layer.weight.add_(0.01)
        graph.replay()
        torch.cuda.synchronize()
        want_y, want_dx, want_dw = _reference_step(x.detach(), layer.weight.detach(), gy)
        assert torch.equal(bits(y.detach()), bits(want_y + layer.bias.detach()))
        assert torch.equal(bits(x.grad), bits(want_dx)) and torch.equal(bits(layer.weight.grad), bits(want_dw))


def _train_mlp(kind: str, steps: int = 300):
    """The 256 -> 512 -> 256 GELU MLP of tests/test_gpu_fp8_train.py, fitted by Adam to a fixed random teacher."""
    torch.manual_seed(0)
    g = torch.Generator(device="cuda").manual_seed(1)
    teacher = [torch.randn((512, 256), device="cuda", generator=g) / 16, torch.randn((256, 512), device="cuda",
                                                                                       generator=g) / 22]
    lins = [torch.nn.Linear(256, 512, device="cuda", dtype=torch.bfloat16),
            torch.nn.Linear(512, 256, device="cuda", dtype=torch.bfloat16)]
    if kind == "bf16":
        layers = [ops.B200Linear.from_linear(lin) for lin in lins]
    else:
        layers = [ops.B200Fp8TrainLinear.from_linear(lin, granularity=kind) for lin in lins]
    model = torch.nn.Sequential(layers[0], torch.nn.GELU(), layers[1])
    opt = torch.optim.Adam(model.parameters(), lr=2e-3)
    losses = []
    for _ in range(steps):
        x = torch.randn((512, 256), device="cuda", generator=g)
        target = F.gelu(x @ teacher[0].t()) @ teacher[1].t()
        loss = F.mse_loss(model(x.bfloat16()).float(), target)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(loss.detach())
    return (float(torch.stack(losses[:20]).mean()), float(torch.stack(losses[-20:]).mean()),
            [p.detach().clone() for p in model.parameters()])


def test_mlp_training_is_deterministic_and_close_to_bf16():
    first, loss_a, params_a = _train_mlp("blockwise")
    _, loss_b, params_b = _train_mlp("blockwise")
    for a, b in zip(params_a, params_b):
        assert torch.equal(bits(a), bits(b))
    first_bf16, loss_bf16, _ = _train_mlp("bf16")
    print(f"MEASURED mlp loss blockwise fp8 {first:.6g} -> {loss_a:.6g}, bf16 {first_bf16:.6g} -> {loss_bf16:.6g}, "
          f"ratio {loss_a / loss_bf16:.4f}")
    assert loss_a < 0.5 * first
    assert loss_a <= LOSS_RATIO * loss_bf16, (loss_a, loss_bf16)
