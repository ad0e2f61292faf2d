"""The e4m3 quantisers of libb200_quant.so on the H100, bit for bit against the torch compositions they replace
(``ops.*_reference``), run on the same device: every granularity and input dtype, 2-D and batched, ragged K and M;
every fp16 and bf16 bit pattern inside blocks; every fp16 and bf16 gate value through the SwiGLU kernel's silu; zero,
-0.0, subnormal, Inf and NaN blocks; masked row counts with NaN sentinels; launch counts, CUDA-graph replay and two
concurrent streams; and B200Fp8GroupedMLP against the same chain built from the torch quantisers."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cuda_l2_b200 import capi, ops

pytestmark = pytest.mark.gpu

DTYPES = (torch.float16, torch.bfloat16, torch.float32)
KS = (16, 128, 300, 7168, 18432)


@pytest.fixture(scope="module", autouse=True)
def _need_h100(built_libs):
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0) != (9, 0):
        pytest.skip("needs an H100")
    torch.cuda.set_device(0)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t.view(torch.int32)


def _same(got, want, what=""):
    """(q, scale) pairs equal bit for bit, with the same shapes, dtypes and strides."""
    for g, w in zip(got, want):
        assert (g.shape, g.dtype, g.stride()) == (w.shape, w.dtype, w.stride()), what
        if not torch.equal(_bits(g), _bits(w)):
            bad = (_bits(g) != _bits(w)).nonzero()[:5].tolist()
            raise AssertionError(f"{what}: {int((_bits(g) != _bits(w)).sum())} elements differ, first at {bad}")


def _activations(shape, dtype, seed):
    """Normal values whose magnitude varies by row over six decades, plus one outlier per row."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g)
    x *= torch.exp(torch.empty(shape[:-1] + (1,), device="cuda").uniform_(-7, 7, generator=g))
    x[..., (seed * 7) % shape[-1]] *= 50
    return x.to(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("k", KS)
def test_every_granularity_against_the_composition(dtype, k):
    for m in (37, 130):
        x = _activations((m, k), dtype, seed=m + k)
        _same(ops.quantize_e4m3(x), ops.quantize_e4m3_reference(x), f"tensor {m}x{k}")
        _same(ops.quantize_e4m3_rowwise(x), ops.quantize_e4m3_rowwise_reference(x), f"rowwise {m}x{k}")
        _same(ops.quantize_e4m3_blockwise(x), ops.quantize_e4m3_blockwise_reference(x), f"blockwise {m}x{k}")
    xb = _activations((3, 37, k), dtype, seed=k)
    _same(ops.quantize_e4m3(xb), ops.quantize_e4m3_reference(xb), f"tensor 3x37x{k}")
    _same(ops.quantize_e4m3_blockwise(xb), ops.quantize_e4m3_blockwise_reference(xb), f"blockwise 3x37x{k}")


@pytest.mark.parametrize("dtype", DTYPES[:2])
@pytest.mark.parametrize("i", KS)
def test_silu_mul_against_the_composition(dtype, i):
    for shape in ((37, 2 * i), (3, 37, 2 * i)):
        h = _activations(shape, dtype, seed=i + len(shape))
        _same(ops.silu_mul_quantize_e4m3_blockwise(h), ops.silu_mul_quantize_e4m3_blockwise_reference(h), str(shape))


def test_unaligned_and_strided_inputs():
    """Element loads where no 16-byte vector fits (a view that starts off the alignment), and non-contiguous views."""
    base = _activations((64, 1040), torch.bfloat16, seed=5)
    x = base[:, 1:1025]   # rows of 1024 starting 2 bytes in: no vector loads, and not contiguous
    for got, want in ((ops.quantize_e4m3(x), ops.quantize_e4m3_reference(x)),
                      (ops.quantize_e4m3_rowwise(x), ops.quantize_e4m3_rowwise_reference(x)),
                      (ops.quantize_e4m3_blockwise(x), ops.quantize_e4m3_blockwise_reference(x)),
                      (ops.silu_mul_quantize_e4m3_blockwise(x), ops.silu_mul_quantize_e4m3_blockwise_reference(x))):
        _same(got, want, "strided")
    flat = base.reshape(-1)[3:3 + 64 * 1024].view(64, 1024)   # contiguous, 6 bytes off a 16-byte boundary
    assert flat.data_ptr() % 16 == 6
    q = torch.empty((64, 1024), dtype=torch.float8_e4m3fn, device="cuda")
    scale = torch.empty(1, device="cuda")
    capi.quantize_e4m3(flat, q, scale, torch.empty(capi.QUANT_TENSOR_WORKSPACE, device="cuda"))
    _same((q, scale), ops.quantize_e4m3_reference(flat), "unaligned tensor")
    scale = torch.empty((64, 1), device="cuda")
    capi.quantize_e4m3_rowwise(flat, q, scale)
    _same((q, scale), ops.quantize_e4m3_rowwise_reference(flat), "unaligned rowwise")
    want = ops.quantize_e4m3_blockwise_reference(flat)
    scale = torch.empty_like(want[1].transpose(0, 1)).transpose(0, 1)   # the same M-major layout
    capi.quantize_e4m3_blockwise(flat, q, scale)
    _same((q, scale), want, "unaligned blockwise")
    want = ops.silu_mul_quantize_e4m3_blockwise_reference(flat)
    q = torch.empty((64, 512), dtype=torch.float8_e4m3fn, device="cuda")
    scale = torch.empty_like(want[1].transpose(0, 1)).transpose(0, 1)
    capi.silu_mul_quantize_e4m3_blockwise(flat, q, scale)
    _same((q, scale), want, "unaligned silu")


def _all_patterns(dtype) -> torch.Tensor:
    """Every 16-bit pattern of ``dtype`` as a CUDA tensor."""
    return torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(dtype)


def _pattern_matrices(dtype) -> list[torch.Tensor]:
    """Every pattern of ``dtype`` inside 1 x 128 blocks, in three arrangements: finite values sorted by magnitude (each
    block's values close to its amax, so the quotients span e4m3's normal range and its rounding boundaries), the
    same values in a random order (quotients deep into e4m3's subnormals and zero), and every pattern, Inf and NaN
    among them, in a random order."""
    v = _all_patterns(dtype)
    finite = v[torch.isfinite(v)]
    finite = finite[torch.argsort(finite.float().abs(), stable=True)]
    g = torch.Generator(device="cuda").manual_seed(11)
    out = []
    for x in (finite, finite[torch.randperm(finite.numel(), device="cuda", generator=g)],
              v[torch.randperm(v.numel(), device="cuda", generator=g)]):
        pad = -x.numel() % 1024
        x = torch.cat([x, torch.zeros(pad, dtype=dtype, device="cuda")])
        out.append(x.view(-1, 1024))
    return out


@pytest.mark.parametrize("dtype", DTYPES[:2])
def test_every_bit_pattern_through_every_quantiser(dtype):
    for i, x in enumerate(_pattern_matrices(dtype)):
        _same(ops.quantize_e4m3_blockwise(x), ops.quantize_e4m3_blockwise_reference(x), f"blockwise {i}")
        _same(ops.quantize_e4m3_rowwise(x), ops.quantize_e4m3_rowwise_reference(x), f"rowwise {i}")
        r = x.view(-1, 128)
        _same(ops.quantize_e4m3_rowwise(r), ops.quantize_e4m3_rowwise_reference(r), f"rowwise 128 {i}")
        for chunk in x.view(16, -1):   # per tensor: 16 tensors, each with its own amax
            _same(ops.quantize_e4m3(chunk), ops.quantize_e4m3_reference(chunk), f"tensor {i}")
        # the SwiGLU quantiser on the same blocks: gate = the patterns, up = the patterns in another order
        h = torch.cat([x, x.flip(0)], dim=1)
        _same(ops.silu_mul_quantize_e4m3_blockwise(h), ops.silu_mul_quantize_e4m3_blockwise_reference(h), f"silu {i}")


@pytest.mark.parametrize("dtype", DTYPES[:2])
def test_every_gate_value_through_the_silu(dtype):
    """Each gate pattern alone in a block, every other gate 0 and every up 1: the block's scale is then
    |RN(silu(g))| * fp32(1/448), which tells every distinct 16-bit |silu(g)| apart, so the scales compare the kernel's
    silu (full-precision expf) with F.silu's, bit for bit, for every gate value; q carries the sign."""
    v = _all_patterns(dtype)
    blocks = 8                                          # blocks per row
    g = torch.zeros((v.numel() // blocks, blocks, 128), dtype=dtype, device="cuda")
    g[:, :, 0] = v.view(-1, blocks)
    g = g.view(g.shape[0], -1)
    h = torch.cat([g, torch.ones_like(g)], dim=1)
    got = ops.silu_mul_quantize_e4m3_blockwise(h)
    want = ops.quantize_e4m3_blockwise_reference(F.silu(g))
    _same(got, want, "silu")
    # and the reference's scales are the silu values themselves, |F.silu(g)| * fp32(1/448)
    s = F.silu(v).float().abs() * torch.tensor(1 / 448, dtype=torch.float32)
    s = torch.where(s < torch.finfo(torch.float32).tiny, torch.finfo(torch.float32).tiny, s)
    finite = torch.isfinite(s)
    assert torch.equal(_bits(got[1].reshape(-1)[finite]), _bits(s[finite].contiguous()))


def _special_blocks(dtype) -> torch.Tensor:
    tiny = torch.finfo(dtype).tiny if dtype != torch.float32 else 1e-40   # a subnormal of each type
    sub = tiny / 8 if dtype != torch.float32 else tiny
    rows = [torch.zeros(128), torch.full((128,), -0.0), torch.full((128,), sub), torch.full((128,), -sub),
            torch.linspace(-sub * 4, sub * 4, 128), torch.ones(128), torch.ones(128), torch.ones(128),
            torch.ones(128), torch.full((128,), 448.0), torch.full((128,), -1e-3)]
    rows[5][17] = float("inf")
    rows[6][3] = float("-inf")
    rows[7][100] = float("nan")
    rows[8][0] = 3e4                                    # one outlier: the rest of its block goes to small codes
    rows[10][64] = -0.0
    x = torch.stack(rows).to(dtype)
    x[2:5, ::3] = -0.0
    return x.cuda()


@pytest.mark.parametrize("dtype", DTYPES)
def test_zero_signed_zero_subnormal_inf_nan_and_outlier_blocks(dtype):
    x = _special_blocks(dtype)
    xb = torch.cat([x, _activations((x.shape[0], 172), dtype, seed=3)], dim=1)   # a second, ragged k-block
    _same(ops.quantize_e4m3_blockwise(xb), ops.quantize_e4m3_blockwise_reference(xb), "blockwise")
    _same(ops.quantize_e4m3_rowwise(x), ops.quantize_e4m3_rowwise_reference(x), "rowwise")
    for r in range(x.shape[0]):
        _same(ops.quantize_e4m3(x[r]), ops.quantize_e4m3_reference(x[r]), f"tensor row {r}")
    q, s = ops.quantize_e4m3_blockwise(x)
    assert (_bits(q[1]) == 0x80).all() and (_bits(q[0]) == 0).all()          # -0.0 keeps its sign, +0.0 stays 0
    assert s[0, 0] == torch.finfo(torch.float32).tiny and torch.isnan(s[7, 0]) and ((_bits(q[7]) & 0x7F) == 0x7F).all()
    if dtype != torch.float32:
        _same(ops.silu_mul_quantize_e4m3_blockwise(torch.cat([x, x.flip(0)], 1)),
              ops.silu_mul_quantize_e4m3_blockwise_reference(torch.cat([x, x.flip(0)], 1)), "silu")


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("k", [128, 300, 7168])
def test_masked_rows_are_identical_and_padding_is_never_written(silu, k):
    bsz, m = 6, 75
    counts = torch.tensor([0, m, m + 9, 33, -4, 1], dtype=torch.int32, device="cuda")
    x = _activations((bsz, m, 2 * k if silu else k), torch.bfloat16, seed=k + silu)
    nkb = capi.num_k_blocks(k)
    q = torch.full((bsz, m, k), 0x7F, dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)   # NaN sentinels
    buf = torch.full((bsz, nkb, 76), float("nan"), device="cuda")
    scale = buf[..., :m].transpose(1, 2)
    before = capi.quant_launch_count()
    call = capi.silu_mul_quantize_e4m3_blockwise if silu else capi.quantize_e4m3_blockwise
    call(x, q, scale, counts)
    torch.cuda.synchronize()
    assert capi.quant_launch_count() - before == 1
    ref = ops.silu_mul_quantize_e4m3_blockwise_reference if silu else ops.quantize_e4m3_blockwise_reference
    want_q, want_s = ref(x)
    for b, c in enumerate(counts.tolist()):
        rows = min(max(c, 0), m)
        assert torch.equal(_bits(q[b, :rows]), _bits(want_q[b, :rows])), b
        assert torch.equal(_bits(scale[b, :rows]), _bits(want_s[b, :rows])), b
        assert (_bits(q[b, rows:]) == 0x7F).all(), b
        assert torch.isnan(scale[b, rows:]).all() and torch.isnan(buf[b, :, m:]).all(), b
    # the operator's valid rows are the same bits
    op = ops.silu_mul_quantize_e4m3_blockwise if silu else ops.quantize_e4m3_blockwise
    got_q, got_s = op(x, counts)
    for b, c in enumerate(counts.tolist()):
        rows = min(max(c, 0), m)
        assert torch.equal(_bits(got_q[b, :rows]), _bits(want_q[b, :rows]))
        assert torch.equal(_bits(got_s[b, :rows]), _bits(want_s[b, :rows]))


def test_one_launch_per_call_two_per_tensor_and_none_for_empty_inputs():
    x = _activations((64, 4096), torch.bfloat16, seed=1)
    for fn, launches in ((ops.quantize_e4m3, 2), (ops.quantize_e4m3_rowwise, 1), (ops.quantize_e4m3_blockwise, 1),
                         (ops.silu_mul_quantize_e4m3_blockwise, 1)):
        before = capi.quant_launch_count()
        fn(x)
        assert capi.quant_launch_count() - before == launches, fn.__name__
    before = capi.quant_launch_count()
    for shape in ((0, 256), (5, 0), (2, 0, 256)):
        e = torch.empty(shape, dtype=torch.bfloat16, device="cuda")
        _same(ops.quantize_e4m3_blockwise(e), ops.quantize_e4m3_blockwise_reference(e), str(shape))
        _same(ops.silu_mul_quantize_e4m3_blockwise(e), ops.silu_mul_quantize_e4m3_blockwise_reference(e), str(shape))
    e = torch.empty((0, 256), dtype=torch.bfloat16, device="cuda")
    _same(ops.quantize_e4m3_rowwise(e), ops.quantize_e4m3_rowwise_reference(e), "rowwise empty")
    assert capi.quant_launch_count() == before


def test_cuda_graph_capture_and_replay():
    x = _activations((96, 2 * 1536), torch.bfloat16, seed=2)
    xb = _activations((4, 40, 1536), torch.bfloat16, seed=4)
    counts = torch.tensor([40, 3, 0, 17], dtype=torch.int32, device="cuda")
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):   # warm-up outside the capture
        ops.quantize_e4m3(x), ops.silu_mul_quantize_e4m3_blockwise(x), ops.quantize_e4m3_blockwise(xb, counts)
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_t = ops.quantize_e4m3(x)
        out_r = ops.quantize_e4m3_rowwise(x)
        out_s = ops.silu_mul_quantize_e4m3_blockwise(x)
        out_m = ops.quantize_e4m3_blockwise(xb, counts)
    for seed in (7, 8):
        x.copy_(_activations(x.shape, torch.bfloat16, seed=seed))
        xb.copy_(_activations(xb.shape, torch.bfloat16, seed=seed + 10))
        counts.copy_(torch.tensor([seed, 40, 41, 0], dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        _same(out_t, ops.quantize_e4m3_reference(x), "graph tensor")
        _same(out_r, ops.quantize_e4m3_rowwise_reference(x), "graph rowwise")
        _same(out_s, ops.silu_mul_quantize_e4m3_blockwise_reference(x), "graph silu")
        want = ops.quantize_e4m3_blockwise_reference(xb)
        for b, c in enumerate(counts.tolist()):
            rows = min(c, 40)
            assert torch.equal(_bits(out_m[0][b, :rows]), _bits(want[0][b, :rows]))
            assert torch.equal(_bits(out_m[1][b, :rows]), _bits(want[1][b, :rows]))


def test_concurrent_calls_on_two_streams():
    xs = [_activations((512, 7168), torch.bfloat16, seed=20 + i) for i in range(2)]
    want = [(ops.quantize_e4m3_reference(x), ops.quantize_e4m3_blockwise_reference(x),
             ops.silu_mul_quantize_e4m3_blockwise_reference(x)) for x in xs]
    streams = [torch.cuda.Stream() for _ in xs]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    outs = [[], []]
    for _ in range(8):
        for i, (x, s) in enumerate(zip(xs, streams)):
            with torch.cuda.stream(s):
                outs[i].append((ops.quantize_e4m3(x), ops.quantize_e4m3_blockwise(x),
                                ops.silu_mul_quantize_e4m3_blockwise(x)))
    torch.cuda.synchronize()
    for i in range(2):
        for got in outs[i]:
            for g, w in zip(got, want[i]):
                _same(g, w, f"stream {i}")


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float16])
def test_grouped_mlp_is_the_chain_of_torch_quantisers(out_dtype):
    g, hid, inter = 5, 512, 384
    gen = torch.Generator(device="cuda").manual_seed(9)
    w13 = (torch.randn((g, 2 * inter, hid), device="cuda", generator=gen) / 16).to(out_dtype)
    w2 = (torch.randn((g, hid, inter), device="cuda", generator=gen) / 16).to(out_dtype)
    mlp = ops.B200Fp8GroupedMLP.from_weights(w13, w2)
    sizes = [37, 0, 130, 1, 90]
    offs = torch.tensor(np.cumsum(sizes).tolist(), dtype=torch.int32, device="cuda")
    t = sum(sizes)
    x = torch.randn((t + 6, hid), device="cuda", generator=gen).to(out_dtype)

    def chain(xq, xs, gemm, quant_silu, *extra):
        h = gemm(xq, mlp.w13_fp8, xs, mlp.w13_scale, *extra)
        pq, ps = quant_silu(h)
        return gemm(pq, mlp.w2_fp8, ps, mlp.w2_scale, *extra)

    before = capi.quant_launch_count()
    y = mlp(x, offs)
    assert capi.quant_launch_count() - before == 2
    want = chain(*ops.quantize_e4m3_blockwise_reference(x), ops.fp8_grouped_gemm,
                 ops.silu_mul_quantize_e4m3_blockwise_reference, offs, out_dtype)
    assert torch.equal(y[:t].view(torch.int16), want[:t].view(torch.int16))
    # the decode layout: one slot of M tokens per expert, counts 0, M, above M and ragged
    m = 48
    counts = torch.tensor([m, 0, 17, m + 3, 1], dtype=torch.int32, device="cuda")
    xm = torch.randn((g, m, hid), device="cuda", generator=gen).to(out_dtype)
    ym = mlp.forward_masked(xm, counts)
    xq, xs = ops.quantize_e4m3_blockwise_reference(xm)
    h = ops.fp8_batched_gemm(xq, mlp.w13_fp8, xs, mlp.w13_scale, out_dtype, counts)
    pq, ps = ops.silu_mul_quantize_e4m3_blockwise_reference(h)
    wm = ops.fp8_batched_gemm(pq, mlp.w2_fp8, ps, mlp.w2_scale, out_dtype, counts)
    for b, c in enumerate(counts.tolist()):
        rows = min(c, m)
        assert torch.equal(ym[b, :rows].view(torch.int16), wm[b, :rows].view(torch.int16)), b


def test_fp8_modules_run_on_the_quantisers():
    """B200Fp8Linear (every granularity) and B200Fp8GroupedLinear (both layouts) quantise through the kernels."""
    lin = torch.nn.Linear(512, 256, dtype=torch.bfloat16, device="cuda")
    x = torch.randn((64, 512), device="cuda", dtype=torch.bfloat16)
    for gran, launches in (("tensor", 2), ("rowwise", 1), ("blockwise", 1)):
        layer = ops.B200Fp8Linear.from_linear(lin, granularity=gran)
        before = capi.quant_launch_count()
        layer(x)
        assert capi.quant_launch_count() - before == launches, gran
    experts = ops.B200Fp8GroupedLinear.from_weights(torch.randn((3, 256, 512), device="cuda", dtype=torch.bfloat16))
    before = capi.quant_launch_count()
    experts(x, torch.tensor([10, 40, 64], dtype=torch.int32, device="cuda"))
    experts.forward_masked(x.view(2, 32, 512).repeat(2, 1, 1)[:3], torch.tensor([5, 0, 32], dtype=torch.int32,
                                                                                   device="cuda"))
    assert capi.quant_launch_count() - before == 2
