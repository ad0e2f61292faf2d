"""fp32 weight-gradient accumulation (libb200_wgrad_accum.so) on the H100, bit for bit:

* Identity: C32 starting at -0.0 ends as S, the fp32 value the wrapped library rounds, so C32 rounded to the 16-bit type
  is that library's output, for every configuration and K-mode of the three kernel families, and on exact-domain data
  S is the float64 product itself;
* Addition: C32 starting at C0 (signed zeros, subnormals, large values that cancel, infinities, NaN) ends as torch's
  fp32 C0 + S; three accumulations are torch's sequential sum;
* guard bands, empty groups and T == 0 (no launch);
* dispatched calls over a token sweep and the training step shapes;
* the fused layers against the unfused ones over 16 micro-batches, and a fused step in a CUDA graph."""
import pytest
import torch

from cuda_l2_b200 import capi, ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
E4M3 = torch.float8_e4m3fn
SENTINEL = 12345.0   # guard bands and untouched matrices


def _configs():
    return capi.configs()


def _kgrouped_ids():
    return [c["id"] for c in _configs() if c["bn"] % 64 == 0]


def _split_k(c):
    return c["cta_group"] == 1 and c["cluster_m"] == c["cluster_n"] == 1 and c["bn"] >= 64 and c["m_rep"] == 1


def _stream_k(c):
    return c["cluster_m"] == c["cluster_n"] == 1 and c["bn"] >= 64 and c["m_rep"] == 1


def _kernels(modes):
    """The (configuration, K-mode) kernels a list of (config id, splits code) runs: one cluster split-K kernel serves
    -2, -4 and -8."""
    return {(cfg, "plain" if sp == 1 else "cluster" if sp < 0 else "stream-K" if sp >= 100 else "workspace")
            for cfg, sp in modes}


def _rowwise_modes():
    """(config id, splits code) covering every compiled (configuration, K-mode) pair: 46 kernels."""
    out = []
    for c in _configs():
        out.append((c["id"], 1))
        if _split_k(c):
            out += [(c["id"], 4), (c["id"], -2), (c["id"], -4), (c["id"], -8)]
        if _stream_k(c):
            out += [(c["id"], 101)]
    return out


def _block_modes():
    out = []
    for c in _configs():
        if c["m_rep"] * c["bn"] <= 128:
            out.append((c["id"], 1))
            if _split_k(c):
                out += [(c["id"], -2), (c["id"], -4), (c["id"], -8)]
    return out


def _guarded(shape, fill=-0.0, band=64):
    """A contiguous fp32 tensor of ``shape`` filled with ``fill``, inside a buffer whose ``band`` floats on each side
    hold SENTINEL; returns (view, buffer)."""
    n = 1
    for d in shape:
        n *= d
    buf = torch.full((n + 2 * band,), SENTINEL, dtype=torch.float32, device=DEV)
    view = buf[band:band + n].view(shape)
    view.fill_(fill)
    return view, buf


def _bands_intact(buf, band=64):
    return bool((buf[:band] == SENTINEL).all() and (buf[-band:] == SENTINEL).all())


def _same_bits(x, y):
    """Bit equality of fp32 tensors, any NaN matching any NaN."""
    nx, ny = torch.isnan(x), torch.isnan(y)
    return bool(torch.equal(nx, ny) and torch.equal(x[~nx].view(torch.int32), y[~ny].view(torch.int32)))


def _as16(x, dtype):
    return x.to(dtype).view(torch.int16)


# ------------------------------------------------------------------------------------------------- K-grouped
def _grouped_operands(dtype, sizes, m, n, seed, exact=False):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    t = sum(sizes) + 5
    if exact:   # small integers: every sum is exact in fp32, so S is the float64 product
        a = torch.randint(-3, 4, (t, m), generator=gen, device=DEV).to(dtype)
        b = torch.randint(-3, 4, (t, n), generator=gen, device=DEV).to(dtype)
    else:
        a = torch.randn((t, m), generator=gen, device=DEV).to(dtype)
        b = torch.randn((t, n), generator=gen, device=DEV).to(dtype)
    ends = torch.tensor(torch.tensor(sizes).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    a[int(ends[-1]):] = float("nan")   # rows past the last end are never read
    b[int(ends[-1]):] = float("inf")
    return a, b, ends


SIZES = [37, 0, 130, 1, 90]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("exact", [False, True])
def test_kgrouped_identity_every_configuration(dtype, exact):
    m, n = 136, 200
    a, b, ends = _grouped_operands(dtype, SIZES, m, n, seed=3, exact=exact)
    g = len(SIZES)
    for cfg in _kgrouped_ids():
        c32, buf = _guarded((g, m, n))
        c32[1] = SENTINEL   # the empty group's matrix stays as it is
        capi.wgrad_accum_grouped(a, b, c32, ends, config_id=cfg)
        want = torch.empty((g, m, n), dtype=dtype, device=DEV)
        capi.gemm_grouped_wgrad(a, b, want, ends, config_id=cfg)
        torch.cuda.synchronize()
        assert _bands_intact(buf), cfg
        assert bool((c32[1] == SENTINEL).all()), cfg
        for i in (0, 2, 3, 4):
            assert torch.equal(_as16(c32[i], dtype), want[i].view(torch.int16)), (cfg, i)
        if exact:
            s = 0
            for i, e in enumerate(ends.tolist()):
                if i != 1:
                    ref = a[s:e].double().t() @ b[s:e].double()
                    assert torch.equal(c32[i].double(), ref), (cfg, i)
                s = e


def test_kgrouped_t0_launches_nothing_and_changes_nothing():
    a = torch.empty((0, 64), dtype=torch.bfloat16, device=DEV)
    b = torch.empty((0, 64), dtype=torch.bfloat16, device=DEV)
    c32 = torch.full((2, 64, 64), -0.0, device=DEV)
    before = capi.wgrad_accum_launch_count()
    capi.wgrad_accum_grouped(a, b, c32, torch.zeros(2, dtype=torch.int32, device=DEV))
    mg = torch.full((64, 64), 3.5, device=DEV)
    ops.wgrad_accumulate_(mg, a, b)
    torch.cuda.synchronize()
    assert capi.wgrad_accum_launch_count() == before
    assert bool((torch.signbit(c32) & (c32 == 0)).all()) and bool((mg == 3.5).all())


# ---------------------------------------------------------------------------------------------- e4m3 families
def _e4m3_operands(m, n, k, seed, form, exact=False):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    if exact:
        a = torch.randint(-4, 5, (m, k), generator=gen, device=DEV).float().to(E4M3)
        b = torch.randint(-4, 5, (n, k), generator=gen, device=DEV).float().to(E4M3)
    else:
        a = (torch.randn((m, k), generator=gen, device=DEV) * 4).to(E4M3)
        b = (torch.randn((n, k), generator=gen, device=DEV) * 4).to(E4M3)
    nkb = -(-k // 128)
    if form == "rowwise":
        pw = (lambda r, c: torch.exp2(torch.randint(-3, 3, (r, c), generator=gen, device=DEV).float())) if exact else \
            (lambda r, c: torch.rand((r, c), generator=gen, device=DEV) + 0.5)
        return a, b, pw(m, 1), pw(1, n)
    sa, sb = capi.empty_m_major((), m, nkb, DEV), capi.empty_m_major((), n, nkb, DEV)
    if exact:   # powers of two, constant over k: the promotion stays exact
        sa.copy_(torch.exp2(torch.randint(-3, 3, (m, 1), generator=gen, device=DEV).float()).expand(m, nkb))
        sb.copy_(torch.exp2(torch.randint(-3, 3, (n, 1), generator=gen, device=DEV).float()).expand(n, nkb))
    else:
        sa.copy_(torch.rand((m, nkb), generator=gen, device=DEV) + 0.5)
        sb.copy_(torch.rand((n, nkb), generator=gen, device=DEV) + 0.5)
    return a, b, sa, sb


def _fp8_identity(form, modes, m, n, k, exact):
    a, b, sa, sb = _e4m3_operands(m, n, k, seed=11, form=form, exact=exact)
    ref = None
    if exact:
        ref = (a.double() @ b.double().t())
        ref = ref * sb.double().reshape(1, -1) * sa.double().reshape(-1, 1) if form == "rowwise" else \
            ref * sa[:, :1].double() * sb[:, :1].double().t()
    for cfg, splits in modes:
        c32, buf = _guarded((m, n))
        capi.wgrad_accum_fp8(a, b, c32, sa, sb, config_id=cfg, splits=splits)
        want = torch.empty((m, n), dtype=torch.bfloat16, device=DEV)
        capi.fp8_gemm(a, b, want, sa, sb, config_id=cfg, splits=splits)
        torch.cuda.synchronize()
        assert _bands_intact(buf), (cfg, splits)
        assert torch.equal(_as16(c32, torch.bfloat16), want.view(torch.int16)), (cfg, splits)
        if exact:
            assert torch.equal(c32.double(), ref), (cfg, splits)


@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("shape", [(1000, 1032, 4096), (256, 264, 8192)])
def test_rowwise_identity_every_configuration_and_k_mode(exact, shape):
    capi.wgrad_accum_prewarm()
    assert len(_kernels(_rowwise_modes())) == 46
    _fp8_identity("rowwise", _rowwise_modes(), *shape, exact)


@pytest.mark.parametrize("exact", [False, True])
def test_block_1d1d_identity_every_configuration_and_k_mode(exact):
    assert len(_kernels(_block_modes())) == 19
    _fp8_identity("blockwise_1d1d", _block_modes(), 392, 264, 2176, exact)


# ------------------------------------------------------------------------------------------------ addition
def _special_c0(shape, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    c0 = torch.randn(shape, generator=gen, device=DEV) * 1e3
    flat = c0.view(-1)
    specials = torch.tensor([0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -5e-39, 3e38, -3e38, float("inf"),
                             float("-inf"), float("nan")], device=DEV)
    idx = torch.randint(0, flat.numel(), (flat.numel() // 3,), generator=gen, device=DEV)
    flat[idx] = specials[torch.randint(0, len(specials), idx.shape, generator=gen, device=DEV)]
    return c0


def _s_of(run, shape):
    s = torch.full(shape, -0.0, device=DEV)
    run(s)
    return s


def _addition_cases():
    m, n, k = 264, 392, 2176
    out = []
    for form in ("rowwise", "blockwise_1d1d"):
        a, b, sa, sb = _e4m3_operands(m, n, k, seed=5, form=form)
        out.append((form, (m, n), lambda c, a=a, b=b, sa=sa, sb=sb, cfg=1, sp=1:
                    capi.wgrad_accum_fp8(a, b, c, sa, sb, config_id=cfg, splits=sp)))
        out.append((form + "-cluster", (m, n), lambda c, a=a, b=b, sa=sa, sb=sb:
                    capi.wgrad_accum_fp8(a, b, c, sa, sb, config_id=1, splits=-4)))
    a, b, sa, sb = _e4m3_operands(m, n, k, seed=5, form="rowwise")
    out.append(("rowwise-workspace", (m, n), lambda c: capi.wgrad_accum_fp8(a, b, c, sa, sb, config_id=1, splits=8)))
    # 40 tiles of 32 k-blocks on 132 workers: planned as stream-K
    sa_, sb_ = torch.rand((1000, 1), device=DEV) + 0.5, torch.rand((1, 1032), device=DEV) + 0.5
    a_, b_ = ((torch.randn(s, device=DEV) * 4).to(E4M3) for s in ((1000, 4096), (1032, 4096)))
    out.append(("rowwise-streamk", (1000, 1032),
                lambda c: capi.wgrad_accum_fp8(a_, b_, c, sa_, sb_, config_id=0, splits=101)))
    ga, gb, ends = _grouped_operands(torch.bfloat16, SIZES, 136, 200, seed=9)
    out.append(("kgrouped", (len(SIZES), 136, 200), lambda c: capi.wgrad_accum_grouped(ga, gb, c, ends, config_id=1)))
    # tiny operands: sums in the subnormal range
    ta = (torch.randn((64, 64), device=DEV) * 1e-20).bfloat16()
    tb = (torch.randn((64, 72), device=DEV) * 1e-20).bfloat16()
    tends = torch.tensor([64], dtype=torch.int32, device=DEV)
    out.append(("kgrouped-subnormal", (1, 64, 72), lambda c: capi.wgrad_accum_grouped(ta, tb, c, tends)))
    return out


@pytest.mark.parametrize("case", range(7))
def test_addition_is_torch_c0_plus_s_and_three_accumulations_are_its_sequential_sum(case):
    name, shape, run = _addition_cases()[case]
    s = _s_of(run, shape)
    c0 = _special_c0(shape, seed=case)
    c = c0.clone()
    run(c)
    torch.cuda.synchronize()
    assert _same_bits(c, c0 + s), name
    if name == "kgrouped":   # the empty group's matrix is not touched: not even -0.0 + 0 -> +0.0
        assert torch.equal(c[1].view(torch.int32), c0[1].view(torch.int32))
    if name == "kgrouped-subnormal":
        assert bool(((s != 0) & (s.abs() < 1.1754944e-38)).any()), "no subnormal sum"
    c = c0.clone()
    for _ in range(3):
        run(c)
    want = ((c0 + s) + s) + s
    torch.cuda.synchronize()
    assert _same_bits(c, want), name


# ---------------------------------------------------------------------------------------------- dispatched
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("t", [1, 7, 63, 65, 193, 4097, 65537])
def test_dispatched_16bit_token_sweep(dtype, t):
    n, k = 264, 136
    gen = torch.Generator(device=DEV).manual_seed(t)
    gy = torch.randn((t, n), generator=gen, device=DEV).to(dtype)
    x = torch.randn((t, k), generator=gen, device=DEV).to(dtype)
    mg = torch.full((n, k), -0.0, device=DEV)
    ops.wgrad_accumulate_(mg, gy, x)
    want = torch.empty((1, n, k), dtype=dtype, device=DEV)
    capi.gemm_grouped_wgrad(gy, x, want, torch.tensor([t], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    assert torch.equal(_as16(mg, dtype), want[0].view(torch.int16))


STEP_SHAPES = [(2048, 4096, 11008), (4096, 11008, 4096), (4096, 4096, 4096), (8192, 3072, 768)]   # tokens, in, out


@pytest.mark.parametrize("tokens", [16, 48, 4096])
@pytest.mark.parametrize("form", ["rowwise", "blockwise_1d1d"])
def test_dispatched_e4m3_token_sweep(tokens, form):
    m, n = 264, 392
    a, b, sa, sb = _e4m3_operands(m, n, tokens, seed=tokens, form=form)
    c32 = torch.full((m, n), -0.0, device=DEV)
    ops.fp8_gemm_accumulate_(c32, a, b, sa, sb)
    want = ops.fp8_gemm(a, b, sa, sb, torch.bfloat16)
    torch.cuda.synchronize()
    assert torch.equal(_as16(c32, torch.bfloat16), want.view(torch.int16))


@pytest.mark.parametrize("shape", STEP_SHAPES)
def test_dispatched_at_the_step_shapes(shape):
    tokens, k_in, n_out = shape
    gen = torch.Generator(device=DEV).manual_seed(tokens + n_out)
    gy = torch.randn((tokens, n_out), generator=gen, device=DEV).bfloat16()
    x = torch.randn((tokens, k_in), generator=gen, device=DEV).bfloat16()
    mg = torch.full((n_out, k_in), -0.0, device=DEV)
    ops.wgrad_accumulate_(mg, gy, x)
    want = torch.empty((1, n_out, k_in), dtype=torch.bfloat16, device=DEV)
    capi.gemm_grouped_wgrad(gy, x, want, torch.tensor([tokens], dtype=torch.int32, device=DEV))
    assert torch.equal(_as16(mg, torch.bfloat16), want[0].view(torch.int16))
    for form in ("rowwise", "blockwise_1d1d"):
        a, b, sa, sb = _e4m3_operands(n_out, k_in, tokens, seed=7, form=form)
        c32 = torch.full((n_out, k_in), -0.0, device=DEV)
        ops.fp8_gemm_accumulate_(c32, a, b, sa, sb)
        want = ops.fp8_gemm(a, b, sa, sb, torch.bfloat16)
        torch.cuda.synchronize()
        assert torch.equal(_as16(c32, torch.bfloat16), want.view(torch.int16)), form


# -------------------------------------------------------------------------------------------- fused layers
MICRO = 16


def _pair(kind, seed):
    torch.manual_seed(seed)
    if kind == "linear":
        lin = torch.nn.Linear(256, 136, device=DEV, dtype=torch.bfloat16)
        fused = ops.B200Linear.from_linear(lin, fuse_wgrad_accumulation=True)
        plain = ops.B200Linear.from_linear(torch.nn.Linear(256, 136, device=DEV, dtype=torch.bfloat16))
        plain.weight, plain.bias = (torch.nn.Parameter(p.detach().clone()) for p in (lin.weight, lin.bias))
    elif kind in ("fp8-rowwise", "fp8-blockwise"):
        gran = kind.split("-")[1]
        lin = torch.nn.Linear(256, 144, device=DEV, dtype=torch.bfloat16)
        fused = ops.B200Fp8TrainLinear.from_linear(lin, gran, fuse_wgrad_accumulation=True)
        plain = ops.B200Fp8TrainLinear.from_linear(torch.nn.Linear(256, 144, device=DEV, dtype=torch.bfloat16), gran)
        plain.weight, plain.bias = (torch.nn.Parameter(p.detach().clone()) for p in (lin.weight, lin.bias))
    else:
        w = torch.randn((4, 136, 256), device=DEV, dtype=torch.bfloat16) * 0.05
        fused = ops.B200GroupedLinear.from_weights(torch.nn.Parameter(w.clone()), fuse_wgrad_accumulation=True)
        plain = ops.B200GroupedLinear.from_weights(torch.nn.Parameter(w.clone()))
    fused.weight.main_grad = torch.zeros(fused.weight.shape, dtype=torch.float32, device=DEV)
    return fused, plain


def _inputs(kind, i):
    gen = torch.Generator(device=DEV).manual_seed(100 + i)
    t = 67 + 16 * i if kind.startswith("fp8") else 61 + 13 * i
    x = torch.randn((t, 256), generator=gen, device=DEV).bfloat16().requires_grad_()
    gy_shape = (t, 144 if kind.startswith("fp8") else 136)
    gy = torch.randn(gy_shape, generator=gen, device=DEV).bfloat16()
    if kind == "grouped":
        cuts = sorted(torch.randint(0, t, (3,), generator=gen, device=DEV).tolist())
        offs = torch.tensor(cuts + [t], dtype=torch.int32, device=DEV)
        return (x, offs), gy
    return (x,), gy


def _s_i(kind, fused, args, gy):
    """The library's own S of one micro-batch, through the same accumulating call into -0.0."""
    s = torch.full(fused.weight.shape, -0.0, device=DEV)
    saved, fused.weight.main_grad = fused.weight.main_grad, s
    y = fused(*(a.detach().requires_grad_() if a.is_floating_point() else a for a in args))
    y.backward(gy)
    fused.weight.main_grad = saved
    if getattr(fused, "bias", None) is not None:
        fused.bias.grad = None
    return s


def _dequantised_t(kind, t):
    """t^T as the FP8 backward's dual quantiser gives it, in float64: q_t times its scales (rowwise: one per row of
    t^T; blockwise: one per row and 128 columns), the padding columns zero."""
    if kind == "fp8-rowwise":
        _, _, q_t, s_t = ops.quantize_e4m3_rowwise_dual(t)
        return q_t.double() * s_t.double().reshape(-1, 1)
    _, _, q_t, s_t = ops.quantize_e4m3_blockwise_dual(t)
    return q_t.double() * s_t.double().repeat_interleave(128, dim=1)[:, :q_t.shape[1]]


@pytest.mark.parametrize("kind", ["linear", "fp8-rowwise", "fp8-blockwise", "grouped"])
def test_fused_layer_against_unfused_over_micro_batches(kind):
    fused, plain = _pair(kind, seed=1)
    want = torch.zeros(fused.weight.shape, dtype=torch.float32, device=DEV)
    ref64 = torch.zeros(fused.weight.shape, dtype=torch.float64, device=DEV)
    for i in range(MICRO):
        args, gy = _inputs(kind, i)
        xf = args[0].detach().clone().requires_grad_()
        xp = args[0].detach().clone().requires_grad_()
        yf = fused(xf, *args[1:])
        yp = plain(xp, *args[1:])
        assert torch.equal(yf.view(torch.int16), yp.view(torch.int16)), i
        yf.backward(gy)
        yp.backward(gy)
        assert torch.equal(xf.grad.view(torch.int16), xp.grad.view(torch.int16)), i
        if getattr(fused, "bias", None) is not None:
            assert torch.equal(fused.bias.grad.view(torch.int16), plain.bias.grad.view(torch.int16)), i
            fused.bias.grad = plain.bias.grad = None   # compared per micro-batch; _s_i runs one more backward
        assert fused.weight.grad is None
        want = want + _s_i(kind, fused, args, gy)
        if kind == "grouped":
            x64, g64 = args[0].detach().double(), gy.double()
            s = 0
            for g, e in enumerate(args[1].tolist()):
                ref64[g] += g64[s:e].t() @ x64[s:e]
                s = e
        elif kind == "linear":
            ref64 += gy.double().t() @ args[0].detach().double()
        else:   # the product of the e4m3 operands the backward quantises, dequantised
            ref64 += _dequantised_t(kind, gy) @ _dequantised_t(kind, args[0].detach()).t()
    torch.cuda.synchronize()
    assert _same_bits(fused.weight.main_grad, want)
    err_fused = (fused.weight.main_grad.double() - ref64).abs().max().item()
    err_plain = (plain.weight.grad.double() - ref64).abs().max().item()
    print(f"{kind}: max |main_grad - fp64| = {err_fused:.3e}, max |bf16 .grad - fp64| = {err_plain:.3e}")
    assert err_fused <= err_plain


@pytest.mark.parametrize("kind", ["linear", "fp8-rowwise", "fp8-blockwise", "grouped"])
def test_fused_step_in_a_cuda_graph_equals_eager_steps(kind):
    """Three replays of a captured fused step equal three eager steps, bit for bit, and two seeded eager runs agree.
    The capture stream's split-K scratch is allocated beforehand, so both run the dispatcher's schedule."""
    def run(capture: bool):
        fused, _ = _pair(kind, seed=2)
        gen = torch.Generator(device=DEV).manual_seed(7)
        x = torch.randn((193, 256), generator=gen, device=DEV).bfloat16().requires_grad_()
        gy = torch.randn((193, fused.weight.shape[-2]), generator=gen, device=DEV).bfloat16()
        extra = (torch.tensor([40, 40, 150, 193], dtype=torch.int32, device=DEV),) if kind == "grouped" else ()

        def step():
            fused(x, *extra).backward(gy)

        if not capture:
            for _ in range(3):
                step()
            torch.cuda.synchronize()
            return fused.weight.main_grad.clone()
        cap = torch.cuda.Stream()
        capi.wgrad_accum_prewarm(cap.cuda_stream)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()   # warm-up outside the graph
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        fused.weight.main_grad.zero_()
        x.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=cap):
            step()
        fused.weight.main_grad.zero_()
        for _ in range(3):
            graph.replay()
        torch.cuda.synchronize()
        return fused.weight.main_grad.clone()

    eager = run(False)
    assert eager.abs().sum() > 0
    assert torch.equal(run(True).view(torch.int32), eager.view(torch.int32))
    assert torch.equal(run(False).view(torch.int32), eager.view(torch.int32))


def test_frozen_weight_gets_nothing_added():
    for kind in ("linear", "grouped", "fp8-rowwise"):
        fused, _ = _pair(kind, seed=3)
        fused.weight.requires_grad_(False)
        args, gy = _inputs(kind, 0)
        before = capi.wgrad_accum_launch_count()
        fused(*args).backward(gy)
        torch.cuda.synchronize()
        assert capi.wgrad_accum_launch_count() == before, kind
        assert not fused.weight.main_grad.any() and args[0].grad is not None, kind


def test_main_grad_is_read_when_the_backward_runs():
    for kind in ("linear", "grouped"):
        fused, _ = _pair(kind, seed=4)
        args, gy = _inputs(kind, 1)
        y = fused(*args)
        first = fused.weight.main_grad
        fused.weight.main_grad = torch.full_like(first, -0.0)
        y.backward(gy)
        torch.cuda.synchronize()
        assert not first.any() and fused.weight.main_grad.abs().sum() > 0, kind
