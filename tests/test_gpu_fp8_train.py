"""FP8 training of linear layers on the H100: the dual-orientation rowwise quantiser (libb200_quant_dual.so) bit for bit
against its torch composition (every input dtype, ragged rows and columns, every fp16 and bf16 bit pattern in both a row
and a column group, zero / -0.0 / subnormal / Inf / NaN rows and columns, the NaN padding of q_t, unaligned inputs,
CUDA-graph replay, two concurrent streams); fp8_linear's y, dX and dW bit for bit against the same chain built from the
torch quantisers and fp8_gemm, for every needs_input_grad combination with its launch counts; its accuracy against a
float64 product and against torch._scaled_mm; B200Fp8TrainLinear against B200Fp8Linear in eval mode; a forward and
backward step captured in one CUDA graph and under FakeTensors; and a small MLP trained twice to the same bits, and to a
loss near the bf16 one."""
import pytest
import torch
import torch.nn.functional as F

from cuda_l2_b200 import capi, ops

pytestmark = pytest.mark.gpu

DTYPES = (torch.float16, torch.bfloat16, torch.float32)
ROWS = (1, 15, 16, 17, 300, 2048, 4104)
COLS = (16, 136, 300, 4096, 11008)
# Measured on an H100 80GB HBM3 (700 W power limit):
# - y, dX and dW of N(0,1) data against the float64 product of the 16-bit operands, max |error| / rms(product):
#   0.158-0.224 over the three shapes of test_accuracy_against_float64_and_torch_scaled_mm, fp16 and bf16.
# - against torch._scaled_mm (rowwise scales, use_fast_accum=True, bf16 out) on the same e4m3 operands: y and dX
#   bit-identical at every shape; dW bit-identical except at 2048 x 4096 x 4096, 0.011 x rms (one bf16 rounding).
RANDOM_TOL = 0.3       # max |got - float64 product| / rms(product)
SCALED_MM_TOL = 0.03   # max |got - torch._scaled_mm| / rms(torch._scaled_mm), bf16 out
LOSS_RATIO = 1.05      # final loss of the FP8-trained MLP over the bf16-trained one: measured 1.0059 (0.1014 / 0.1008)


@pytest.fixture(scope="module", autouse=True)
def _need_h100(built_libs):
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0) != (9, 0):
        pytest.skip("needs an H100")
    torch.cuda.set_device(0)


def _bits(t: torch.Tensor) -> torch.Tensor:
    if t.dtype == torch.float8_e4m3fn:
        return t.view(torch.uint8)
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _same(got, want, what=""):
    """Tensors equal bit for bit, with the same shapes, dtypes and strides."""
    for i, (g, w) in enumerate(zip(got, want)):
        assert (g.shape, g.dtype, g.stride()) == (w.shape, w.dtype, w.stride()), (what, i)
        if not torch.equal(_bits(g), _bits(w)):
            bad = (_bits(g) != _bits(w)).nonzero()[:5].tolist()
            raise AssertionError(f"{what} result {i}: {int((_bits(g) != _bits(w)).sum())} elements differ, first at {bad}")


def _activations(shape, dtype, seed):
    """Normal values whose magnitude varies by row and by column over several decades, plus one outlier per row, all
    finite in fp16."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g)
    x *= torch.exp(torch.empty((shape[0], 1), device="cuda").uniform_(-4, 4, generator=g))
    x *= torch.exp(torch.empty((1, shape[1]), device="cuda").uniform_(-2, 2, generator=g))
    x[torch.arange(shape[0], device="cuda"), (torch.arange(shape[0], device="cuda") * 7 + seed) % shape[1]] *= 8
    return x.to(dtype)


def _dual_same(x, what=""):
    _same(ops.quantize_e4m3_rowwise_dual(x), ops.quantize_e4m3_rowwise_dual_reference(x), what)


# ------------------------------------------------------------------------------------------------ the dual quantiser
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows", ROWS)
def test_dual_quantiser_against_the_composition(dtype, rows):
    for cols in COLS:
        _dual_same(_activations((rows, cols), dtype, seed=rows + cols), f"{rows}x{cols} {dtype}")


def _all_patterns(dtype) -> torch.Tensor:
    return torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(dtype)


@pytest.mark.parametrize("dtype", DTYPES[:2])
def test_every_bit_pattern_in_a_row_and_a_column_group(dtype):
    """Every 16-bit pattern as a [256, 256] matrix, so each is in one row and one column group, in three arrangements:
    finite values sorted by magnitude (row and column maxima near their members), the same shuffled, and every pattern,
    Inf and NaN among them, shuffled. Ragged shapes (17 x 512, 300 x 200) exercise the tile edges."""
    v = _all_patterns(dtype)
    finite = v[torch.isfinite(v)]
    finite = finite[torch.argsort(finite.float().abs(), stable=True)]
    g = torch.Generator(device="cuda").manual_seed(11)
    for i, x in enumerate((finite, finite[torch.randperm(finite.numel(), device="cuda", generator=g)],
                           v[torch.randperm(v.numel(), device="cuda", generator=g)])):
        x = torch.cat([x, torch.zeros(-x.numel() % 65536, dtype=dtype, device="cuda")]).view(256, 256)
        _dual_same(x, f"patterns {i}")
        _dual_same(x.t().contiguous(), f"patterns {i} transposed")
        _dual_same(x.reshape(128, 512)[:17].contiguous(), f"patterns {i} 17 rows")
        _dual_same(x.reshape(-1)[:300 * 200].view(300, 200), f"patterns {i} 300 x 200")


def _special(dtype, rows: int, cols: int) -> torch.Tensor:
    """Activations with whole rows and whole columns of zero, -0.0, subnormals, Inf and NaN."""
    sub = 1e-40 if dtype == torch.float32 else torch.finfo(dtype).tiny / 8
    x = _activations((rows, cols), torch.float32, seed=rows).to(dtype)
    x[1] = 0.0
    x[2] = -0.0
    x[3] = sub
    x[4, ::2] = -sub
    x[5, 3] = float("inf")
    x[6, 9] = float("-inf")
    x[7, 11] = float("nan")
    x[:, 0] = 0.0
    x[:, 1] = -0.0
    x[:, 2] = sub
    x[10, 4] = float("inf")
    x[12, 5] = float("nan")
    x[:, 8] = 448.0
    return x


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows", [17, 16, 300])
def test_zero_signed_zero_subnormal_inf_nan_rows_and_columns(dtype, rows):
    x = _special(dtype, rows, 136)
    _dual_same(x, "special")
    q, s, q_t, s_t = ops.quantize_e4m3_rowwise_dual(x)
    ld_t = capi.dual_ld_t(rows)
    assert q_t.shape == (136, ld_t)
    assert torch.isnan(s_t[11]) and torch.isnan(s_t[5]) and torch.isnan(s[7]) and torch.isnan(s[12])
    if ld_t > rows:   # the padding: e4m3(0 / s), 0x00, and the NaN code in NaN columns
        pad = _bits(q_t[:, rows:])
        nan_cols = torch.isnan(s_t)
        assert (pad[nan_cols] == 0x7F).all() and (pad[~nan_cols] == 0).all()
    assert (_bits(q_t[1][:rows]) == 0x80).all() and (_bits(q_t[0]) == 0).all()   # -0.0 keeps its sign


def test_unaligned_inputs_take_the_element_path():
    base = _activations((300, 1040), torch.bfloat16, seed=5)
    flat = base.reshape(-1)[3:3 + 300 * 1024].view(300, 1024)   # 6 bytes off a 16-byte boundary
    assert flat.data_ptr() % 16 == 6
    _dual_same(flat, "unaligned")
    _dual_same(base[:, 1:1025], "strided")
    for dtype in DTYPES:
        x = _activations((2000, 1040), dtype, seed=9).reshape(-1)[1:1 + 37 * 4100].view(37, 4100)
        _dual_same(x, f"unaligned {dtype}")
    # and through the C ABI with a q_t that is not 16-byte aligned: refused
    q = torch.empty((300, 1024), dtype=torch.float8_e4m3fn, device="cuda")
    q_t = torch.empty(304 * 1024 + 16, dtype=torch.uint8, device="cuda")[8:8 + 1024 * 304].view(torch.float8_e4m3fn)
    with pytest.raises(capi.B200HgemmError, match="16-byte"):
        capi.quantize_e4m3_rowwise_dual(flat, q, torch.empty(300, device="cuda"), q_t.view(1024, 304),
                                        torch.empty(1024, device="cuda"), torch.empty(1324, device="cuda"))


def test_two_launches_per_call():
    x = _activations((64, 4096), torch.bfloat16, seed=1)
    before = capi.quant_dual_launch_count()
    ops.quantize_e4m3_rowwise_dual(x)
    assert capi.quant_dual_launch_count() - before == 2


def test_cuda_graph_capture_and_replay():
    x = _activations((300, 1536), torch.bfloat16, seed=2)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        ops.quantize_e4m3_rowwise_dual(x)
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.quantize_e4m3_rowwise_dual(x)
    for seed in (7, 8):
        x.copy_(_activations(x.shape, torch.bfloat16, seed=seed))
        if seed == 8:
            x[:, 5] = float("nan")
        graph.replay()
        torch.cuda.synchronize()
        _same(out, ops.quantize_e4m3_rowwise_dual_reference(x), f"graph {seed}")


def test_concurrent_calls_on_two_streams():
    xs = [_activations((4104, 4096), torch.bfloat16, seed=20 + i) for i in range(2)]
    want = [ops.quantize_e4m3_rowwise_dual_reference(x) for x in xs]
    streams = [torch.cuda.Stream() for _ in xs]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    outs = [[], []]
    for _ in range(6):
        for i, (x, s) in enumerate(zip(xs, streams)):
            with torch.cuda.stream(s):
                outs[i].append(ops.quantize_e4m3_rowwise_dual(x))
    torch.cuda.synchronize()
    for i in range(2):
        for got in outs[i]:
            _same(got, want[i], f"stream {i}")


# ------------------------------------------------------------------------------------------------ fp8_linear
def _reference_step(x2, w, gy, launches=None):
    """y, dX, dW of fp8_linear built from the torch quantisers and fp8_gemm; ``launches`` (a list) receives the GEMM
    library's launches of each of the three products."""
    xq, xs, xqt, xst = ops.quantize_e4m3_rowwise_dual_reference(x2)
    wq, ws, wqt, wst = ops.quantize_e4m3_rowwise_dual_reference(w)
    gq, gs, gqt, gst = ops.quantize_e4m3_rowwise_dual_reference(gy)
    out = []
    for a, b, sa, sb, dtype in ((xq, wq, xs, ws, x2.dtype), (gq, wqt, gs, wst, x2.dtype), (gqt, xqt, gst, xst, w.dtype)):
        before = capi.launch_count()
        out.append(ops.fp8_gemm(a, b, sa.reshape(-1, 1), sb.reshape(1, -1), dtype))
        if launches is not None:
            launches.append(capi.launch_count() - before)
    return out


def _counts():
    return capi.quant_dual_launch_count(), capi.quant_launch_count(), capi.launch_count()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("lead", [(300,), (37,), (3, 45), (2048,)])
@pytest.mark.parametrize("need", [(True, True), (True, False), (False, True), (False, False)])
def test_fp8_linear_is_the_chain_of_torch_quantisers_and_fp8_gemm(dtype, lead, need):
    n, k = 272, 1024
    x = _activations((*lead, k) if len(lead) == 1 else (lead[0] * lead[1], k), dtype, seed=3).view(*lead, k)
    w = (_activations((n, k), torch.float32, seed=4) / 64).to(dtype)
    gy = _activations((x.numel() // k, n), dtype, seed=5)
    launches = []
    want_y, want_dx, want_dw = _reference_step(x.reshape(-1, k), w, gy, launches)
    x.requires_grad_(need[0])
    w.requires_grad_(need[1])
    before = _counts()
    y = ops.fp8_linear(x, w)
    assert y.shape == (*lead, n)
    assert torch.equal(_bits(y.detach().reshape(-1, n)), _bits(want_y))
    if any(need):
        y.backward(gy.view(*lead, n))
    dual, quant, gemm = (a - b for a, b in zip(_counts(), before))
    if need[0]:
        assert torch.equal(_bits(x.grad.reshape(-1, k)), _bits(want_dx)) and x.grad.dtype == dtype
    if need[1]:
        assert torch.equal(_bits(w.grad), _bits(want_dw)) and w.grad.dtype == dtype
    # transposed copies only for the gradients asked for: x's for dW, W's for dX, dY's for dW
    want_dual = 2 * (2 * need[1] + need[0])
    want_quant = {(True, True): 0, (True, False): 2, (False, True): 1, (False, False): 2}[need]
    assert (dual, quant) == (want_dual, want_quant), need
    assert gemm == launches[0] + need[0] * launches[1] + need[1] * launches[2], (gemm, launches)


def test_zero_tokens_launch_nothing():
    w = torch.randn((64, 128), device="cuda", dtype=torch.bfloat16).requires_grad_()
    x = torch.empty((0, 128), device="cuda", dtype=torch.bfloat16).requires_grad_()
    w.grad = None
    before = _counts()
    y = ops.fp8_linear(x, w)
    y.sum().backward()
    assert _counts() == before
    assert y.shape == (0, 64) and x.grad.shape == (0, 128)
    assert w.grad.shape == (64, 128) and not w.grad.view(torch.int16).any()
    with torch.no_grad():
        assert ops.fp8_linear(x, w).shape == (0, 64)


def _rel(got, truth):
    return float((got.double() - truth).abs().max() / truth.pow(2).mean().sqrt())


@pytest.mark.parametrize("mnk", [(2048, 4096, 4096), (4096, 1024, 2048), (333, 768, 512)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_accuracy_against_float64_and_torch_scaled_mm(mnk, dtype):
    m, n, k = mnk
    g = torch.Generator(device="cuda").manual_seed(m + n)
    x = torch.randn((m, k), device="cuda", generator=g).to(dtype).requires_grad_()
    w = torch.randn((n, k), device="cuda", generator=g).to(dtype).requires_grad_()
    gy = torch.randn((m, n), device="cuda", generator=g).to(dtype)
    y = ops.fp8_linear(x, w)
    y.backward(gy)
    xd, wd, gd = x.detach().double(), w.detach().double(), gy.double()
    errs = {"y": _rel(y.detach(), xd @ wd.t()), "dx": _rel(x.grad, gd @ wd), "dw": _rel(w.grad, gd.t() @ xd)}
    # torch._scaled_mm, rowwise scales and fast accumulation, on the same e4m3 operands
    xq, xs, xqt, xst = ops.quantize_e4m3_rowwise_dual(x.detach())
    wq, ws, wqt, wst = ops.quantize_e4m3_rowwise_dual(w.detach())
    gq, gs, gqt, gst = ops.quantize_e4m3_rowwise_dual(gy)
    smm = {"y": (xq, wq, xs, ws), "dx": (gq, wqt, gs, wst), "dw": (gqt, xqt, gst, xst)}
    got = {"y": y.detach(), "dx": x.grad, "dw": w.grad}
    diffs = {}
    for name, (a, b, sa, sb) in smm.items() if dtype == torch.bfloat16 else ():   # torch's rowwise form: bf16 out
        ref = torch._scaled_mm(a, b.t(), scale_a=sa.reshape(-1, 1), scale_b=sb.reshape(1, -1), out_dtype=dtype,
                               use_fast_accum=True)
        diffs[name] = float((got[name].float() - ref.float()).abs().max() / ref.float().pow(2).mean().sqrt())
    print(f"MEASURED accuracy {mnk} {dtype}: float64 {errs} scaled_mm {diffs}")
    for name in errs:
        assert errs[name] <= RANDOM_TOL, (name, errs)
    for name in diffs:
        assert diffs[name] <= SCALED_MM_TOL, (name, diffs)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_eval_mode_is_b200_fp8_linear_rowwise(dtype):
    lin = torch.nn.Linear(1024, 512, device="cuda", dtype=dtype)
    train = ops.B200Fp8TrainLinear.from_linear(lin)
    infer = ops.B200Fp8Linear.from_linear(lin, granularity="rowwise")
    x = _activations((300, 1024), dtype, seed=6).view(3, 100, 1024)
    want = infer(x)
    train.eval()
    with torch.no_grad():
        before = _counts()
        got = train(x)
        assert _counts()[0] == before[0]   # no transposed copy without a gradient
    assert torch.equal(_bits(got), _bits(want))
    assert torch.equal(_bits(train(x).detach()), _bits(want))   # and with one prepared, the same bits


def test_training_step_captured_in_a_cuda_graph():
    layer = ops.B200Fp8TrainLinear(1024, 768, device="cuda")
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
        assert torch.equal(_bits(y.detach()), _bits(want_y + layer.bias.detach()))
        assert torch.equal(_bits(x.grad), _bits(want_dx)) and torch.equal(_bits(layer.weight.grad), _bits(want_dw))
        assert torch.equal(_bits(layer.bias.grad), _bits(gy.sum(0)))


def test_forward_and_backward_trace_under_fake_tensors():
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        for shape in ((37, 64), (3, 5, 64)):
            x = torch.empty(shape, dtype=torch.bfloat16, device="cuda").requires_grad_()
            w = torch.empty((48, 64), dtype=torch.bfloat16, device="cuda").requires_grad_()
            y = ops.fp8_linear(x, w)
            y.sum().backward()
            assert y.shape == (*shape[:-1], 48) and x.grad.shape == x.shape and w.grad.shape == w.shape


# ------------------------------------------------------------------------------------------------ training
def _train_mlp(kind: str, steps: int = 300) -> tuple[float, float, list[torch.Tensor]]:
    """A 256 -> 512 -> 256 GELU MLP (bf16, with biases) fitted by Adam to a fixed random teacher; returns the mean loss
    of the first and of the last 20 steps, and the final parameters."""
    torch.manual_seed(0)
    g = torch.Generator(device="cuda").manual_seed(1)
    teacher = [torch.randn((512, 256), device="cuda", generator=g) / 16, torch.randn((256, 512), device="cuda",
                                                                                       generator=g) / 22]
    lins = [torch.nn.Linear(256, 512, device="cuda", dtype=torch.bfloat16),
            torch.nn.Linear(512, 256, device="cuda", dtype=torch.bfloat16)]
    cls = ops.B200Fp8TrainLinear if kind == "fp8" else ops.B200Linear
    model = torch.nn.Sequential(cls.from_linear(lins[0]), torch.nn.GELU(), cls.from_linear(lins[1]))
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
    first, loss_a, params_a = _train_mlp("fp8")
    _, loss_b, params_b = _train_mlp("fp8")
    for a, b in zip(params_a, params_b):
        assert torch.equal(_bits(a), _bits(b))
    assert loss_a == loss_b
    first_bf16, loss_bf16, _ = _train_mlp("bf16")
    print(f"MEASURED mlp loss fp8 {first:.6g} -> {loss_a:.6g}, bf16 {first_bf16:.6g} -> {loss_bf16:.6g}, "
          f"ratio {loss_a / loss_bf16:.4f}")
    assert loss_a < 0.5 * first   # it learns
    assert loss_a <= LOSS_RATIO * loss_bf16, (loss_a, loss_bf16)
