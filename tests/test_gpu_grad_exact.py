"""The 16-bit training products on the H100, bit for bit: y, dX, dW and dbias of every differentiable operator and of
the modules built on them, against a float64 reference rounded once (tests/grad_domain.py's exact gradient domain).

Token counts M that are not a multiple of 8 are the point: the weight gradient reduces over M, and at such M it runs
the K-grouped weight-gradient kernel (one group, or one per batch) instead of the row-major B kernel on a transposed
copy. Aligned M are the controls and must keep their launches. The cases cover M from 1 to 65537 at feature counts from
24 x 64 to 11008 x 4096 (at most MAX_FLOP per product), every gradient request with its launch counts, strided and
transposed inputs, expanded and transposed output gradients, CUDA-graph capture of a ragged step, grouped_linear's
ragged groups, gelu_tanh and N(0,1) data within test_gpu_nn.GRAD_TOL, and a short training run on 3 x 67-token
batches.
"""
import itertools

import pytest
import torch
import torch.nn.functional as F

import dispatch_sweep as ds
import grad_domain as gd
from cuda_l2_b200 import capi, ops
from test_gpu_nn import GRAD_TOL

pytestmark = pytest.mark.gpu

RAGGED = (1, 7, 9, 63, 65, 193, 4097, 65537)
ALIGNED = (8, 200, 4096, 65536)
FEATURES = ((24, 64), (64, 136), (1024, 4096), (4096, 1024))     # (N, K): out_features, in_features
WIDE = (11008, 4096)                                              # at M <= 4097
MAX_FLOP = 2 ** 40                                                # 2 B M N K of one case
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
# Aligned M whose weight gradient (the NN problem M' = N, N' = K, K' = M) the NN dispatcher plans as cluster split-K
# or stream-K at 132 SMs (asserted by test_grad_exact_cpu.py, run here by every operator variant).
SPLIT_SHAPE = (65536, 24, 64)

# Every differentiable operator, with the variants this file runs: (kind, forward acc, activation, batch).
OPERATORS = {
    "hgemm": [("fp16", "fp32", "none", 1), ("fp16", "fp16", "none", 1), ("bf16", "fp32", "none", 1)],
    "hgemm_nn": [("fp16", "fp32", "none", 1), ("bf16", "fp32", "none", 1)],
    "hgemm_batched": [("fp16", "fp32", "none", 1), ("bf16", "fp32", "none", 3), ("fp16", "fp32", "none", 8)],
    "hgemm_bias_act": [("fp16", "fp32", "none", 1), ("bf16", "fp32", "relu", 1), ("fp16", "fp32", "relu", 1)],
    "grouped_linear": [("fp16", "fp32", "none", 1), ("bf16", "fp32", "none", 1)],
}


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def bits(x):
    return x.detach().view(torch.int16)


def check(got, want64, kind, what):
    """``got`` has the operand dtype and the reference's shape, and is bit for bit ``want64`` rounded once."""
    assert got is not None, what
    assert got.dtype == DTYPES[kind] and tuple(got.shape) == tuple(want64.shape), (what, got.dtype, got.shape)
    want = ds.round_to(torch, want64, kind)
    if not torch.equal(bits(got), want):
        bad = (bits(got) != want).nonzero()
        raise AssertionError(f"{what}: {len(bad)} of {want.numel()} elements differ, first at {bad[0].tolist()}")


def counts():
    torch.cuda.synchronize()
    return capi.launch_count(), capi.batched_launch_count(), capi.grouped_bwd_launch_count()


# ------------------------------------------------------------------------------------------------- one step
def _operands(kind, bsz, m, n, k, seed, bias=False):
    """Per-batch exact-domain operands (a list of B GradOperands)."""
    return [gd.operands(torch, m, n, k, kind, seed + 7919 * b, bias=bias) for b in range(bsz)]


def _reference(obs, activation="none", batched=False):
    """float64 (y, dX, dW, dbias), stacked over the batch if ``batched``."""
    refs = [gd.exact(torch, o, activation) for o in obs]
    if not batched:
        (ref,) = refs
        return ref
    return tuple(None if r[0] is None else torch.stack(r) for r in zip(*refs))


def _step(op, kind, acc, activation, obs, need=(True, True, True)):
    """One forward and backward of ``op`` on the operands, the inputs requiring a gradient as ``need`` says (x, w,
    bias). Returns (y, dX, dW as [N, K], dbias)."""
    leaf = lambda t, flag: t.detach().clone().requires_grad_(flag)  # noqa: E731
    if op == "hgemm_batched":
        a = leaf(torch.stack([o.a for o in obs]), need[0])
        bt = leaf(torch.stack([o.bt for o in obs]), need[1])
        y = ops.hgemm_batched(a, bt, acc)
        dy = torch.stack([o.dy for o in obs])
    else:
        (o,) = obs
        a, dy = leaf(o.a, need[0]), o.dy
        if op == "hgemm_nn":
            bt = leaf(o.bt.t().contiguous(), need[1])          # B [K, N] row-major
            y = ops.hgemm_nn(a, bt, acc)
        else:
            bt = leaf(o.bt, need[1])
            if op == "hgemm":
                y = ops.hgemm(a, bt, acc)
            else:
                bias = None if o.bias is None else leaf(o.bias, need[2])
                y = ops.hgemm_bias_act(a, bt, bias, activation)
    if y.requires_grad:
        y.backward(dy)
    dw = bt.grad
    if op == "hgemm_nn" and dw is not None:
        dw = dw.t()
    db = None if op != "hgemm_bias_act" or o.bias is None else bias.grad
    return y, a.grad, dw, db


def _check_step(got, want, kind, acc, what):
    y, dx, dw, db = got
    wy, wdx, wdw, wdb = want
    if acc == "fp32":                       # an fp16-accumulating forward is not on the exact domain
        check(y, wy, kind, f"{what} y")
    check(dx, wdx, kind, f"{what} dX")
    check(dw, wdw, kind, f"{what} dW")
    if wdb is not None:
        check(db, wdb, kind, f"{what} dbias")


def _cases():
    out = []
    for op, variants in OPERATORS.items():
        if op == "grouped_linear":
            continue
        for (kind, acc, act, bsz), m, (n, k) in itertools.product(variants, RAGGED + ALIGNED, FEATURES + (WIDE,)):
            if (n, k) == WIDE and m > 4097 or 2 * bsz * m * n * k > MAX_FLOP:
                continue
            out.append(pytest.param(op, kind, acc, act, bsz, m, n, k,
                                    id=f"{op}-{kind}-acc{acc}-{act}-B{bsz}-{m}x{n}x{k}"))
    return out


@pytest.mark.parametrize("op, kind, acc, activation, bsz, m, n, k", _cases())
def test_training_products_are_one_rounding_of_the_exact_value(op, kind, acc, activation, bsz, m, n, k):
    bias = op == "hgemm_bias_act" and (activation == "none" or m % 2 == 1)   # relu also runs without a bias
    obs = _operands(kind, bsz, m, n, k, ds.shape_seed(m, n, k, bsz), bias=bias)
    got = _step(op, kind, acc, activation, obs)
    _check_step(got, _reference(obs, activation, op == "hgemm_batched"), kind, acc, f"{op} {kind} M={m}")


# ------------------------------------------------------------------------------------------ gradient requests
@pytest.mark.parametrize("op", ["hgemm", "hgemm_nn", "hgemm_batched", "hgemm_bias_act"])
@pytest.mark.parametrize("m", [193, 200])
def test_every_gradient_request_and_its_launches(op, m):
    """Each combination of inputs requiring a gradient gives exactly those gradients, bit for bit, with the launches of
    its path: dX one launch of its kernel; dW one row-major B (or batched) launch at aligned M, and at ragged M one
    K-grouped launch and none of the library the aligned path uses."""
    kind, n, k = "bf16", 64, 136
    bsz = 3 if op == "hgemm_batched" else 1
    obs = _operands(kind, bsz, m, n, k, 11 + m, bias=op == "hgemm_bias_act")
    want = _reference(obs, batched=op == "hgemm_batched")
    inputs = 3 if op == "hgemm_bias_act" else 2
    for need in itertools.product((False, True), repeat=inputs):
        need = need + (False,) * (3 - inputs)
        before = counts()
        # the forward alone: its launches are not what this counts
        y, dx, dw, db = _step(op, kind, "fp32", "none", obs, need)
        after = counts()
        check(y, want[0], kind, f"{op} {need} y")
        for flag, g, w, name in ((need[0], dx, want[1], "dX"), (need[1], dw, want[2], "dW"), (need[2], db, want[3], "db")):
            if flag:
                check(g, w, kind, f"{op} {need} {name}")
            else:
                assert g is None, (op, need, name)
        fwd = {"hgemm": (1, 0), "hgemm_nn": (1, 0), "hgemm_batched": (0, 1), "hgemm_bias_act": (0, 0)}[op]
        lib = 1 if op == "hgemm_batched" else 0               # the counter of dX's and the aligned dW's kernel
        want_counts = [fwd[0], fwd[1], 0]
        want_counts[lib] += need[0]
        if need[1]:
            want_counts[lib if m % 8 == 0 else 2] += 1
        assert [b - a for a, b in zip(before, after)] == want_counts, (op, m, need)


# ------------------------------------------------------------------------------------------------- layouts
@pytest.mark.parametrize("kind", ["fp16", "bf16"])
@pytest.mark.parametrize("m", [193, 4096])
def test_strided_inputs_and_output_gradients(kind, m):
    """x as a row slice of a wider tensor and as a transposed view; dY expanded along the tokens (stride 0, as a
    .sum() or a broadcast gives) and as a transposed view. Through ops.linear and B200Linear."""
    n, k = 64, 136
    (o,) = _operands(kind, 1, m, n, k, 5 + m, bias=True)
    wide = torch.zeros((m, k + 24), dtype=o.a.dtype, device="cuda")
    wide[:, 8:8 + k] = o.a
    xs = {"row slice": wide[:, 8:8 + k], "transposed": o.a.t().contiguous().t()}
    dys = {"expanded": o.dy[:1].expand(m, n), "transposed": o.dy.t().contiguous().t()}
    for (xname, x), (dname, dy), module in itertools.product(xs.items(), dys.items(), (False, True)):
        assert not x.is_contiguous() and not dy.is_contiguous()
        ref = gd.GradOperands(o.a, o.bt, dy.contiguous(), o.bias, o.r, o.c, o.q, o.limits)
        _, wdx, wdw, wdb = gd.exact(torch, ref)
        x = x.detach().requires_grad_()
        w, b = o.bt.clone().requires_grad_(), o.bias.clone().requires_grad_()
        if module:
            lin = ops.B200Linear(k, n, device="cuda", dtype=o.a.dtype)
            lin.weight, lin.bias = torch.nn.Parameter(w), torch.nn.Parameter(b)
            lin(x).backward(dy)
            w, b = lin.weight, lin.bias
        else:
            ops.linear(x, w, b).backward(dy)
        what = f"{xname} x, {dname} dY, module={module}"
        check(x.grad, wdx, kind, f"{what} dX")
        check(w.grad, wdw, kind, f"{what} dW")
        check(b.grad, wdb, kind, f"{what} dbias")


@pytest.mark.parametrize("kind", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", [(193,), (3, 67), (4097,)])
def test_b200linear_with_bias(kind, shape):
    """B200Linear (2-D and 3-D input): y = round(round(x W^T) + b) as torch adds the bias, dX, dW and dbias exact."""
    m, n, k = int(torch.tensor(shape).prod()), 1024, 4096
    (o,) = _operands(kind, 1, m, n, k, 3 + m, bias=True)
    lin = ops.B200Linear(k, n, device="cuda", dtype=o.a.dtype)
    with torch.no_grad():
        lin.weight.copy_(o.bt)
        lin.bias.copy_(o.bias)
    x = o.a.reshape(*shape, k).clone().requires_grad_()
    y = lin(x)
    y.backward(o.dy.reshape(*shape, n))
    ref = gd.GradOperands(o.a, o.bt, o.dy, None, o.r, o.c, o.q, o.limits)
    wy, wdx, wdw, _ = gd.exact(torch, ref)
    want_y = ds.round_to(torch, wy, kind).view(o.a.dtype) + o.bias
    assert y.shape == (*shape, n) and torch.equal(bits(y.reshape(m, n)), bits(want_y))
    check(x.grad.reshape(m, k), wdx, kind, "dX")
    check(lin.weight.grad, wdw, kind, "dW")
    check(lin.bias.grad, o.dy.double().sum(0), kind, "dbias")


# ------------------------------------------------------------------------------------------------- grouped_linear
@pytest.mark.parametrize("kind", ["fp16", "bf16"])
@pytest.mark.parametrize("t, sizes", [(193, [0, 1, 37, 0, 100, 1, 50]), (4097, [1, 0, 2048, 7, 1999, 0, 1])])
def test_grouped_linear_ragged_groups(kind, t, sizes):
    """Empty and one-row groups, starts off every multiple of 8, and a last end before T: rows past it get a zero dX
    and their dY is never read (NaN there)."""
    g, n, k = len(sizes), 64, 136
    (o,) = _operands(kind, 1, t, g * n, k, 17 + t)
    ends = torch.tensor(sizes).cumsum(0)
    offs = ends.to(torch.int32).cuda()
    w = o.bt.view(g, n, k).clone().requires_grad_()
    x = o.a.clone().requires_grad_()
    dy = torch.empty((t, n), dtype=o.a.dtype, device="cuda").fill_(float("nan"))
    a64, w64, dy64 = o.a.double(), o.bt.double().view(g, n, k), torch.zeros((t, n), dtype=torch.float64, device="cuda")
    want_y, want_dx = torch.zeros_like(dy64), torch.zeros((t, k), dtype=torch.float64, device="cuda")
    want_dw = torch.zeros((g, n, k), dtype=torch.float64, device="cuda")
    start = 0
    for j, end in enumerate(ends.tolist()):
        dy[start:end] = o.dy[start:end, j * n:(j + 1) * n]
        dy64[start:end] = dy[start:end].double()
        want_y[start:end] = a64[start:end] @ w64[j].T
        want_dx[start:end] = dy64[start:end] @ w64[j]
        want_dw[j] = dy64[start:end].T @ a64[start:end]
        start = end
    y = ops.grouped_linear(x, w, offs)
    y.backward(dy)
    used = int(ends[-1])
    check(y[:used], want_y[:used].add_(0.0), kind, "y")
    check(x.grad, want_dx.add_(0.0), kind, "dX")
    check(w.grad, want_dw.add_(0.0), kind, "dW")


# ------------------------------------------------------------------------------------------------- N(0,1) data
def _randn(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dtype)


def _rel_err(got, ref):
    return float((got.double() - ref).abs().max() / ref.pow(2).mean().sqrt())


@pytest.mark.parametrize("kind", ["fp16", "bf16"])
@pytest.mark.parametrize("m", [65, 193, 4096])
def test_gelu_tanh_gradients_within_tolerance(kind, m):
    """gelu_tanh's dZ is not on the exact domain: dX, dW and dbias against float64 within GRAD_TOL x rms."""
    dtype, n, k = DTYPES[kind], 1024, 1024
    a = _randn((m, k), dtype, 1).requires_grad_()
    bt = _randn((n, k), dtype, 2, k ** -0.5).requires_grad_()
    bias = _randn((n,), dtype, 3).requires_grad_()
    dy = _randn((m, n), dtype, 4)
    ops.linear(a, bt, bias, "gelu_tanh").backward(dy)
    a64, bt64 = a.detach().double(), bt.detach().double()
    z = a64 @ bt64.T + bias.detach().double()
    dz = torch.ops.aten.gelu_backward(dy.double(), z, approximate="tanh")
    for got, ref in ((a.grad, dz @ bt64), (bt.grad, dz.T @ a64), (bias.grad, dz.sum(0))):
        assert got.dtype == dtype and got.shape == ref.shape
        assert _rel_err(got, ref) <= GRAD_TOL[dtype], (kind, m, _rel_err(got, ref))


@pytest.mark.parametrize("kind, m, k, n", [("bf16", 4097, 4096, 11008), ("fp16", 193, 1024, 1024)])
def test_randn_gradients_within_tolerance(kind, m, k, n):
    """B200Linear's dX and dW on N(0,1) data against float64, at a ragged M (the K-grouped weight gradient)."""
    dtype = DTYPES[kind]
    lin = ops.B200Linear(k, n, bias=False, device="cuda", dtype=dtype)
    with torch.no_grad():
        lin.weight.copy_(_randn((n, k), dtype, 5, k ** -0.5))
    x = _randn((m, k), dtype, 6).requires_grad_()
    dy = _randn((m, n), dtype, 7)
    lin(x).backward(dy)
    x64, w64, dy64 = x.detach().double(), lin.weight.detach().double(), dy.double()
    for got, ref in ((x.grad, dy64 @ w64), (lin.weight.grad, dy64.T @ x64)):
        assert got.dtype == dtype and got.shape == ref.shape
        assert _rel_err(got, ref) <= GRAD_TOL[dtype], (kind, _rel_err(got, ref))


# ------------------------------------------------------------------------------------------------- CUDA graph
@pytest.mark.parametrize("kind", ["fp16", "bf16"])
def test_ragged_training_step_captured_in_a_cuda_graph(kind):
    """A B200Linear step at M = 193 (the K-grouped weight gradient, its group end written on the device) captured in
    a CUDA graph and replayed twice gives the eager bits."""
    m, n, k = 193, 1024, 4096
    (o,) = _operands(kind, 1, m, n, k, 23, bias=True)
    lin = ops.B200Linear(k, n, device="cuda", dtype=o.a.dtype)
    with torch.no_grad():
        lin.weight.copy_(o.bt)
        lin.bias.copy_(o.bias)
    x = o.a.clone().requires_grad_()
    dy = o.dy.clone()
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for _ in range(2):                  # eager steps on a side stream (the warm-up torch.cuda.graph asks for)
            lin.zero_grad(set_to_none=True)
            x.grad = None
            y = lin(x)
            y.backward(dy)
            eager = [y.detach().clone(), x.grad.clone(), lin.weight.grad.clone(), lin.bias.grad.clone()]
    torch.cuda.current_stream().wait_stream(stream)
    del y                                   # its autograd graph would tie the captured AccumulateGrad to the side stream
    lin.zero_grad(set_to_none=True)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = lin(x)
        y.backward(dy)
    for _ in range(2):
        for t in (x.grad, lin.weight.grad, lin.bias.grad):
            t.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        for got, want in zip((y.detach(), x.grad, lin.weight.grad, lin.bias.grad), eager):
            assert torch.equal(bits(got), bits(want))
    ref = gd.GradOperands(o.a, o.bt, o.dy, None, o.r, o.c, o.q, o.limits)
    _, wdx, wdw, _ = gd.exact(torch, ref)
    check(eager[1], wdx, kind, "dX")
    check(eager[2], wdw, kind, "dW")


# ------------------------------------------------------------------------------------------------- training
def _train(kind: str, seed: int, steps: int = 50) -> tuple[list[float], list[torch.Tensor]]:
    """A 256 -> 512 -> 256 GELU MLP (bf16, with biases) fitted by Adam to a fixed random teacher on batches of
    3 x 67 tokens; ``kind`` "b200" swaps its layers with replace_linear_modules. Returns the losses and the final
    parameters."""
    torch.manual_seed(seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    teacher = [torch.randn((512, 256), device="cuda", generator=g) / 16,
               torch.randn((256, 512), device="cuda", generator=g) / 22]
    model = torch.nn.Sequential(torch.nn.Linear(256, 512), torch.nn.GELU(), torch.nn.Linear(512, 256))
    model = model.to(device="cuda", dtype=torch.bfloat16)
    if kind == "b200":
        assert ops.replace_linear_modules(model) == ["0", "2"]
    opt = torch.optim.Adam(model.parameters(), lr=2e-3)
    losses = []
    for _ in range(steps):
        x = torch.randn((3, 67, 256), device="cuda", generator=g)
        target = F.gelu(x @ teacher[0].t()) @ teacher[1].t()
        loss = F.mse_loss(model(x.bfloat16()).float(), target)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    return losses, [p.detach().clone() for p in model.parameters()]


def test_mlp_training_on_ragged_batches_is_deterministic_and_close_to_bf16():
    losses_a, params_a = _train("b200", 0)
    losses_b, params_b = _train("b200", 0)
    assert losses_a == losses_b
    for p, q in zip(params_a, params_b):
        assert torch.equal(bits(p), bits(q))
    losses_ref, _ = _train("torch", 0)
    final, final_ref = sum(losses_a[-10:]) / 10, sum(losses_ref[-10:]) / 10
    assert final < losses_a[0], (losses_a[0], final)                 # it trains
    assert abs(final - final_ref) <= 0.01 * final_ref, (final, final_ref)
