"""The 16-bit operators on empty shapes give torch's answer without a library launch: M, N or B == 0 an empty result,
K == 0 (an empty reduction) zeros. The backward of each on an empty batch gives zero weight gradients and empty input
gradients, as nn.Linear's does; a training step on an empty micro-batch must not raise."""
import pytest
import torch
from torch import nn

from cuda_l2_b200 import capi, ops

pytestmark = pytest.mark.gpu

DTYPES = (torch.float16, torch.bfloat16)
MNK = {"M": (0, 24, 32), "N": (16, 0, 32), "K": (16, 24, 0)}


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def counters():
    return (capi.launch_count(), capi.batched_launch_count(), capi.grouped_launch_count(),
            capi.grouped_bwd_launch_count())


def rand(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, device="cuda", generator=g).to(dtype)


def same_as(got, want, dtype):
    """Shape and dtype of torch's result, and its values (zeros or nothing)."""
    assert got.dtype == dtype and got.shape == want.shape, (got.shape, want.shape)
    assert torch.equal(got.float(), want), got
    assert not got.view(torch.int16).any()          # +0.0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("zero", sorted(MNK))
def test_2d_operators(zero, dtype):
    m, n, k = MNK[zero]
    a, bt = rand((m, k), dtype, 1), rand((n, k), dtype, 2)
    before = counters()
    want = torch.matmul(a.float(), bt.float().t())
    same_as(ops.hgemm(a, bt), want, dtype)
    same_as(ops.hgemm_nn(a, bt.t().contiguous()), want, dtype)
    if dtype == torch.float16:
        same_as(ops.hgemm(a, bt, "fp16"), want, dtype)
        same_as(ops.hgemm_nn(a, bt.t().contiguous(), "fp16"), want, dtype)
    torch.cuda.synchronize()
    assert counters() == before


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("zero", ["B", "M", "N", "K"])
def test_batched_operator(zero, dtype):
    b, m, n, k = {"B": (0, 8, 16, 32), "M": (3, 0, 16, 32), "N": (3, 8, 0, 32), "K": (3, 8, 16, 0)}[zero]
    a, bt = rand((b, m, k), dtype, 3), rand((b, n, k), dtype, 4)
    before = counters()
    want = torch.bmm(a.float(), bt.float().transpose(1, 2))
    same_as(ops.hgemm_batched(a, bt), want, dtype)
    if b:
        masked = torch.full((b,), m, dtype=torch.int32, device="cuda")
        same_as(ops.hgemm_batched(a, bt, masked_m=masked), want, dtype)
    torch.cuda.synchronize()
    assert counters() == before


@pytest.mark.parametrize("dtype", DTYPES)
def test_grouped_operators_with_an_empty_reduction_or_no_column(dtype):
    offs = torch.tensor([3, 3, 10], dtype=torch.int32, device="cuda")
    t = 10
    before = counters()
    for n, k in ((16, 0), (0, 16)):
        x, w = rand((t, k), dtype, 5), rand((3, n, k), dtype, 6)
        want = torch.zeros((t, n))
        same_as(ops.hgemm_grouped(x, w, offs), want.cuda(), dtype)
        same_as(ops.hgemm_grouped_nn(x, w.transpose(1, 2).contiguous(), offs), want.cuda(), dtype)
        same_as(ops.grouped_linear(x, w, offs), want.cuda(), dtype)
    torch.cuda.synchronize()
    assert counters() == before


@pytest.mark.parametrize("dtype", DTYPES)
def test_grouped_linear_backward_with_an_empty_reduction(dtype):
    offs = torch.tensor([3, 3, 10], dtype=torch.int32, device="cuda")
    for n, k in ((16, 0), (0, 16)):
        x = rand((10, k), dtype, 7).requires_grad_()
        w = rand((3, n, k), dtype, 8).requires_grad_()
        before = counters()
        ops.grouped_linear(x, w, offs).sum().backward()
        torch.cuda.synchronize()
        assert counters() == before
        assert x.grad.shape == x.shape and not x.grad.view(torch.int16).any()
        assert w.grad.shape == w.shape and not w.grad.view(torch.int16).any()


def check_grads(ours, theirs):
    for (name, p), (_, q) in zip(ours, theirs):
        assert p.grad is not None and p.grad.shape == q.grad.shape and p.grad.dtype == p.dtype, name
        assert torch.equal(p.grad.float(), q.grad.float()), name
        assert not p.grad.view(torch.int16).any(), name


@pytest.mark.parametrize("dtype", DTYPES)
def test_operator_backward_on_an_empty_batch(dtype):
    k, n = 24, 32
    for op, b_shape, ref in ((ops.hgemm, (n, k), lambda a, b: a @ b.t()),
                             (ops.hgemm_nn, (k, n), lambda a, b: a @ b)):
        a = rand((0, k), dtype, 9).requires_grad_()
        b = rand(b_shape, dtype, 10).requires_grad_()
        a2, b2 = a.detach().float().requires_grad_(), b.detach().float().requires_grad_()
        before = counters()
        op(a, b).sum().backward()
        torch.cuda.synchronize()
        assert counters() == before
        ref(a2, b2).sum().backward()
        check_grads([("a", a), ("b", b)], [("a", a2), ("b", b2)])
    a = rand((3, 0, k), dtype, 11).requires_grad_()
    bt = rand((3, n, k), dtype, 12).requires_grad_()
    a2, bt2 = a.detach().float().requires_grad_(), bt.detach().float().requires_grad_()
    before = counters()
    ops.hgemm_batched(a, bt).sum().backward()
    torch.cuda.synchronize()
    assert counters() == before
    torch.bmm(a2, bt2.transpose(1, 2)).sum().backward()
    check_grads([("a", a), ("bt", bt)], [("a", a2), ("bt", bt2)])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(0, 5, 64), (4, 0, 64), (0, 64)])
def test_linear_training_step_on_an_empty_micro_batch(shape, dtype):
    torch.manual_seed(0)
    lin = nn.Linear(64, 48, bias=True).to("cuda", dtype)
    ref = nn.Linear(64, 48, bias=True).to("cuda", torch.float32)
    with torch.no_grad():
        ref.weight.copy_(lin.weight)
        ref.bias.copy_(lin.bias)
    layer = ops.B200Linear.from_linear(lin)
    x = torch.zeros(shape, dtype=dtype, device="cuda", requires_grad=True)
    x2 = torch.zeros(shape, dtype=torch.float32, device="cuda", requires_grad=True)
    before = counters()
    y = layer(x)
    y.sum().backward()
    torch.cuda.synchronize()
    assert counters() == before
    y2 = ref(x2)
    y2.sum().backward()
    assert y.shape == y2.shape and y.dtype == dtype
    assert x.grad.shape == x.shape
    check_grads([("weight", lin.weight), ("bias", lin.bias)], [("weight", ref.weight), ("bias", ref.bias)])
