"""Without a GPU: which kernels the 16-bit backward runs at ragged and aligned token counts (recorded on meta tensors),
the exact gradient domain of tests/grad_domain.py, and that tests/test_gpu_grad_exact.py covers every differentiable
operator."""
import numpy as np
import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode

import dispatch_sweep as ds
import exact_domain as ed
import grad_domain as gd
import test_gpu_grad_exact as gpu
from cuda_l2_b200 import ops
from test_op_registry_cpu import SCHEMAS, WHY

_OURS = {"hgemm", "hgemm_nn", "hgemm_batched", "hgemm_grouped_wgrad", "hgemm_bias_act"}


class _Calls(TorchDispatchMode):
    """Records (operator name, shapes of its tensor arguments, offs length) of every cuda_l2_b200 call."""

    def __init__(self):
        super().__init__()
        self.calls = []

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        if func.namespace == "cuda_l2_b200":
            self.calls.append((func.__name__.split(".")[0],
                               tuple(tuple(a.shape) for a in args if isinstance(a, torch.Tensor))))
        return func(*args, **(kwargs or {}))


def _meta(*shape, dtype=torch.bfloat16):
    return torch.empty(shape, dtype=dtype, device="meta", requires_grad=True)


def _backward_calls(op: str, m: int, bsz: int = 3):
    n, k = 24, 32
    if op == "hgemm_batched":
        a, b = _meta(bsz, m, k), _meta(bsz, n, k)
        y = ops.hgemm_batched(a, b)
    elif op == "hgemm_nn":
        a, b = _meta(m, k), _meta(k, n)
        y = ops.hgemm_nn(a, b)
    elif op == "hgemm_bias_act":
        a, b = _meta(m, k), _meta(n, k)
        y = ops.hgemm_bias_act(a, b, _meta(n), "relu")
    else:
        a, b = _meta(m, k), _meta(n, k)
        y = ops.hgemm(a, b)
    with _Calls() as rec:
        grads = torch.autograd.grad(y.sum(), (a, b))
    assert grads[0].shape == a.shape and grads[1].shape == b.shape
    return [c for c in rec.calls if c[0] in _OURS]


@pytest.mark.parametrize("op", ["hgemm", "hgemm_nn", "hgemm_batched", "hgemm_bias_act"])
@pytest.mark.parametrize("m", [1, 7, 41, 193])
def test_a_ragged_weight_gradient_runs_the_k_grouped_kernel_once(op, m):
    """At M % 8 != 0: dX as before, and dW from one hgemm_grouped_wgrad call with G = 1 (G = B batched) that reads
    the output gradient and the input in place; no row-major B or batched call for it."""
    bsz = 3
    calls = _backward_calls(op, m, bsz)
    wgrad = [c for c in calls if c[0] == "hgemm_grouped_wgrad"]
    assert len(wgrad) == 1, calls
    rows = bsz * m if op == "hgemm_batched" else m
    n, k = 24, 32
    a_shape, b_shape = ((rows, k), (rows, n)) if op == "hgemm_nn" else ((rows, n), (rows, k))
    assert wgrad[0][1] == (a_shape, b_shape, (bsz if op == "hgemm_batched" else 1,)), wgrad
    dx = {"hgemm": "hgemm_nn", "hgemm_bias_act": "hgemm_nn", "hgemm_nn": "hgemm", "hgemm_batched": "hgemm_batched"}[op]
    assert [c[0] for c in calls if c[0] != "hgemm_grouped_wgrad"] == [dx], calls


@pytest.mark.parametrize("op, want", [
    ("hgemm", [("hgemm_nn", ((40, 24), (24, 32))), ("hgemm_nn", ((24, 40), (40, 32)))]),
    ("hgemm_bias_act", [("hgemm_nn", ((40, 24), (24, 32))), ("hgemm_nn", ((24, 40), (40, 32)))]),
    ("hgemm_nn", [("hgemm", ((40, 24), (32, 24))), ("hgemm_nn", ((32, 40), (40, 24)))]),
    ("hgemm_batched", [("hgemm_batched", ((3, 40, 24), (3, 32, 24))), ("hgemm_batched", ((3, 24, 40), (3, 32, 40)))]),
])
def test_an_aligned_weight_gradient_keeps_its_calls(op, want):
    """At M = 40 the backward calls exactly what it called before ragged M had a path: the row-major B (or batched)
    products on dC^T / A^T."""
    assert _backward_calls(op, 40) == want


# ------------------------------------------------------------------------------------------------- the domain
SHAPES = [(193, 64, 136), (200, 1024, 4096)]


@pytest.mark.parametrize("kind", ["fp16", "bf16"])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("m, n, k", SHAPES + [(1, 24, 64), (65537, 24, 64), (4097, 11008, 4096)])
def test_domain_bounds_and_operands(kind, bias, m, n, k):
    """The three sum bounds hold (from the integers, not the limits), and every operand is exact and zero or normal."""
    if m * n * k > 2 ** 30:
        li, lj, lh = gd.limits(m, n, k, bias)          # too large to build here: the limits alone
        assert k * li * lj < ed.EXACT_SUM_BOUND and n * lh * lj < ed.EXACT_SUM_BOUND and m * lh * li < ed.EXACT_SUM_BOUND
        return
    o = gd.operands(torch, m, n, k, kind, 3, bias=bias, device="cpu")
    ia = o.a.double() / torch.exp2(o.r.double())[:, None]
    jb = o.bt.double() / torch.exp2(o.c.double())[:, None]
    h = o.dy.double() / torch.exp2((o.q - o.r[:, None] - o.c[None, :]).double())
    for x in (ia, jb, h):
        assert torch.equal(x, x.round()) and int(x.abs().max()) <= 2 ** gd.LIM_BITS - 1
    assert float((ia.abs() @ jb.abs().T).max()) < ed.EXACT_SUM_BOUND
    assert float((h.abs() @ jb.abs()).max()) < ed.EXACT_SUM_BOUND
    assert float((h.abs().T @ ia.abs()).max()) < ed.EXACT_SUM_BOUND
    lo, hi = 2.0 ** gd.NORMAL[kind][0], float(torch.finfo(o.a.dtype).max)
    for t in (o.a, o.bt, o.dy) + ((o.bias,) if bias else ()):
        v = t.double().abs()
        assert bool(((v == 0) | ((v >= lo) & (v <= hi))).all())
    assert float((o.dy != 0).double().mean()) > 0.2   # most of dY is not zero-masked


@pytest.mark.parametrize("kind", ["fp16", "bf16"])
@pytest.mark.parametrize("m, n, k", SHAPES)
def test_domain_reaches_every_rounding_case(kind, m, n, k):
    """y, dX and dW each round up, round down and tie. In fp16, y has subnormal outputs, overflows to inf and rounds
    nonzero values to zero (the relu mask is read from the rounded output); dX and dW reach subnormals and inf at the
    larger shape, whose sums spread wider."""
    o = gd.operands(torch, m, n, k, kind, ds.shape_seed(m, n, k, 1), device="cpu")
    y, dx, dw, _ = gd.exact(torch, o)
    for name, x in (("y", y), ("dX", dx), ("dW", dw)):
        c = gd.classify(x.numpy(), kind)
        assert c["up"] and c["down"] and c["tie"], (name, c)
        if kind == "fp16" and (name == "y" or (m, n, k) == SHAPES[-1]):
            assert c["subnormal"] and c["inf"], (name, c)
    assert gd.classify(y.numpy(), "fp16")["zero"] if kind == "fp16" else True


@pytest.mark.parametrize("kind", ["fp16", "bf16"])
@pytest.mark.parametrize("m", [193, 4097])
def test_bias_gradient_is_exact_in_fp32(kind, m):
    """With bias=True the fp32 column sum of dY (any order) equals the float64 one, and z = A Bt^T + bias is exact in
    fp32; the relu mask then differs from z > 0 exactly where a positive z rounds to zero."""
    n, k = 64, 136
    o = gd.operands(torch, m, n, k, kind, 9, bias=True, device="cpu")
    d64 = o.dy.double()
    assert torch.equal(o.dy.float().sum(0).double(), d64.sum(0))
    assert torch.equal(o.dy.float().flip(0).cumsum(0)[-1].double(), d64.sum(0))
    z = o.a.double() @ o.bt.double().T + o.bias.double()
    assert torch.equal(z.float().double(), z)
    y, _, _, db = gd.exact(torch, o, "relu")
    assert torch.equal(db, (d64 * (y.float().to(o.a.dtype) > 0)).sum(0))


@pytest.mark.parametrize("kind", ["fp16", "bf16"])
def test_reference_equals_numpy_rounded_once(kind):
    """The reference the GPU tests use (torch float64, dispatch_sweep.round_to) equals numpy float64 rounded once."""
    m, n, k = 193, 64, 136
    o = gd.operands(torch, m, n, k, kind, 4, bias=True, device="cpu")
    y, dx, dw, db = gd.exact(torch, o)
    a, bt, dy = (t.double().numpy() for t in (o.a, o.bt, o.dy))
    want = {"y": a @ bt.T + o.bias.double().numpy(), "dx": dy @ bt, "dw": dy.T @ a, "db": dy.sum(0)}
    rnd = ed.round_fp16_bits if kind == "fp16" else ed.round_bf16_bits
    with np.errstate(over="ignore"):
        for name, got in (("y", y), ("dx", dx), ("dw", dw), ("db", db)):
            ours = ds.round_to(torch, got, kind).numpy().view(np.uint16)
            assert np.array_equal(ours, rnd(want[name] + 0.0)), name


# ------------------------------------------------------------------------------------------------- coverage
def test_every_differentiable_operator_is_in_the_gpu_table():
    assert set(SCHEMAS) - set(WHY) == set(gpu.OPERATORS)


def test_an_aligned_weight_gradient_is_planned_with_a_k_split(built_libs):
    """SPLIT_SHAPE's weight gradient (an NN problem N x K reducing over M = 65536) runs cluster split-K or stream-K."""
    m, n, k = gpu.SPLIT_SHAPE
    for leg in ("nn_fp16", "nn_bf16"):
        cfg, _, splits, _ = ds.nn_choice(leg, n, k, m)
        mode, _ = ds.plan(leg, cfg, n, k, m, splits)
        assert mode in ("cluster-split-k", "stream-k"), (leg, cfg, splits, mode)
