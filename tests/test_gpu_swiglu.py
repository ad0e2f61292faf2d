"""The SwiGLU library (libb200_swiglu.so) on the H100: every gated configuration against the TN kernel and torch's
composition bit for bit, the dispatched calls at the benchmark shapes, every 16-bit value of the gate through the
epilogue and the backward, the trainable layer's gradients, and a training step captured in a CUDA graph."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from cuda_l2_b200 import capi, ops
from swiglu_ref import cuda_exp, swiglu_grad_reference

pytestmark = pytest.mark.gpu

DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
NP16 = {torch.float16: np.float16, torch.bfloat16: "bfloat16"}
GATED = [c["id"] for c in capi.configs() if c["bn"] in (128, 256)] if torch.cuda.is_available() else []


def _split(h: torch.Tensor):
    """(g, u) views of an interleaved h [M, 2I]."""
    m, n = h.shape
    v = h.view(m, n // 128, 2, 64)
    return v[:, :, 0].reshape(m, n // 2), v[:, :, 1].reshape(m, n // 2)


def _same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Equal bit for bit, except that any NaN matches any NaN."""
    nan = torch.isnan(a)
    return bool(torch.equal(nan, torch.isnan(b)) and torch.equal(a[~nan].view(torch.int16), b[~nan].view(torch.int16)))


def _canaried(shape, dtype, pad=64):
    """A contiguous tensor of ``shape`` inside a NaN-filled buffer with ``pad`` elements on both sides."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * pad,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[pad:pad + n].view(shape)


def _canaries_intact(buf, pad=64) -> bool:
    return bool(torch.isnan(buf[:pad]).all() and torch.isnan(buf[-pad:]).all())


def _operands(m, i, k, dtype, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn((m, k), device="cuda", generator=gen) / 4).to(dtype)
    w = (torch.randn((2 * i, k), device="cuda", generator=gen) / (k ** 0.5) * 8).to(dtype)
    return x, w


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("cfg", GATED)
def test_every_configuration_is_the_tn_kernel_and_torch(cfg, dtype):
    """h is capi.gemm_kmajor's output on the same configuration (plain, splits code 1), y is F.silu(g) * u on that h,
    a launch without h gives the same y, and nothing outside [M, I] / [M, 2I] is written."""
    dt = DTYPES[dtype]
    for m in (1, 129, 200):
        for i in (64, 192, 320):
            for k in (72, 520, 4096):
                x, w = _operands(m, i, k, dt, seed=m + i + k)
                hbuf, h = _canaried((m, 2 * i), dt)
                ybuf, y = _canaried((m, i), dt)
                capi.swiglu(x, w, y, h, config_id=cfg, splits=1)
                want_h = torch.empty((m, 2 * i), dtype=dt, device="cuda")
                capi.gemm_kmajor(x, w, want_h, config_id=cfg, splits=1)
                y2buf, y2 = _canaried((m, i), dt)
                capi.swiglu(x, w, y2, None, config_id=cfg)
                g, u = _split(h)
                where = (cfg, dtype, m, i, k)
                assert torch.equal(h.view(torch.int16), want_h.view(torch.int16)), where
                assert _same_bits(y, F.silu(g) * u), where
                assert torch.equal(y.view(torch.int16), y2.view(torch.int16)), where
                assert _canaries_intact(hbuf) and _canaries_intact(ybuf) and _canaries_intact(y2buf), where


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("cfg", [0, 1, 3, 4, 26])
def test_split_and_stream_k_requests_run_the_plain_schedule(cfg, dtype):
    """Every non-plain splits code (workspace split-K 4 and 32, cluster split-K -2 / -8, stream-K 100 / 101) at shapes
    where the TN kernel would take them (few tiles with a long K; a ragged last wave) runs the plain schedule: h and y
    are the splits = 1 launch's, bit for bit."""
    dt = DTYPES[dtype]
    for m, i, k in ((200, 192, 8192), (1000, 2560, 2048)):
        x, w = _operands(m, i, k, dt, seed=cfg + m)
        h1 = torch.empty((m, 2 * i), dtype=dt, device="cuda")
        y1 = torch.empty((m, i), dtype=dt, device="cuda")
        capi.swiglu(x, w, y1, h1, config_id=cfg, splits=1)
        for splits in (4, 32, -2, -8, capi.STREAMK_TAIL, capi.STREAMK_TAIL_PLUS_WAVE):
            h = torch.full((m, 2 * i), float("nan"), dtype=dt, device="cuda")
            y = torch.full((m, i), float("nan"), dtype=dt, device="cuda")
            capi.swiglu(x, w, y, h, config_id=cfg, splits=splits)
            where = (cfg, dtype, m, i, k, splits)
            assert torch.equal(h.view(torch.int16), h1.view(torch.int16)), where
            assert torch.equal(y.view(torch.int16), y1.view(torch.int16)), where


BENCH_SHAPES = [(16, 11008, 4096), (2048, 11008, 4096), (8192, 11008, 4096), (16, 14336, 4096), (2048, 14336, 4096),
                (8192, 14336, 4096), (16, 1408, 2048)]


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("m,i,k", BENCH_SHAPES)
def test_dispatched_calls_at_the_benchmark_shapes(m, i, k, dtype):
    """y of the dispatched call is the composition over capi.gemm_kmajor with the gated choice, bit for bit, and within
    the 16-bit rounding bound of a float64 SwiGLU of the float64 product."""
    dt = DTYPES[dtype]
    x, w = _operands(m, i, k, dt, seed=m + i)
    y = torch.empty((m, i), dtype=dt, device="cuda")
    capi.swiglu(x, w, y)
    cid, gm, splits = capi.swiglu_select(capi.swiglu_variant(dt), m, i, k)
    assert splits == 1
    h = torch.empty((m, 2 * i), dtype=dt, device="cuda")
    capi.gemm_kmajor(x, w, h, config_id=cid, group_m=gm, splits=1)
    g, u = _split(h)
    assert _same_bits(y, F.silu(g) * u)
    g64, u64 = _split(x.double() @ w.double().t())
    ag, au = _split(x.double().abs() @ w.double().abs().t())
    y64 = F.silu(g64) * u64
    eps = 2.0 ** -(11 if dt == torch.float16 else 8)
    # four roundings (g, u, silu, the product), each at most eps relative; g's carries into silu with the factor
    # 1 + g (1 - sigmoid(g)), at most 1 + |g|. The fp32 sums of g and u carry an absolute error of order
    # 2^-24 sqrt(K) sum |x w| (8 times that here), which matters where g or u is small by cancellation; a floor for the
    # 16-bit subnormal range.
    acc = 2.0 ** -24 * 8 * k ** 0.5
    bound = (eps * y64.abs() * (4 + g64.abs()) + acc * (1.1 * u64.abs() * ag + F.silu(g64).abs() * au) +
             1e-6 * y64.abs().max())
    assert bool(((y.double() - y64).abs() <= bound).all())


def _all_patterns(dt):
    """Every 16-bit pattern as a tensor of dt, [1024, 64]."""
    return torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(dt).view(1024, 64)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_every_gate_value_through_the_epilogue(dtype):
    """Each row of 64 gate values (every 16-bit pattern, ±Inf and NaN included) is one launch with M = 1 and a one-hot
    x, so h is the weight's column exactly, with the sum's own conventions: -0.0 comes out as +0.0 (1 * -0.0 plus the
    +0.0 products of the zero columns) and a NaN as the canonical NaN. y is F.silu(g) * u on that h, bit for bit."""
    dt = DTYPES[dtype]
    gate = _all_patterns(dt)
    gen = torch.Generator(device="cuda").manual_seed(3)
    up = (torch.randn((1024, 64), device="cuda", generator=gen) * 3).to(dt)
    x = torch.zeros((1, 8), dtype=dt, device="cuda")
    x[0, 0] = 1
    y = torch.empty((1024, 64), dtype=dt, device="cuda")
    h = torch.empty((1024, 128), dtype=dt, device="cuda")
    for r in range(1024):
        w = torch.zeros((128, 8), dtype=dt, device="cuda")
        w[:64, 0], w[64:, 0] = gate[r], up[r]
        capi.swiglu(x, w, y[r:r + 1], h[r:r + 1], config_id=1)
    want = torch.where(gate == 0, torch.zeros_like(gate), gate)   # -0.0 -> +0.0
    assert _same_bits(h[:, :64], want) and torch.equal(h[:, 64:].view(torch.int16), up.view(torch.int16))
    assert _same_bits(y, F.silu(h[:, :64]) * h[:, 64:])


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_every_gate_value_through_the_backward(dtype):
    """dh for every 16-bit pattern of g: du and dg are torch autograd's bit for bit, and the numpy reference's (CUDA's
    expf). The kernel's order of operations, fmaf contraction included, is torch's silu_backward's: a change to either
    that moves a last bit fails here."""
    dt = DTYPES[dtype]
    g = _all_patterns(dt)
    gen = torch.Generator(device="cuda").manual_seed(4)
    u = (torch.randn((1024, 64), device="cuda", generator=gen) * 3).to(dt)
    dy = (torch.randn((1024, 64), device="cuda", generator=gen)).to(dt)
    h = torch.stack((g, u), dim=1).reshape(1024, 128).contiguous()
    dh = torch.empty_like(h)
    capi.swiglu_backward(dy, h, dh)
    dg, du = dh[:, :64], dh[:, 64:]
    gt, ut = g.clone().requires_grad_(), u.clone().requires_grad_()
    (F.silu(gt) * ut).backward(dy)
    assert _same_bits(du, ut.grad)
    ref_dg, ref_du = swiglu_grad_reference(dy.float().cpu().numpy(), g.float().cpu().numpy(), u.float().cpu().numpy(),
                                           NP16[dt], exp=cuda_exp)
    assert _same_bits(dg.float().cpu(), torch.from_numpy(ref_dg))
    assert _same_bits(du.float().cpu(), torch.from_numpy(ref_du))
    assert _same_bits(dg, gt.grad)


def _ref_dh(h, dy, dt):
    g, u = _split(h)
    dg, du = swiglu_grad_reference(dy.float().cpu().numpy(), g.float().cpu().numpy(), u.float().cpu().numpy(),
                                   NP16[dt], exp=cuda_exp)
    m, i = dy.shape
    dh = torch.stack((torch.from_numpy(dg).view(m, i // 64, 64), torch.from_numpy(du).view(m, i // 64, 64)), dim=2)
    return dh.reshape(m, 2 * i).to(dt).cuda()


@pytest.mark.parametrize("m", [1, 41, 2048])
def test_layer_gradients_are_the_product_grads_of_the_reference_dh(m):
    dt, hid, i = torch.bfloat16, 512, 320
    layer = ops.B200SwiGLULinear(hid, i, device="cuda", dtype=dt)
    gen = torch.Generator(device="cuda").manual_seed(m)
    x = torch.randn((m, hid), device="cuda", generator=gen).to(dt).requires_grad_()
    dy = torch.randn((m, i), device="cuda", generator=gen).to(dt)
    y = layer(x)
    y.backward(dy)
    h = torch.empty((m, 2 * i), dtype=dt, device="cuda")
    y_ref = torch.empty((m, i), dtype=dt, device="cuda")
    capi.swiglu(x.detach(), layer.weight.detach(), y_ref, h)
    assert torch.equal(y.view(torch.int16), y_ref.view(torch.int16))
    dx, dw = ops._product_grads(x.detach(), layer.weight.detach(), _ref_dh(h, dy, dt), True, True)
    assert torch.equal(x.grad.view(torch.int16), dx.view(torch.int16))
    assert torch.equal(layer.weight.grad.view(torch.int16), dw.view(torch.int16))
    # against a float64 layer: the 16-bit roundings of h, y and dh only
    x64, w64 = x.detach().double().requires_grad_(), layer.weight.detach().double().requires_grad_()
    g64, u64 = _split(x64 @ w64.t())
    (F.silu(g64) * u64).backward(dy.double())
    for got, want in ((y.double(), (F.silu(g64) * u64).detach()), (x.grad.double(), x64.grad),
                      (layer.weight.grad.double(), w64.grad)):
        assert float((got.detach() - want).norm() / want.norm()) < 2e-2


def test_from_linears_is_the_two_linear_composition():
    dt = torch.bfloat16
    gate, up = nn.Linear(256, 192, bias=False, device="cuda", dtype=dt), nn.Linear(256, 192, bias=False, device="cuda",
                                                                                    dtype=dt)
    layer = ops.B200SwiGLULinear.from_linears(gate, up)
    w_g, w_u = ops.split_gate_up(layer.weight.detach())
    assert torch.equal(w_g, gate.weight) and torch.equal(w_u, up.weight)
    x = torch.randn((3, 37, 256), device="cuda").to(dt)
    y = layer(x)
    assert y.shape == (3, 37, 192)
    ref = (F.silu(gate(x).double()) * up(x).double())
    assert float((y.detach().double() - ref.detach()).norm() / ref.norm()) < 1e-2
    # a Llama MLP: the down projection as a B200Linear
    down = ops.B200Linear(192, 256, bias=False, device="cuda", dtype=dt)
    assert down(layer(x)).shape == x.shape


def test_empty_and_inference_calls():
    dt = torch.float16
    w = (torch.randn((256, 64), device="cuda") / 8).to(dt).requires_grad_()
    before = capi.swiglu_launch_count()
    y = ops.swiglu_linear(torch.empty((0, 64), dtype=dt, device="cuda"), w)
    assert y.shape == (0, 128) and capi.swiglu_launch_count() == before
    w0 = torch.empty((256, 0), dtype=dt, device="cuda", requires_grad=True)
    x0 = torch.empty((5, 0), dtype=dt, device="cuda", requires_grad=True)
    y0 = ops.swiglu_linear(x0, w0)
    assert y0.shape == (5, 128) and not y0.view(torch.int16).any()
    y0.sum().backward()
    assert w0.grad.shape == w0.shape and x0.grad.shape == x0.shape
    before = capi.swiglu_launch_count()   # the backward above ran the dh kernel once
    with torch.no_grad():
        x = torch.randn((7, 64), device="cuda").to(dt)
        y = ops.swiglu_linear(x, w)
    assert capi.swiglu_launch_count() == before + 1   # y only: one launch
    h = torch.empty((7, 256), dtype=dt, device="cuda")
    want = torch.empty((7, 128), dtype=dt, device="cuda")
    capi.swiglu(x, w.detach(), want, h)
    assert torch.equal(y.view(torch.int16), want.view(torch.int16))


def test_training_step_captured_in_a_cuda_graph():
    dt, m, hid, i = torch.bfloat16, 67, 256, 192
    layer = ops.B200SwiGLULinear(hid, i, device="cuda", dtype=dt)
    x = torch.randn((m, hid), device="cuda").to(dt).requires_grad_()
    dy = torch.randn((m, i), device="cuda").to(dt)

    def step():
        x.grad = None
        layer.weight.grad = None
        layer(x).backward(dy)
        return x.grad.clone(), layer.weight.grad.clone()

    want = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    x.grad = layer.weight.grad = None
    with torch.cuda.graph(graph, stream=s):
        layer(x).backward(dy)
    x.grad.zero_()
    layer.weight.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(x.grad.view(torch.int16), want[0].view(torch.int16))
    assert torch.equal(layer.weight.grad.view(torch.int16), want[1].view(torch.int16))
