"""Grouped fp16 / bf16 SwiGLU GEMM over contiguous row groups on the H100 (libb200_grouped_swiglu.so).

The anchor: a gated grouped launch runs Grouped<>'s main loop and tile list unchanged, so h must be BIT-IDENTICAL to
libb200_grouped.so with the same configuration, and y to torch's `F.silu(g) * u` on that h; each group's y must also be
the 2-D fused call (libb200_swiglu.so) on that group's rows with the same configuration. Group sizes: empty groups,
one-row groups, ends inside a 16-row box, groups longer than a 512-row pair block, and a last end before T. Output
buffers start as NaN canaries, and rows at or past the last end must keep them. Then: clamped and device-written
offsets, CUDA-graph replays with changing offsets, the dispatched call at the benchmark shapes, the backward over the
groups' rows only, and the layer's gradients against the grouped kernels on the reference dh, bit for bit.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cuda_l2_b200 import capi, ops

pytestmark = pytest.mark.gpu

DTYPES = {0: torch.float16, 2: torch.bfloat16}
TOL = {torch.float16: 0.005, torch.bfloat16: 0.03}   # max |y - ref| / rms(ref), as the grouped tests allow
# empty, one row, an end inside a 16-row box, longer than a 512-row pair block; the last end stays 23 rows before T
SIZES = [0, 1, 37, 300, 0, 17, 530, 1, 128, 0, 1100, 15]
T_PAD = 23


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def randn(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dtype)


def nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def bits(x):
    return x.view(torch.int16)


def split_h(h):
    """(g, u) [T, I] of h [T, 2I] in the interleaved layout"""
    t, n = h.shape
    g, u = h.view(t, n // 128, 2, 64).unbind(2)
    return g.reshape(t, n // 2), u.reshape(t, n // 2)


def swiglu_ref(h):
    g, u = split_h(h)
    return F.silu(g) * u


def problem(dtype, g_sizes, i, k, seed):
    ends = [int(v) for v in np.cumsum(g_sizes)]
    t = ends[-1] + T_PAD
    x = randn((t, k), dtype, seed, 0.5)
    w = randn((len(g_sizes), 2 * i, k), dtype, seed + 1, 1 / 8)
    return x, w, torch.tensor(ends, dtype=torch.int32, device="cuda"), ends, t


def test_every_configuration_against_the_grouped_kernel_and_torch():
    """For every gated configuration and both dtypes: h is libb200_grouped.so's output with the same configuration, y is
    torch's F.silu(g) * u on that h and each group's 2-D fused call, all bit for bit; without h, y is the same and the h
    buffer untouched; rows at or past the last end keep their NaN canaries."""
    i, k = 192, 136
    cfgs = [c["id"] for c in capi.configs() if c["bn"] in (128, 256)]
    assert len(cfgs) == 18
    for variant, dtype in DTYPES.items():
        x, w, offs, ends, t = problem(dtype, SIZES, i, k, 10 + variant)
        last = ends[-1]
        for cid in cfgs:
            h, y, y2, h_ref = nan((t, 2 * i), dtype), nan((t, i), dtype), nan((t, i), dtype), nan((t, 2 * i), dtype)
            h_untouched = nan((t, 2 * i), dtype)
            before = capi.grouped_swiglu_launch_count()
            capi.grouped_swiglu(x, w, offs, y, h, config_id=cid)
            capi.grouped_swiglu(x, w, offs, y2, None, config_id=cid)
            assert capi.grouped_swiglu_launch_count() - before == 2
            capi.gemm_grouped(x, w, h_ref, offs, config_id=cid)
            torch.cuda.synchronize()
            assert torch.equal(bits(h[:last]), bits(h_ref[:last])), (cid, dtype)
            assert torch.equal(bits(y[:last]), bits(swiglu_ref(h[:last]))), (cid, dtype)
            assert torch.equal(bits(y2), bits(y)), (cid, dtype)
            assert torch.isnan(h[last:]).all() and torch.isnan(y[last:]).all(), (cid, dtype)
            assert torch.isnan(h_untouched).all()
            for grp, (s, e) in enumerate(zip([0] + ends[:-1], ends)):
                if e > s:
                    y_2d = torch.empty((e - s, i), dtype=dtype, device="cuda")
                    capi.swiglu(x[s:e].contiguous(), w[grp], y_2d, config_id=cid)
                    torch.cuda.synchronize()
                    assert torch.equal(bits(y[s:e]), bits(y_2d)), (cid, dtype, s, e)


@pytest.mark.parametrize("offs_list", [[300, 100, 900, 900], [-5, 40, 2000, 3000], [0, 0, 0, 0],
                                       [1500, 1500, 1500, 1500]])
def test_clamped_offsets_behave_as_the_grouped_kernel(offs_list):
    """Decreasing, negative and too-large offsets clamp as hgemm_grouped's do: h matches it row for row below the last
    clamped end, y matches torch on that h, and nothing at or past that end is written."""
    dtype, i, k, t = torch.bfloat16, 128, 64, 1000
    x = randn((t, k), dtype, 3, 0.5)
    w = randn((4, 2 * i, k), dtype, 4, 1 / 8)
    offs = torch.tensor(offs_list, dtype=torch.int32, device="cuda")
    last = min(max(0, *offs_list), t)
    h, y, h_ref = nan((t, 2 * i), dtype), nan((t, i), dtype), nan((t, 2 * i), dtype)
    capi.grouped_swiglu(x, w, offs, y, h, config_id=1)
    capi.gemm_grouped(x, w, h_ref, offs, config_id=1)
    torch.cuda.synchronize()
    assert torch.equal(bits(h), bits(h_ref))   # NaN canaries included: the same rows are written
    assert torch.equal(bits(y[:last]), bits(swiglu_ref(h[:last])))
    assert torch.isnan(y[last:]).all()


def test_offsets_written_just_before_the_launch_and_graph_replays():
    dtype, i, k = torch.float16, 128, 128
    sizes = [40, 0, 200, 7]
    x, w, _, _, t = problem(dtype, sizes, i, k, 21)
    offs = torch.zeros(len(sizes), dtype=torch.int32, device="cuda")
    y = nan((t, i), dtype)
    src = torch.tensor([int(v) for v in np.cumsum(sizes)], dtype=torch.int32, device="cuda")
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        offs.copy_(src * 1)   # a kernel writes the offsets right before the launch on the same stream
        capi.grouped_swiglu(x, w, offs, y, stream=stream.cuda_stream, config_id=1)
    stream.synchronize()
    want = nan((t, i), dtype)
    capi.grouped_swiglu(x, w, src, want, config_id=1)
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(want))
    # a captured launch reads the offsets of each replay
    graph = torch.cuda.CUDAGraph()
    out = nan((t, i), dtype)
    with torch.cuda.graph(graph):
        capi.grouped_swiglu(x, w, offs, out, stream=torch.cuda.current_stream().cuda_stream, config_id=1)
    for ends in ([10, 20, 30, 200], [0, 150, 150, 247], [247, 247, 247, 247]):
        offs.copy_(torch.tensor(ends, dtype=torch.int32))
        out.fill_(float("nan"))
        graph.replay()
        ref = nan((t, i), dtype)
        capi.grouped_swiglu(x, w, offs, ref, config_id=1)
        torch.cuda.synchronize()
        assert torch.equal(bits(out), bits(ref)), ends


@pytest.mark.parametrize("g,t,i,k", [(8, 4096, 14336, 4096), (64, 16384, 1408, 2048)])
def test_dispatched_call_at_the_benchmark_shapes(g, t, i, k):
    """The dispatched call is the sibling configuration's bit for bit (h against libb200_grouped.so), and y is within
    the grouped tests' 16-bit tolerance of a float64 reference on uneven groups with an empty one, each element's error
    measured against |ref| + rms(ref)."""
    dtype = torch.bfloat16
    rng = np.random.default_rng(g + t)
    sizes = rng.multinomial(t - 64, rng.dirichlet(np.ones(g) * 0.5))
    sizes[1] = 0
    ends = [int(v) for v in np.cumsum(sizes)]
    offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
    x = randn((t, k), dtype, 5, 0.5)
    w = randn((g, 2 * i, k), dtype, 6, k ** -0.5)
    cid, gm = capi.grouped_swiglu_select(2, g, t, i, k)
    y, h = nan((t, i), dtype), nan((t, 2 * i), dtype)
    capi.grouped_swiglu(x, w, offs, y, h)
    h_ref, y_pin = nan((t, 2 * i), dtype), nan((t, i), dtype)
    capi.gemm_grouped(x, w, h_ref, offs, config_id=cid, group_m=gm)
    capi.grouped_swiglu(x, w, offs, y_pin, config_id=cid, group_m=gm)
    torch.cuda.synchronize()
    last = ends[-1]
    assert torch.equal(bits(h[:last]), bits(h_ref[:last])) and torch.equal(bits(y[:last]), bits(y_pin[:last]))
    # float64 reference on a sample of rows of every non-empty group
    for e_idx, (s, e) in enumerate(zip([0] + ends[:-1], ends)):
        if e == s:
            continue
        rows = torch.arange(s, e, max(1, (e - s) // 16), device="cuda")
        hr = x[rows].double() @ w[e_idx].double().t()
        ref = swiglu_ref(hr)
        # per element against |ref| + rms(ref): y is a product of two rounded factors, heavy-tailed where g is large
        err = ((y[rows].double() - ref).abs() / (ref.abs() + ref.pow(2).mean().sqrt())).max()
        assert err <= TOL[dtype], (e_idx, float(err))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_backward_is_torch_autograd_bit_for_bit_for_every_gate_value(dtype):
    """dh = torch's autograd through F.silu(g) * u for all 65536 16-bit gate values, with rows past the last end set to
    NaN in dy and h (they change nothing) and dh's rows there left as they were."""
    i = 256
    allv = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(dtype)
    rows = allv.numel() // i
    sizes = [rows // 3, 0, rows - rows // 3]
    t = rows + 5
    g_val = torch.empty((t, i), dtype=dtype, device="cuda")
    g_val[:rows] = allv.view(rows, i)
    u_val = randn((t, i), dtype, 7)
    dy = randn((t, i), dtype, 8)
    h = torch.empty((t, 2 * i), dtype=dtype, device="cuda")
    hv = h.view(t, i // 64, 2, 64)
    hv[:, :, 0] = g_val.view(t, i // 64, 64)
    hv[:, :, 1] = u_val.view(t, i // 64, 64)
    h[rows:] = float("nan")
    dy[rows:] = float("nan")
    offs = torch.tensor([int(v) for v in np.cumsum(sizes)], dtype=torch.int32, device="cuda")
    dh = torch.full((t, 2 * i), 1.5, dtype=dtype, device="cuda")
    before = capi.grouped_swiglu_launch_count()
    capi.grouped_swiglu_backward(dy, h, dh, offs)
    assert capi.grouped_swiglu_launch_count() - before == 1
    gg, uu = (v.detach().clone().requires_grad_() for v in split_h(h[:rows]))
    (F.silu(gg) * uu).backward(dy[:rows])
    torch.cuda.synchronize()
    dg, du = split_h(dh[:rows])
    for got, want in ((dg, gg.grad), (du, uu.grad)):
        nans = torch.isnan(want)
        assert torch.equal(torch.isnan(got), nans)
        assert torch.equal(bits(got[~nans]), bits(want[~nans]))
    assert (dh[rows:] == 1.5).all()
    # T == 0 launches nothing
    before = capi.grouped_swiglu_launch_count()
    e = torch.empty((0, i), dtype=dtype, device="cuda")
    capi.grouped_swiglu_backward(e, torch.empty((0, 2 * i), dtype=dtype, device="cuda"),
                                 torch.empty((0, 2 * i), dtype=dtype, device="cuda"), offs)
    assert capi.grouped_swiglu_launch_count() == before


def _layer_problem(dtype, seed):
    sizes = [37, 0, 130, 1, 90]
    g, i, k = len(sizes), 128, 64
    ends = [int(v) for v in np.cumsum(sizes)]
    t = ends[-1] + 9
    x = randn((t, k), dtype, seed, 0.5)
    wg, wu = randn((g, i, k), dtype, seed + 1, 1 / 8), randn((g, i, k), dtype, seed + 2, 1 / 8)
    offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
    return x, wg, wu, offs, ends, t


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_layer_gradients_are_the_grouped_kernels_on_the_reference_dh(dtype):
    x, wg, wu, offs, ends, t = _layer_problem(dtype, 30)
    last = ends[-1]
    layer = ops.B200GroupedSwiGLULinear.from_weights(wg, wu)
    xr = x.clone().requires_grad_()
    y = layer(xr, offs)
    dy = randn(y.shape, dtype, 33)
    dy[last:] = float("nan")   # never read
    y.backward(dy)
    torch.cuda.synchronize()
    # the reference: h from the grouped kernel, dh from torch's autograd, then the grouped backward kernels
    h = nan((t, 2 * 128), dtype)
    capi.gemm_grouped(x, layer.weight.detach(), h, offs)
    gg, uu = (v.detach().clone().requires_grad_() for v in split_h(h[:last]))
    (F.silu(gg) * uu).backward(dy[:last])
    dh = torch.zeros((t, 2 * 128), dtype=dtype, device="cuda")
    dhv = dh[:last].view(last, 2, 2, 64)
    dhv[:, :, 0] = gg.grad.view(last, 2, 64)
    dhv[:, :, 1] = uu.grad.view(last, 2, 64)
    dx_ref = ops._grouped_input_grad(dh, x, layer.weight.detach(), offs, "fp32")
    dw_ref = ops.hgemm_grouped_wgrad(dh, x, offs)
    assert torch.equal(bits(xr.grad), bits(dx_ref)) and not xr.grad[last:].any()
    assert torch.equal(bits(layer.weight.grad), bits(dw_ref))
    # y against the per-expert torch composition of the gate and up weights
    for e_idx, (s, e) in enumerate(zip([0] + ends[:-1], ends)):
        if e > s:
            hg, hu = (torch.empty((e - s, 128), dtype=dtype, device="cuda") for _ in range(2))
            capi.gemm_kmajor(x[s:e].contiguous(), wg[e_idx].contiguous(), hg)
            capi.gemm_kmajor(x[s:e].contiguous(), wu[e_idx].contiguous(), hu)
            assert torch.equal(bits(y[s:e].detach()), bits(F.silu(hg) * hu)), e_idx


def test_one_forward_and_one_dh_launch_per_call_and_a_captured_training_step():
    dtype = torch.bfloat16
    x, wg, wu, offs, ends, t = _layer_problem(dtype, 40)
    layer = ops.B200GroupedSwiGLULinear.from_weights(wg, wu)
    xr = x.clone().requires_grad_()
    before = capi.grouped_swiglu_launch_count()
    y = layer(xr, offs)
    assert capi.grouped_swiglu_launch_count() - before == 1
    y.backward(torch.ones_like(y))
    assert capi.grouped_swiglu_launch_count() - before == 2
    with torch.no_grad():
        layer(x, offs)
    assert capi.grouped_swiglu_launch_count() - before == 3
    del y   # its autograd graph, and the weight's gradient node on this stream with it
    # a training step of a fresh layer captured in a CUDA graph, replayed with changing offsets, against eager steps
    layer = ops.B200GroupedSwiGLULinear.from_weights(wg, wu)
    static_x = x.clone().requires_grad_()
    static_offs = offs.clone()
    static_dy = randn((t, 128), dtype, 41)
    layer.weight.grad = None
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):   # warm up on a side stream
            layer.weight.grad = None
            static_x.grad = None
            layer(static_x, static_offs).backward(static_dy)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    layer.weight.grad = None
    static_x.grad = None
    with torch.cuda.graph(graph):
        static_y = layer(static_x, static_offs)
        static_y.backward(static_dy)
    for new_ends in ([10, 10, 100, 101, 200], [0, 50, 60, 61, 258], ends):
        static_offs.copy_(torch.tensor(new_ends, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        eager_x = x.clone().requires_grad_()
        w2 = layer.weight.detach().clone().requires_grad_()
        e_offs = torch.tensor(new_ends, dtype=torch.int32, device="cuda")
        ey = ops.grouped_swiglu_linear(eager_x, w2, e_offs)
        ey.backward(static_dy)
        torch.cuda.synchronize()
        last = new_ends[-1]
        assert torch.equal(bits(static_y[:last]), bits(ey[:last].detach())), new_ends
        assert torch.equal(bits(static_x.grad), bits(eager_x.grad)), new_ends
        assert torch.equal(bits(layer.weight.grad), bits(w2.grad)), new_ends
