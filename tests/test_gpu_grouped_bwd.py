"""The backward of the grouped GEMM on the H100 (libb200_grouped_bwd.so).

The anchors, bit for bit on N(0,1) data with ragged groups (empty, one row, 37 rows, 100 rows, longer than a k-block
run of a tile) and NaN / Inf in the rows past the last group:
- the K-grouped weight gradient dW[g] = dY[s:e]^T X[s:e] against the 2-D K-major kernel (the same configuration and
  group_m, splits = 1) on the group's rows transposed and zero-padded to a multiple of 8, for every configuration with
  a row-major B kernel and both types, with all SMs and with a two-worker CTA cap; an empty group gives +0.0;
- the grouped row-major B input gradient dX[s:e] = dY[s:e] W[g] against the grouped forward kernel (same
  configuration) on W transposed to K-major.
Then: exactness on 0/1 operands, clamped offsets, guard bands around C and T == 0, offsets written by a torch kernel
just before the launch and changed between CUDA-graph replays, one launch per call, the operators against fp32
torch.matmul per group and torch._grouped_mm (bf16), and grouped_linear's gradients against an fp32 reference.
"""
import numpy as np
import pytest
import torch

from cuda_l2_b200 import capi, ops

pytestmark = pytest.mark.gpu

NN_CONFIGS = [c for c in range(31) if c not in (12, 13, 14)]   # BN = 32 has no row-major B kernel
VARIANTS = {0: torch.float16, 2: torch.bfloat16}
SIZES = [0, 1, 37, 100, 0, 530, 64, 1]
FP16_TOL, BF16_TOL = 0.005, 0.03
SENTINEL = 0x7BCD


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def randn(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, device="cuda", generator=g).to(dtype)


def sentinel(shape, dtype):
    return torch.full(shape, SENTINEL, dtype=torch.int16, device="cuda").view(dtype)


def bits(x):
    return x.view(torch.int16)


def clamped_groups(offs, t):
    out, s = [], 0
    for o in offs:
        e = min(max(o, s), t)
        out.append((s, e))
        s = e
    return out


def offs_tensor(offs):
    return torch.tensor(offs, dtype=torch.int32, device="cuda")


def cta_count(config_id):
    c = capi.configs()[config_id]
    return c["cta_group"] * c["cluster_m"] * c["cluster_n"]


def poisoned(t, cols, dtype, seed, last_end):
    x = randn((t, cols), dtype, seed)
    x[last_end:] = float("nan")
    x[last_end::2] = float("inf")
    return x


def wgrad_reference(dy, x, offs, config_id, group_m=0):
    """The 2-D K-major kernel on each group's rows, transposed and zero-padded along T to a multiple of 8."""
    t, m = dy.shape
    n = x.shape[1]
    want = torch.zeros((len(offs), m, n), dtype=dy.dtype, device="cuda")
    for g, (s, e) in enumerate(clamped_groups(offs, t)):
        if e > s:
            pad = -(-(e - s) // 8) * 8
            a = torch.zeros((m, pad), dtype=dy.dtype, device="cuda")
            bt = torch.zeros((n, pad), dtype=dy.dtype, device="cuda")
            a[:, :e - s] = dy[s:e].t()
            bt[:, :e - s] = x[s:e].t()
            capi.gemm_kmajor(a, bt, want[g], "fp32", config_id=config_id, group_m=group_m, splits=1)
    return want


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("config_id", NN_CONFIGS)
def test_wgrad_is_bit_identical_to_the_2d_kernel(config_id, variant):
    dtype = VARIANTS[variant]
    offs = [int(v) for v in np.cumsum(SIZES)]
    t, m, n = offs[-1] + 29, 136, 264
    dy, x = poisoned(t, m, dtype, config_id, offs[-1]), poisoned(t, n, dtype, config_id + 50, offs[-1])
    want = wgrad_reference(dy, x, offs, config_id)
    o = offs_tensor(offs)
    for max_ctas in (0, 2 * cta_count(config_id)):
        c = sentinel((len(offs), m, n), dtype)
        capi.gemm_grouped_wgrad(dy, x, c, o, config_id=config_id, max_ctas=max_ctas)
        torch.cuda.synchronize()
        assert torch.equal(bits(c), bits(want)), (config_id, variant, max_ctas)
        for g, (s, e) in enumerate(clamped_groups(offs, t)):
            if e == s:
                assert not bits(c[g]).any(), (config_id, g)   # +0.0, not -0.0


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("config_id", NN_CONFIGS)
def test_grouped_nn_is_bit_identical_to_the_grouped_forward(config_id, variant):
    dtype = VARIANTS[variant]
    offs = [int(v) for v in np.cumsum(SIZES)]
    t, nm, km = offs[-1] + 29, 136, 264                          # dY [T, N_model], W [G, N_model, K_model]
    dy = poisoned(t, nm, dtype, config_id + 7, offs[-1])
    w = randn((len(offs), nm, km), dtype, config_id + 8)
    want = sentinel((t, km), dtype)
    o = offs_tensor(offs)
    capi.gemm_grouped(dy, w.transpose(1, 2).contiguous(), want, o, "fp32", config_id=config_id)
    for max_ctas in (0, 2 * cta_count(config_id)):
        c = sentinel((t, km), dtype)
        capi.gemm_grouped_nn(dy, w, c, o, config_id=config_id, max_ctas=max_ctas)
        torch.cuda.synchronize()
        assert torch.equal(bits(c), bits(want)), (config_id, variant, max_ctas)


def test_exact_on_zero_one_operands():
    rng = np.random.default_rng(3)
    sizes, m, n = [70, 0, 1, 129, 200, 64], 136, 200
    offs = [int(v) for v in np.cumsum(sizes)]
    t = offs[-1]
    a = rng.integers(0, 2, size=(t, m)).astype(np.float32)
    b = rng.integers(0, 2, size=(t, n)).astype(np.float32)
    w = rng.integers(0, 2, size=(len(sizes), m, n)).astype(np.float32)
    for dtype in VARIANTS.values():
        c = sentinel((len(sizes), m, n), dtype)
        capi.gemm_grouped_wgrad(torch.from_numpy(a).cuda().to(dtype), torch.from_numpy(b).cuda().to(dtype), c,
                                offs_tensor(offs))
        dx = sentinel((t, n), dtype)
        capi.gemm_grouped_nn(torch.from_numpy(a).cuda().to(dtype), torch.from_numpy(w).cuda().to(dtype), dx,
                             offs_tensor(offs))
        torch.cuda.synchronize()
        for g, (s, e) in enumerate(clamped_groups(offs, t)):
            assert np.array_equal(c[g].float().cpu().numpy(), a[s:e].T @ b[s:e]), (dtype, g)   # sums <= 200: exact
            assert np.array_equal(dx[s:e].float().cpu().numpy(), a[s:e] @ w[g]), (dtype, g)


def test_clamped_offsets_guard_bands_and_empty_reduction():
    dtype, m, n, t = torch.bfloat16, 64, 72, 300
    dy, x = randn((t, m), dtype, 1), randn((t, n), dtype, 2)
    for offs in ([100, 50, 400, -3], [-5, 10, 10, 290], [t + 100, 0, 5, 7]):   # decreasing, negative, past T
        guard = 4096
        buf = sentinel((2 * guard + len(offs) * m * n,), dtype)
        c = buf[guard:guard + len(offs) * m * n].view(len(offs), m, n)
        capi.gemm_grouped_wgrad(dy, x, c, offs_tensor(offs), config_id=2)
        torch.cuda.synchronize()
        assert torch.equal(bits(c), bits(wgrad_reference(dy, x, offs, 2))), offs
        assert (bits(buf[:guard]) == SENTINEL).all() and (bits(buf[-guard:]) == SENTINEL).all(), offs
    # T == 0: every matrix is zero, and no kernel runs
    c = sentinel((3, m, n), dtype)
    before = capi.grouped_bwd_launch_count()
    capi.gemm_grouped_wgrad(dy[:0], x[:0], c, offs_tensor([0, 0, 0]))
    torch.cuda.synchronize()
    assert capi.grouped_bwd_launch_count() == before
    assert not bits(c).any()
    assert ops.hgemm_grouped_nn(dy[:0], randn((3, m, n), dtype, 3), offs_tensor([0, 0, 0])).shape == (0, n)
    assert ops.hgemm_grouped_wgrad(dy[:0], x[:0], offs_tensor([0, 0, 0])).count_nonzero() == 0
    torch.cuda.synchronize()
    assert capi.grouped_bwd_launch_count() == before


def test_offsets_written_by_a_kernel_just_before_the_launch():
    dtype, m, n = torch.float16, 128, 192
    sizes = torch.tensor([3, 0, 200, 77, 1], dtype=torch.int32, device="cuda")
    t = 300
    dy, x = randn((t, m), dtype, 4), randn((t, n), dtype, 5)
    torch.cuda.synchronize()
    torch.cuda._sleep(20_000_000)                   # the cumsum below still waits when the launch is issued
    o = torch.cumsum(sizes, 0, dtype=torch.int32)
    c = torch.empty((5, m, n), dtype=dtype, device="cuda")
    capi.gemm_grouped_wgrad(dy, x, c, o, config_id=1, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(bits(c), bits(wgrad_reference(dy, x, o.tolist(), 1)))


def test_cuda_graph_replays_read_the_current_offsets():
    dtype, m, n, t = torch.bfloat16, 128, 128, 400
    dy, x = randn((t, m), dtype, 6), randn((t, n), dtype, 7)
    o = offs_tensor([100, 100, 350])
    c = torch.empty((3, m, n), dtype=dtype, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        capi.gemm_grouped_wgrad(dy, x, c, o, config_id=4, stream=s.cuda_stream)   # warm: attributes, maps
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        capi.gemm_grouped_wgrad(dy, x, c, o, config_id=4, stream=s.cuda_stream)
    for offs in ([10, 200, 400], [0, 0, 1], [390, 395, 400]):
        o.copy_(offs_tensor(offs))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(c), bits(wgrad_reference(dy, x, offs, 4))), offs


def test_one_launch_per_call():
    dtype = torch.bfloat16
    dy, x, w = randn((500, 128), dtype, 8), randn((500, 256), dtype, 9), randn((4, 128, 256), dtype, 10)
    o = offs_tensor([100, 250, 250, 480])
    before = capi.grouped_bwd_launch_count()
    ops.hgemm_grouped_wgrad(dy, x, o)
    ops.hgemm_grouped_nn(dy, w, o)
    capi.gemm_grouped_wgrad(dy, x, torch.empty((4, 128, 256), dtype=dtype, device="cuda"), o, config_id=0)
    torch.cuda.synchronize()
    assert capi.grouped_bwd_launch_count() - before == 3


@pytest.mark.parametrize("dtype,tol", [(torch.float16, FP16_TOL), (torch.bfloat16, BF16_TOL)])
def test_operators_against_torch(dtype, tol):
    sizes, m, n = [300, 0, 1000, 17, 600], 512, 768
    offs = [int(v) for v in np.cumsum(sizes)]
    t = offs[-1]
    dy, x, w = randn((t, m), dtype, 11), randn((t, n), dtype, 12), randn((len(sizes), m, n), dtype, 13)
    o = offs_tensor(offs)
    dw = ops.hgemm_grouped_wgrad(dy, x, o)
    dx = ops.hgemm_grouped_nn(dy, w, o)
    for g, (s, e) in enumerate(clamped_groups(offs, t)):
        ref = dy[s:e].float().t() @ x[s:e].float()
        scale = max(ref.pow(2).mean().sqrt().item(), 1.0)
        assert (dw[g].float() - ref).abs().max().item() / scale <= tol, g
        if e > s:
            ref = dy[s:e].float() @ w[g].float()
            assert (dx[s:e].float() - ref).abs().max().item() / ref.pow(2).mean().sqrt().item() <= tol, g
    if dtype == torch.bfloat16:
        tw = torch._grouped_mm(dy.t(), x, offs=o)
        assert (dw.float() - tw.float()).abs().max().item() / tw.float().pow(2).mean().sqrt().item() <= tol
        tx = torch._grouped_mm(dy, w, offs=o)
        assert (dx.float() - tx.float()).abs().max().item() / tx.float().pow(2).mean().sqrt().item() <= tol


@pytest.mark.parametrize("dtype,tol", [(torch.float16, FP16_TOL), (torch.bfloat16, BF16_TOL)])
def test_grouped_linear_gradients(dtype, tol):
    sizes, k, n = [200, 0, 333, 64], 256, 384
    offs = [int(v) for v in np.cumsum(sizes)]
    t = offs[-1] + 40                                 # 40 rows past the last group
    o = offs_tensor(offs)
    x = randn((t, k), dtype, 14).requires_grad_()
    layer = ops.B200GroupedLinear.from_weights(randn((len(sizes), n, k), dtype, 15))
    y = layer(x, o)
    assert torch.equal(bits(y[:offs[-1]]), bits(ops.hgemm_grouped(x.detach(), layer.weight.detach(), o)[:offs[-1]]))
    gy = randn((t, n), dtype, 16)
    gy[offs[-1]:] = float("nan")                      # rows past the last end must not leak
    y.backward(gy)
    assert not bits(x.grad[offs[-1]:]).any()          # +0.0
    xf, wf, gf = x.detach().float(), layer.weight.detach().float(), gy.float()
    for g, (s, e) in enumerate(clamped_groups(offs, t)):
        ref_w = gf[s:e].t() @ xf[s:e]
        assert torch.isfinite(layer.weight.grad[g].float()).all()
        assert (layer.weight.grad[g].float() - ref_w).abs().max().item() / max(ref_w.pow(2).mean().sqrt().item(), 1) <= tol
        if e > s:
            ref_x = gf[s:e] @ wf[g]
            assert (x.grad[s:e].float() - ref_x).abs().max().item() / ref_x.pow(2).mean().sqrt().item() <= tol


def test_hgemm_grouped_stays_inference_only():
    x = randn((64, 64), torch.float16, 17).requires_grad_()
    y = ops.hgemm_grouped(x, randn((1, 64, 64), torch.float16, 18), offs_tensor([64]))
    with pytest.raises(capi.B200HgemmError, match="inference only"):
        y.sum().backward()
