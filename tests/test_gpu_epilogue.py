"""The fused bias + activation epilogue on the H100 (libb200_epilogue.so, csrc/b200_epilogue.h).

The anchor: with a bias of -0.0 and no activation, a BiasAct<> kernel computes what the TN kernel of the same
configuration, K-mode and type computes, bit for bit (x + -0.0 == x, -0.0 included): every configuration, every K-mode
it carries, all four variants (e4m3 per tensor and rowwise), pinned through run_config, and the dispatched call. Then,
on tests/exact_domain.py's operands, every configuration and K-mode bit-exact against tests/epilogue_ref.py with a bias
and none / relu, gelu_tanh against the float64 tanh form over z in [-8, 8], guard bands, N(0,1) data against fp32
torch and against torch._addmm_activation (cuBLASLt's epilogue), the gradients, one launch per call, empty shapes,
CUDA-graph capture, and one production-scale case whose output passes 2^31 elements.
"""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import epilogue_ref as ref
import exact_domain as ed
import scale_cases as sc
from conftest import REPO
from cuda_l2_b200 import capi, ops

pytestmark = pytest.mark.gpu

WORKSPACE, CLUSTER, STREAM_K = 3, -2, capi.STREAMK_TAIL
OUT = {torch.float16: "fp16", torch.bfloat16: "bf16"}
TOL = {torch.float16: 0.005, torch.bfloat16: 0.03}           # max |err| / rms(ref) against fp32 torch
GRAD_TOL = {torch.float16: 0.01, torch.bfloat16: 0.05}
SENTINEL = {torch.float16: 0x7D5A, torch.bfloat16: 0x7FA5}   # NaN payloads no kernel produces
E4M3 = torch.float8_e4m3fn


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def randn(shape, dtype, seed):
    return torch.randn(shape, device="cuda", generator=gen(seed)).to(dtype)


def bits(x):
    return x.view(torch.int16)


def cases():
    """(config, group_m, splits, M, N, K, K-mode the plan runs) for every configuration and every K-mode its kernels
    carry, ragged in M and N (N % 8 == 0, not a multiple of BN) and K, with K % 16 == 0 for the e4m3 variants."""
    out, seen = [], set()
    for c in capi.configs():
        cid, bn, cg, cm, cn, mr = c["id"], c["bn"], c["cta_group"], c["cluster_m"], c["cluster_n"], c["m_rep"]
        stream_k = cm * cn == 1 and bn >= 64 and mr == 1
        tile_m = 128 * mr * cg * cm
        wanted = [(1, "plain", 2 * tile_m + 72, 2 * bn * cn + 40, 208 + 16 * cid)]
        if stream_k:   # 20 tiles on 132 / cg workers: stream-K over all of them
            wanted.append((STREAM_K, "stream-k", 4 * 128 * cg - 56, 5 * bn - 24, 1744 + 16 * cid))
        if stream_k and cg == 1:
            wanted.append((WORKSPACE, "split-k", 200, bn + 40, 1008 + 16 * cid))
            wanted.append((CLUSTER, "cluster-split-k", 200, bn + 40, 1024 + 16 * cid))
        for i, (splits, mode, m, n, k) in enumerate(wanted):
            while (m, n, k) in seen:
                k += 16
            seen.add((m, n, k))
            out.append((cid, 4 * ((cid + i) % 3), splits, m, n, k, mode))
    return out


CASES = cases()


def test_cases_run_their_k_mode():
    for (cid, _, splits, m, n, k, mode) in CASES:
        assert capi.schedule(cid, m, n, k, splits)["mode"] == mode, (cid, splits, m, n, k)
    assert {c[0] for c in CASES} == set(range(len(capi.configs())))
    assert len(CASES) == 46


def e4m3_scales(m, n, rowwise, seed):
    g = gen(seed)
    if rowwise:
        sa = torch.rand((m, 1), device="cuda", generator=g) + 0.5
        sb = torch.rand((1, n), device="cuda", generator=g) + 0.5
    else:
        sa = torch.rand((1,), device="cuda", generator=g) + 0.5
        sb = torch.rand((1,), device="cuda", generator=g) + 0.5
    return sa, sb


# ------------------------------------------------------------------------------------------------------------ anchor
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"cfg{c[0]}-{c[6]}")
def test_anchor_is_the_tn_kernel_bit_for_bit(case):
    cid, gm, splits, m, n, k, mode = case
    pin = dict(config_id=cid, group_m=gm, splits=splits)
    for dtype in (torch.float16, torch.bfloat16):
        a, bt = randn((m, k), dtype, m + k), randn((n, k), dtype, n + 3 * k)
        neg0 = torch.full((n,), -0.0, dtype=dtype, device="cuda")
        want = torch.full((m, n), float("nan"), dtype=dtype, device="cuda")
        capi.gemm_kmajor(a, bt, want, "fp32", **pin)
        for bias in (neg0, None):
            got = torch.full((m, n), float("nan"), dtype=dtype, device="cuda")
            capi.gemm_bias_act(a, bt, got, bias, "none", **pin)
            assert torch.equal(bits(got), bits(want)), (case, dtype, bias is None)
    for out in (torch.float16, torch.bfloat16):
        a = randn((m, k), torch.float32, m).to(E4M3)
        bt = randn((n, k), torch.float32, n).to(E4M3)
        neg0 = torch.full((n,), -0.0, dtype=out, device="cuda")
        for rowwise in (False, True):
            sa, sb = e4m3_scales(m, n, rowwise, m + n)
            want = torch.full((m, n), float("nan"), dtype=out, device="cuda")
            capi.fp8_gemm(a, bt, want, sa, sb, **pin)
            got = torch.full((m, n), float("nan"), dtype=out, device="cuda")
            capi.gemm_bias_act(a, bt, got, neg0, "none", sa, sb, **pin)
            assert torch.equal(bits(got), bits(want)), (case, out, rowwise)


@pytest.mark.parametrize("shape", [(4096, 4096, 4096), (8192, 3072, 768), (16, 4096, 4096), (200, 328, 1040),
                                   (77, 1000, 8192), (1, 8, 16)])
def test_anchor_dispatched(shape):
    m, n, k = shape
    for dtype in (torch.float16, torch.bfloat16):
        a, bt = randn((m, k), dtype, 1), randn((n, k), dtype, 2)
        want = torch.empty((m, n), dtype=dtype, device="cuda")
        capi.gemm_kmajor(a, bt, want, "fp32")
        got = torch.empty((m, n), dtype=dtype, device="cuda")
        capi.gemm_bias_act(a, bt, got, torch.full((n,), -0.0, dtype=dtype, device="cuda"), "none")
        assert torch.equal(bits(got), bits(want)), (shape, dtype)
    a, bt = randn((m, k), torch.float32, 3).to(E4M3), randn((n, k), torch.float32, 4).to(E4M3)
    for rowwise in (False, True):
        sa, sb = e4m3_scales(m, n, rowwise, 5)
        want = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
        capi.fp8_gemm(a, bt, want, sa, sb)
        got = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
        capi.gemm_bias_act(a, bt, got, torch.full((n,), -0.0, dtype=torch.bfloat16, device="cuda"), "none", sa, sb)
        assert torch.equal(bits(got), bits(want)), (shape, rowwise)


# ------------------------------------------------------------------------------------------------------ exact domain
def bias_values(n, dtype, seed, lo=-64.0, hi=64.0):
    """N bias values of ``dtype`` (as a CUDA tensor) and their fp32 values (numpy)."""
    rng = np.random.default_rng(seed)
    b = torch.from_numpy(rng.uniform(lo, hi, size=n).astype(np.float32)).to(dtype)
    return b.cuda(), b.float().numpy()


def bits_np(x):
    return bits(x).cpu().numpy().view(np.uint16)


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"cfg{c[0]}-{c[6]}")
def test_exact_domain_none_and_relu_bit_exact(case):
    cid, gm, splits, m, n, k, mode = case
    pin = dict(config_id=cid, group_m=gm, splits=splits)
    for dtype in (torch.float16, torch.bfloat16):
        kind = OUT[dtype]
        o = ed.operands16(m, n, k, kind, seed=cid + 7 * k)
        a = torch.from_numpy(o.a).to(dtype).cuda()
        bt = torch.from_numpy(o.bt).to(dtype).cuda()
        bias, bias32 = bias_values(n, dtype, cid + k)
        for act in ("none", "relu"):
            got = torch.full((m, n), float("nan"), dtype=dtype, device="cuda")
            capi.gemm_bias_act(a, bt, got, bias, act, **pin)
            want = ref.reference(o.a, o.bt, bias32, act, kind)
            assert np.array_equal(bits_np(got), want), (case, kind, act)
    a64, bt64 = ed.operands_e4m3(m, n, k, seed=cid + 11 * k)
    a, bt = torch.from_numpy(a64).to(E4M3).cuda(), torch.from_numpy(bt64).to(E4M3).cuda()
    for out, (rowwise, act) in ((torch.float16, (False, "relu")), (torch.bfloat16, (True, "none")),
                                (torch.float16, (True, "relu"))):
        kind = OUT[out]
        if rowwise:
            sa_np, sb_np = ed.e4m3_rowwise_scales(m, n, kind)
            sa, sb = torch.from_numpy(sa_np).cuda().view(m, 1), torch.from_numpy(sb_np).cuda().view(1, n)
        else:
            sa_np, sb_np = (np.float32(v) for v in ed.e4m3_tensor_scales(kind)[1])
            sa, sb = torch.tensor([sa_np], device="cuda"), torch.tensor([sb_np], device="cuda")
        bias, bias32 = bias_values(n, out, cid + 5 * k, -4.0, 4.0)
        got = torch.full((m, n), float("nan"), dtype=out, device="cuda")
        capi.gemm_bias_act(a, bt, got, bias, act, sa, sb, **pin)
        want = ref.reference(a64, bt64, bias32, act, kind, sa_np, sb_np, rowwise)
        assert np.array_equal(bits_np(got), want), (case, kind, rowwise, act)


GELU_CASES = [c for c in CASES if c[0] in (0, 1, 3, 12, 26, 29)]


@pytest.mark.parametrize("case", GELU_CASES, ids=lambda c: f"cfg{c[0]}-{c[6]}")
def test_gelu_tanh_against_the_float64_reference(case):
    """z spread over [-8, 8]: small exact sums (|s| <= 1) plus a bias drawn from [-8, 8]. Every element within one unit
    in the last place of the float64 tanh form, or, where 1 + tanh(u) has cancelled in fp32, within the fp32 form's
    absolute error (epilogue_ref.gelu_excess). The counts of elements one unit off and past one unit are printed."""
    cid, gm, splits, m, n, k, mode = case
    pin = dict(config_id=cid, group_m=gm, splits=splits)
    rng = np.random.default_rng(cid + k)
    a64 = rng.integers(-1, 2, size=(m, k)) / 8.0
    bt64 = rng.integers(-1, 2, size=(n, k)) / 8.0 * (np.arange(k) < 64)   # at most 64 products per sum: |s| <= 1
    counts = {}

    def check(got, kind, a, bt, bias32, sa=None, sb=None):
        z = ref.pre_activation(a, bt, bias32, sa, sb)
        gb = bits_np(got)
        excess = ref.gelu_excess(gb, z, kind)
        assert excess.max() <= 0, (case, kind, float(excess.max()), float(z.reshape(-1)[excess.argmax()]))
        d = ref.ulp_distance(gb, ref.round_out(ref.gelu_tanh(z), kind))
        counts[kind if sa is None else "e4m3->" + kind] = (int((d == 1).sum()), int((d > 1).sum()))

    for dtype in (torch.float16, torch.bfloat16):
        kind = OUT[dtype]
        bias, bias32 = bias_values(n, dtype, cid, -8.0, 8.0)
        got = torch.full((m, n), float("nan"), dtype=dtype, device="cuda")
        capi.gemm_bias_act(torch.from_numpy(a64).to(dtype).cuda(), torch.from_numpy(bt64).to(dtype).cuda(), got,
                           bias, "gelu_tanh", **pin)
        check(got, kind, a64, bt64, bias32)
    a8, bt8 = torch.from_numpy(a64 * 8).to(E4M3).cuda(), torch.from_numpy(bt64 * 8).to(E4M3).cuda()
    sa, sb = torch.tensor([0.125], device="cuda"), torch.tensor([0.125], device="cuda")
    bias, bias32 = bias_values(n, torch.bfloat16, cid + 1, -8.0, 8.0)
    got = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
    capi.gemm_bias_act(a8, bt8, got, bias, "gelu_tanh", sa, sb, **pin)
    check(got, "bf16", a64 * 8, bt64 * 8, bias32, np.float32(0.125), np.float32(0.125))
    print(f"\nGELU cfg {cid} {mode} {m}x{n}x{k}: (one unit off, more than one unit off) of {m * n} each: {counts}")


# ------------------------------------------------------------------------------------------------------ guard bands
@pytest.mark.parametrize("cid,splits", [(1, 1), (2, WORKSPACE), (2, CLUSTER), (0, STREAM_K), (26, 1), (13, 1)])
def test_guard_bands_and_the_bias_past_n(cid, splits):
    for dtype in (torch.float16, torch.bfloat16):
        for (m, n, k) in ((77, 72, 64), (300, 520, 208), (1000, 136, 2064)):
            a, bt = randn((m, k), dtype, m), randn((n, k), dtype, n)
            guard = 4096
            buf = torch.full((2 * guard + m * n,), SENTINEL[dtype], dtype=torch.int16, device="cuda").view(dtype)
            c = buf[guard:guard + m * n].view(m, n)
            bias_buf = torch.full((n + 64,), float("nan"), dtype=dtype, device="cuda")   # NaN past N: never read
            bias_buf[:n] = randn((n,), dtype, 7)
            for act in ("none", "relu"):   # relu would turn a NaN read from past N into +0.0; none keeps it
                buf.view(torch.int16).fill_(SENTINEL[dtype])
                capi.gemm_bias_act(a, bt, c, bias_buf[:n], act, config_id=cid, splits=splits)
                torch.cuda.synchronize()
                assert bool((bits(buf[:guard]) == SENTINEL[dtype]).all())
                assert bool((bits(buf[guard + m * n:]) == SENTINEL[dtype]).all())
                assert not bool(c.isnan().any()), (cid, splits, dtype, m, n, k, act)


# ------------------------------------------------------------------------------------------------------ N(0, 1) data
def torch_ref(x, w, bias, act):
    z = F.linear(x.float(), w.float(), None if bias is None else bias.float())
    return ops._activate(z, act)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("act", ref.ACTIVATIONS)
def test_against_fp32_torch(dtype, act):
    for (m, n, k) in ((256, 512, 1024), (2048, 128, 2048), (333, 200, 1024), (16, 4096, 4096)):
        x, w, b = randn((m, k), dtype, m), randn((n, k), dtype, n), randn((n,), dtype, k)
        want = torch_ref(x, w, b, act)
        got = ops.hgemm_bias_act(x, w, b, act)
        assert got.shape == (m, n) and got.dtype == dtype
        err = float((got.float() - want).abs().max() / want.pow(2).mean().sqrt())
        assert err <= TOL[dtype], (m, n, k, act, err)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_against_addmm_activation(dtype):
    """cuBLASLt's bias epilogues (torch._addmm_activation, F.linear): where the two libraries' plain products agree bit
    for bit, the none and relu results are at most one unit in the last place apart. cuBLASLt's GELU epilogue is its own
    evaluation, not torch's F.gelu form: measured on the H100 it lies up to 17 fp16 units from this kernel in the tail
    where 1 + tanh(u) cancels, while this kernel stays within its allowance of the float64 reference there
    (test_gelu_tanh_against_the_float64_reference). For gelu_tanh the bound is one unit plus |z| 2^-17, eight times the
    two evaluations' own absolute allowances. Counts and sizes of all differences are printed."""
    m, n, k = 2048, 3072, 768
    x, w, b = randn((m, k), dtype, 1), randn((n, k), dtype, 2), randn((n,), dtype, 3)
    ours_plain = ops.hgemm(x, w)
    agree = (bits(ours_plain) == bits(x @ w.t())).cpu().numpy()
    z = (ours_plain.double() + b.double()).cpu().numpy()
    for act in ref.ACTIVATIONS:
        if act == "none":
            theirs = F.linear(x, w, b)
        else:
            theirs = torch._addmm_activation(b, x, w.t(), use_gelu=act == "gelu_tanh")
        ours = ops.hgemm_bias_act(x, w, b, act)
        d = ref.ulp_distance(bits_np(ours), bits_np(theirs))
        ok = d <= 1
        if act == "gelu_tanh":
            gap = np.abs(ours.double().cpu().numpy() - theirs.double().cpu().numpy())
            ok |= gap <= ref.ulp_at(theirs.double().cpu().numpy(), OUT[dtype]) + 2.0 ** -17 * np.abs(z)
        print(f"\nADDMM {dtype} {act}: {int((d > 0).sum())} of {d.size} differ, max {int(d.max())} ulp; where the "
              f"products agree ({int(agree.sum())}): max {int(d[agree].max())} ulp, {int((d[agree] > 1).sum())} past one")
        assert ok[agree].all(), (act, int((~ok & agree).sum()))


# ------------------------------------------------------------------------------------------------------ gradients
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("act", ref.ACTIVATIONS)
def test_gradients_against_torch(dtype, act):
    m, n, k = 192, 256, 136
    x = randn((2, m // 2, k), dtype, 20).requires_grad_(True)
    w = randn((n, k), dtype, 21).requires_grad_(True)
    b = randn((n,), dtype, 22).requires_grad_(True)
    gy = randn((2, m // 2, n), dtype, 23)
    y = ops.linear(x, w, b, act)
    assert y.shape == (2, m // 2, n)
    before = capi.epilogue_launch_count()
    y.backward(gy)
    torch.cuda.synchronize()
    # gelu_tanh recomputes its pre-activation: one launch of the fused kernel in the backward, none otherwise
    assert capi.epilogue_launch_count() - before == (1 if act == "gelu_tanh" else 0)
    xf, wf, bf = (t.detach().float().requires_grad_(True) for t in (x, w, b))
    torch_ref(xf, wf, bf, act).backward(gy.float())
    for got, want in ((x.grad, xf.grad), (w.grad, wf.grad), (b.grad, bf.grad)):
        assert got.dtype == dtype and got.shape == want.shape
        err = float((got.float() - want).abs().max() / want.pow(2).mean().sqrt())
        assert err <= GRAD_TOL[dtype], (act, err)


def test_relu_mask_comes_from_the_output():
    x = torch.tensor([[1.0, 0.0]], dtype=torch.half, device="cuda").repeat(8, 4)
    w = torch.eye(8, dtype=torch.half, device="cuda")
    b = torch.tensor([-1.0, 1.0] * 4, dtype=torch.half, device="cuda").requires_grad_(True)
    xr = x.clone().requires_grad_(True)
    y = ops.hgemm_bias_act(xr, w, b, "relu")   # z = 0 in the even columns: no gradient there
    assert torch.equal(y, torch.tensor([[0.0, 1.0] * 4], dtype=torch.half, device="cuda").repeat(8, 1))
    y.sum().backward()
    assert torch.equal(b.grad, torch.tensor([0.0, 8.0] * 4, dtype=torch.half, device="cuda"))


# ------------------------------------------------------------------------------------------------------ launches
def test_one_launch_per_forward_and_empty_shapes():
    x, w, b = randn((100, 64), torch.half, 1), randn((72, 64), torch.half, 2), randn((72,), torch.half, 3)
    for act in ref.ACTIVATIONS:
        before = capi.epilogue_launch_count()
        ops.hgemm_bias_act(x, w, b, act)
        ops.hgemm_bias_act(x, w, None, act)
        torch.cuda.synchronize()
        assert capi.epilogue_launch_count() - before == 2
    before = capi.epilogue_launch_count()
    for dtype in (torch.float16, torch.bfloat16):
        bias = torch.tensor([-3.0, -0.5, 0.0, 0.25, 1.0, 2.5, -1.0, 7.0], dtype=dtype, device="cuda")
        assert ops.hgemm_bias_act(torch.empty((0, 16), dtype=dtype, device="cuda"),
                                  torch.empty((8, 16), dtype=dtype, device="cuda"), bias, "relu").shape == (0, 8)
        assert ops.hgemm_bias_act(torch.empty((5, 16), dtype=dtype, device="cuda"),
                                  torch.empty((0, 16), dtype=dtype, device="cuda"), None, "gelu_tanh").shape == (5, 0)
        for act in ref.ACTIVATIONS:
            a0, w0 = torch.empty((5, 0), dtype=dtype, device="cuda"), torch.empty((8, 0), dtype=dtype, device="cuda")
            got = ops.hgemm_bias_act(a0, w0, bias, act)
            want = ops._activate(bias.float(), act).to(dtype).expand(5, 8)
            assert torch.equal(got, want), (dtype, act)
            assert torch.equal(ops.hgemm_bias_act(a0, w0, None, act), torch.zeros((5, 8), dtype=dtype, device="cuda"))
            e = torch.empty((5, 0), device="cuda").to(E4M3)
            got = ops.fp8_gemm_bias_act(e, torch.empty((8, 0), device="cuda").to(E4M3), torch.ones(1, device="cuda"),
                                        torch.ones(1, device="cuda"), bias, act, dtype)
            assert torch.equal(got, want), (dtype, act)
    torch.cuda.synchronize()
    assert capi.epilogue_launch_count() == before


GRAPH = textwrap.dedent("""
    import sys
    import torch
    sys.path.insert(0, {repo!r})
    from cuda_l2_b200 import capi
    torch.cuda.set_device(0)
    m, n, k = 256, 512, 4096     # 2 x 2 tiles of configuration 1: B200_HGEMM_FORCE asks for workspace split-K
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn((m, k), device="cuda", generator=g).half()
    bt = torch.randn((n, k), device="cuda", generator=g).half()
    bias = torch.randn((n,), device="cuda", generator=g).half()
    def eager(splits):
        c = torch.empty((m, n), dtype=torch.half, device="cuda")
        capi.gemm_bias_act(a, bt, c, bias, "gelu_tanh", config_id=1, splits=splits)
        return c
    ok = []
    c = torch.full((m, n), float("nan"), dtype=torch.half, device="cuda")
    capi.gemm_bias_act(a[:128], bt[:64], c[:128, :64].contiguous(), bias[:64], "relu", config_id=1)  # loads the library
    torch.cuda.synchronize()
    for prewarm in (False, True):
        s = torch.cuda.Stream()
        if prewarm:
            capi.epilogue_prewarm(s.cuda_stream)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            before = capi.epilogue_launch_count()
            with torch.cuda.graph(graph, stream=s):
                capi.gemm_bias_act(a, bt, c, bias, "gelu_tanh", stream=s.cuda_stream)
            ok.append(capi.epilogue_launch_count() - before == 1)
        # without prewarm the capture finds no scratch and runs the undivided schedule; with it, split-K
        for step in range(2):
            a.copy_(torch.randn((m, k), device="cuda", generator=g).half())   # new inputs before each replay
            bias.copy_(torch.randn((n,), device="cuda", generator=g).half())
            c.fill_(float("nan"))
            graph.replay()
            torch.cuda.synchronize()
            ok.append(bool(torch.equal(c.view(torch.int16), eager(3 if prewarm else 1).view(torch.int16))))
    capi.epilogue_release()
    print("RESULT", ok)
""")


def test_cuda_graph_capture_with_and_without_prewarm():
    env = dict(os.environ, B200_HGEMM_FORCE="1,0,3")
    env.pop("B200_HGEMM_TABLE", None)
    r = subprocess.run([sys.executable, "-c", GRAPH.format(repo=str(REPO))], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    assert r.stdout.split("RESULT", 1)[1].strip() == str([True] * 6), r.stdout


# ------------------------------------------------------------------------------------------------------ e4m3
@pytest.mark.parametrize("out", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("rowwise", [False, True])
def test_fp8_operator_against_fp8_gemm_plus_bias(out, rowwise):
    """fp8_gemm's output s' (s rounded once) plus the bias in fp32, activated and rounded again, against the fused
    result, which rounds once: they differ by the two extra roundings at most, |d| <= 2^-p (|s'| + |b|) * 2 with p the
    output's significand bits, plus the smallest subnormal (a unit in the last place of the result alone means nothing
    where s' and b nearly cancel). The activations' slopes are at most 1.13."""
    m, n, k = 1000, 1032, 2048
    x, w = randn((m, k), torch.float32, 1), randn((n, k), torch.float32, 2)
    if rowwise:
        xq, sx = ops.quantize_e4m3_rowwise(x)
        wq, sw = ops.quantize_e4m3_rowwise(w)
        sa, sb = sx, sw.view(1, n)
    else:
        xq, sa = ops.quantize_e4m3(x)
        wq, sb = ops.quantize_e4m3(w)
    b = randn((n,), out, 3)
    p, tiny = (11, 2.0 ** -24) if out == torch.float16 else (8, 2.0 ** -133)
    plain = ops.fp8_gemm(xq, wq, sa, sb, out).double()
    for act in ref.ACTIVATIONS:
        got = ops.fp8_gemm_bias_act(xq, wq, sa, sb, b, act, out).double()
        want = ops._activate(plain + b.double(), act)
        bound = 2.0 ** -p * (plain.abs() + b.double().abs()) * 2 * 1.13 + tiny
        excess = float(((got - want).abs() - bound).max())
        assert excess <= 0, (out, rowwise, act, excess)


# ------------------------------------------------------------------------------------------------------ scale
def test_output_past_2_31_with_bias_and_relu():
    """sc.CASES['tn'] (C [24600, 131080], 3.2e9 elements) with an integer bias and relu, fp16, dispatched, bit-compared
    band by band against relu(float64 product + bias), rounded once; guard bands intact."""
    case = sc.CASES["tn"]
    need = case.memory_bytes() + 4 * case.tensor("c").shape[1]
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    assert free >= need, f"the case needs {need} bytes of device memory, {free} are free"
    d = sc.allocate(case, torch.float16)
    dom = sc.DOMAINS["fp16"]
    sc.fill_ints_(d["a"], dom["a"], sc.generator(60))
    sc.fill_ints_(d["bt"], dom["b"], sc.generator(61))
    n = d["c"].shape[1]
    bias = torch.empty((n,), dtype=torch.float16, device="cuda").random_(-2000, 2001, generator=sc.generator(62))
    assert d["c"].numel() > 2 ** 31
    capi.gemm_bias_act(d["a"], d["bt"], d["c"], bias, "relu")
    bias64 = bias.to(torch.float64)
    msg = sc.first_mismatch(d["c"], lambda r0, r1: torch.relu(sc.matmul64(d["a"][r0:r1], d["bt"].t()) + bias64),
                            what="fp16 bias relu")
    assert msg is None, msg
    assert sc.guards_intact(d["c:buf"])
    del d
    torch.cuda.empty_cache()
