"""Row-major B (NN) fp16 / bf16 GEMM on the H100 (libb200_nn.so, reached through the drop-in entry points of
libb200_hgemm.so with B_rowmajor and no B_kmajor).

The anchor: an NN launch runs the TN kernel's schedule, K-block partition, wgmma sequence and epilogues unchanged; only
B's shared-memory layout (MN-major atom columns instead of K-major rows) and its load differ. So on N(0,1) data the NN
result must be BIT-IDENTICAL to b200_hgemm_run_config / b200_bgemm_run_config with the same configuration (after the
BN = 32 sibling map), group_m and splits on b.t().contiguous(): for every configuration, every K-mode it carries and all
three types. The dispatched NN call takes the TN choice, so one subprocess points B200_HGEMM_TABLE at a table that maps
one distinct ragged shape to each (configuration, group_m, splits). Then: exactness against the oracle on the
reference's 0/1 domain, ragged shapes, guard bands, CUDA-graph capture with and without prewarm, the operator and its
gradients against fp32 torch.matmul (test_gpu_batched.py's tolerances), hgemm's backward against the parent formula
(TN on transposed copies) bit for bit, and one launch per call.
"""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import oracle
from conftest import REPO
from cuda_l2_b200 import capi, ops

pytestmark = pytest.mark.gpu

TYPES = {"fp16": (torch.float16, "fp32"), "fp16acc16": (torch.float16, "fp16"), "bf16": (torch.bfloat16, "fp32")}
FP16_TOL, BF16_TOL, FP16_ACC16_TOL = 0.005, 0.03, 0.1
GRAD_TOL = {torch.float16: 0.01, torch.bfloat16: 0.05}
SENTINEL = 0x7BCD
WORKSPACE, CLUSTER, STREAM_K = 3, -2, capi.STREAMK_TAIL


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def randn(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, device="cuda", generator=g).to(dtype)


def bits(x):
    return x.view(torch.int16)


def nn_sibling(cfgs, cid):
    """The NN stand-in of a configuration (hgemm_configs.cuh nn::sibling)."""
    c = cfgs[cid]
    if c["bn"] % 64 == 0:
        return cid
    cands = [d for d in cfgs if d["bn"] == 64 and d["cta_group"] == c["cta_group"] and d["cluster_m"] == c["cluster_m"]
             and d["m_rep"] == c["m_rep"] and d["cluster_n"] <= c["cluster_n"]]
    return max(cands, key=lambda d: d["cluster_n"])["id"]


def table_cases():
    """(config, group_m, splits, M, N, K, K-mode the plan runs) for every configuration and every K-mode its kernels
    carry, each with a shape of its own (ragged in M, N and K) that the configuration's pair / cluster fits."""
    cfgs = capi.configs()
    cases, seen = [], set()
    for c in cfgs:
        cid, bn, cg, cm, cn, mr = c["id"], c["bn"], c["cta_group"], c["cluster_m"], c["cluster_n"], c["m_rep"]
        stream_k = cm * cn == 1 and bn >= 64 and mr == 1
        tile_m = 128 * mr * cg * cm
        wanted = [(1, "plain", 2 * tile_m + 72, 2 * bn * cn + 40, 200 + 8 * cid)]
        if bn == 32:   # the dispatcher's split request is dropped with the sibling map (a BN = 32 kernel runs plain)
            wanted.append((-4, "plain", tile_m + 24, bn * cn * 3 + 8, 1000 + 8 * cid))
        if stream_k:
            workers = 132 // cg
            wanted.append((STREAM_K, "stream-k", 10 * 128 * cg - 56, 14 * bn - 24, 4264 + 8 * cid))
            assert (10 * 14) % workers
        if stream_k and cg == 1:
            wanted.append((WORKSPACE, "split-k", 200, bn + 40, 1000 + 8 * cid))
            wanted.append((CLUSTER, "cluster-split-k", 200, bn + 40, 1008 + 8 * cid))
        for i, (splits, mode, m, n, k) in enumerate(wanted):
            while (m, n, k) in seen:
                k += 8
            seen.add((m, n, k))
            cases.append((cid, 4 * ((cid + i) % 3), splits, m, n, k, mode))
    return cases


SWEEP = textwrap.dedent("""
    import json, sys
    import torch
    sys.path.insert(0, {repo!r})
    from cuda_l2_b200 import capi
    cases, siblings, types = json.loads(sys.argv[1])
    torch.cuda.set_device(0)
    out = []
    for (cid, gm, splits, m, n, k, mode) in cases:
        sib = siblings[str(cid)]
        for name, (dt, acc) in types.items():
            dtype = getattr(torch, dt)
            g = torch.Generator(device="cuda").manual_seed(m * 7 + n * 3 + k)
            a = torch.randn((m, k), device="cuda", generator=g).to(dtype)
            b = torch.randn((k, n), device="cuda", generator=g).to(dtype)
            nn = torch.full((m, n), float("nan"), dtype=dtype, device="cuda")
            before = capi.launch_count()
            capi.gemm_rowmajor(a, b, nn, acc)
            launches = capi.launch_count() - before
            bt = b.t().contiguous()
            tn = torch.full((m, n), float("nan"), dtype=dtype, device="cuda")
            capi.gemm_kmajor(a, bt, tn, acc, config_id=sib, group_m=gm, splits=splits if sib == cid else 1)
            same = bool(torch.equal(nn.view(torch.int16), tn.view(torch.int16)))
            if sib != cid:   # and what the TN call of the dispatched configuration itself computes
                tn0 = torch.full((m, n), float("nan"), dtype=dtype, device="cuda")
                capi.gemm_kmajor(a, bt, tn0, acc, config_id=cid, group_m=gm, splits=splits)
                same = same and bool(torch.equal(nn.view(torch.int16), tn0.view(torch.int16)))
            ref = a.float() @ b.float()
            err = float((nn.float() - ref).abs().max() / ref.pow(2).mean().sqrt())
            out.append([cid, gm, splits, m, n, k, mode, name, same, launches, err])
    torch.cuda.synchronize()
    print("RESULT " + json.dumps(out))
""")


def test_every_configuration_and_k_mode_is_bit_identical_to_tn(tmp_path):
    cases = table_cases()
    cfgs = capi.configs()
    for (cid, gm, splits, m, n, k, mode) in cases:   # the plan really runs the K-mode each case is for
        sched = capi.schedule(nn_sibling(cfgs, cid), m, n, k, splits if cfgs[cid]["bn"] % 64 == 0 else 1)
        assert sched["mode"] == mode, (cid, splits, m, n, k, sched["mode"])
    table = tmp_path / "nn_table.txt"
    table.write_text("".join(f"{m} {n} {k} {cid} {gm} {sp} {cid} {gm} {sp}\n" for (cid, gm, sp, m, n, k, _) in cases))
    siblings = {str(c["id"]): nn_sibling(cfgs, c["id"]) for c in cfgs}
    types = {name: (str(dt).split(".")[-1], acc) for name, (dt, acc) in TYPES.items()}
    env = dict(os.environ, B200_HGEMM_TABLE=str(table))
    env.pop("B200_HGEMM_FORCE", None)
    r = subprocess.run([sys.executable, "-c", SWEEP.format(repo=str(REPO)), json.dumps([cases, siblings, types])],
                       env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    rows = json.loads(r.stdout.split("RESULT ", 1)[1])
    assert len(rows) == 3 * len(cases)
    assert {row[0] for row in rows} == set(range(len(cfgs)))
    for (cid, gm, splits, m, n, k, mode, name, same, launches, err) in rows:
        assert same, f"config {cid} {mode} (splits {splits}, group_m {gm}) {name} at {m}x{n}x{k}: NN != TN"
        assert launches == 1, (cid, name, launches)
        if name != "fp16acc16":   # fp16 accumulation over the long K of the stream-K shapes has no fixed bound here
            assert err <= (BF16_TOL if name == "bf16" else FP16_TOL), (cid, mode, name, err)


@pytest.mark.parametrize("acc", ["fp32", "fp16"])
def test_golden_zero_one_vectors_bit_exact(zero_one_cases, acc):
    """The reference's 0/1 domain: the fixtures hold B [K,N] row-major, read here as it is."""
    for c in zero_one_cases:
        if c["k"] % 8 or c["n"] % 8:
            continue
        a = torch.from_numpy(c["a"]).cuda()
        b = torch.from_numpy(np.ascontiguousarray(c["b"])).cuda()
        out = torch.empty((c["m"], c["n"]), dtype=torch.half, device="cuda")
        capi.gemm_rowmajor(a, b, out, acc)
        got = out.cpu().numpy()
        truth = c["truth"]
        keep = np.abs(truth.astype(np.float32)) <= 2047
        assert np.array_equal(got[keep], truth[keep]), (acc, c["m"], c["n"], c["k"])
        if acc == "fp32":
            assert np.array_equal(got.view(np.uint16), truth.view(np.uint16))


def test_ragged_shapes_against_the_oracle():
    """0/1 operands (exact with fp32 accumulation) on ragged M, N and K, against the C oracle."""
    for (m, n, k) in [(1, 8, 8), (200, 328, 72), (129, 136, 520), (77, 1000, 1032), (513, 72, 4104)]:
        a = oracle.fill_zero_one((m, k), 2, seed=m + k)
        b = oracle.fill_zero_one((k, n), 2, seed=n + 3 * k)
        want = oracle.hgemm_f32acc(a, np.ascontiguousarray(b.T), fast=True)
        out = torch.full((m, n), float("nan"), dtype=torch.half, device="cuda")
        capi.gemm_rowmajor(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), out, "fp32")
        assert np.array_equal(out.cpu().numpy().view(np.uint16), want.view(np.uint16)), (m, n, k)


def test_guard_bands_around_c():
    for name, (dtype, acc) in TYPES.items():
        for (m, n, k) in [(77, 72, 64), (300, 520, 200), (1000, 136, 2056)]:
            a, b = randn((m, k), dtype, m), randn((k, n), dtype, n)
            guard = 4096
            buf = torch.full((2 * guard + m * n,), SENTINEL, dtype=torch.int16, device="cuda").view(dtype)
            c = buf[guard:guard + m * n].view(m, n)
            capi.gemm_rowmajor(a, b, c, acc)
            torch.cuda.synchronize()
            assert bool((bits(buf[:guard]) == SENTINEL).all()) and bool((bits(buf[guard + m * n:]) == SENTINEL).all())
            assert not bool((bits(c) == SENTINEL).any()), (name, m, n, k)


GRAPH = textwrap.dedent("""
    import sys
    import torch
    sys.path.insert(0, {repo!r})
    from cuda_l2_b200 import capi
    torch.cuda.set_device(0)
    m, n, k = 256, 512, 4096     # 2 x 2 tiles of configuration 1: B200_HGEMM_FORCE asks for workspace split-K
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn((m, k), device="cuda", generator=g).half()
    b = torch.randn((k, n), device="cuda", generator=g).half()
    bt = b.t().contiguous()
    def tn(splits):
        c = torch.empty((m, n), dtype=torch.half, device="cuda")
        capi.gemm_kmajor(a, bt, c, "fp32", config_id=1, splits=splits)
        return c
    ok = []
    c = torch.full((m, n), float("nan"), dtype=torch.half, device="cuda")
    capi.gemm_rowmajor(a, b, c, "fp32")   # loads the library and its kernels, on another stream than the captures
    torch.cuda.synchronize()
    for prewarm in (False, True):
        s = torch.cuda.Stream()
        if prewarm:
            capi.prewarm(s.cuda_stream)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            before = capi.launch_count()
            with torch.cuda.graph(graph, stream=s):
                capi.gemm_rowmajor(a, b, c, "fp32", stream=s.cuda_stream)
            ok.append(capi.launch_count() - before == 1)   # the capture's one launch
        c.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        # without prewarm the capture finds no scratch and runs the undivided schedule; with it, split-K
        want = tn(3 if prewarm else 1)
        ok.append(bool(torch.equal(c.view(torch.int16), want.view(torch.int16))))
        a.mul_(-1)                 # a replay reads the operands' current contents
        graph.replay()
        torch.cuda.synchronize()
        ok.append(bool(torch.equal(c.view(torch.int16), tn(3 if prewarm else 1).view(torch.int16))))
    print("RESULT", ok)
""")


def test_cuda_graph_capture_with_and_without_prewarm():
    env = dict(os.environ, B200_HGEMM_FORCE="1,0,3")
    env.pop("B200_HGEMM_TABLE", None)
    r = subprocess.run([sys.executable, "-c", GRAPH.format(repo=str(REPO))], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    assert r.stdout.split("RESULT", 1)[1].strip() == str([True] * 6), r.stdout


@pytest.mark.parametrize("dtype,acc,tol", [(torch.float16, "fp32", FP16_TOL), (torch.float16, "fp16", FP16_ACC16_TOL),
                                           (torch.bfloat16, "fp32", BF16_TOL)])
def test_operator_against_torch_matmul(dtype, acc, tol):
    for (m, n, k) in ((256, 512, 1024), (2048, 128, 2048), (333, 200, 1024), (64, 4096, 64)):
        a, b = randn((m, k), dtype, m), randn((k, n), dtype, n)
        ref = a.float() @ b.float()
        got = ops.hgemm_nn(a, b, acc)
        assert got.shape == (m, n) and got.dtype == dtype
        err = float((got.float() - ref).abs().max() / ref.pow(2).mean().sqrt())
        assert err <= tol, (m, n, k, err)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_gradients_against_torch_matmul(dtype):
    m, n, k = 192, 256, 136
    a = randn((m, k), dtype, 20).requires_grad_(True)
    b = randn((k, n), dtype, 21).requires_grad_(True)
    w = randn((m, n), torch.float32, 22)
    (ops.hgemm_nn(a, b).float() * w).sum().backward()
    a32, b32 = a.detach().float().requires_grad_(True), b.detach().float().requires_grad_(True)
    ((a32 @ b32) * w).sum().backward()
    tol = GRAD_TOL[dtype]
    for got, ref in ((a.grad, a32.grad), (b.grad, b32.grad)):
        assert got.dtype == dtype and got.shape == ref.shape
        assert float((got.float() - ref).abs().max() / ref.pow(2).mean().sqrt()) <= tol


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_hgemm_backward_is_bit_identical_to_the_transposed_copy_formula(dtype):
    """hgemm's backward reads b_kmajor and a in place through the NN kernels; it must compute exactly what the TN
    kernels compute on the transposed copies (the formula it replaces), including where the dispatcher picks a BN = 32
    configuration (small N) and a split or stream-K schedule."""
    for i, (m, n, k) in enumerate([(64, 64, 64), (200, 328, 72), (256, 1024, 512), (2048, 4096, 1024),
                                   (4096, 64, 4096), (128, 11008, 4096)]):
        a = randn((m, k), dtype, 30 + i).requires_grad_(True)
        bt = randn((n, k), dtype, 40 + i).requires_grad_(True)
        g = randn((m, n), dtype, 50 + i)
        ops.hgemm(a, bt).backward(g)
        want_a = ops.hgemm(g, bt.detach().t().contiguous())
        want_b = ops.hgemm(g.t().contiguous(), a.detach().t().contiguous())
        assert torch.equal(bits(a.grad), bits(want_a)), (m, n, k)
        assert torch.equal(bits(bt.grad), bits(want_b)), (m, n, k)


def test_one_launch_per_call():
    a, b = randn((300, 264), torch.float16, 1), randn((264, 520), torch.float16, 2)
    for acc in ("fp32", "fp16"):
        before = capi.launch_count()
        ops.hgemm_nn(a, b, acc)
        torch.cuda.synchronize()
        assert capi.launch_count() - before == 1
    a, b = a.bfloat16(), b.bfloat16()
    before = capi.launch_count()
    ops.hgemm_nn(a, b)
    torch.cuda.synchronize()
    assert capi.launch_count() - before == 1
