"""The DISPATCHED row-major B (NN), bias + activation and grouped-backward calls, bit-exact at the tuned grid, at the
off-grid samples and at MoE-shaped samples of dispatch_sweep.py, against the exact product (float64 on the GPU).

Each leg calls what users call, with no configuration or split pinned: ``capi.gemm_rowmajor`` (B [K, N] row-major: the
TN choice mapped through select_rowmajor, BN = 32 configurations to their BN = 64 sibling), ``capi.gemm_bias_act``
(bias + none / relu / gelu_tanh, the activation drawn per shape; fp16, bf16, e4m3 per tensor and rowwise),
``capi.gemm_grouped_nn`` and ``capi.gemm_grouped_wgrad`` (grouped_linear's backward). As in test_gpu_dispatch_sweep.py,
C sits in a guarded buffer pre-filled with a NaN sentinel, and a leg collects every failing shape with the choice, the
planned K-mode and stream-K tiles and the first bad element, and asserts once.

The bias legs keep the exact domain: z = fp32(s) + fp32(bias) is one IEEE fp32 addition on the device, s the exact
(scaled) product; none and relu must match bit for bit, gelu_tanh stays within epilogue_ref.gelu_excess's allowance of
the float64 tanh form. A few rows per shape are recomputed with epilogue_ref in numpy.

The heuristic never reaches the BN = 32 cluster configurations 13 and 14; a subprocess points B200_HGEMM_TABLE at
entries naming them, where their NN sibling (8: four CTAs of BN = 64 along N) spans more columns than N has.
test_dispatch_sweep_late_cpu.py checks without a GPU that these lists reach every K-mode, configuration and tier.
"""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import dispatch_sweep as ds
from conftest import REPO
from cuda_l2_b200 import capi
from test_gpu_dispatch_sweep import SENTINEL, first_bad, guarded, guards_intact

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def _rows_cols(m, n, probe_rows, seed):
    return ds.sample_rows(m, probe_rows.tolist(), seed), ds.sample_cols(n, seed)


# ------------------------------------------------------------------------------------------------- NN
def run_nn(leg: str, m: int, n: int, k: int):
    """The dispatched NN call of ``leg`` on (M, N, K): None, or a failure report."""
    spec = ds.NN_LEGS[leg]
    seed = ds.shape_seed(m, n, k)
    out = spec["out"]
    ops = ds.operands16(torch, m, n, k, spec["operand"], seed, acc16=spec["acc"] == "fp16")
    b = ops.bt.t().contiguous()                         # [K, N] row-major
    buf, c = guarded(m, n, out)
    capi.gemm_rowmajor(ops.a, b, c, spec["acc"])
    del b
    got = c.view(torch.int16)
    errs = [] if guards_intact(buf) else ["guard band written"]
    total, first = 0, None
    rows, cols = _rows_cols(m, n, ops.probe_rows, seed)
    want_rows = {}
    for lo, hi, want in ds.reference_blocks(torch, ops, out):
        cnt, fb = first_bad(got[lo:hi], want)
        if cnt and first is None:
            first = (fb[0] + lo,) + fb[1:]
        total += cnt
        for r in rows:
            if lo <= r < hi:
                want_rows[r] = want[r - lo, cols].cpu().numpy().view(np.uint16)
    if total:
        errs.append(f"{total} mismatches, first (row, col, got, want) {first}")
    if not np.array_equal(np.stack([want_rows[r] for r in rows]), ds.numpy_rows(torch, ops, rows, cols, out)):
        errs.append(f"device reference differs from numpy at rows {rows}")
    if not errs:
        return None
    cfg, gm, sp, tn = ds.nn_choice(leg, m, n, k)
    mode, sk = ds.plan(leg, cfg, m, n, k, sp)
    return (f"{(m, n, k)}: TN cfg {tn} -> NN cfg {cfg} group_m {gm} splits {sp} -> {mode} sk_tiles {sk}: "
            + "; ".join(errs))


@pytest.mark.parametrize("leg,shapes", [(leg, lst) for leg in ds.NN_LEGS for lst in ds.LATE_LEG_LISTS[leg]])
def test_dispatched_nn_call_is_exact(leg, shapes):
    failures = []
    for m, n, k in (ds.grid_shapes() if shapes == "grid" else ds.offgrid_shapes(leg)):
        r = run_nn(leg, m, n, k)
        if r:
            failures.append(r)
    torch.cuda.synchronize()
    assert not failures, f"{leg} {shapes}: {len(failures)} shapes fail:\n" + "\n".join(failures[:40])


# ------------------------------------------------------------------------------------------------- bias + activation
def run_epi(leg: str, m: int, n: int, k: int, act: str | None = None):
    """The dispatched bias + activation call of ``leg`` on (M, N, K) with activation ``act`` (default: the leg's draw
    for the shape): None, or a failure report."""
    spec = ds.EPI_LEGS[leg]
    seed = ds.shape_seed(m, n, k)
    out = spec["out"]
    act = act or ds.epi_activation(leg, m, n, k)
    scales = None
    if spec["operand"] == "e4m3":
        ops = ds.operands_e4m3(torch, m, n, k, seed)
        sa_t, sb_t, sa, sb = ds.e4m3_scales(torch, spec["scales"], m, n, k, out, seed)
        scales = (sa, sb)
    else:
        ops = ds.operands16(torch, m, n, k, spec["operand"], seed)
        sa_t = sb_t = None
    bias = ds.epi_bias(torch, leg, ops, scales, n, k, seed)
    buf, c = guarded(m, n, out)
    capi.gemm_bias_act(ops.a, ops.bt, c, bias, act, sa_t, sb_t)
    got = c.view(torch.int16)
    errs = [] if guards_intact(buf) else ["guard band written"]
    total, first = 0, None
    rows, cols = _rows_cols(m, n, ops.probe_rows, seed)
    z_rows, want_rows = {}, {}
    for lo, hi, z in ds.epilogue_blocks(torch, ops, bias, scales, spec["scales"]):
        g = got[lo:hi]
        if act == "gelu_tanh":
            bad = ~ds.gelu_ok(torch, g, z, out)
            cnt = int(bad.sum())
            if cnt and first is None:
                r, col = (int(x) for x in bad.nonzero()[0])
                first = (r + lo, col, hex(int(g[r, col]) & 0xFFFF), f"z {float(z[r, col])!r}")
        else:
            want = ds.activated_bits(torch, z, act, out)
            cnt, fb = first_bad(g, want)
            if cnt and first is None:
                first = (fb[0] + lo,) + fb[1:]
        total += cnt
        for r in rows:
            if lo <= r < hi:
                z_rows[r] = z[r - lo, cols].cpu().numpy()
                if act != "gelu_tanh":
                    want_rows[r] = want[r - lo, cols].cpu().numpy().view(np.uint16)
    if total:
        errs.append(f"{total} mismatches, first (row, col, got, want) {first}")
    host_z, host_bits = ds.epilogue_numpy_rows(torch, ops, rows, cols, bias, act, out, scales, spec["scales"])
    if not np.array_equal(np.stack([z_rows[r] for r in rows]).view(np.uint32), host_z.view(np.uint32)) or (
            host_bits is not None and not np.array_equal(np.stack([want_rows[r] for r in rows]), host_bits)):
        errs.append(f"device reference differs from epilogue_ref at rows {rows}")   # the reference itself is wrong
    if not errs:
        return None
    cfg, gm, sp = ds.epi_choice(leg, m, n, k)
    mode, sk = ds.plan(leg, cfg, m, n, k, sp)
    return f"{(m, n, k)} {act}: cfg {cfg} group_m {gm} splits {sp} -> {mode} sk_tiles {sk}: " + "; ".join(errs)


@pytest.mark.parametrize("leg,shapes", [(leg, lst) for leg in ds.EPI_LEGS for lst in ds.LATE_LEG_LISTS[leg]])
def test_dispatched_bias_act_call_is_exact(leg, shapes):
    failures = []
    for m, n, k in (ds.grid_shapes() if shapes == "grid" else ds.offgrid_shapes(leg)):
        r = run_epi(leg, m, n, k)
        if r:
            failures.append(r)
    torch.cuda.synchronize()
    assert not failures, f"{leg} {shapes}: {len(failures)} shapes fail:\n" + "\n".join(failures[:40])


# ------------------------------------------------------------------------------------------------- grouped backward
def _offs(case):
    return torch.tensor(case["offs"], dtype=torch.int32, device="cuda")


def run_grouped_nn(kind: str, case: dict):
    """dX = dY @ W[g] per group: a [T, d_out] by b [G, d_out, d_in] row-major."""
    g, t, n, k, offs = case["g"], case["t"], case["d_in"], case["d_out"], case["offs"]
    a, b = ds.grouped_nn_operands(torch, t, g, n, k, kind, ds.shape_seed(g, t, n, k))
    buf, c = guarded(t, n, kind)
    capi.gemm_grouped_nn(a, b, c, _offs(case))
    got = c.view(torch.int16)
    errs = [] if guards_intact(buf) else ["guard band written"]
    start = 0
    for i, end in enumerate(offs):
        if end > start:
            cnt, fb = first_bad(got[start:end], ds.grouped_nn_reference(torch, a, b, start, end, i, kind))
            if cnt:
                errs.append(f"group {i} (rows {start}:{end}): {cnt} mismatches, first {fb}")
        start = max(start, end)
    if not bool((got[offs[-1]:] == SENTINEL).all()):
        errs.append(f"rows from the last end {offs[-1]} written")
    if not errs:
        return None
    cfg, gm = capi.grouped_nn_select(ds.GROUPED_BWD_VARIANTS[kind], g, t, n, k)
    return f"grouped nn {(g, t, n, k)}: cfg {cfg} group_m {gm}: " + "; ".join(errs[:5])


def run_wgrad(kind: str, case: dict):
    """dW[g] = dY[s:e]^T X[s:e] per group: a [T, d_out], b [T, d_in], c [G, d_out, d_in]; an empty group +0.0."""
    g, t, m, n, offs = case["g"], case["t"], case["d_out"], case["d_in"], case["offs"]
    a, b = ds.wgrad_operands(torch, t, m, n, kind, ds.shape_seed(g, t, m, n, 1))
    buf, c = guarded(m, n, kind, (g,))
    capi.gemm_grouped_wgrad(a, b, c, _offs(case))
    got = c.view(torch.int16)
    errs = [] if guards_intact(buf) else ["guard band written"]
    start = 0
    for i, end in enumerate(offs):
        end = max(start, end)
        if end > start:
            cnt, fb = first_bad(got[i], ds.wgrad_reference(torch, a, b, start, end, kind))
        else:
            cnt, fb = first_bad(got[i], torch.zeros((m, n), dtype=torch.int16, device="cuda"))
        if cnt:
            errs.append(f"group {i} (rows {start}:{end}): {cnt} mismatches, first {fb}")
        start = end
    if not errs:
        return None
    cfg, gm = capi.grouped_wgrad_select(ds.GROUPED_BWD_VARIANTS[kind], g, t, m, n)
    return f"grouped wgrad {(g, t, m, n)}: cfg {cfg} group_m {gm}: " + "; ".join(errs[:5])


@pytest.mark.parametrize("kind", list(ds.GROUPED_BWD_VARIANTS))
def test_dispatched_grouped_backward_calls_are_exact(kind):
    failures = []
    for case in ds.grouped_bwd_cases():
        for run in ((run_grouped_nn, run_wgrad) if case["t"] else (run_wgrad,)):
            r = run(kind, case)
            if r:
                failures.append(f"{r} offs {case['offs'][:8]}...")
    torch.cuda.synchronize()
    assert not failures, f"{kind}: {len(failures)} problems fail:\n" + "\n".join(failures[:40])


# ------------------------------------------------------------------------------------------------- BN = 32 clusters
# (table config, M, N, K, group_m, splits): configuration 13 (BN = 32, cluster_n = 4) at N <= 192, where its NN sibling
# 8 (BN = 64, cluster_n = 4) has fewer N tiles than CTAs in its cluster; configuration 14 (cluster_n = 8), mapped to
# the same sibling with half its cluster, ragged N included. A split code in the entry is dropped with the map.
BN32_ENTRIES = [
    (13, 77, 104, 1040, 0, 1), (13, 200, 112, 64, 4, -4), (13, 1, 136, 4096, 0, 1), (13, 1000, 136, 200, 8, 100),
    (13, 640, 168, 2056, 0, -2), (13, 3000, 192, 520, 4, 1), (13, 129, 184, 8192, 0, 101), (13, 256, 120, 1000, 0, 1),
    (14, 100, 232, 512, 0, 1), (14, 200, 256, 1040, 4, -4), (14, 1000, 264, 72, 0, 1), (14, 33, 392, 4096, 8, 100),
    (14, 513, 520, 200, 0, 1), (14, 2048, 1000, 1024, 4, -8),
]

BN32_SWEEP = textwrap.dedent("""
    import json, sys
    sys.path[:0] = [{repo!r}, {tests!r}]
    import torch
    torch.cuda.set_device(0)
    import dispatch_sweep as ds
    import test_gpu_dispatch_sweep_late as late
    from cuda_l2_b200 import capi
    out = []
    for cfg, m, n, k, gm, sp in json.loads(sys.argv[1]):
        chosen = [list(capi.select(acc, m, n, k)) for acc in ("fp32", "fp16")]
        mapped = list(ds.nn_choice("nn_fp16", m, n, k)[:3])
        grouped = list(capi.grouped_nn_select(0, 1, m, n, k))
        fails = [late.run_nn(leg, m, n, k) for leg in ds.NN_LEGS]
        fails += [late.run_epi(leg, m, n, k, act) for leg in ("epi_fp16", "epi_bf16") for act in ds.ACTIVATIONS]
        out.append([cfg, m, n, k, chosen, mapped, grouped, [f for f in fails if f]])
    torch.cuda.synchronize()
    print("RESULT " + json.dumps(out))
""")


def test_bn32_cluster_entries_of_a_runtime_table(tmp_path):
    cfgs = capi.configs()
    for cfg, m, n, k, gm, sp in BN32_ENTRIES:
        assert ds.usable(cfgs[cfg], m, n) and ds.nn_sibling(cfgs, cfg) == 8, (cfg, m, n)
    assert any(not ds.usable(cfgs[8], m, n) for cfg, m, n, *_ in BN32_ENTRIES if cfg == 13)
    table = tmp_path / "bn32_table.txt"
    table.write_text("".join(f"{m} {n} {k} {c} {gm} {sp} {c} {gm} {sp}\n" for c, m, n, k, gm, sp in BN32_ENTRIES))
    env = dict(os.environ, B200_HGEMM_TABLE=str(table))
    env.pop("B200_HGEMM_FORCE", None)
    r = subprocess.run([sys.executable, "-c", BN32_SWEEP.format(repo=str(REPO), tests=str(REPO / "tests")),
                        json.dumps(BN32_ENTRIES)], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"the sweep process died (status {r.returncode}):\n{r.stderr[-4000:]}"
    rows = json.loads(r.stdout.split("RESULT ", 1)[1])
    assert len(rows) == len(BN32_ENTRIES)
    failures = []
    for (cfg, m, n, k, chosen, mapped, grouped, fails), (_, _, _, _, gm, sp) in zip(rows, BN32_ENTRIES):
        sp = sp or 1
        assert chosen == [[cfg, gm, sp]] * 2, (cfg, m, n, k, chosen)     # the runtime entry decides
        assert mapped == [8, gm, 1] and grouped == [8, gm], (cfg, m, n, k, mapped, grouped)
        failures += [f"table cfg {cfg}: {f}" for f in fails]
    assert not failures, f"{len(failures)} calls fail:\n" + "\n".join(failures[:40])
