"""The dispatch sweep without a GPU (its results are test_gpu_dispatch_sweep.py's):

* the torch generator and reference of dispatch_sweep.py, run on the CPU at small sizes, meet exact_domain's bounds,
  plant every rounding target, and give exactly exact_domain's and the FP8 references' bits;
* the sweep is not vacuous: over each leg's shapes the dispatched choices and their plans cover every K-mode, every
  configuration the table names, the L2-hint branch of the launcher and every tier of the dispatcher;
* the selectors are total: every ``*_select`` entry point on extreme in-range shapes returns a valid choice, and the
  dispatched batched and grouped calls refuse shapes past the tile bound before any device call (run in a subprocess, so
  that a trap in the dispatcher is a failure and not the end of the test session).
"""
import json
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest
import torch

import dispatch_sweep as ds
import exact_domain as ed
from conftest import REPO
from cuda_l2_b200 import capi
from fp8_block_ref import fp8gemm_f32acc_block
from fp8_rowwise_ref import fp8gemm_f32acc_rowwise
from oracle import fp8 as fp8_oracle

SMALL = ((45, 120, 256), (64, 72, 1000), (13, 200, 48))


def _np(x: torch.Tensor) -> np.ndarray:
    return x.to(torch.float32).numpy().astype(np.float64)


def _ref_bits(ops, out, scales=None, granularity=None) -> np.ndarray:
    blocks = list(ds.reference_blocks(torch, ops, out, scales, granularity, rows_per_block=16))
    return np.concatenate([b.numpy().view(np.uint16) for _, _, b in blocks])


@pytest.mark.parametrize("m,n,k", SMALL)
@pytest.mark.parametrize("variant", ["fp16", "bf16", "fp16acc16"])
def test_torch_operands_and_reference_match_exact_domain(m, n, k, variant):
    kind = "bf16" if variant == "bf16" else "fp16"
    acc16 = variant == "fp16acc16"
    ops = ds.operands16(torch, m, n, k, kind, seed=ds.shape_seed(m, n, k), acc16=acc16, device="cpu")
    r, c = ops.row_exp.numpy(), ops.col_exp.numpy()
    probe = ops.probe_rows.numpy()
    targets = ed.rounding_targets(kind)
    ref_ops = ed.Operands(_np(ops.a), _np(ops.bt), r, c, probe, [targets[j % len(targets)] for j in range(n)])
    assert ref_ops.sum_bound() < (ed.FP16_ACC_SUM_BOUND if acc16 else ed.EXACT_SUM_BOUND)
    if not acc16:
        # probe rows times column n: +-target[n] * 2^(r + c), every target planted
        units = np.exp2(r[probe][:, None] + c[None, :])
        planted = np.abs(ref_ops.exact()[probe]) / units
        assert np.array_equal(planted, np.broadcast_to(np.array(ref_ops.targets, float), planted.shape))
        if n >= len(targets):
            assert set(targets) <= set(planted[0].astype(np.int64).tolist())
    with np.errstate(over="ignore"):
        want = ed.reference16(ref_ops, kind)
    assert np.array_equal(_ref_bits(ops, kind), want)
    rows, cols = ds.sample_rows(m, probe, 1), ds.sample_cols(n, 1, limit=50)
    assert np.array_equal(ds.numpy_rows(torch, ops, rows, cols, kind), want[np.ix_(rows, cols)])


@pytest.mark.parametrize("m,n,k", [(45, 136, 256), (13, 264, 1024)])
@pytest.mark.parametrize("granularity", ["tensor", "rowwise", "block"])
@pytest.mark.parametrize("out", ["fp16", "bf16"])
def test_torch_e4m3_operands_and_scales_match_the_fp8_references(m, n, k, granularity, out):
    ops = ds.operands_e4m3(torch, m, n, k, seed=ds.shape_seed(m, n, k), device="cpu")
    ca, cb = ops.a.view(torch.uint8).numpy(), ops.bt.view(torch.uint8).numpy()
    a, bt = _np(ops.a), _np(ops.bt)
    assert (np.abs(a) @ np.abs(bt).T).max() <= ed.E4M3_SUM_BOUND
    for seed in (0, 1):
        sa_t, sb_t, sa, sb = ds.e4m3_scales(torch, granularity, m, n, k, out, seed, device="cpu")
        with np.errstate(over="ignore"):
            if granularity == "tensor":
                want = fp8_oracle.fp8gemm_f32acc(ca, cb, float(sa), float(sb), out == "bf16")
            elif granularity == "rowwise":
                want = fp8gemm_f32acc_rowwise(ca, cb, sa.astype(np.float32), sb.astype(np.float32), out == "bf16")
            else:
                want = fp8gemm_f32acc_block(ca, cb, sa.astype(np.float32), sb.astype(np.float32), out == "bf16")
        assert np.array_equal(_ref_bits(ops, out, (sa, sb), granularity), want)
        rows, cols = ds.sample_rows(m, ops.probe_rows.numpy(), 2), ds.sample_cols(n, 2, limit=64)
        assert np.array_equal(ds.numpy_rows(torch, ops, rows, cols, out, (sa, sb), granularity), want[np.ix_(rows, cols)])


def test_offgrid_samples_follow_the_shape_rules():
    for leg, spec in ds.LEGS.items():
        shapes = ds.offgrid_shapes(leg)
        assert 250 <= len(shapes) <= 400, (leg, len(shapes))
        assert not set(shapes) & set(ds.grid_shapes())
        for m, n, k in shapes:
            assert m >= 1 and n % 8 == 0 and k % spec["k_align"] == 0 and k >= 16, (leg, m, n, k)
            assert 2 * m * n * k <= ds.OFFGRID_MAX_FLOP
        ms = {s[0] for s in shapes}
        assert set(range(1, 17)) <= ms and any(m % 2 and m > 16 for m in ms)
        assert any(n % 16 for _, n, _ in shapes) and any(k % 64 for _, _, k in shapes)


# ------------------------------------------------------------------------------------------------- coverage
def _legal_splits(sp: int, block: bool) -> bool:
    if block:
        return sp in (1, -2, -4, -8)
    return sp in (1, -2, -4, -8, 100, 101) or 2 <= sp <= 127


@pytest.mark.parametrize("leg", list(ds.LEGS))
def test_sweep_covers_every_k_mode_configuration_tier_and_l2_hint(leg, built_libs):
    spec = ds.LEGS[leg]
    configs = capi.configs()
    block = spec["scales"] == "block"
    col = 0 if spec["acc"] == "fp32" else 1
    table_cfgs = {e[col][0] for e in ds.tuned_table().values()}
    if block:   # the block-scaled stand-in of each configuration (b200_fp8_block_capi.cu)
        def sibling(cid):
            c = configs[cid]
            return next(d["id"] for d in configs if (d["cta_group"], d["cluster_m"], d["cluster_n"], d["m_rep"], d["bn"])
                        == (c["cta_group"], c["cluster_m"], c["cluster_n"], 1, min(c["bn"], 128)))
        table_cfgs = {sibling(c) for c in table_cfgs}
    op_bytes = 1 if spec["operand"] == "e4m3" else 2
    # the two block-scaled legs share one selector (the output type does not enter it): their lists are covered together
    shapes = (ds.leg_shapes("e4m3_block_fp16") + ds.leg_shapes("e4m3_block_bf16")) if block else ds.leg_shapes(leg)
    modes, cfgs, tiers, hints = Counter(), Counter(), Counter(), 0
    for m, n, k in shapes:
        cfg, gm, sp = ds.choice(leg, m, n, k)
        assert 0 <= cfg < len(configs) and _legal_splits(sp, block) and ds.usable(configs[cfg], m, n), (m, n, k, cfg, sp)
        t, entry = ds.tier(configs, spec["acc"], m, n, k, spec["k_div"])
        if entry is not None and not block:      # the dispatcher took the entry the tier names
            assert (cfg, gm, sp) == entry, (leg, m, n, k, t, entry, (cfg, gm, sp))
        tiers[t] += 1
        modes[ds.plan(leg, cfg, m, n, k, sp)[0]] += 1
        cfgs[cfg] += 1
        hints += ds.l2_hint(configs[cfg], m, n, k, op_bytes)
    print(f"\n{leg}: {sum(cfgs.values())} shapes; K-modes {dict(modes)}; tiers {dict(tiers)}; "
          f"{len(cfgs)} configurations; L2-hint shapes {hints}")
    # Workspace split-K comes only from a table entry with a split code in 2..99 (the shipped table has none) or from the
    # heuristic's split branch, which needs at most two tiles: there, the nearest grid entry is always usable, so the
    # heuristic never decides. It is demanded once the table names it.
    ws = any(2 <= e[col][2] < 100 for e in ds.tuned_table().values())
    want_modes = {"plain", "cluster-split-k"} if block else {"plain", "cluster-split-k", "stream-k"} | ({"split-k"} if ws else set())
    assert want_modes <= set(modes), modes
    assert table_cfgs <= set(cfgs), sorted(table_cfgs - set(cfgs))
    assert hints > 0
    assert {"exact", "nearest", "heuristic"} <= set(tiers), tiers


def test_tile_list_sample_covers_dense_masked_and_skewed_groups(built_libs):
    cases = ds.tile_list_cases()
    batched = [c for c in cases if c["kind"] == "batched"]
    grouped = [c for c in cases if c["kind"] == "grouped"]
    assert any(c["counts"] is None for c in batched) and any(c["counts"] for c in batched)
    assert any(0 in c["counts"] for c in batched if c["counts"]) and any(
        c["m"] in c["counts"] for c in batched if c["counts"])
    sizes = [np.diff([0] + c["offs"]) for c in grouped]
    assert max(c["g"] for c in grouped) == 256 and any((s == 0).any() for s in sizes)
    assert any(c["offs"][-1] < c["t"] for c in grouped) and any(c["offs"][-1] == c["t"] for c in grouped)
    assert all((s >= 0).all() for s in sizes) and any(s.max() > 4 * max(1, s.mean()) for s in sizes)
    rows = [c["b"] * c["m"] for c in batched] + [c["t"] for c in grouped]
    assert min(rows) >= 64 and max(rows) >= 20000
    chosen = Counter()
    for name, variant in ds.TILE_LIST_VARIANTS.items():
        for c in batched:
            chosen[(name, capi.batched_select(variant, c["b"], c["m"], c["n"], c["k"])[0])] += 1
        for c in grouped:
            chosen[(name, capi.grouped_select(variant, c["g"], c["t"], c["n"], c["k"])[0])] += 1
    print(f"\ntile lists: {len(batched)} batched, {len(grouped)} grouped; "
          f"configurations per variant {dict(Counter(v for v, _ in chosen))}")


# ------------------------------------------------------------------------------------------------- totality
INT_MAX = 2 ** 31 - 1

_TOTALITY = r"""
import ctypes, json, sys
sys.path.insert(0, {repo!r})
from cuda_l2_b200 import capi
INT_MAX = 2 ** 31 - 1
dims = (1, 7, 64, 1000, 16384, 2 ** 20, 10 ** 9, INT_MAX)
ks = (16, 64, 4096, 16384, 2 ** 24, INT_MAX - 15)
out = {{"select": [], "fp8": [], "block": [], "batched": [], "grouped": [], "gemm": []}}
i = ctypes.c_int
def sel(fn, *args):
    c, g, s = i(-99), i(-99), i(-99)
    st = fn(*args, ctypes.byref(c), ctypes.byref(g), ctypes.byref(s))
    return [st, c.value, g.value, s.value]
lib, blk = capi.hgemm_lib(), capi.fp8block_lib()
for m in dims:
    for n in (8, 64, 1000, 16384, INT_MAX - 7):
        for k in ks:
            for acc in (32, 16):
                out["select"].append([acc, m, n, k] + sel(lib.b200_hgemm_select, acc, m, n, k))
            out["fp8"].append([m, n, k] + sel(lib.b200_fp8gemm_select, m, n, k))
            out["block"].append([m, n, k] + sel(blk.b200_fp8gemm_blockwise_select, m, n, k))
tl = [(1, 1), (1, INT_MAX), (2, INT_MAX), (INT_MAX, 1), (INT_MAX, INT_MAX), (2 * 10 ** 9, 2 * 10 ** 9),
      (256, 10 ** 9), (3, 10 ** 9), (10 ** 6, 4096)]
for name, lib2 in (("batched", capi.batched_lib()), ("grouped", capi.grouped_lib())):
    fn = getattr(lib2, "b200_%s_select" % name)
    for v in (0, 1, 2):
        for a, b in tl:
            for n in (8, 64, 4096, INT_MAX - 7):
                for k in (16, 4096, INT_MAX - 7):
                    c, g = i(-99), i(-99)
                    st = fn(v, a, b, n, k, ctypes.byref(c), ctypes.byref(g))
                    out[name].append([v, a, b, n, k, st, c.value, g.value])
buf = ctypes.create_string_buffer(1 << 12)
p = (ctypes.addressof(buf) + 15) & ~15
# the dispatched tile-list calls on shapes whose every configuration's tile list passes INT_MAX: refused before any
# device call
for v in (0, 1, 2):
    for g, t, n in ((2 * 10 ** 9, 2 * 10 ** 9, 1024), (INT_MAX, INT_MAX, 4096), (2, INT_MAX, INT_MAX - 7)):
        st = capi.grouped_lib().b200_grouped_gemm(v, p, p, p, p, g, t, n, 64, None)
        out["gemm"].append(["grouped", v, g, t, n, st])
    for b, m, n in ((2 * 10 ** 9, 2 * 10 ** 9, 1024), (INT_MAX, INT_MAX, 64), (3, INT_MAX, INT_MAX - 7)):
        st = capi.batched_lib().b200_batched_gemm(v, p, p, p, None, b, m, n, 64, None)
        out["gemm"].append(["batched", v, b, m, n, st])
print(json.dumps(out))
"""


def test_selectors_are_total_and_tile_list_calls_refuse_before_the_device(built_libs):
    r = subprocess.run([sys.executable, "-c", _TOTALITY.format(repo=str(REPO))], capture_output=True, text=True,
                       timeout=600, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, f"the selector process died (status {r.returncode}):\n{r.stderr[-2000:]}"
    out = json.loads(r.stdout)
    configs = capi.configs()

    def valid(cfg, sp, m, n, block=False):
        return 0 <= cfg < len(configs) and _legal_splits(sp, block) and ds.usable(configs[cfg], m, n)

    for acc, m, n, k, st, cfg, gm, sp in out["select"]:
        assert st == 0 and valid(cfg, sp, m, n) and gm >= 0, (acc, m, n, k, cfg, gm, sp)
    for key in ("fp8", "block"):
        for m, n, k, st, cfg, gm, sp in out[key]:
            assert st == 0 and valid(cfg, sp, m, n, key == "block") and gm >= 0, (key, m, n, k, cfg, sp)
    for key in ("batched", "grouped"):
        for v, a, b, n, k, st, cfg, gm in out[key]:
            rows = b if key == "batched" else -(-b // a)      # per matrix; grouped: ceil(T / G)
            assert st == 0 and valid(cfg, 1, rows, n) and gm >= 0, (key, v, a, b, n, k, cfg)
    assert len(out["gemm"]) == 18
    for kind, v, a, b, n, st in out["gemm"]:
        assert st == -1, (kind, v, a, b, n, st)                # kBadShape
