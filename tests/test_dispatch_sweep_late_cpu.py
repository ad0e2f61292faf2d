"""The NN, bias + activation and grouped-backward sweep without a GPU (its results are test_gpu_dispatch_sweep_late.py's):

* the legs of test_gpu_dispatch_sweep.py are untouched: their fields, lists, off-grid samples and tile-list cases hash
  to what they were when the new legs were added;
* the Python mirror of select_rowmajor is the library's choice (the grouped NN select of one group reduces to it);
* the sweep is not vacuous: the NN legs reach every NN configuration the mapped table names, the BN = 32 -> sibling map
  with both accumulators, every K-mode and stream-K code, the L2-hint branch and every tier; the bias legs reach every
  configuration the table names and every K-mode it reaches, each activation in each K-mode, sign flips of z, and
  (configuration, K-mode, stream-K tiles, ragged M, ragged N) tuples beyond test_gpu_epilogue.py's pinned cases; the
  grouped-backward cases hold every edge and make both selects choose more than one configuration;
* the torch generators and references of the new legs give exactly epilogue_ref's and exact_domain's bits.
"""
import hashlib
import json
from collections import Counter

import numpy as np
import pytest
import torch

import dispatch_sweep as ds
import epilogue_ref
import exact_domain as ed
from cuda_l2_b200 import capi

# sha256 of the existing legs (LEGS, LEG_LISTS), their off-grid samples and tile_list_cases(), as the parent of the NN
# / bias + activation / grouped-backward legs generated them
EXISTING_LEGS_SHA256 = "8b48257232bf055e1012abf1a87f16b78f3bc9281906ce94ad68d8bd2c401a8b"


def test_existing_legs_lists_and_seeds_are_unchanged(built_libs):
    blob = json.dumps({"legs": ds.LEGS, "lists": ds.LEG_LISTS, "offgrid": {leg: ds.offgrid_shapes(leg) for leg in ds.LEGS},
                       "tile_list": ds.tile_list_cases()}, sort_keys=True)
    assert hashlib.sha256(blob.encode()).hexdigest() == EXISTING_LEGS_SHA256
    assert not set(ds.LEGS) & set(ds.LATE_LEGS) and set(ds.LATE_LEG_LISTS) == set(ds.LATE_LEGS)


def test_late_offgrid_samples_follow_the_shape_rules(built_libs):
    for leg, spec in ds.LATE_LEGS.items():
        shapes = ds.offgrid_shapes(leg)
        assert 250 <= len(shapes) <= 400, (leg, len(shapes))
        assert not set(shapes) & set(ds.grid_shapes())
        for m, n, k in shapes:
            assert m >= 1 and n % 8 == 0 and k % spec["k_align"] == 0 and k >= 16, (leg, m, n, k)
            assert 2 * m * n * k <= ds.OFFGRID_MAX_FLOP
        assert set(range(1, 17)) <= {s[0] for s in shapes}


# ------------------------------------------------------------------------------------------------- NN
def test_nn_mirror_is_the_library_choice(built_libs):
    """With one group the grouped NN select's tile-list rule reduces to select and nn::sibling: it is the dispatched
    NN call's choice, computed by the library."""
    for leg, variant in (("nn_fp16", 0), ("nn_bf16", 2)):
        for m, n, k in ds.leg_shapes(leg):
            cfg, gm, _, _ = ds.nn_choice(leg, m, n, k)
            assert (cfg, gm) == capi.grouped_nn_select(variant, 1, m, n, k), (leg, m, n, k)


@pytest.mark.parametrize("acc,legs", [("fp32", ("nn_fp16", "nn_bf16")), ("fp16", ("nn_fp16acc16",))])
def test_nn_legs_cover_every_mapped_configuration_k_mode_tier_and_l2_hint(acc, legs, built_libs):
    configs = capi.configs()
    col = 0 if acc == "fp32" else 1
    table_cfgs = {ds.nn_sibling(configs, e[col][0]) for e in ds.tuned_table().values()}
    modes, codes, cfgs, tiers, hints, mapped, mapped_grid = Counter(), Counter(), Counter(), Counter(), 0, 0, 0
    grid = set(ds.grid_shapes())
    for leg in legs:
        seen = (Counter(modes), Counter(tiers), Counter(cfgs), hints)
        for m, n, k in ds.leg_shapes(leg):
            cfg, gm, sp, tn = ds.nn_choice(leg, m, n, k)
            assert configs[cfg]["bn"] % 64 == 0 and ds.usable(configs[tn], m, n), (leg, m, n, k, tn, cfg)
            mode = ds.plan(leg, cfg, m, n, k, sp)[0]
            modes[mode] += 1
            if mode == "stream-k":
                codes[sp] += 1
            cfgs[cfg] += 1
            tiers[ds.tier(configs, acc, m, n, k)[0]] += 1
            hints += ds.l2_hint(configs[cfg], m, n, k, 2)
            mapped += cfg != tn
            mapped_grid += cfg != tn and (m, n, k) in grid
        print(f"\n{leg}: K-modes {dict(modes - seen[0])}; tiers {dict(tiers - seen[1])}; configurations "
              f"{sorted(cfgs - seen[2])}; L2-hint shapes {hints - seen[3]}")
    print(f"\nNN {acc} ({', '.join(legs)}): {sum(cfgs.values())} shapes; K-modes {dict(modes)}; stream-K codes "
          f"{dict(codes)}; tiers {dict(tiers)}; configurations {sorted(cfgs)}; BN = 32 mapped {mapped} "
          f"({mapped_grid} on the grid); L2-hint shapes {hints}; mapped table configurations not run "
          f"{sorted(table_cfgs - set(cfgs))}")
    assert {"plain", "cluster-split-k", "stream-k"} <= set(modes), modes
    assert mapped > 0 and hints > 0
    if acc == "fp32":   # the grid: every entry of the column, both stream-K codes, every tier
        assert table_cfgs <= set(cfgs), sorted(table_cfgs - set(cfgs))
        assert {100, 101} <= set(codes) and mapped_grid > 0, codes
        assert {"exact", "nearest", "heuristic"} <= set(tiers), tiers
    else:               # the off-grid sample only: borrowed entries and the heuristic
        assert {"nearest", "heuristic"} <= set(tiers) and len(cfgs) >= 6, (tiers, cfgs)


def test_bn32_map_is_reached_on_the_grid_with_both_accumulators(built_libs):
    """The tuned table names a BN = 32 configuration at grid shapes of both columns, and the NN legs run some of them
    (nn_fp16acc16 runs the off-grid sample: its nearest-entry tier borrows those grid entries)."""
    configs = capi.configs()
    for acc, leg in (("fp32", "nn_fp16"), ("fp16", "nn_fp16acc16")):
        col = 0 if acc == "fp32" else 1
        named = [s for s, e in ds.tuned_table().items() if configs[e[col][0]]["bn"] == 32]
        runs = [s for s in ds.leg_shapes(leg)
                if ds.tier(configs, acc, *s)[0] != "heuristic" and configs[ds.nn_choice(leg, *s)[3]]["bn"] == 32]
        print(f"\n{acc}: table entries naming BN = 32: {len(named)}; {leg} shapes mapped from one: {len(runs)}")
        assert named and runs, (acc, len(named), len(runs))


# ------------------------------------------------------------------------------------------------- bias + activation
def _epi_runs():
    """(leg, M, N, K, cfg, splits, K-mode, sk_tiles, activation) of every shape of the bias + activation legs."""
    runs = []
    for leg in ds.EPI_LEGS:
        for m, n, k in ds.leg_shapes(leg):
            cfg, _, sp = ds.epi_choice(leg, m, n, k)
            mode, sk = ds.plan(leg, cfg, m, n, k, sp)
            runs.append((leg, m, n, k, cfg, sp, mode, sk, ds.epi_activation(leg, m, n, k)))
    return runs


def _tuple(configs, cfg, mode, sk, m, n):
    c = configs[cfg]
    return cfg, mode, sk > 0, m % (128 * c["m_rep"] * c["cta_group"]) != 0, n % c["bn"] != 0


def test_bias_legs_cover_every_configuration_k_mode_and_activation(built_libs):
    import test_gpu_epilogue
    configs = capi.configs()
    runs = _epi_runs()
    table_cfgs = {e[0][0] for e in ds.tuned_table().values()}
    ws = any(2 <= e[0][2] < 100 for e in ds.tuned_table().values())
    want_modes = {"plain", "cluster-split-k", "stream-k"} | ({"split-k"} if ws else set())
    cfgs = Counter(r[4] for r in runs)
    modes = Counter(r[6] for r in runs)
    per_mode = Counter((r[6], r[8]) for r in runs)
    tiers, hints = Counter(), 0
    per_leg = {leg: (Counter(), Counter(), set(), [0]) for leg in ds.EPI_LEGS}
    for leg, m, n, k, cfg, sp, mode, sk, act in runs:
        spec = ds.EPI_LEGS[leg]
        t = ds.tier(configs, "fp32", m, n, k, spec["k_div"])[0]
        h = ds.l2_hint(configs[cfg], m, n, k, 1 if spec["operand"] == "e4m3" else 2)
        tiers[t] += 1
        hints += h
        lm, lt, lc, lh = per_leg[leg]
        lm[mode] += 1
        lt[t] += 1
        lc.add(cfg)
        lh[0] += h
    for leg, (lm, lt, lc, lh) in per_leg.items():
        print(f"\n{leg}: K-modes {dict(lm)}; tiers {dict(lt)}; configurations {sorted(lc)}; L2-hint shapes {lh[0]}")
    pinned = {_tuple(configs, cid, mode, capi.schedule(cid, m, n, k, sp)["sk_tiles"], m, n)
              for (cid, _, sp, m, n, k, mode) in test_gpu_epilogue.CASES}
    swept = {_tuple(configs, r[4], r[6], r[7], r[1], r[2]) for r in runs}
    print(f"\nbias legs: {len(runs)} shapes; K-modes {dict(modes)}; tiers {dict(tiers)}; {len(cfgs)} configurations; "
          f"L2-hint shapes {hints}; (K-mode, activation) {dict(per_mode)}")
    print(f"coverage delta: {len(swept - pinned)} (configuration, K-mode, sk_tiles > 0, ragged M, ragged N) tuples run "
          f"beyond test_gpu_epilogue.py's {len(test_gpu_epilogue.CASES)} pinned cases ({len(swept)} in all)")
    assert table_cfgs <= set(cfgs), sorted(table_cfgs - set(cfgs))
    assert want_modes <= set(modes), modes
    assert all(per_mode[(mode, act)] for mode in modes for act in ds.ACTIVATIONS), per_mode
    assert {"exact", "nearest", "heuristic"} <= set(tiers) and hints > 0, tiers
    assert len(swept - pinned) >= 45


@pytest.mark.parametrize("leg", list(ds.EPI_LEGS))
def test_bias_flips_the_sign_of_z(leg, built_libs):
    """On a CPU-sized shape of each leg: relu zeroes a real fraction of z, and the bias turns the product's sign on some
    rows of both signs; a quarter of the columns keep the product (bias -0.0)."""
    m, n, k = 200, 264, 1024
    spec = ds.EPI_LEGS[leg]
    ops, scales = _operands(leg, m, n, k, 9)
    bias = ds.epi_bias(torch, leg, ops, scales, n, k, 9, device="cpu")
    s = np.concatenate([y.numpy() for _, _, y in ds.exact_blocks(torch, ops, scales, spec["scales"])])
    z = np.concatenate([z.numpy() for _, _, z in ds.epilogue_blocks(torch, ops, bias, scales, spec["scales"])])
    b = bias.to(torch.float32).numpy()
    neg0 = (b == 0) & np.signbit(b)
    assert 0.15 < neg0.mean() < 0.35 and ((b == 0) & ~np.signbit(b)).any()
    zeroed = (z <= 0).mean()
    up, down = ((s < 0) & (z > 0)).mean(), ((s > 0) & (z <= 0)).mean()
    print(f"\n{leg}: relu zeroes {zeroed:.3f} of z; the bias turns {up:.3f} of s < 0 up and {down:.3f} of s > 0 down")
    assert 0.1 < zeroed < 0.9 and up > 0.01 and down > 0.01


# ------------------------------------------------------------------------------------------------- grouped backward
def test_grouped_backward_cases_hold_every_edge_and_reach_several_configurations(built_libs):
    cases = ds.grouped_bwd_cases()
    assert {c["g"] for c in cases} == {1, 8, 64, 256} and max(c["t"] for c in cases) == 65536
    starts, sizes = [], []
    for c in cases:
        g, t, offs = c["g"], c["t"], c["offs"]
        assert len(offs) == g and all(a <= b for a, b in zip([0] + offs, offs)) and offs[-1] <= t
        assert 2 * t * c["d_in"] * c["d_out"] <= 2 ** 37 and g * c["d_in"] * c["d_out"] <= ds.GROUPED_BWD_OUT_MAX
        assert c["d_in"] % 8 == 0 and c["d_out"] % 8 == 0 and (t == 0 or t >= 16)
        sz = np.diff([0] + offs)
        sizes.append(sz)
        starts += [s for s, z in zip([0] + offs[:-1], sz) if z > 0]
    assert any((s == 0).any() for s in sizes) and any((s == 1).any() for s in sizes)
    assert any(s % 8 for s in starts) and any(s % 16 == 8 for s in starts) and any(s % 64 in (16, 32, 48) for s in starts)
    assert any(c["offs"][-1] < c["t"] for c in cases) and any(c["offs"][-1] == c["t"] > 0 for c in cases)
    assert any(c["t"] == 0 for c in cases) and any(c["t"] > 0 and c["offs"][-1] == 0 for c in cases)
    dims = {d for c in cases for d in (c["d_in"], c["d_out"])}
    assert {1408, 2816} & dims and max(dims) >= 4096
    chosen = Counter()
    for kind, v in ds.GROUPED_BWD_VARIANTS.items():
        for c in cases:
            if c["t"]:
                chosen[("nn", capi.grouped_nn_select(v, c["g"], c["t"], c["d_in"], c["d_out"])[0])] += 1
            chosen[("wgrad", capi.grouped_wgrad_select(v, c["g"], c["t"], c["d_out"], c["d_in"])[0])] += 1
    nn = sorted({cfg for (kind, cfg) in chosen if kind == "nn"})
    wg = sorted({cfg for (kind, cfg) in chosen if kind == "wgrad"})
    print(f"\ngrouped backward: {len(cases)} cases; grouped NN configurations {nn}; weight-gradient configurations {wg}")
    assert len(nn) >= 2 and len(wg) >= 2


# ------------------------------------------------------------------------------------------------- references
def _operands(leg, m, n, k, seed):
    spec = ds.EPI_LEGS[leg]
    if spec["operand"] == "e4m3":
        ops = ds.operands_e4m3(torch, m, n, k, seed, device="cpu")
        _, _, sa, sb = ds.e4m3_scales(torch, spec["scales"], m, n, k, spec["out"], seed, device="cpu")
        return ops, (sa, sb)
    return ds.operands16(torch, m, n, k, spec["operand"], seed, device="cpu"), None


def _np(x):
    return x.to(torch.float32).numpy().astype(np.float64)


@pytest.mark.parametrize("m,n,k", [(45, 136, 256), (13, 264, 1024)])
@pytest.mark.parametrize("leg", list(ds.EPI_LEGS))
def test_bias_leg_reference_matches_epilogue_ref(leg, m, n, k):
    spec = ds.EPI_LEGS[leg]
    out = spec["out"]
    for seed in (0, 1, 2):
        ops, scales = _operands(leg, m, n, k, seed)
        bias = ds.epi_bias(torch, leg, ops, scales, n, k, seed, device="cpu")
        b32 = bias.to(torch.float32).numpy()
        sa = sb = None
        if spec["scales"] == "tensor":
            sa, sb = np.float32(scales[0]), np.float32(scales[1])
        elif spec["scales"] == "rowwise":
            sa, sb = scales
        rowwise = spec["scales"] == "rowwise"
        z = np.concatenate([z.numpy() for _, _, z in ds.epilogue_blocks(torch, ops, bias, scales, spec["scales"], 16)])
        with np.errstate(over="ignore", invalid="ignore"):
            want_z = epilogue_ref.pre_activation(_np(ops.a), _np(ops.bt), b32, sa, sb, rowwise)
        assert np.array_equal(z.view(np.uint32), want_z.view(np.uint32)), (leg, seed)
        rows, cols = ds.sample_rows(m, ops.probe_rows.numpy(), seed), ds.sample_cols(n, seed, limit=64)
        for act in ds.ACTIVATIONS:
            with np.errstate(over="ignore", invalid="ignore"):
                want = epilogue_ref.reference(_np(ops.a), _np(ops.bt), b32, act, out, sa, sb, rowwise)
            hz, hbits = ds.epilogue_numpy_rows(torch, ops, rows, cols, bias, act, out, scales, spec["scales"])
            assert np.array_equal(hz.view(np.uint32), want_z[np.ix_(rows, cols)].view(np.uint32))
            if act == "gelu_tanh":
                # the torch check is epilogue_ref.gelu_excess's: it passes the reference's own rounding, and fails a
                # result two units off wherever that lies outside the allowance
                tz = torch.from_numpy(want_z)
                assert bool(ds.gelu_ok(torch, torch.from_numpy(want.view(np.int16)), tz, out).all())
                off = (want.astype(np.int32) + 2).astype(np.uint16)
                with np.errstate(invalid="ignore"):
                    allowed = epilogue_ref.gelu_excess(off, want_z, out) <= 0
                got = ds.gelu_ok(torch, torch.from_numpy(off.view(np.int16)), tz, out).numpy()
                fin = np.isfinite(epilogue_ref.bits_to_f64(off, out)) & np.isfinite(want_z)
                assert np.array_equal(got[fin], allowed[fin]) and not allowed[fin].all(), (leg, seed)
            else:
                bits = ds.activated_bits(torch, torch.from_numpy(z), act, out).numpy().view(np.uint16)
                assert np.array_equal(bits, want), (leg, seed, act)
                assert np.array_equal(hbits, want[np.ix_(rows, cols)])


def _clamped(offs, t):
    out, s = [], 0
    for o in offs:
        e = min(max(o, s), t)
        out.append((s, e))
        s = e
    return out


@pytest.mark.parametrize("kind", ["fp16", "bf16"])
def test_grouped_backward_references_match_exact_domain(kind):
    """The wgrad transpose keeps every group's partial sum exact, and both references give exact_domain's rounding
    of the float64 product, group by group (an empty weight-gradient group: +0.0)."""
    rnd = ed.round_fp16_bits if kind == "fp16" else ed.round_bf16_bits
    t, m, n, offs = 300, 72, 136, [0, 1, 37, 37, 100, 163, 250]
    a, b = ds.wgrad_operands(torch, t, m, n, kind, 5, device="cpu")
    assert a.shape == (t, m) and b.shape == (t, n)
    a64, b64 = _np(a), _np(b)
    ops = ds.operands16(torch, m, n, t, kind, 5, device="cpu")
    assert torch.equal(a, ops.a.t()) and torch.equal(b, ops.bt.t())
    ia = np.abs(a64) / np.exp2(ops.row_exp.numpy())[None, :]
    jb = np.abs(b64) / np.exp2(ops.col_exp.numpy())[None, :]
    for s, e in _clamped(offs, t):
        assert (ia[s:e].T @ jb[s:e]).max(initial=0) < ed.EXACT_SUM_BOUND        # a subset of an exact row sum
        got = ds.wgrad_reference(torch, a, b, s, e, kind).numpy().view(np.uint16)
        assert np.array_equal(got, rnd(a64[s:e].T @ b64[s:e])), (s, e)
        if e == s:
            assert not got.any()
    g, k = len(offs), 200
    a, bb = ds.grouped_nn_operands(torch, t, g, n, k, kind, 6, device="cpu")
    assert a.shape == (t, k) and bb.shape == (g, k, n) and bb.is_contiguous()
    for i, (s, e) in enumerate(_clamped(offs, t)):
        if e > s:
            got = ds.grouped_nn_reference(torch, a, bb, s, e, i, kind).numpy().view(np.uint16)
            assert np.array_equal(got, rnd(_np(a[s:e]) @ _np(bb[i]))), (i, s, e)
    assert ds.wgrad_operands(torch, 0, m, n, kind, 1, device="cpu")[0].shape == (0, m)
