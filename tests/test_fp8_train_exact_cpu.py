"""CPU companion of test_gpu_fp8_train_exact.py: the fixtures, plans and samples of the 1 x 128 x 1 x 128 GEMM's tests
are not vacuous.

* The 1D1D fixtures reach every rounding case for fp16 and bf16 out, stay exact in fp32, and keep every promotion exact.
* They catch what the kernel's new device code can get wrong: a scale of A or Bt read for a k-block 1..9 or 32 away, a
  swapped pair of Bt's scales, a column of another pair group, the row 8 below each row of A; each changes the rounded
  output somewhere.
* The steady-state cases run one worker on several tiles with the ring (the 1D1D stage count) wrapping; the K-mode,
  non-finite and edge cases are planned as named.
* The dispatched samples reach both compiled K-modes and every configuration the tuned table's block-scaled stand-ins
  name, and the torch reference of the block_1d1d granularity gives exact_domain's bits.
* The legs, lists and seeds of the earlier sweeps are unchanged.
"""
import hashlib
import re
import json
from collections import Counter

import numpy as np
import pytest
import torch

import dispatch_sweep as ds
import exact_domain as ed
import scale_cases as sc
import test_gpu_fp8_train_exact as g
from cuda_l2_b200 import capi

SMEM_LIMIT, EPI_BYTES, BAR_BYTES = 232448, 8 * 16 * 64 * 2, 256      # hgemm_sm90.cuh
# sha256 of NN_LEGS, EPI_LEGS, LATE_LEG_LISTS and their off-grid samples, as they were when TRAIN_LEGS was added (LEGS,
# LEG_LISTS and their samples are pinned by test_dispatch_sweep_late_cpu.py)
# eligible configurations the dispatched call never chooses (no tuned-table entry's block-scaled stand-in)
UNREACHED_BY_THE_SELECTOR = (7, 8, 9, 11, 13, 14, 15, 16, 30)
LATE_LEGS_SHA256 = "ad254f7110eb96e5ca5d0173cc9c409ac31db29e256071fdc447fb4450936d12"


@pytest.fixture(scope="module", autouse=True)
def _libs(built_libs):
    return built_libs


def stages_1d1d(cfg: int) -> int:
    """The ring depth of a BlockScaled1D1D<> configuration (hgemm_sm90.cuh): the e4m3 Config's depth, capped again for
    the stage's scale slice of CTA_M + BN floats."""
    c = capi.configs()[cfg]
    cta_m = 128 * c["m_rep"]
    stage = (cta_m + c["bn"]) * 64 * 2
    base = min(c["stages_requested"], (SMEM_LIMIT - 1024 - EPI_BYTES - BAR_BYTES) // stage)
    return min(base, (SMEM_LIMIT - 1024 - EPI_BYTES - BAR_BYTES) // (stage + (cta_m + c["bn"]) * 4))


def fixture(m, n, k, out, seed=None):
    a, bt = ed.operands_e4m3(m, n, k, seed=m + 5 * n + 3 * k if seed is None else seed)
    sa, sb = ed.e4m3_block_1d1d_scales(m, n, k, out)
    return a, bt, sa, sb


def rounded(y, out):
    with np.errstate(over="ignore"):
        return ed.round_fp16_bits(y) if out == "fp16" else ed.round_bf16_bits(y)


@pytest.mark.parametrize("out", ["fp16", "bf16"])
def test_1d1d_fixtures_reach_the_full_output_range(out):
    for m, n, k in (g.STEADY_MNK, g.SPLIT_MNK):
        a, bt, sa, sb = fixture(m, n, k, out)
        y = ed.exact_1d1d(a, bt, sa, sb)
        assert np.array_equal(y.astype(np.float32).astype(np.float64), y)        # exact in fp32 as well
        r = np.minimum(ed._cycle(ed.E4M3_ROW_EXP, np.arange(m) // 4), 103)
        unit = np.exp2(r[:, None] + ed._cycle(ed.E4M3_COL_EXP, np.arange(n))[None, :])
        with np.errstate(over="ignore"):
            c = ed.classify(y, out, unit)
        assert any(v.any() for v in c["tie_up"].values()) and any(v.any() for v in c["tie_down"].values()), (m, n, k)
        assert c["rounds"].any()
        if out == "fp16":                 # bf16 keeps no subnormal and, below the per-tensor scales, no overflow
            assert c["inf"].any() and (c["subnormal"] & c["rounds"]).any(), (m, n, k)
            assert (y == 65520).any() or (y == -65520).any()
        # the probe rows hold their planted targets: u = t = 0 on the probe positions' k-blocks
        u, t = ed.e4m3_1d1d_kb_bits(k)
        assert not any(u[p // 128] or t[p // 128] for p in ed.probe_positions(k))


@pytest.mark.parametrize("out", ["fp16", "bf16"])
def test_every_promotion_is_exact(out):
    m, n, k = g.STEADY_MNK
    a, bt, sa, sb = fixture(m, n, k, out)
    u, t = ed.e4m3_1d1d_kb_bits(k)
    assert ((u + t) <= 1).all() and u.any() and t.any()
    ia = np.abs(a)
    bound = np.zeros((m, n))
    q = ed.e4m3_row_q(m, out)
    for kb in range(len(u)):
        sl = slice(kb * 128, (kb + 1) * 128)
        bound += (ia[:, sl] @ np.abs(bt[:, sl]).T) * q[:, None] * 2.0 ** (u[kb] + t[kb])
    assert bound.max() < 2 ** 24


def _shift_kb(s, d):
    """Scales read for the k-block d away (a stale stage or the wrong k-block): column kb takes kb - d where it exists
    (d < 0: a later k-block, a stage already refilled)."""
    out = s.copy()
    if d > 0:
        out[:, d:] = s[:, :-d]
    else:
        out[:, :d] = s[:, -d:]
    return out


def test_1d1d_scales_catch_wrong_k_blocks_columns_and_rows():
    m, n, k = g.STEADY_MNK
    for out in ("fp16", "bf16"):
        a, bt, sa, sb = fixture(m, n, k, out)
        want = rounded(ed.exact_1d1d(a, bt, sa, sb), out)
        differs = lambda sa2, sb2: not np.array_equal(rounded(ed.exact_1d1d(a, bt, sa2, sb2), out), want)
        for d in (*range(1, 10), 32):
            assert differs(_shift_kb(sa, d), sb), ("A's scales", d, out)
            assert differs(sa, _shift_kb(sb, d)), ("Bt's scales", d, out)
            assert differs(_shift_kb(sa, d), _shift_kb(sb, d)), ("both", d, out)
            assert differs(_shift_kb(sa, -d), _shift_kb(sb, -d)), ("both, a later k-block", d, out)
        cols = np.arange(n)
        swapped = cols ^ 1                                            # sb.x <-> sb.y in every pair
        assert differs(sa, sb[swapped]), out
        for shift in (8, 16, 24):                                     # a column of another pair group of the tile
            other = (cols // 32) * 32 + (cols % 32 + shift) % 32
            assert differs(sa, sb[np.minimum(other, n - 1)]), (shift, out)
        rows = np.arange(m)
        hi_as_lo = np.where(rows % 16 >= 8, rows - 8, rows)           # sa_hi read as sa_lo
        assert differs(sa[hi_as_lo], sb), out
        # within every 8-column group adjacent columns differ, and so do columns 8 apart
        c = sb[:, 0]
        assert (c[:-1] != c[1:]).all() and (c[:-8] != c[8:]).all()


def test_steady_state_runs_one_worker_over_several_tiles_and_wraps_the_1d1d_ring():
    m, n, k = g.STEADY_MNK
    configs = capi.configs()
    for cfg in g.ELIGIBLE:
        s = capi.schedule(cfg, m, n, k // 2, 1, num_sms=g.cluster_ctas(cfg))
        c = configs[cfg]
        assert s["mode"] == "plain" and s["workers"] == 1, cfg
        assert max(len(u) for u in s["units"]) >= 2, cfg
        per_unit = [kb1 - kb0 for u in s["units"] for _, kb0, kb1, _ in u]
        assert min(per_unit) > 32 and min(per_unit) > stages_1d1d(cfg) >= 2, (cfg, stages_1d1d(cfg))
        assert stages_1d1d(cfg) <= c["stages"]
        assert m % (128 * c["m_rep"]) and n % c["bn"], cfg


def test_k_mode_and_edge_cases_are_planned_as_named():
    m, n, k = g.SPLIT_MNK
    for cfg in g.SPLIT_K:
        for splits in (-2, -4, -8):
            assert g.planned_splits(cfg, m, n, k, splits) == -splits
            assert g.planned_splits(cfg, 200, g.EDGE_N, 8576, splits) == -splits
    for cfg, splits in g.NONFINITE_CASES + g.GUARD_CASES:
        assert g.planned_splits(cfg, m, n, k, splits) == max(1, -splits), (cfg, splits)
    nan_kb = (k - 40) // 128                                        # the NaN of A: in the last split's k-blocks
    for cfg, splits in g.NONFINITE_CASES:
        plan = capi.schedule(cfg, m, n, k // 2, splits)
        ranges = sorted((kb0, kb1) for units in plan["units"] for tile, kb0, kb1, _ in units if tile == 0)
        assert len(ranges) == max(1, -splits) and ranges[-1][0] <= nan_kb < ranges[-1][1], (cfg, splits, ranges)
        if len(ranges) > 1:                                        # the NaN scales: one in an early split, one later
            assert ranges[0][0] <= 1 < ranges[0][1] and not ranges[0][0] <= (k // 128 + 1) // 2 < ranges[0][1]
    assert set(g.UNCOMPILED) == {4, 16, 64, 100, 101}
    assert {capi.schedule(1, m, n, k // 2, sp)["mode"] for sp in g.UNCOMPILED} == {"split-k", "stream-k"}
    for cfg in g.ELIGIBLE:
        assert g.EDGE_N % capi.configs()[cfg]["bn"] == 8
    assert 193 % 64 == 1 and 193 % 128 != 1


def test_sweep_samples_reach_both_k_modes_and_every_configuration_the_selector_can_choose():
    configs = capi.configs()
    shapes = ds.leg_shapes("e4m3_1d1d_fp16") + ds.leg_shapes("e4m3_1d1d_bf16") + ds.dw_shapes()
    cfgs, modes = Counter(), Counter()
    for m, n, k in shapes:
        cfg, gm, sp = ds.choice("e4m3_1d1d_fp16", m, n, k)
        assert (cfg, gm, sp) == capi.fp8_blockwise_select(m, n, k)
        assert cfg in g.ELIGIBLE and sp in (1, -2, -4, -8), (m, n, k, cfg, sp)
        mode = ds.plan("e4m3_1d1d_fp16", cfg, m, n, k, sp)[0]
        cfgs[cfg] += 1
        modes[(cfg, mode)] += 1

    def sibling(cid):   # the block-scaled stand-in of each configuration (b200_fp8_block_capi.cu)
        c = configs[cid]
        return next(d["id"] for d in configs if (d["cta_group"], d["cluster_m"], d["cluster_n"], d["m_rep"], d["bn"])
                    == (c["cta_group"], c["cluster_m"], c["cluster_n"], 1, min(c["bn"], 128)))
    table_cfgs = {sibling(e[0][0]) for e in ds.tuned_table().values()}
    print(f"\n1D1D sweep: {len(shapes)} shapes; configurations {dict(sorted(cfgs.items()))}; (configuration, K-mode) "
          f"{dict(sorted(modes.items()))}")
    # The selector is the e4m3 dispatcher's choice mapped to its block-scaled stand-in (block::select). The stand-ins of
    # what the tuned table names are the configurations reached; the other eligible ones are no stand-in of a table
    # entry and the heuristic picks none of them, so only the pinned tests of test_gpu_fp8_train_exact.py run them.
    assert set(cfgs) == table_cfgs, (sorted(cfgs), sorted(table_cfgs))
    assert set(g.ELIGIBLE) - set(cfgs) == set(UNREACHED_BY_THE_SELECTOR)
    assert {mode for _, mode in modes} == {"plain", "cluster-split-k"}
    assert {cfg for cfg, mode in modes if mode == "cluster-split-k"} == set(g.SPLIT_K)


def test_weight_gradient_samples():
    dw = ds.dw_shapes()
    assert len(dw) == len(ds.DW_FEATURES) * len(ds.DW_TOKENS)
    for (m, n, k), (t, (fm, fn)) in zip(dw, [(t, f) for f in ds.DW_FEATURES for t in ds.DW_TOKENS]):
        assert (m, n) == (fm, fn) and k == capi.dual_ld_t(t) and k % 16 == 0 and t % 128 and k % 128
    offgrid = ds.offgrid_shapes("e4m3_1d1d_bf16")
    assert 250 <= len(offgrid) <= 400 and not set(offgrid) & set(ds.grid_shapes())
    assert all(k % 16 == 0 and n % 8 == 0 for _, n, k in offgrid)


@pytest.mark.parametrize("m,n,k", [(45, 136, 256), (13, 264, 1040)])
@pytest.mark.parametrize("out", ["fp16", "bf16"])
def test_block_1d1d_torch_reference_is_exact_domains(m, n, k, out):
    operands = ds.operands_e4m3(torch, m, n, k, seed=ds.shape_seed(m, n, k), device="cpu")
    sa_t, sb_t, sa, sb = ds.e4m3_scales(torch, "block_1d1d", m, n, k, out, 3, device="cpu")
    assert sa_t.stride() == (1, -(-m // 4) * 4) and sb_t.stride() == (1, -(-n // 4) * 4)
    assert capi.scale_granularity(m, n, sa_t, sb_t, k=k) == "blockwise_1d1d"
    a = operands.a.to(torch.float32).numpy().astype(np.float64)
    bt = operands.bt.to(torch.float32).numpy().astype(np.float64)
    want = rounded(ed.exact_1d1d(a, bt, sa, sb), out)
    got = np.concatenate([b.numpy().view(np.uint16) for _, _, b in
                          ds.reference_blocks(torch, operands, out, (sa, sb), "block_1d1d", rows_per_block=16)])
    assert np.array_equal(got, want)
    rows, cols = ds.sample_rows(m, operands.probe_rows.numpy(), 2), ds.sample_cols(n, 2, limit=64)
    assert np.array_equal(ds.numpy_rows(torch, operands, rows, cols, out, (sa, sb), "block_1d1d"),
                          want[np.ix_(rows, cols)])


def test_scale_cases_of_the_weight_gradient():
    m, n, k = sc.FP8_DW
    assert k == capi.dual_ld_t(sc.FP8_DW_TOKENS) and sc.FP8_DW_TOKENS % 128
    assert m * k > 2 ** 31 and sc.CASES["fp8_dw"].tensor("a").shape == (m, k)
    # the domain: at most 128 unit products per k-block, scales 2^-1..2^1 on both operands: |sum| / 2^-2 < 2^24 for a
    # row of A with fewer than 2^20 nonzeros, which p = 0.2 of 2/3 gives with a wide margin at this K
    p = sc.DOMAINS["e4m3"]["a"][2]
    mean = k * p * 2 / 3
    assert (mean + 10 * (mean ** 0.5)) * 16 < 2 ** 24
    assert sc.CASES["fp8_dw_out"].tensor("c").numel > 2 ** 31


def test_earlier_legs_lists_and_seeds_are_unchanged():
    blob = json.dumps({"nn": ds.NN_LEGS, "epi": ds.EPI_LEGS, "lists": ds.LATE_LEG_LISTS,
                       "offgrid": {leg: ds.offgrid_shapes(leg) for leg in ds.LATE_LEGS}}, sort_keys=True)
    assert hashlib.sha256(blob.encode()).hexdigest() == LATE_LEGS_SHA256
    assert not set(ds.TRAIN_LEGS) & (set(ds.LEGS) | set(ds.LATE_LEGS))


def _promotion_1d1d(path) -> tuple[str, str]:
    """(the block-scaled main loop up to the 1D1D promotion, the 1D1D promotion through its `continue`) of the kernel
    body at ``path``."""
    text = path.read_text()
    loop = text.index("block-scaled main loop")
    start = text.index("if constexpr (k1D1D) {", loop)
    return text[loop:start], text[start:text.index("continue;", start)]


def test_1d1d_promotion_releases_its_stage_after_reading_the_scales():
    """The stage holding a k-block's scales goes back to the producer only after the promotion has read them: a release
    before the last shared-memory read lets the producer refill the stage under the reads. The window is too short for
    a run to show it reliably, so the order is checked in the source (the 1D1D kernels are outside the SASS digest)."""
    before, promotion = _promotion_1d1d(ds.REPO / "cuda_l2_b200" / "csrc" / "hgemm_tn_kernel_body.inc")
    reads = [m.end() for m in re.finditer(r"\bld_shared_(?:f32|v2f)\(", promotion)]
    releases = [m.start() for m in re.finditer(r"\brelease\(stage\)", promotion)]
    assert len(reads) >= 3 and len(releases) == 1 and releases[0] > max(reads), (reads, releases)
    assert not re.search(r"\brelease\(", before[before.index("for (int kb = u.kb0"):])


@pytest.mark.parametrize("kind", sc.QUANTISERS)
@pytest.mark.parametrize("band_rows", [128, 256, 1024])
def test_banded_quantiser_reference_is_the_unbanded_one(kind, band_rows):
    """scale_cases.quant_bands, assembled band by band, is the unbanded *_reference bit for bit: the per-tensor amax and
    the rowwise dual's column maxima reduced over all bands, q_t's padding columns included, every element covered
    exactly once. x: rows % 16 != 0, cols % 128 != 0, rows and columns of very different magnitudes, a NaN."""
    from cuda_l2_b200 import ops
    rows, cols = 300, 392
    g_ = torch.Generator().manual_seed(5)
    x = torch.randn((rows, cols), generator=g_)
    x *= torch.exp(torch.empty((rows, 1)).uniform_(-4, 4, generator=g_))
    x *= torch.exp(torch.empty((1, cols)).uniform_(-3, 3, generator=g_))
    x[17, 33] = x[290, 40] = float("nan")                          # the first and the last (padded) row group
    x = x.bfloat16()
    ref = {"tensor": lambda: dict(zip(("q", "scale"), ops.quantize_e4m3_reference(x))),
           "rowwise": lambda: dict(zip(("q", "scale"), ops.quantize_e4m3_rowwise_reference(x))),
           "blockwise": lambda: dict(zip(("q", "scale"), ops.quantize_e4m3_blockwise_reference(x))),
           "silu_mul": lambda: dict(zip(("q", "scale"), ops.silu_mul_quantize_e4m3_blockwise_reference(x))),
           "rowwise_dual": lambda: dict(zip(("q", "scale", "q_t", "scale_t"), ops.quantize_e4m3_rowwise_dual_reference(x))),
           "blockwise_dual": lambda: dict(zip(("q", "scale", "q_t", "scale_t"),
                                              ops.quantize_e4m3_blockwise_dual_reference(x))),
           "block128x128_dual": lambda: dict(zip(("q", "scale", "q_t", "scale_t"),
                                                 ops.quantize_e4m3_block128x128_dual_reference(x)))}[kind]()
    raw = lambda t: t.contiguous().view(torch.uint8 if t.element_size() == 1 else torch.int32)
    want = {name: raw(t) for name, t in ref.items()}
    got = {name: torch.zeros_like(t) for name, t in want.items()}
    seen = {name: torch.zeros(t.shape, dtype=torch.int32) for name, t in want.items()}
    for name, idx, part in sc.quant_bands(kind, x, band_rows):
        got[name][idx] = raw(part)
        seen[name][idx] += 1
    for name in want:
        assert bool((seen[name] == 1).all()), (kind, name)
        g_, w_ = got[name], want[name]
        if ref[name].dtype == torch.float32:   # a NaN scale: any encoding (which sign a reduction's NaN has is torch's)
            nan_g, nan_w = g_.view(torch.float32).isnan(), w_.view(torch.float32).isnan()
            assert torch.equal(nan_g, nan_w), (kind, name)
            g_, w_ = g_[~nan_g], w_[~nan_w]
        assert torch.equal(g_, w_), (kind, name)
    if kind in ("rowwise_dual", "blockwise_dual"):
        assert want["q_t"].shape == (cols, capi.dual_ld_t(rows)) and capi.dual_ld_t(rows) > rows
        assert (want["q_t"][40, rows:] == 0x7F).all() and (want["q_t"][34, rows:] == 0).all()    # NaN column padding
