"""The DISPATCHED calls, bit-exact at every tuned-grid shape and at the off-grid and tile-list samples of
dispatch_sweep.py, against the one rounding of the exact product (computed on the GPU in float64).

Each leg calls what users call, with no configuration or split pinned: ``capi.hgemm`` (fp16, fp32 and fp16
accumulation), ``capi.gemm_kmajor`` (bf16), ``capi.fp8_gemm`` (e4m3 per tensor, rowwise, block-scaled),
``capi.gemm_batched`` and ``capi.gemm_grouped``. C sits in a guarded buffer pre-filled with a NaN sentinel: an element
left unwritten fails, and the guard bands must stay untouched. A leg collects every failing shape with the dispatcher's
choice, the planned K-mode and stream-K tiles and the first bad element, and asserts once. test_dispatch_sweep_cpu.py
checks without a GPU that these lists reach every K-mode, configuration and tier the dispatcher has.
"""
import numpy as np
import pytest
import torch

import dispatch_sweep as ds
import exact_domain as ed
from cuda_l2_b200 import capi

pytestmark = pytest.mark.gpu

GUARD = 64                      # elements of sentinel before and after C (128 bytes: C stays 16-byte aligned)
SENTINEL = 0x7E55               # a NaN in fp16 and in bf16
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def test_device_rounding_equals_exact_domain():
    """The reference's one rounding on the device (float64 -> fp32 -> fp16 / bf16) against exact_domain's, for every
    rounding target at every exponent the operands reach, both signs, and the e4m3 targets times the scale multipliers."""
    for kind in ("fp16", "bf16"):
        exps = sorted({r + c for r in ed.ROW_EXP[kind] for c in ed.COL_EXP[kind]}
                      | ({r + c for r in ed.ROW_EXP_ACC16 for c in ed.COL_EXP_ACC16} if kind == "fp16" else set()))
        t = np.array(ed.rounding_targets(kind), dtype=np.float64)
        vals = np.concatenate([t * 2.0 ** e for e in exps])
        q = np.array([q * 2.0 ** e for q in ed.E4M3_Q[kind] for e in range(-40, 20)])
        vals = np.concatenate([vals, np.outer(np.array(ed.E4M3_TARGETS, float), q).ravel()])
        vals = np.concatenate([vals, -vals])
        got = ds.round_to(torch, torch.from_numpy(vals).cuda(), kind).cpu().numpy().view(np.uint16)
        with np.errstate(over="ignore"):
            want = ed.round_fp16_bits(vals) if kind == "fp16" else ed.round_bf16_bits(vals)
        assert np.array_equal(got, want), kind


def guarded(rows: int, n: int, out: str, lead=()):
    """(buffer, C view): C [*lead, rows, n] inside GUARD sentinel elements on each side, all of it sentinel."""
    count = int(np.prod(lead, dtype=np.int64)) * rows * n
    buf = torch.full((count + 2 * GUARD,), SENTINEL, dtype=torch.int16, device="cuda")
    return buf, buf[GUARD:GUARD + count].view(DTYPES[out]).view(*lead, rows, n)


def guards_intact(buf) -> bool:
    return bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all())


def first_bad(got, want):
    """(mismatch count, (row, col, got bits, want bits) of the first)."""
    bad = got != want
    cnt = int(bad.sum())
    if not cnt:
        return 0, None
    r, c = (int(x) for x in bad.nonzero()[0])
    return cnt, (r, c, hex(int(got[r, c]) & 0xFFFF), hex(int(want[r, c]) & 0xFFFF))


def run_2d(leg: str, m: int, n: int, k: int):
    """The dispatched call of ``leg`` on (M, N, K): None, or a failure report."""
    spec = ds.LEGS[leg]
    seed = ds.shape_seed(m, n, k)
    out = spec["out"]
    scales = None
    if spec["operand"] == "e4m3":
        ops = ds.operands_e4m3(torch, m, n, k, seed)
        sa_t, sb_t, sa, sb = ds.e4m3_scales(torch, spec["scales"], m, n, k, out, seed)
        scales = (sa, sb)
    else:
        ops = ds.operands16(torch, m, n, k, spec["operand"], seed, acc16=spec["acc"] == "fp16")
    buf, c = guarded(m, n, out)
    if spec["operand"] == "e4m3":
        capi.fp8_gemm(ops.a, ops.bt, c, sa_t, sb_t)
    elif spec["operand"] == "bf16":
        capi.gemm_kmajor(ops.a, ops.bt, c)
    else:
        capi.hgemm(ops.a, ops.bt.view(k, n), c, spec["acc"])   # b_col_major: labelled [K, N], the memory of Bt [N, K]
    got = c.view(torch.int16)
    errs = []
    if not guards_intact(buf):
        errs.append("guard band written")
    total, first = 0, None
    rows = ds.sample_rows(m, ops.probe_rows.tolist(), seed)
    cols = ds.sample_cols(n, seed)
    want_rows = {}
    for lo, hi, want in ds.reference_blocks(torch, ops, out, scales, spec["scales"]):
        cnt, fb = first_bad(got[lo:hi], want)
        if cnt and first is None:
            first = (fb[0] + lo,) + fb[1:]
        total += cnt
        for r in rows:
            if lo <= r < hi:
                want_rows[r] = want[r - lo, cols].cpu().numpy().view(np.uint16)
    if total:
        errs.append(f"{total} mismatches, first (row, col, got, want) {first}")
    host = ds.numpy_rows(torch, ops, rows, cols, out, scales, spec["scales"])
    if not np.array_equal(np.stack([want_rows[r] for r in rows]), host):
        errs.append(f"device reference differs from numpy at rows {rows}")   # the reference itself is wrong
    if not errs:
        return None
    cfg, gm, sp = ds.choice(leg, m, n, k)
    mode, sk = ds.plan(leg, cfg, m, n, k, sp)
    return f"{(m, n, k)}: cfg {cfg} group_m {gm} splits {sp} -> {mode} sk_tiles {sk}: " + "; ".join(errs)


@pytest.mark.parametrize("leg,shapes", [(leg, lst) for leg in ds.LEGS for lst in ds.LEG_LISTS[leg]])
def test_dispatched_2d_call_is_exact(leg, shapes):
    failures = []
    for m, n, k in (ds.grid_shapes() if shapes == "grid" else ds.offgrid_shapes(leg)):
        r = run_2d(leg, m, n, k)
        if r:
            failures.append(r)
    torch.cuda.synchronize()
    assert not failures, f"{leg} {shapes}: {len(failures)} shapes fail:\n" + "\n".join(failures[:40])


# ------------------------------------------------------------------------------------------------- tile lists
def run_batched(variant: str, case: dict):
    b, m, n, k, counts = case["b"], case["m"], case["n"], case["k"], case["counts"]
    kind = "bf16" if variant == "bf16" else "fp16"
    seed = ds.shape_seed(b, m, n, k)
    # rows and columns of all matrices drawn as one 2-D problem: [B*M, K] and [B*N, K]
    ops = ds.operands16(torch, b * m, b * n, k, kind, seed, acc16=variant == "fp16acc16")
    a, bt = ops.a.view(b, m, k), ops.bt.view(b, n, k)
    buf, c = guarded(m, n, kind, (b,))
    mm = None if counts is None else torch.tensor(counts, dtype=torch.int32, device="cuda")
    capi.gemm_batched(a, bt, c, "fp16" if variant == "fp16acc16" else "fp32", masked_m=mm)
    got = c.view(torch.int16)
    errs = [] if guards_intact(buf) else ["guard band written"]
    for i in range(b):
        want = ds.round_to(torch, a[i].to(torch.float64) @ bt[i].to(torch.float64).T, kind)
        valid = m if counts is None else min(max(counts[i], 0), m)
        cnt, fb = first_bad(got[i, :valid], want[:valid])
        if cnt:
            errs.append(f"batch {i} (rows {valid}): {cnt} mismatches, first {fb}")
        untouched = min(m, -(-valid // 16) * 16)          # no 16-row store box starting at or past the count
        if not bool((got[i, untouched:] == SENTINEL).all()):
            errs.append(f"batch {i}: rows from {untouched} written")
    if not errs:
        return None
    cfg, gm = capi.batched_select(ds.TILE_LIST_VARIANTS[variant], b, m, n, k)
    return f"batched {(b, m, n, k)} counts {counts}: cfg {cfg} group_m {gm}: " + "; ".join(errs[:5])


def run_grouped(variant: str, case: dict):
    g, t, n, k, offs = case["g"], case["t"], case["n"], case["k"], case["offs"]
    kind = "bf16" if variant == "bf16" else "fp16"
    seed = ds.shape_seed(g, t, n, k)
    ops = ds.operands16(torch, t, g * n, k, kind, seed, acc16=variant == "fp16acc16")
    a, bt = ops.a, ops.bt.view(g, n, k)
    buf, c = guarded(t, n, kind)
    capi.gemm_grouped(a, bt, c, torch.tensor(offs, dtype=torch.int32, device="cuda"),
                      "fp16" if variant == "fp16acc16" else "fp32")
    got = c.view(torch.int16)
    errs = [] if guards_intact(buf) else ["guard band written"]
    start = 0
    for i, end in enumerate(offs):
        if end > start:
            want = ds.round_to(torch, a[start:end].to(torch.float64) @ bt[i].to(torch.float64).T, kind)
            cnt, fb = first_bad(got[start:end], want)
            if cnt:
                errs.append(f"group {i} (rows {start}:{end}): {cnt} mismatches, first {fb}")
        start = max(start, end)
    if not bool((got[offs[-1]:] == SENTINEL).all()):
        errs.append(f"rows from the last end {offs[-1]} written")
    if not errs:
        return None
    cfg, gm = capi.grouped_select(ds.TILE_LIST_VARIANTS[variant], g, t, n, k)
    return f"grouped {(g, t, n, k)}: cfg {cfg} group_m {gm}: " + "; ".join(errs[:5])


@pytest.mark.parametrize("variant", list(ds.TILE_LIST_VARIANTS))
def test_dispatched_tile_list_calls_are_exact(variant):
    failures = []
    for case in ds.tile_list_cases():
        r = run_batched(variant, case) if case["kind"] == "batched" else run_grouped(variant, case)
        if r:
            failures.append(r)
    torch.cuda.synchronize()
    assert not failures, f"{variant}: {len(failures)} problems fail:\n" + "\n".join(failures[:40])
