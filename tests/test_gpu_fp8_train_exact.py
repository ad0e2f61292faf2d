"""The GEMM with 1 x 128 scales on both operands (libb200_fp8block_1d1d.so, the weight gradient of blockwise FP8
training) on the H100, bit-exact against a plain float64 reference on the exact domain of ``exact_domain.py``.

The operands are exact_domain's e4m3 integers and its probe rows; the scales are ``e4m3_block_1d1d_scales``: Q_m 2^r_m
per row of A and 2^c_n per row of Bt, with an extra bit along K on A's even k-blocks and Bt's odd ones. Every
promotion is then exact, the output is one rounding of the float64 product, and the fixtures reach ties at every
number of dropped bits, fp16 subnormals and fp16 overflow to inf. Because adjacent columns, columns 8 apart and
k-blocks 1..9 and 32 apart all carry different scales, a swapped pair of Bt's scales, a scale of the wrong pair group,
a row's scale of A taken for the row 8 below it, and a scale read from a stale stage or the wrong k-block each change
some output.

* Steady state: every eligible configuration with ``max_ctas`` limiting the launch to one worker, which walks every
  tile of a ragged problem with 34 k-blocks per tile, so the ring wraps many times within and across tiles.
* Cluster split-K -2/-4/-8 at the full output range, against tests/fp8_block_1d1d_ref.c with the planner's split count.
* K-mode requests the library does not compile (workspace split-K 4/16/64, stream-K 100/101) run plain: the plain bits,
  one launch each.
* Non-finite values: an e4m3 NaN in A in a late split's k-range, a NaN in scale_a[m, kb] and one in scale_b[n, kb] make
  exactly their row / column NaN; every other element stays exact. Plain and cluster split-K.
* Guard bands around C; N = 8 mod BN (the last tile reads fewer than BN rows of Bt's scales); ld_b = N, N + 4 and far
  past N with NaN in the padding; M = 1 and M = 1 mod 64.
* Scales written by a kernel just before the launch, and graph replays reading the current scales.
* The dispatched call (no configuration pinned) at every tuned-grid shape (fp16 out), the off-grid sample (bf16 out) and
  weight-gradient shapes (M = out_features, N = in_features, K = dual_ld_t(T)), as test_gpu_dispatch_sweep_late.py does.
* Production scale (scale_cases.py): A past 2^31 bytes along K, and C past 2^31 elements; and one bf16 activation past
  2^31 elements (rows % 16 != 0, cols % 128 != 0) through each of the seven e4m3 quantisers, every result bit-exact
  against its torch reference applied in row bands, q and q_t inside guarded buffers.

test_fp8_train_exact_cpu.py checks without a GPU that these fixtures and plans hold what is claimed here.
"""
import functools
import time

import numpy as np
import pytest
import torch

import dispatch_sweep as ds
import exact_domain as ed
import scale_cases as sc
from cuda_l2_b200 import capi, ops
from test_gpu_dispatch_sweep import first_bad, guarded, guards_intact
from test_gpu_fp8_train_blockwise import ELIGIBLE, SPLIT_K, ref_1d1d

pytestmark = pytest.mark.gpu

E4 = torch.float8_e4m3fn
KINDS = ("fp16", "bf16")
STEADY_MNK = (600, 392, 4288)             # M, N off every tile multiple; 34 k-blocks per tile
SPLIT_MNK = (520, 392, 8576)              # 67 k-blocks, few tiles
UNCOMPILED = (4, 16, 64, 100, 101)        # workspace split-K and stream-K requests: the library runs them plain
NONFINITE_CASES = ((1, 1), (12, 1), (1, -4), (2, -8))
GUARD_CASES = ((1, 1), (2, 1), (4, 1), (12, 1), (14, 1), (30, 1), (1, -4), (2, -8))
EDGE_N = 264                              # 8 mod 32, 64, 128 and 256: the last tile holds 8 columns
NAN_ROW, NAN_SA_ROW, NAN_COL = 7, 11, 13


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)


def cluster_ctas(cfg: int) -> int:
    c = capi.configs()[cfg]
    return c["cta_group"] * c["cluster_m"] * c["cluster_n"]


def out_dtype(kind: str):
    return torch.bfloat16 if kind == "bf16" else torch.float16


def bits(c: torch.Tensor) -> np.ndarray:
    return c.view(torch.int16).cpu().numpy().view(np.uint16)


def round_bits(y: np.ndarray, kind: str) -> np.ndarray:
    with np.errstate(over="ignore"):
        return ed.round_fp16_bits(y) if kind == "fp16" else ed.round_bf16_bits(y)


def planned_splits(cfg: int, m: int, n: int, k: int, splits: int) -> int:
    """How many cluster split-K splits the launch runs (1: plain); e4m3 plans as the 16-bit problem of K / 2."""
    s = capi.schedule(cfg, m, n, k // 2, splits)
    if s["mode"] != "cluster-split-k":
        return 1
    return sum(1 for units in s["units"] for u in units if u[0] == 0)


class Case:
    """Exact-domain operands and 1D1D scales of one (M, N, K, output type), on the host and the device."""

    def __init__(self, m, n, k, kind, seed=None):
        self.m, self.n, self.k, self.kind = m, n, k, kind
        self.a, self.bt = ed.operands_e4m3(m, n, k, seed=m + 5 * n + 3 * k if seed is None else seed)
        self.sa, self.sb = ed.e4m3_block_1d1d_scales(m, n, k, kind)
        self.da = torch.from_numpy(self.a.astype(np.float32)).to(E4).cuda()
        self.dbt = torch.from_numpy(self.bt.astype(np.float32)).to(E4).cuda()
        self.exact = ed.exact_1d1d(self.a, self.bt, self.sa, self.sb)
        self.want = round_bits(self.exact, kind)

    def run(self, sa=None, sb=None, c=None, **kw) -> np.ndarray:
        sa = ds.m_major(torch, self.sa) if sa is None else sa
        sb = ds.m_major(torch, self.sb) if sb is None else sb
        if c is None:
            c = torch.full((self.m, self.n), float("nan"), dtype=out_dtype(self.kind), device="cuda")
        capi.fp8_gemm(self.da, self.dbt, c, sa, sb, **kw)
        torch.cuda.synchronize()
        return bits(c)


@functools.lru_cache(maxsize=None)
def case(m, n, k, kind) -> Case:
    return Case(m, n, k, kind)


# ------------------------------------------------------------------------------------------------ pinned launches
@pytest.mark.parametrize("kind", KINDS)
def test_steady_state_every_eligible_configuration(kind):
    c = case(*STEADY_MNK, kind)
    for cfg in ELIGIBLE:
        got = c.run(config_id=cfg, max_ctas=cluster_ctas(cfg))
        assert np.array_equal(got, c.want), (cfg, kind, first_bad(torch.from_numpy(got.view(np.int16)),
                                                                   torch.from_numpy(c.want.view(np.int16))))


@pytest.mark.parametrize("cfg", SPLIT_K)
@pytest.mark.parametrize("splits", [-2, -4, -8])
def test_cluster_split_k_full_range(cfg, splits):
    m, n, k = SPLIT_MNK
    s = planned_splits(cfg, m, n, k, splits)
    assert s == -splits
    for kind in KINDS:
        c = case(m, n, k, kind)
        got = c.run(config_id=cfg, splits=splits)
        want = ref_1d1d(c.da, c.dbt, torch.from_numpy(c.sa), torch.from_numpy(c.sb), out_dtype(kind), s)
        assert np.array_equal(want, c.want), "the C reference is not the one rounding on the exact domain"
        assert np.array_equal(got, want), (cfg, splits, kind)


@pytest.mark.parametrize("splits", UNCOMPILED)
def test_uncompiled_k_mode_requests_run_plain(splits):
    m, n, k = SPLIT_MNK
    for kind in KINDS:
        c = case(m, n, k, kind)
        for cfg in SPLIT_K:
            before = capi.fp8block_1d1d_launch_count()
            got = c.run(config_id=cfg, splits=splits)
            assert capi.fp8block_1d1d_launch_count() - before == 1, (cfg, splits)
            assert np.array_equal(got, c.run(config_id=cfg, splits=1)), (cfg, splits, kind)
            assert np.array_equal(got, c.want), (cfg, splits, kind)


def nan_mask(got: np.ndarray, kind: str) -> np.ndarray:
    if kind == "fp16":
        return np.isnan(got.view(np.float16))
    return np.isnan((got.astype(np.uint32) << 16).view(np.float32))


@pytest.mark.parametrize("cfg,splits", NONFINITE_CASES)
def test_nan_in_a_or_either_scale_makes_exactly_its_row_or_column_nan(cfg, splits):
    m, n, k = SPLIT_MNK
    s = planned_splits(cfg, m, n, k, splits)
    assert s == max(1, -splits)
    nkb = -(-k // 128)
    for kind in KINDS:
        c = case(m, n, k, kind)
        a = c.da.clone()
        a[NAN_ROW, k - 40] = float("nan")                  # inside the last split's k-range for any split count
        assert a.view(torch.uint8)[NAN_ROW, k - 40] == 0x7F
        sa, sb = c.sa.copy(), c.sb.copy()
        sa[NAN_SA_ROW, nkb // 2] = np.nan
        sb[NAN_COL, 1] = np.nan                            # an early split's k-block
        out = torch.full((m, n), float("nan"), dtype=out_dtype(kind), device="cuda")
        capi.fp8_gemm(a, c.dbt, out, ds.m_major(torch, sa), ds.m_major(torch, sb), config_id=cfg, splits=splits)
        torch.cuda.synchronize()
        got = bits(out)
        expect = np.zeros((m, n), dtype=bool)
        expect[[NAN_ROW, NAN_SA_ROW], :] = True
        expect[:, NAN_COL] = True
        assert np.array_equal(nan_mask(got, kind), expect), (cfg, splits, kind)
        assert np.array_equal(got[~expect], c.want[~expect]), (cfg, splits, kind)


@pytest.mark.parametrize("cfg,splits", GUARD_CASES)
def test_guard_bands(cfg, splits):
    m, n, k = SPLIT_MNK
    c = case(m, n, k, "fp16")
    pad = 4096
    buf = torch.full((m * n + 2 * pad,), -7.0, dtype=torch.float16, device="cuda")
    out = buf[pad:pad + m * n].view(m, n)
    out.fill_(float("nan"))
    got = c.run(c=out, config_id=cfg, splits=splits)
    assert np.array_equal(got, c.want), (cfg, splits)
    assert bool((buf[:pad] == -7).all()) and bool((buf[pad + m * n:] == -7).all()), (cfg, splits)


def test_last_tile_reads_fewer_rows_of_bt_scales():
    """N = 264: every BN leaves 8 columns in the last tile, whose bulk copy of Bt's scales holds 8 rows (ld_b = N)."""
    for kind in KINDS:
        c = case(200, EDGE_N, 8576, kind)
        for cfg in ELIGIBLE:
            bn = capi.configs()[cfg]["bn"]
            assert EDGE_N % bn == 8
            assert np.array_equal(c.run(config_id=cfg), c.want), (cfg, kind)
        for cfg in SPLIT_K:
            for splits in (-2, -4, -8):
                assert planned_splits(cfg, c.m, c.n, c.k, splits) == -splits
                assert np.array_equal(c.run(config_id=cfg, splits=splits), c.want), (cfg, splits, kind)


@pytest.mark.parametrize("cfg", [1, 4, 12, 14, 30])
def test_row_stride_of_bt_scales(cfg):
    c = case(200, EDGE_N, 1040, "fp16")
    for ld_b in (EDGE_N, EDGE_N + 4, 4096):
        sb = ds.m_major(torch, c.sb, ld=ld_b)              # NaN in the padding rows: never read into an output
        assert sb.stride() == (1, ld_b)
        assert np.array_equal(c.run(sb=sb, config_id=cfg), c.want), (cfg, ld_b)


@pytest.mark.parametrize("m", [1, 193])
def test_m_1_and_1_mod_64(m):
    for kind in KINDS:
        c = case(m, 392, 1040, kind)
        for cfg in ELIGIBLE:
            assert np.array_equal(c.run(config_id=cfg), c.want), (m, cfg, kind)
        assert np.array_equal(c.run(), c.want), (m, kind)


def _scale_variants(c: Case):
    """Exact-domain scale pairs other than the case's own: its rows rolled."""
    for v in (1, 5, 8):
        yield np.roll(c.sa, v, axis=0), np.roll(c.sb, v, axis=0)


def test_scales_written_just_before_the_gemm_are_the_ones_used():
    c = case(256, 392, 1040, "fp16")
    sa, sb = ds.m_major(torch, c.sa), ds.m_major(torch, c.sb)
    ops.fp8_gemm(c.da, c.dbt, sa, sb, torch.float16)
    for new_a, new_b in _scale_variants(c):
        sa.copy_(torch.from_numpy(new_a)); sb.copy_(torch.from_numpy(new_b))   # torch kernels, same stream, just before
        y = ops.fp8_gemm(c.da, c.dbt, sa, sb, torch.float16)
        assert np.array_equal(bits(y), round_bits(ed.exact_1d1d(c.a, c.bt, new_a, new_b), "fp16"))


@pytest.mark.parametrize("mnk", [(512, 512, 8192), (256, 392, 1040)])
def test_graph_replay_reads_the_current_scales(mnk):
    c = case(*mnk, "bf16")
    sa, sb = ds.m_major(torch, c.sa), ds.m_major(torch, c.sb)
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        y = ops.fp8_gemm(c.da, c.dbt, sa, sb, torch.bfloat16)
    for new_a, new_b in _scale_variants(c):
        sa.copy_(torch.from_numpy(new_a)); sb.copy_(torch.from_numpy(new_b))
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(bits(y), round_bits(ed.exact_1d1d(c.a, c.bt, new_a, new_b), "bf16")), mnk


# ------------------------------------------------------------------------------------------------ the dispatched call
def run_dispatched(leg: str, m: int, n: int, k: int):
    """The dispatched 1D1D call of ``leg`` on (M, N, K): None, or a failure report."""
    spec = ds.TRAIN_LEGS[leg]
    seed = ds.shape_seed(m, n, k)
    out = spec["out"]
    operands = ds.operands_e4m3(torch, m, n, k, seed)
    sa_t, sb_t, sa, sb = ds.e4m3_scales(torch, "block_1d1d", m, n, k, out, seed)
    buf, c = guarded(m, n, out)
    capi.fp8_gemm(operands.a, operands.bt, c, sa_t, sb_t)
    got = c.view(torch.int16)
    errs = [] if guards_intact(buf) else ["guard band written"]
    total, first = 0, None
    rows, cols = ds.sample_rows(m, operands.probe_rows.tolist(), seed), ds.sample_cols(n, seed)
    want_rows = {}
    for lo, hi, want in ds.reference_blocks(torch, operands, out, (sa, sb), "block_1d1d"):
        cnt, fb = first_bad(got[lo:hi], want)
        if cnt and first is None:
            first = (fb[0] + lo,) + fb[1:]
        total += cnt
        for r in rows:
            if lo <= r < hi:
                want_rows[r] = want[r - lo, cols].cpu().numpy().view(np.uint16)
    if total:
        errs.append(f"{total} mismatches, first (row, col, got, want) {first}")
    host = ds.numpy_rows(torch, operands, rows, cols, out, (sa, sb), "block_1d1d")
    if not np.array_equal(np.stack([want_rows[r] for r in rows]), host):
        errs.append(f"device reference differs from numpy at rows {rows}")
    if not errs:
        return None
    cfg, gm, sp = ds.choice(leg, m, n, k)
    mode, _ = ds.plan(leg, cfg, m, n, k, sp)
    return f"{(m, n, k)}: cfg {cfg} group_m {gm} splits {sp} -> {mode}: " + "; ".join(errs)


@pytest.mark.parametrize("leg,shapes", [(leg, lst) for leg in ds.TRAIN_LEGS for lst in ds.TRAIN_LEG_LISTS[leg]]
                         + [("e4m3_1d1d_bf16", "dw")])
def test_dispatched_1d1d_call_is_exact(leg, shapes):
    lst = {"grid": ds.grid_shapes, "offgrid": lambda: ds.offgrid_shapes(leg), "dw": ds.dw_shapes}[shapes]()
    failures = []
    t0 = time.perf_counter()
    for m, n, k in lst:
        r = run_dispatched(leg, m, n, k)
        if r:
            failures.append(r)
    torch.cuda.synchronize()
    print(f"\nSWEEP {leg} {shapes}: {len(lst)} shapes in {time.perf_counter() - t0:.1f} s, {len(failures)} failing")
    assert not failures, f"{leg} {shapes}: {len(failures)} shapes fail:\n" + "\n".join(failures[:40])


# ------------------------------------------------------------------------------------------------ production scale
@pytest.fixture
def scale_case(request):
    c = sc.CASES[request.param]
    torch.cuda.empty_cache()
    need = c.memory_bytes()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"case {c.name} needs {need} bytes of device memory, {free} are free")
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield c
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print(f"\nSCALE {c.name}: {time.perf_counter() - t0:.1f} s, peak {peak / 2 ** 30:.2f} GiB "
          f"(budget {need / 2 ** 30:.2f} GiB)")
    torch.cuda.empty_cache()
    assert peak <= need, (c.name, peak, need)


def _fill_1d1d(d: dict, m: int, n: int, seed: int):
    """Exact-domain e4m3 operands and power-of-two 1D1D scales: (scale_a, scale_b) as [M, nkb] / [N, nkb] views."""
    dom = sc.DOMAINS["e4m3"]
    sc.fill_ints_(d["a"], dom["a"], sc.generator(seed))
    sc.fill_ints_(d["bt"], dom["b"], sc.generator(seed + 1))
    sc.pow2_scales_(d["sa"], sc.generator(seed + 2))
    sc.pow2_scales_(d["sb"], sc.generator(seed + 3))
    return d["sa"][:, :m].t(), d["sb"][:, :n].t()


def _scaled64(x, s, r0, r1, k0, k1):
    """Rows [r0, r1), k [k0, k1) of e4m3 ``x`` times its 1 x 128 scales ``s`` [R, nkb], float64 (k0 % 128 == 0)."""
    y = x[r0:r1, k0:k1].to(torch.float64)
    y.mul_(sc.block_expand(s[r0:r1, k0 // 128:-(-k1 // 128)], r1 - r0, k1 - k0))
    return y


@pytest.mark.parametrize("scale_case", ["fp8_dw"], indirect=True)
def test_weight_gradient_with_a_past_2_31_bytes(scale_case):
    """K = dual_ld_t of FP8_DW_TOKENS: A [M, K] passes 2^31 bytes; every k-block sum and every promotion stays exact
    (at most 128 unit products per k-block, power-of-two scales, sum_k |p| 2^2 < 2^24), bf16 out."""
    d = sc.allocate(scale_case)
    m, n, k = sc.FP8_DW
    sa, sb = _fill_1d1d(d, m, n, 70)
    nnz = max(int((d["a"][r0:r0 + 8].float() != 0).sum(1).max()) for r0 in range(0, m, 8))   # -0.0 is no nonzero
    assert nnz * 16 < 2 ** 24, nnz                         # |sum| / smallest unit, with scale ratios up to 2^4
    capi.fp8_gemm(d["a"], d["bt"], d["c"], sa, sb)
    kc = max(128, (sc.BAND_BYTES // (8 * max(m, n))) // 128 * 128)

    def ref(r0, r1):
        out = torch.zeros((r1 - r0, n), dtype=torch.float64, device="cuda")
        for k0 in range(0, k, kc):
            k1 = min(k, k0 + kc)
            b = _scaled64(d["bt"], sb, 0, n, k0, k1)
            out.addmm_(_scaled64(d["a"], sa, r0, r1, k0, k1), b.t())
            del b
        return out
    torch.cuda.synchronize()
    msg = sc.first_mismatch(d["c"], ref, what="1D1D weight gradient, A past 2^31 bytes")
    assert msg is None, msg
    assert sc.guards_intact(d["c:buf"])


@pytest.mark.parametrize("scale_case", ["fp8_dw_out"], indirect=True)
def test_1d1d_output_past_2_31(scale_case):
    d = sc.allocate(scale_case)
    m, n, k = sc.TN
    sa, sb = _fill_1d1d(d, m, n, 80)
    capi.fp8_gemm(d["a"], d["bt"], d["c"], sa, sb)
    bt = _scaled64(d["bt"], sb, 0, n, 0, k)               # scales folded in: exact

    def ref(r0, r1):
        return sc.matmul64(_scaled64(d["a"], sa, r0, r1, 0, k), bt.t())
    torch.cuda.synchronize()
    msg = sc.first_mismatch(d["c"], ref, what="1D1D, C past 2^31 elements")
    assert msg is None, msg
    assert sc.guards_intact(d["c:buf"])


def _quant_outputs(d: dict, kind: str, rows: int, cols: int):
    """The kernel call of quantiser ``kind`` on d["x"], writing into the case's buffers, and its results as the
    reference lays them out: {result: view}."""
    nkb = lambda c: -(-c // 128)
    ld = lambda r: -(-r // 4) * 4
    flat_s, flat_t = d["scale"].view(-1), d["scale_t"].view(-1)
    m_major = lambda flat, r, c: flat[:nkb(c) * ld(r)].view(nkb(c), ld(r))[:, :r].t()
    x, q, ld_t = d["x"], d["q"], capi.dual_ld_t(rows)
    if kind == "tensor":
        out = {"q": q, "scale": flat_s[:1]}
        capi.quantize_e4m3(x, q, out["scale"], d["workspace"][:capi.QUANT_TENSOR_WORKSPACE])
    elif kind == "rowwise":
        out = {"q": q, "scale": flat_s[:rows].view(rows, 1)}
        capi.quantize_e4m3_rowwise(x, q, out["scale"])
    elif kind == "blockwise":
        out = {"q": q, "scale": m_major(flat_s, rows, cols)}
        capi.quantize_e4m3_blockwise(x, q, out["scale"])
    elif kind == "silu_mul":
        i = cols // 2
        out = {"q": q.view(-1)[:rows * i].view(rows, i), "scale": m_major(flat_s, rows, i)}
        capi.silu_mul_quantize_e4m3_blockwise(x, out["q"], out["scale"])
    elif kind == "rowwise_dual":
        out = {"q": q, "scale": flat_s[:rows], "q_t": d["q_t"], "scale_t": flat_t[:cols]}
        capi.quantize_e4m3_rowwise_dual(x, q, out["scale"], d["q_t"], out["scale_t"],
                                        d["workspace"][:capi.quant_dual_workspace(rows, cols)])
    elif kind == "blockwise_dual":
        out = {"q": q, "scale": m_major(flat_s, rows, cols), "q_t": d["q_t"], "scale_t": m_major(flat_t, cols, rows)}
        capi.quantize_e4m3_blockwise_dual(x, q, out["scale"], d["q_t"], out["scale_t"])
    else:
        nr, nc = nkb(rows), nkb(cols)
        out = {"q": q, "scale": flat_s[:nr * nc].view(nr, nc), "q_t": d["q_t"].view(-1)[:cols * rows].view(cols, rows),
               "scale_t": flat_t[:nc * nr].view(nc, nr)}
        capi.quantize_e4m3_block128x128_dual(x, q, out["scale"], out["q_t"], out["scale_t"])
    assert "q_t" not in out or out["q_t"].shape[1] in (ld_t, rows)
    return out


def _all_sentinel(b: torch.Tensor, chunk: int = 1 << 28) -> bool:
    """Whether every byte of ``b`` (uint8) holds the e4m3 sentinel, checked in chunks (no full-size temporary)."""
    s = sc.SENTINEL[torch.float8_e4m3fn]
    return all(bool((b[i:i + chunk] == s).all()) for i in range(0, b.numel(), chunk))


def _raw(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.uint8) if t.element_size() == 1 else t.view(torch.int32)


@pytest.mark.parametrize("scale_case", ["quant"], indirect=True)
def test_every_quantiser_on_an_input_past_2_31_elements(scale_case):
    """One bf16 activation past 2^31 elements through every quantiser that takes it, in turn. Each writes into the same
    guarded q / q_t buffers (refilled with the sentinel first) and scale buffers; every result is compared bit for bit
    with its torch reference applied in row bands (scale_cases.quant_bands), and every byte of q's and q_t's buffers
    that the call does not own must keep the sentinel."""
    d = sc.allocate(scale_case)
    rows, cols = sc.QUANT
    x = d["x"]
    x.normal_(generator=sc.generator(90))
    x[::97].mul_(1000)                                    # outlier rows, and whole 128-row groups' scales move with them
    x[:, 5::211].mul_(1e-3)                               # small columns: the transposed copies' scales differ widely
    band = sc.quant_band_rows(cols)
    for kind in sc.QUANTISERS:
        for name in ("q", "q_t"):
            d[f"{name}:buf"].view(torch.uint8).fill_(sc.SENTINEL[torch.float8_e4m3fn])
        d["scale"].fill_(float("nan")); d["scale_t"].fill_(float("nan"))
        t0 = time.perf_counter()
        out = _quant_outputs(d, kind, rows, cols)
        torch.cuda.synchronize()
        ran = time.perf_counter() - t0
        failures = []
        for name, idx, want in sc.quant_bands(kind, x, band):
            got = out[name][idx]
            bad = _raw(got) != _raw(want.contiguous())
            if bool(bad.any()):
                j = [int(v) for v in bad.nonzero()[0]]
                failures.append(f"{name}{[(s.start, s.stop) for s in idx]}: {int(bad.sum())} differ, first at {j}")
                if len(failures) > 5:
                    break
        for name in ("q", "q_t"):                        # the bytes of the guarded buffers the call does not own
            buf, view = d[f"{name}:buf"].view(torch.uint8), out.get(name)
            start = 0 if view is None else view.data_ptr() - buf.data_ptr()
            end = start if view is None else start + view.numel()
            if not (_all_sentinel(buf[:start]) and _all_sentinel(buf[end:])):
                failures.append(f"{name}: a byte outside the result was written")
        print(f"\nSCALE quant {kind}: kernel {ran:.2f} s")
        assert not failures, f"{kind}: " + "; ".join(failures)
