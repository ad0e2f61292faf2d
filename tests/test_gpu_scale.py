"""Every kernel family at production scale, where a 32-bit element or byte index would wrap, bit-exact against a
float64 reference over the whole output (scale_cases.py: the cases, operands, reference and guard bands).

Each case's outputs live inside NaN-sentinel guard bands, which must be intact afterwards; an element never written
keeps the sentinel, which no exact-domain result equals. A case needs up to about 14 GB of device memory
(``Case.memory_bytes``, asserted against torch's peak) and is skipped, naming the bytes, when the device has less
free. Run with ``-s`` to see each case's wall time and peak memory.
"""
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import pytest
import torch

import scale_cases as sc
from cuda_l2_b200 import capi

pytestmark = pytest.mark.gpu

HERE = Path(__file__).resolve().parent
VARIANTS16 = {"fp16": (torch.float16, "fp32"), "fp16acc16": (torch.float16, "fp16"), "bf16": (torch.bfloat16, "fp32")}
# pinned configurations of the 2-D TN case (each asserted to run its K-mode in test_scale_cpu.py)
TN_PINNED = ((3, 1, "plain"), (10, 1, "plain"), (0, capi.STREAMK_TAIL_PLUS_WAVE, "stream-k"))
# pinned cluster split-K and stream-K of the NN long reduction, run through B200_HGEMM_FORCE in a child process
NN_LONG_PINNED = ((1, -4, "cluster-split-k"), (0, capi.STREAMK_TAIL, "stream-k"))


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        pytest.skip("needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)
    free, total = torch.cuda.mem_get_info()
    print(f"\nSCALE device {torch.cuda.get_device_name(0)}: {free / 2 ** 30:.1f} GiB free of {total / 2 ** 30:.1f}")


@pytest.fixture
def case(request):
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


def cases(*names):
    return pytest.mark.parametrize("case", names, indirect=True)


def expect_equal(out, ref_rows, **kw):
    torch.cuda.synchronize()
    msg = sc.first_mismatch(out, ref_rows, **kw)
    assert msg is None, msg


def t_of(x):
    return x.t()


# ------------------------------------------------------------------------------------------------------ 2-D
@cases("tn")
def test_2d_tn_output_past_2_31(case):
    d = {}
    for i, (variant, (dtype, acc)) in enumerate(VARIANTS16.items()):
        d = sc.allocate(case, dtype)
        dom = sc.DOMAINS[variant]
        sc.fill_ints_(d["a"], dom["a"], sc.generator(10 + i))
        sc.fill_ints_(d["bt"], dom["b"], sc.generator(20 + i))
        runs = [(None, 1)] + ([(cfg, sp) for cfg, sp, _ in TN_PINNED] if variant == "fp16" else [])
        for cfg, sp in runs:
            d["c:buf"].view(torch.int16).fill_(sc.SENTINEL[dtype])
            kw = {} if cfg is None else dict(config_id=cfg, splits=sp)
            capi.gemm_kmajor(d["a"], d["bt"], d["c"], acc, **kw)
            expect_equal(d["c"], lambda r0, r1: sc.matmul64(d["a"][r0:r1], d["bt"].t()), what=f"{variant} {kw}")
            assert sc.guards_intact(d["c:buf"]), (variant, kw)
        del d


@cases("nn")
def test_2d_nn_output_past_2_31(case):
    for i, variant in enumerate(("fp16", "bf16")):
        dtype, acc = VARIANTS16[variant]
        d = sc.allocate(case, dtype)
        dom = sc.DOMAINS[variant]
        sc.fill_ints_(d["a"], dom["a"], sc.generator(30 + i))
        sc.fill_ints_(d["b"], dom["b"], sc.generator(40 + i))
        capi.gemm_rowmajor(d["a"], d["b"], d["c"], acc)
        expect_equal(d["c"], lambda r0, r1: sc.matmul64(d["a"][r0:r1], d["b"]), what=variant)
        assert sc.guards_intact(d["c:buf"]), variant
        del d


@cases("block")
def test_block_scaled_2d_output_past_2_31(case):
    d = sc.allocate(case)
    m, n, k = sc.TN
    dom = sc.DOMAINS["e4m3"]
    sc.fill_ints_(d["a"], dom["a"], sc.generator(50))
    sc.fill_ints_(d["bt"], dom["b"], sc.generator(51))
    sc.pow2_scales_(d["sa"], sc.generator(52))
    sc.pow2_scales_(d["sb"], sc.generator(53))
    sa = d["sa"][:, :m].t()                                  # M-major [M, nkb]
    capi.fp8_gemm(d["a"], d["bt"], d["c"], sa, d["sb"])
    bt = d["bt"].to(torch.float64).mul_(sc.block_expand(d["sb"], n, k, 128))   # scales folded in: exact

    def ref(r0, r1):
        return sc.matmul64(d["a"][r0:r1].to(torch.float64) * sc.block_expand(sa[r0:r1], r1 - r0, k), bt.t())
    expect_equal(d["c"], ref, what="block-scaled")
    assert sc.guards_intact(d["c:buf"])


@cases("tall")
def test_2d_tn_operand_past_2_31(case):
    d = sc.allocate(case)
    dom = sc.DOMAINS["tall"]
    sc.fill_ints_(d["a"], dom["a"], sc.generator(60))
    sc.fill_ints_(d["bt"], dom["b"], sc.generator(61))
    capi.gemm_kmajor(d["a"], d["bt"], d["c"], "fp32")
    expect_equal(d["c"], lambda r0, r1: sc.matmul64(d["a"][r0:r1], d["bt"].t()), what="tall A")
    assert sc.guards_intact(d["c:buf"])


def nn_long_runs(variants=("fp16", "bf16")) -> list:
    """The NN long-reduction case for each variant with the dispatcher's choice (or B200_HGEMM_FORCE's): mismatch
    messages, None where bit-exact and the guards intact."""
    case = sc.CASES["nn_long"]
    out = []
    for i, variant in enumerate(variants):
        dtype, acc = VARIANTS16[variant]
        d = sc.allocate(case, dtype)
        dom = sc.DOMAINS["nn_long"]
        sc.fill_ints_(d["a"], dom["a"], sc.generator(70 + i))
        sc.fill_ints_(d["b"], dom["b"], sc.generator(80 + i))
        assert float(d["a"].float().sum(1).max()) < 65504        # every sum below fp16's largest finite value
        capi.gemm_rowmajor(d["a"], d["b"], d["c"], acc)
        torch.cuda.synchronize()
        msg = sc.first_mismatch(d["c"], lambda r0, r1: sc.matmul64(d["a"][r0:r1], d["b"]), what=variant)
        out.append(msg or (None if sc.guards_intact(d["c:buf"]) else f"{variant}: guard band overwritten"))
        del d
        torch.cuda.empty_cache()
    return out


CHILD = """
import json, sys
sys.path.insert(0, {tests!r}); sys.path.insert(0, {repo!r})
import torch
torch.cuda.set_device(0)
import test_gpu_scale as t
print("RESULT " + json.dumps(t.nn_long_runs()))
"""


@cases("nn_long")
def test_nn_long_reduction_operand_past_2_31(case):
    assert nn_long_runs() == [None, None]
    torch.cuda.empty_cache()
    for cfg, splits, mode in NN_LONG_PINNED:
        env = dict(os.environ, B200_HGEMM_FORCE=f"{cfg},0,{splits}")
        env.pop("B200_HGEMM_TABLE", None)
        r = subprocess.run([sys.executable, "-c", CHILD.format(tests=str(HERE), repo=str(HERE.parent))], env=env,
                           capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-4000:]
        assert json.loads(r.stdout.split("RESULT ", 1)[1]) == [None, None], (cfg, splits, mode)


# ------------------------------------------------------------------------------------------------------ batched
@cases("batched")
def test_batched_output_past_2_31(case):
    b, m, k = case.tensor("a").shape
    for i, (variant, masked) in enumerate((("fp16", False), ("bf16", True))):
        dtype, acc = VARIANTS16[variant]
        d = sc.allocate(case, dtype)
        dom = sc.DOMAINS[variant]
        sc.fill_ints_(d["a"], dom["a"], sc.generator(90 + i))
        sc.fill_ints_(d["bt"], dom["b"], sc.generator(95 + i))
        counts = sc.masked_counts(b, m, seed=5) if masked else [m] * b
        d["masked_m"].copy_(torch.tensor(counts, dtype=torch.int32))
        capi.gemm_batched(d["a"], d["bt"], d["c"], acc, masked_m=d["masked_m"] if masked else None)
        torch.cuda.synchronize()
        n = d["c"].shape[2]
        for j in range(b):
            rows = min(max(counts[j], 0), m)
            expect_equal(d["c"][j], lambda r0, r1, j=j: sc.matmul64(d["a"][j, r0:r1], d["bt"][j].t()), rows=rows,
                         base=j * m * n, what=f"{variant} batch {j} (count {counts[j]})")
        assert sc.guards_intact(d["c:buf"]), variant
        del d


# ------------------------------------------------------------------------------------------------------ grouped
def fill_grouped(case, dtype, seed):
    d = sc.allocate(case, dtype)
    dom = sc.DOMAINS["fp16" if dtype == torch.float16 else "bf16"]
    sc.fill_ints_(d["a"], dom["a"], sc.generator(seed))
    sc.fill_ints_(d["bt" if "bt" in d else "b"], dom["b"], sc.generator(seed + 1))
    ends = sc.group_ends(sc.histogram("grouped"))
    d["offs"].copy_(torch.tensor(ends, dtype=torch.int32))
    return d, ends


@cases("grouped")
def test_grouped_forward_output_past_2_31(case):
    d, ends = fill_grouped(case, torch.float16, 100)
    capi.gemm_grouped(d["a"], d["bt"], d["c"], d["offs"], "fp32")
    expect_equal(d["c"], sc.grouped_rows(d["a"], lambda g: d["bt"][g].t(), ends), what="grouped")
    assert sc.guards_intact(d["c:buf"])


@cases("grouped_nn")
def test_grouped_nn_output_past_2_31(case):
    d, ends = fill_grouped(case, torch.bfloat16, 110)
    capi.gemm_grouped_nn(d["a"], d["b"], d["c"], d["offs"])
    expect_equal(d["c"], sc.grouped_rows(d["a"], lambda g: d["b"][g], ends), what="grouped NN")
    assert sc.guards_intact(d["c:buf"])


@cases("wgrad")
def test_grouped_wgrad_output_past_2_32(case):
    d = sc.allocate(case)
    dom = sc.DOMAINS["wgrad"]
    sc.fill_ints_(d["dy"], dom["a"], sc.generator(120))
    sc.fill_ints_(d["x"], dom["b"], sc.generator(121))
    ends = sc.group_ends(sc.histogram("wgrad"))
    d["offs"].copy_(torch.tensor(ends, dtype=torch.int32))
    capi.gemm_grouped_wgrad(d["dy"], d["x"], d["c"], d["offs"])
    torch.cuda.synchronize()
    _, m, n = d["c"].shape
    for g, (s, e) in enumerate(zip([0] + ends[:-1], ends)):
        expect_equal(d["c"][g], lambda r0, r1, s=s, e=e: sc.matmul64(d["dy"][s:e, r0:r1].t(), d["x"][s:e]),
                     base=g * m * n, boundary=2 ** 31 if g < 200 else 2 ** 32, what=f"group {g} ({e - s} rows)")
    assert sc.guards_intact(d["c:buf"])
    # T == 0: the same output zero-filled, no kernel launched
    before = capi.grouped_bwd_launch_count()
    d["offs"].zero_()
    capi.gemm_grouped_wgrad(d["dy"][:0], d["x"][:0], d["c"], d["offs"])
    torch.cuda.synchronize()
    assert capi.grouped_bwd_launch_count() == before
    assert not bool(d["c"].view(torch.int16).any())
    assert sc.guards_intact(d["c:buf"])


@cases("wgrad_long")
def test_grouped_wgrad_long_reductions_operand_past_2_31(case):
    d = sc.allocate(case)
    dom = sc.DOMAINS["wgrad_long"]
    sc.fill_ints_(d["dy"], dom["a"], sc.generator(130))
    sc.fill_ints_(d["x"], dom["b"], sc.generator(131))
    ends = sc.group_ends(sc.WGRAD_LONG_SIZES)
    d["offs"].copy_(torch.tensor(ends, dtype=torch.int32))
    capi.gemm_grouped_wgrad(d["dy"], d["x"], d["c"], d["offs"])
    torch.cuda.synchronize()
    _, m, n = d["c"].shape
    for g, (s, e) in enumerate(zip([0] + ends[:-1], ends)):
        expect_equal(d["c"][g], lambda r0, r1, s=s, e=e: sc.matmul64(d["dy"][s:e, r0:r1].t(), d["x"][s:e]),
                     base=g * m * n, what=f"group {g} ({e - s} rows)")
    assert sc.guards_intact(d["c:buf"])


# ------------------------------------------------------------------------------------------------------ FP8 experts
@cases("fp8_experts")
def test_fp8_expert_stack_past_2_32_bytes(case):
    d = sc.allocate(case)
    e = sc.FP8_EXPERTS
    g, n, k, t, slots = e["g"], e["n"], e["k"], e["t"], e["slots"]
    dom = sc.DOMAINS["e4m3"]
    sc.fill_ints_(d["bt"], dom["b"], sc.generator(140))
    sc.fill_ints_(d["a"], dom["a"], sc.generator(141))
    sc.fill_ints_(d["ab"], dom["a"], sc.generator(142))
    for name, seed in (("sb", 143), ("sa", 144), ("sab", 145)):
        sc.pow2_scales_(d[name], sc.generator(seed))
    for x in (d["a"], d["ab"].view(-1, k)):                  # the e4m3 domain: at most 2047 nonzeros per row of A
        assert int((x.view(torch.uint8) & 0x7F).ne(0).sum(1).max()) <= 2047
    ends = sc.group_ends(sc.histogram("fp8_experts"))
    d["offs"].copy_(torch.tensor(ends, dtype=torch.int32))
    counts = sc.masked_counts(g, slots, seed=6)
    d["masked_m"].copy_(torch.tensor(counts, dtype=torch.int32))
    sa, sab = d["sa"].t(), d["sab"].transpose(1, 2)          # M-major [T, nkb] and [G, slots, nkb]
    capi.fp8_grouped_gemm(d["a"], d["bt"], d["c"], sa, d["sb"], d["offs"])
    capi.fp8_batched_gemm(d["ab"], d["bt"], d["cb"], sab, d["sb"], masked_m=d["masked_m"])
    torch.cuda.synchronize()
    got_rows = [int(v) for v in torch.tensor(ends).diff(prepend=torch.tensor([0]))]
    assert got_rows[117] > 0 and got_rows[234] > 0
    scaled = {}

    def bt64(j):   # expert j's weight with its block scales folded in (exact), one expert at a time
        if j not in scaled:
            scaled.clear()
            scaled[j] = d["bt"][j].to(torch.float64).mul_(sc.block_expand(d["sb"][j], n, k, 128)).t()
        return scaled[j]

    def a64(x, s, r0, r1):
        return x[r0:r1].to(torch.float64) * sc.block_expand(s[r0:r1], r1 - r0, k)

    starts = [0] + ends[:-1]

    def grouped_ref(r0, r1):
        out = torch.empty((r1 - r0, n), dtype=torch.float64, device="cuda")
        for j, (s, en) in enumerate(zip(starts, ends)):
            lo, hi = max(s, r0), min(en, r1)
            if lo < hi:
                out[lo - r0:hi - r0] = sc.matmul64(a64(d["a"], sa, lo, hi), bt64(j))
        return out
    expect_equal(d["c"], grouped_ref, what="fp8 grouped")
    for j in range(g):
        rows = min(max(counts[j], 0), slots)
        expect_equal(d["cb"][j], lambda r0, r1, j=j: sc.matmul64(a64(d["ab"][j], sab[j], r0, r1), bt64(j)),
                     rows=rows, what=f"fp8 batched expert {j} (count {counts[j]})")
    assert sc.guards_intact(d["c:buf"]) and sc.guards_intact(d["cb:buf"])
