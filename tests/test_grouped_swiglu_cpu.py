"""The grouped SwiGLU library (libb200_grouped_swiglu.so) without a GPU: exports against the ABI table and the internal
header, the build entry, the kernel count, registers and local memory against the Grouped<> kernels the gated ones
wrap, every (configuration, variant) through run_config in a process that sees no device, the dispatcher's choice,
argument statuses in order before any CUDA call, the stacked gate / up weight layout, and the layer on the meta
device."""
import json
import os
import re
import shutil
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from conftest import REPO
from cuda_l2_b200 import build, capi, ops

KNULL, KBADSHAPE, KBADALIGN, KBADCONFIG, KNOTHOPPER, KBADWIDTH, KBADDTYPE = -5, -1, -2, -6, -7, -14, -15
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
CUFILT = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
X, W, H, Y, OFFS = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000   # fake, never dereferenced addresses
HEADER = build.CSRC / "b200_grouped_swiglu.h"
GATED_BN = (128, 256)


@pytest.fixture(scope="module")
def libs(built_libs):
    return built_libs


def _exports(path) -> list[str]:
    out = subprocess.run(["nm", "-D", "--defined-only", str(path)], capture_output=True, text=True, check=True).stdout
    return [line.split()[-1] for line in out.splitlines() if line.strip()]


def test_exports_are_the_table_and_the_internal_header(libs):
    table = capi.INTERNAL_ABI[capi.GROUPED_SWIGLU_LIB]
    names = _exports(libs["grouped_swiglu"])
    assert not [s for s in names if s.startswith("b200_")]
    assert sorted(s for s in names if s.startswith("cuda_l2_b200_")) == sorted(table)
    assert all(s.startswith("cuda_l2_b200_grouped_swiglu_") for s in table)
    assert capi.GROUPED_SWIGLU_LIB not in capi.ABI
    assert not any("grouped_swiglu" in h.read_text() for h in (REPO / "include").glob("*.h"))
    text = re.sub(r"//[^\n]*", "", HEADER.read_text())
    protos = dict(re.findall(r"(cuda_l2_b200_grouped_swiglu_\w+)\(([^)]*)\);", text))
    assert sorted(protos) == sorted(table)
    for sym, params in protos.items():
        count = 0 if params.strip() in ("", "void") else params.count(",") + 1
        assert count == len(table[sym][0]), sym


def test_build_entry():
    name, objects, link_flags = build.LIBRARIES["grouped_swiglu"]
    assert name == capi.GROUPED_SWIGLU_LIB and link_flags == []
    assert [(src.name, defines) for src, defines in objects] == \
        [("b200_grouped_swiglu.cu", [f"-DB200_VARIANT={v}"]) for v in (0, 2)]


def _resources(path) -> dict:
    """{demangled kernel name without parameters: (registers, stack bytes, local bytes)} from cuobjdump -res-usage."""
    out = subprocess.run([CUOBJDUMP, "-res-usage", str(path)], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    res = {}
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            res[m.group(1)] = tuple(int(re.search(k + r":(\d+)", lines[i + 1]).group(1)) for k in ("REG", "STACK", "LOCAL"))
    names = subprocess.run([CUFILT], input="\n".join(res), capture_output=True, text=True, check=True).stdout.splitlines()
    out = {}
    for d, v in zip(names, res.values()):
        depth = 0
        for i, ch in enumerate(d):
            depth += (ch == "<") - (ch == ">")
            if ch == "(" and depth == 0 and i > 0 and d[i - 1] == ">":
                d = d[:i]
                break
        out[re.sub(r"\((?:int|bool)\)", "", d).replace("void ", "", 1)] = v
    return out


@pytest.mark.skipif(not Path(CUOBJDUMP).exists(), reason="cuobjdump not available")
def test_kernel_count_registers_and_local_memory_against_the_grouped_kernels(libs):
    """18 gated grouped kernels per variant (the BN = 128 and 256 configurations) and the backward kernel of each
    variant; no gated grouped kernel uses more than 168 registers, nor more stack or local memory than the Grouped<>
    kernel of its configuration in libb200_grouped.so."""
    res = _resources(libs["grouped_swiglu"])
    gated = {k: v for k, v in res.items() if k.startswith("b200::hgemm_grouped_gated_kernel<")}
    backward = [k for k in res if "grouped_swiglu_backward_kernel" in k]
    assert len(gated) == 36 and len(backward) == 2 and len(res) == 38
    grouped = _resources(libs["grouped"])
    for name, (regs, stack, local) in gated.items():
        m = re.fullmatch(r"b200::hgemm_grouped_gated_kernel<b200::Gated<b200::Grouped<(b200::Config<[^>]*>)>>, 0>", name)
        assert m, name
        sib = grouped[f"b200::hgemm_tn_kernel<b200::Grouped<{m.group(1)}>, 0>"]
        assert regs <= 168, name
        assert stack <= sib[1] and local <= sib[2], (name, (stack, local), sib)


def _sibling(cfgs: list[dict], cid: int) -> int:
    """gated::sibling, written again: itself for BN = 128 / 256, else the BN = 128 configuration with the same CTA
    group and M_REP and the largest cluster no wider in M or N."""
    c = cfgs[cid]
    if c["bn"] in GATED_BN:
        return cid
    cands = [d for d in cfgs if d["bn"] == 128 and d["cta_group"] == c["cta_group"] and d["m_rep"] == c["m_rep"] and
             d["cluster_m"] <= c["cluster_m"] and d["cluster_n"] <= c["cluster_n"]]
    return max(cands, key=lambda d: (d["cluster_m"] * d["cluster_n"], -d["id"]))["id"]


def _run_config(cfg, variant=0, x=X, w=W, h=H, y=Y, offs=OFFS, g=4, t=64, i=64, k=64):
    return capi.grouped_swiglu_lib().cuda_l2_b200_grouped_swiglu_run_config(variant, cfg, x, w, h, y, offs, g, t, i, k,
                                                                             0, 0, None)


# Every (configuration, variant) through cuda_l2_b200_grouped_swiglu_run_config on fake addresses, in a process that sees
# no device: a configuration with a gated kernel gets as far as the device query (kNotHopper), one without is kBadConfig.
_NO_DEVICE = """
import json, sys
sys.path.insert(0, {repo!r})
from cuda_l2_b200 import capi
lib = capi.grouped_swiglu_lib()
out = []
for variant in (0, 2):
    for cfg in range(-1, 32):
        st = lib.cuda_l2_b200_grouped_swiglu_run_config(variant, cfg, {x}, {w}, {h}, {y}, {offs}, 4, 64, 64, 64, 0, 0,
                                                        None)
        out.append([variant, cfg, st])
print(json.dumps(out))
"""


def test_every_configuration_and_variant_maps_to_a_gated_kernel(libs):
    """All 31 configurations in both variants: those with BN = 128 or 256 have a gated grouped kernel, the others are
    kBadConfig, and their sibling is a BN = 128 one. The launches run on fake addresses, so they run in a process with
    CUDA_VISIBLE_DEVICES="", where a launch with a kernel stops at the device query (kNotHopper) on any machine. In this
    process only the refusals are called: kBadConfig comes back before any CUDA call."""
    cfgs = capi.configs()
    assert len(cfgs) == 31
    r = subprocess.run([sys.executable, "-c", _NO_DEVICE.format(repo=str(REPO), x=X, w=W, h=H, y=Y, offs=OFFS)],
                       capture_output=True, text=True, timeout=300, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-2000:]
    seen = json.loads(r.stdout)
    assert len(seen) == 2 * 33
    for variant, cfg, st in seen:
        gated = 0 <= cfg < 31 and cfgs[cfg]["bn"] in GATED_BN
        assert st == (KNOTHOPPER if gated else KBADCONFIG), (variant, cfg, st)
    for c in cfgs:
        if c["bn"] not in GATED_BN:
            assert _run_config(c["id"]) == KBADCONFIG and _run_config(c["id"], variant=2) == KBADCONFIG, c
        s = cfgs[_sibling(cfgs, c["id"])]
        assert s["bn"] in GATED_BN and s["cta_group"] == c["cta_group"] and s["m_rep"] == c["m_rep"]
    assert _run_config(31) == KBADCONFIG and _run_config(-1) == KBADCONFIG


SHAPES = [(8, 4096, 14336, 4096), (8, 16384, 14336, 4096), (64, 16384, 1408, 2048), (1, 1, 64, 64), (3, 200, 192, 520),
          (128, 4096, 768, 2048), (60, 8192, 1408, 2048), (16, 64, 11008, 4096), (2, 100000, 64, 8)]


@pytest.mark.parametrize("variant", [0, 2])
def test_select_is_the_grouped_choice_of_the_doubled_width_mapped_to_its_sibling(libs, variant):
    cfgs = capi.configs()
    for g, t, i, k in SHAPES:
        cid, gm = capi.grouped_select(variant, g, t, 2 * i, k)
        assert capi.grouped_swiglu_select(variant, g, t, i, k) == (_sibling(cfgs, cid), gm), (g, t, i, k)


def test_statuses_come_back_in_order_before_any_cuda_call(libs):
    lib = capi.grouped_swiglu_lib()
    before = capi.grouped_swiglu_launch_count()
    for cfg in (None, 1):
        def run(variant=0, x=X, w=W, h=H, y=Y, offs=OFFS, g=4, t=64, i=64, k=64):
            if cfg is None:
                return lib.cuda_l2_b200_grouped_swiglu_run(variant, x, w, h, y, offs, g, t, i, k, None)
            return _run_config(cfg, variant, x, w, h, y, offs, g, t, i, k)
        for variant in (1, 3, 5, -1):
            assert run(variant) == KBADDTYPE
            assert run(variant, x=None, t=-1, i=96) == KBADDTYPE            # the variant first
        for ptr in ("x", "w", "y", "offs"):
            assert run(**{ptr: None}) == KNULL
            assert run(**{ptr: None}, t=-1, i=96, k=60) == KNULL            # then null pointers
        for g, t, i, k in ((0, 64, 64, 64), (4, -1, 64, 64), (4, 64, 0, 64), (4, 64, 64, 0), (-1, 64, 64, 64),
                           (4, 64, 2 ** 30, 64)):
            assert run(g=g, t=t, i=i, k=k) == KBADSHAPE, (g, t, i, k)
        assert run(t=-1, i=96, k=60) == KBADSHAPE                             # then the shape
        assert run(i=96) == KBADWIDTH and run(i=32) == KBADWIDTH
        assert run(i=96, k=60, x=X + 8) == KBADWIDTH                          # then I % 64
        assert run(k=60) == KBADALIGN
        for ptr in ("x", "w", "h", "y"):
            assert run(**{ptr: {"x": X, "w": W, "h": H, "y": Y}[ptr] + 8}) == KBADALIGN
        assert run(offs=OFFS + 2) == KBADALIGN and run(offs=OFFS + 2, k=60) == KBADALIGN
        # the worst-case tile list: (T / 256 + G) * 2I / 256 tiles for the widest configurations
        assert run(g=2 ** 30, t=2 ** 30, i=2 ** 20, k=64) == KBADSHAPE
        assert run(t=0) == 0 and run(t=0, h=None) == 0                        # T == 0: nothing to do, no launch
    bwd = lib.cuda_l2_b200_grouped_swiglu_backward
    assert bwd(1, X, H, W, OFFS, 4, 64, 64, None) == KBADDTYPE
    for args in ((None, H, W, OFFS), (X, None, W, OFFS), (X, H, None, OFFS), (X, H, W, None)):
        assert bwd(0, *args, 4, 64, 64, None) == KNULL
    assert bwd(0, X, H, W, OFFS, 4, -1, 64, None) == KBADSHAPE and bwd(0, X, H, W, OFFS, 4, 64, 0, None) == KBADSHAPE
    assert bwd(0, X, H, W, OFFS, 0, 64, 64, None) == KBADSHAPE
    assert bwd(0, X, H, W, OFFS, 4, 64, 96, None) == KBADWIDTH
    assert bwd(0, X + 8, H, W, OFFS, 4, 64, 64, None) == KBADALIGN
    assert bwd(0, X, H, W, OFFS + 2, 4, 64, 64, None) == KBADALIGN
    assert bwd(0, X, H, W, OFFS, 4, 0, 64, None) == 0        # T == 0: nothing to do, no launch
    assert bwd(0, None, None, None, OFFS, 4, 0, 64, None) == 0 and bwd(0, None, None, None, None, 4, 0, 64, None) == KNULL
    sel = lib.cuda_l2_b200_grouped_swiglu_select
    assert sel(1, 4, 64, 64, 64, None, None) == KBADDTYPE
    assert sel(0, 0, 64, 64, 64, None, None) == KBADSHAPE and sel(0, 4, 0, 64, 64, None, None) == KBADSHAPE
    assert sel(0, 4, 64, 96, 64, None, None) == KBADWIDTH
    assert capi.grouped_swiglu_launch_count() == before
    # each status decoded by the library's own strerror
    for st, words in ((KBADWIDTH, "multiple of 64"), (KBADDTYPE, "fp16"), (KBADSHAPE, "positive"),
                      (KNOTHOPPER, "compute capability")):
        assert words in lib.cuda_l2_b200_grouped_swiglu_strerror(st).decode()
    with pytest.raises(capi.B200HgemmError, match="multiple of 64"):
        capi._check(KBADWIDTH, "cuda_l2_b200_grouped_swiglu_run")


def test_python_argument_rules():
    x = torch.empty((4, 64), dtype=torch.bfloat16)
    offs = torch.empty((3,), dtype=torch.int32)
    w = torch.empty((3, 128, 64), dtype=torch.bfloat16)
    assert capi.check_grouped_swiglu_operands(x, w, offs) == (3, 4, 64, 64)
    with pytest.raises(capi.B200HgemmError, match="I % 64"):
        capi.check_grouped_swiglu_operands(x, torch.empty((3, 96, 64), dtype=torch.bfloat16), offs)
    with pytest.raises(capi.B200HgemmError, match="share a dtype"):
        capi.check_grouped_swiglu_operands(x, w.half(), offs)
    with pytest.raises(capi.B200HgemmError, match="fp16 or bf16"):
        capi.check_grouped_swiglu_operands(x.float(), w.float(), offs)
    with pytest.raises(capi.B200HgemmError, match="int32"):
        capi.check_grouped_swiglu_operands(x, w, offs[:2])
    with pytest.raises(capi.B200HgemmError, match="expected"):
        capi.check_grouped_swiglu_operands(x, w[0], offs)
    with pytest.raises(capi.B200HgemmError, match="no CPU implementation"):
        ops.grouped_swiglu_linear(x, w, offs)


@pytest.mark.parametrize("i", [64, 192, 1408])
def test_stacked_interleave_and_split_round_trip(i):
    g, h = 3, 24
    wg = torch.randn((g, i, h)).bfloat16()
    wu = torch.randn((g, i, h)).bfloat16()
    w = ops.interleave_gate_up(wg, wu)
    assert w.shape == (g, 2 * i, h) and w.is_contiguous()
    for e in range(g):
        assert torch.equal(w[e], ops.interleave_gate_up(wg[e], wu[e]))   # each expert is the 2-D layout
    g2, u2 = ops.split_gate_up(w)
    assert torch.equal(g2, wg) and torch.equal(u2, wu) and g2.is_contiguous() and u2.is_contiguous()
    assert g2.data_ptr() != w.data_ptr()
    # a vLLM-style w13 stack (all gate rows, then all up rows) through the one-liner of the layer
    w13 = torch.cat((wg, wu), dim=1)
    assert torch.equal(ops.interleave_gate_up(w13[:, :i], w13[:, i:]), w)
    with pytest.raises(capi.B200HgemmError):
        ops.interleave_gate_up(wg[:, :32], wu[:, :32])
    with pytest.raises(capi.B200HgemmError):
        ops.interleave_gate_up(wg, wu[:2])
    with pytest.raises(capi.B200HgemmError):
        ops.split_gate_up(w[:, :64])


def test_two_dimensional_layout_and_errors_are_unchanged():
    """The 2-D results are the block interleave written out, and the 2-D refusals keep their words."""
    i, h = 192, 24
    wg, wu = torch.randn((i, h)), torch.randn((i, h))
    w = ops.interleave_gate_up(wg, wu)
    want = torch.cat([t for b in range(i // 64) for t in (wg[64 * b:64 * b + 64], wu[64 * b:64 * b + 64])])
    assert torch.equal(w, want) and w.shape == (2 * i, h)
    assert all(torch.equal(a, b) for a, b in zip(ops.split_gate_up(w), (wg, wu)))
    with pytest.raises(capi.B200HgemmError, match=r"gate and up weights must both be \[I, H\] with I % 64 == 0"):
        ops.interleave_gate_up(wg[:32], wu[:32])
    with pytest.raises(capi.B200HgemmError, match=r"w_gu must be \[2I, H\] with I % 64 == 0"):
        ops.split_gate_up(w[:64])
    with pytest.raises(capi.B200HgemmError, match=r"must both be \[I, H\]"):
        ops.interleave_gate_up(wg[None, None], wu[None, None])


def test_layer_on_the_meta_device():
    layer = ops.B200GroupedSwiGLULinear(8, 4096, 14336, device="meta", dtype=torch.bfloat16)
    assert [(n, tuple(p.shape), p.dtype) for n, p in layer.named_parameters()] == \
        [("weight", (8, 28672, 4096), torch.bfloat16)]
    assert "num_groups=8" in repr(layer) and "intermediate_features=14336" in repr(layer)
    for bad in ((0, 4096, 128, torch.bfloat16), (8, 4096, 100, torch.bfloat16), (8, 4100, 128, torch.bfloat16),
                (8, 4096, 128, torch.float32)):
        with pytest.raises(capi.B200HgemmError):
            ops.B200GroupedSwiGLULinear(*bad[:3], device="meta", dtype=bad[3])
    wg = torch.empty((4, 128, 64), device="meta", dtype=torch.float16)
    wu = torch.empty((4, 128, 64), device="meta", dtype=torch.float16)
    layer = ops.B200GroupedSwiGLULinear.from_weights(wg, wu)
    assert layer.weight.shape == (4, 256, 64) and layer.weight.dtype == torch.float16
    assert (layer.num_groups, layer.in_features, layer.intermediate_features) == (4, 64, 128)
    with pytest.raises(capi.B200HgemmError, match="one dtype and device"):
        ops.B200GroupedSwiGLULinear.from_weights(wg, wu.bfloat16())
    with pytest.raises(capi.B200HgemmError):
        ops.B200GroupedSwiGLULinear.from_weights(wg[0], wu[0])
    with pytest.raises(capi.B200HgemmError):
        ops.B200GroupedSwiGLULinear.from_weights(wg[:, :96], wu[:, :96])
