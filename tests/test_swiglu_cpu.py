"""The SwiGLU library (libb200_swiglu.so) without a GPU: exports against the ABI table and the internal header, the build
entry, the kernel count, registers and local memory against the TN kernels the gated ones wrap, the configuration
mapping and the dispatcher's choice, argument statuses before any CUDA call, the gate / up weight layout, the layer's
parameters on the meta device, and the float32 reference of the backward against torch's autograd."""
import json
import os
import re
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from torch import nn

from conftest import REPO
from cuda_l2_b200 import build, capi, ops
from swiglu_ref import swiglu_grad_reference

KNULL, KBADSHAPE, KBADALIGN, KBADCONFIG, KNOTHOPPER, KBADWIDTH, KBADDTYPE = -5, -1, -2, -6, -7, -14, -15
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
CUFILT = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
X, W, H, Y = 0x10000, 0x20000, 0x30000, 0x40000   # fake, never dereferenced addresses
HEADER = build.CSRC / "b200_swiglu.h"
GATED_BN = (128, 256)


@pytest.fixture(scope="module")
def libs(built_libs):
    return built_libs


def _exports(path) -> list[str]:
    out = subprocess.run(["nm", "-D", "--defined-only", str(path)], capture_output=True, text=True, check=True).stdout
    return [line.split()[-1] for line in out.splitlines() if line.strip()]


def test_exports_are_the_table_and_the_internal_header(libs):
    table = capi.INTERNAL_ABI[capi.SWIGLU_LIB]
    names = _exports(libs["swiglu"])
    assert not [s for s in names if s.startswith("b200_")]
    assert sorted(s for s in names if s.startswith("cuda_l2_b200_")) == sorted(table)
    assert capi.SWIGLU_LIB not in capi.ABI
    assert not any("swiglu" in h.read_text() for h in (REPO / "include").glob("*.h"))
    text = re.sub(r"//[^\n]*", "", HEADER.read_text())
    protos = dict(re.findall(r"(cuda_l2_b200_swiglu_\w+)\(([^)]*)\);", text))
    assert sorted(protos) == sorted(table)
    for sym, params in protos.items():
        count = 0 if params.strip() in ("", "void") else params.count(",") + 1
        assert count == len(table[sym][0]), sym


def test_build_entry():
    name, objects, link_flags = build.LIBRARIES["swiglu"]
    assert name == capi.SWIGLU_LIB and link_flags == []
    assert [(src.name, defines) for src, defines in objects] == \
        [("b200_swiglu.cu", [f"-DB200_VARIANT={v}"]) for v in (0, 2)]


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
def test_kernel_count_registers_and_local_memory_against_the_tn_kernels(libs):
    """18 gated kernels per variant (the BN = 128 and 256 configurations, plain schedule) and the backward kernel of
    each variant; no gated kernel uses more than 168 registers, nor more stack or local memory than the plain TN kernel
    of its configuration in libb200_hgemm.so."""
    res = _resources(libs["swiglu"])
    gated = {k: v for k, v in res.items() if k.startswith("b200::hgemm_gated_kernel<")}
    backward = [k for k in res if "swiglu_backward_kernel" in k]
    assert len(gated) == 36 and len(backward) == 2 and len(res) == 38
    tn = _resources(libs["capi"])
    for name, (regs, stack, local) in gated.items():
        m = re.fullmatch(r"b200::hgemm_gated_kernel<b200::Gated<(b200::Config<[^>]*>)>, 0>", name)
        assert m, name
        sib = tn[f"b200::hgemm_tn_kernel<{m.group(1)}, 0>"]
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


def _run_config(cfg, variant=0, x=X, w=W, h=H, y=Y, m=64, i=64, k=64, splits=1):
    return capi.swiglu_lib().cuda_l2_b200_swiglu_run_config(variant, cfg, x, w, h, y, m, i, k, 0, splits, 0, None)


# Every (configuration, splits code) through cuda_l2_b200_swiglu_run_config on fake addresses, in a process that sees no
# device: a configuration with a gated kernel gets as far as the device query (kNotHopper), one without is kBadConfig.
_NO_DEVICE = """
import json, sys
sys.path.insert(0, {repo!r})
from cuda_l2_b200 import capi
lib = capi.swiglu_lib()
out = []
for cfg in range(-1, 32):
    for splits in (1, -2, 4, capi.STREAMK_TAIL, capi.STREAMK_TAIL_PLUS_WAVE):
        st = lib.cuda_l2_b200_swiglu_run_config(0, cfg, {x}, {w}, {h}, {y}, 64, 64, 64, 0, splits, 0, None)
        out.append([cfg, splits, st])
print(json.dumps(out))
"""


def test_every_configuration_maps_to_a_gated_kernel(libs):
    """All 31 configurations: those with BN = 128 or 256 have a gated kernel for every splits code, the others are
    kBadConfig, and their sibling is a BN = 128 one. The launches run on fake addresses, so they run in a process with
    CUDA_VISIBLE_DEVICES="", where a launch with a kernel stops at the device query (kNotHopper) on any machine. In this
    process only the refusals are called: kBadConfig comes back before any CUDA call."""
    cfgs = capi.configs()
    assert len(cfgs) == 31
    r = subprocess.run([sys.executable, "-c", _NO_DEVICE.format(repo=str(REPO), x=X, w=W, h=H, y=Y)],
                       capture_output=True, text=True, timeout=300, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-2000:]
    for cfg, splits, st in json.loads(r.stdout):
        gated = 0 <= cfg < 31 and cfgs[cfg]["bn"] in GATED_BN
        assert st == (KNOTHOPPER if gated else KBADCONFIG), (cfg, splits, st)
    for c in cfgs:
        if c["bn"] not in GATED_BN:
            assert _run_config(c["id"]) == KBADCONFIG, c
        s = cfgs[_sibling(cfgs, c["id"])]
        assert s["bn"] in GATED_BN and s["cta_group"] == c["cta_group"] and s["m_rep"] == c["m_rep"]
    assert _run_config(31) == KBADCONFIG and _run_config(-1) == KBADCONFIG


SHAPES = [(1, 64, 64), (16, 1408, 2048), (16, 11008, 4096), (129, 192, 520), (2048, 11008, 4096), (8192, 14336, 4096),
          (200, 320, 72), (4096, 64, 8192), (513, 2048, 1024), (1, 18944, 3584)]


@pytest.mark.parametrize("variant", [0, 2])
def test_select_is_the_tn_choice_of_the_doubled_width_mapped_to_its_sibling(libs, variant):
    cfgs = capi.configs()
    for m, i, k in SHAPES:
        cid, gm, _ = capi.select("fp32", m, 2 * i, k)
        assert capi.swiglu_select(variant, m, i, k) == (_sibling(cfgs, cid), gm, 1), (m, i, k)


def test_statuses_come_back_before_any_cuda_call(libs):
    lib = capi.swiglu_lib()
    before = capi.swiglu_launch_count()
    for cfg in (None, 1):
        def run(variant=0, x=X, w=W, h=H, y=Y, m=64, i=64, k=64):
            if cfg is None:
                return lib.cuda_l2_b200_swiglu_run(variant, x, w, h, y, m, i, k, None)
            return _run_config(cfg, variant, x, w, h, y, m, i, k)
        for variant in (1, 3, 5, -1):
            assert run(variant) == KBADDTYPE
        assert run(x=None) == KNULL and run(w=None) == KNULL and run(y=None) == KNULL
        for m, i, k in ((0, 64, 64), (64, 0, 64), (64, 64, 0), (-1, 64, 64)):
            assert run(m=m, i=i, k=k) == KBADSHAPE
        assert run(i=96) == KBADWIDTH and run(i=32) == KBADWIDTH
        assert run(k=60) == KBADALIGN
        for ptr in ("x", "w", "h", "y"):
            assert run(**{ptr: {"x": X, "w": W, "h": H, "y": Y}[ptr] + 8}) == KBADALIGN
    bwd = lib.cuda_l2_b200_swiglu_backward
    assert bwd(1, X, H, W, 64, 64, None) == KBADDTYPE
    assert bwd(0, None, H, W, 64, 64, None) == KNULL
    assert bwd(0, X, H, W, -1, 64, None) == KBADSHAPE and bwd(0, X, H, W, 64, 0, None) == KBADSHAPE
    assert bwd(0, X, H, W, 64, 96, None) == KBADWIDTH
    assert bwd(0, X + 8, H, W, 64, 64, None) == KBADALIGN
    assert bwd(0, X, H, W, 0, 64, None) == 0        # M == 0: nothing to do, no launch
    sel = lib.cuda_l2_b200_swiglu_select
    assert sel(1, 64, 64, 64, None, None, None) == KBADDTYPE
    assert sel(0, 0, 64, 64, None, None, None) == KBADSHAPE
    assert sel(0, 64, 96, 64, None, None, None) == KBADWIDTH
    assert capi.swiglu_launch_count() == before
    # each status decoded by the library's own strerror
    for st, words in ((KBADWIDTH, "multiple of 64"), (KBADDTYPE, "fp16"), (KBADSHAPE, "positive"),
                      (KNOTHOPPER, "compute capability")):
        assert words in lib.cuda_l2_b200_swiglu_strerror(st).decode()
    with pytest.raises(capi.B200HgemmError, match="multiple of 64"):
        capi._check(KBADWIDTH, "cuda_l2_b200_swiglu_run")


def test_python_argument_rules():
    x = torch.empty((4, 64), dtype=torch.bfloat16)
    with pytest.raises(capi.B200HgemmError, match="I % 64"):
        capi.check_swiglu_operands(x, torch.empty((96, 64), dtype=torch.bfloat16))
    with pytest.raises(capi.B200HgemmError, match="share a dtype"):
        capi.check_swiglu_operands(x, torch.empty((128, 64), dtype=torch.float16))
    with pytest.raises(capi.B200HgemmError, match="fp16 or bf16"):
        capi.check_swiglu_operands(x.float(), torch.empty((128, 64)))
    assert capi.check_swiglu_operands(x, torch.empty((256, 64), dtype=torch.bfloat16)) == (4, 128, 64)
    with pytest.raises(capi.B200HgemmError, match="no CPU implementation"):
        ops.swiglu_linear(x, torch.empty((128, 64), dtype=torch.bfloat16))


@pytest.mark.parametrize("i", [64, 192, 11008])
def test_interleave_and_split_round_trip(i):
    h = 24
    wg = torch.randn((i, h)).bfloat16()
    wu = torch.randn((i, h)).bfloat16()
    w = ops.interleave_gate_up(wg, wu)
    assert w.shape == (2 * i, h)
    for b in range(i // 64):
        assert torch.equal(w[128 * b:128 * b + 64], wg[64 * b:64 * b + 64])
        assert torch.equal(w[128 * b + 64:128 * b + 128], wu[64 * b:64 * b + 64])
    g2, u2 = ops.split_gate_up(w)
    assert torch.equal(g2, wg) and torch.equal(u2, wu)
    assert g2.data_ptr() != w.data_ptr() and g2.is_contiguous() and u2.is_contiguous()
    g2.zero_()
    assert torch.equal(w[:64], wg[:64])   # copies: the fused weight is untouched
    with pytest.raises(capi.B200HgemmError):
        ops.interleave_gate_up(wg[:32], wu[:32])
    with pytest.raises(capi.B200HgemmError):
        ops.split_gate_up(w[:64])


def test_layer_parameters_on_the_meta_device():
    layer = ops.B200SwiGLULinear(4096, 11008, device="meta", dtype=torch.bfloat16)
    assert [(n, tuple(p.shape), p.dtype) for n, p in layer.named_parameters()] == \
        [("weight", (22016, 4096), torch.bfloat16)]
    assert "intermediate_features=11008" in repr(layer)
    for bad in ((4096, 100, torch.bfloat16), (4100, 128, torch.bfloat16), (4096, 128, torch.float32)):
        with pytest.raises(capi.B200HgemmError):
            ops.B200SwiGLULinear(*bad[:2], device="meta", dtype=bad[2])


def test_from_linears_refuses_biased_or_misfitting_projections():
    mk = lambda i, bias=False, dtype=torch.bfloat16: nn.Linear(64, i, bias=bias, dtype=dtype)   # noqa: E731
    with pytest.raises(capi.B200HgemmError, match="bias-free"):
        ops.B200SwiGLULinear.from_linears(mk(128, bias=True), mk(128))
    with pytest.raises(capi.B200HgemmError, match="match"):
        ops.B200SwiGLULinear.from_linears(mk(128), mk(192))
    with pytest.raises(capi.B200HgemmError, match="match"):
        ops.B200SwiGLULinear.from_linears(mk(128), mk(128, dtype=torch.float16))
    with pytest.raises(capi.B200HgemmError):
        ops.B200SwiGLULinear.from_linears(mk(96), mk(96))
    g, u = mk(128), mk(128)
    layer = ops.B200SwiGLULinear.from_linears(g, u)
    assert torch.equal(layer.weight, ops.interleave_gate_up(g.weight, u.weight)) and layer.weight.requires_grad


def test_numpy_backward_reference_against_torch_autograd_in_fp32():
    """The reference's operation order, run on fp32 inputs without the 16-bit roundings, is torch's fp32 autograd of
    F.silu(g) * u to within fp32 rounding (torch's CPU kernels may contract or vectorise differently)."""
    rng = np.random.default_rng(0)
    g = (rng.standard_normal(4096) * 4).astype(np.float32)
    u = rng.standard_normal(4096).astype(np.float32)
    dy = rng.standard_normal(4096).astype(np.float32)
    dg, du = swiglu_grad_reference(dy, g, u, dtype=np.float32)
    gt, ut = torch.from_numpy(g).requires_grad_(), torch.from_numpy(u).requires_grad_()
    (torch.nn.functional.silu(gt) * ut).backward(torch.from_numpy(dy))
    np.testing.assert_allclose(du, ut.grad.numpy(), rtol=2e-6, atol=1e-30)
    np.testing.assert_allclose(dg, gt.grad.numpy(), rtol=1e-5, atol=1e-30)
