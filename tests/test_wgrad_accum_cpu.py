"""fp32 weight-gradient accumulation (libb200_wgrad_accum.so) without a GPU: exports against the ABI table and the
internal header, the build entry, the kernel count, local memory against the wrapped kernels, argument statuses before
any CUDA call, the dispatchers' choices, and the Python argument rules and meta-device gradients of the fused layers."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest
import torch

from conftest import REPO
from cuda_l2_b200 import build, capi, ops

KNULL, KBADSHAPE, KBADALIGN, KBADCONFIG, KBADFP8K, KBADLD, KBADLDB = -5, -1, -2, -6, -9, -10, -13
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
CUFILT = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
A, B, C, S, SB, OFFS = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000   # fake, never dereferenced addresses
ROWWISE, BLOCK_1D1D = 1, 3
HEADER = build.CSRC / "b200_wgrad_accum.h"


@pytest.fixture(scope="module")
def libs(built_libs):
    return built_libs


def _grouped(variant=0, cfg=-1, a=A, b=B, c=C, offs=OFFS, g=2, t=64, m=64, n=64):
    return capi.wgrad_accum_lib().cuda_l2_b200_wgrad_accum_grouped(variant, cfg, a, b, c, offs, g, t, m, n, 0, 0, None)


def _fp8(form=ROWWISE, cfg=-1, a=A, b=B, c=C, sa=S, ld_a=64, sb=SB, ld_b=64, m=64, n=64, k=128):
    return capi.wgrad_accum_lib().cuda_l2_b200_wgrad_accum_fp8(form, cfg, a, b, c, sa, ld_a, sb, ld_b, m, n, k, 0, 0, 1,
                                                               None)


def _exports(path) -> list[str]:
    out = subprocess.run(["nm", "-D", "--defined-only", str(path)], capture_output=True, text=True, check=True).stdout
    return [line.split()[-1] for line in out.splitlines() if line.strip()]


def test_exports_are_the_table_and_the_internal_header(libs):
    table = capi.INTERNAL_ABI[capi.WGRAD_ACCUM_LIB]
    names = _exports(libs["wgrad_accum"])
    assert not [s for s in names if s.startswith("b200_")]
    assert sorted(s for s in names if s.startswith("cuda_l2_b200_")) == sorted(table)
    assert capi.WGRAD_ACCUM_LIB not in capi.ABI
    assert not any("wgrad_accum" in h.read_text() for h in (REPO / "include").glob("*.h"))
    # every prototype of the header, with as many parameters as its argtypes
    text = re.sub(r"//[^\n]*", "", HEADER.read_text())
    protos = dict(re.findall(r"(cuda_l2_b200_wgrad_accum_\w+)\(([^)]*)\);", text))
    assert sorted(protos) == sorted(table)
    for sym, params in protos.items():
        count = 0 if params.strip() in ("", "void") else params.count(",") + 1
        assert count == len(table[sym][0]), sym


def test_build_entry():
    name, objects, link_flags = build.LIBRARIES["wgrad_accum"]
    assert name == capi.WGRAD_ACCUM_LIB and link_flags == []
    assert [(src.name, defines) for src, defines in objects] == \
        [("b200_wgrad_accum.cu", [f"-DB200_VARIANT={v}"]) for v in (0, 2, 3, 7)]


def _resources(path) -> dict:
    """{demangled kernel name: (registers, stack bytes, local bytes)} from cuobjdump -res-usage."""
    out = subprocess.run([CUOBJDUMP, "-res-usage", str(path)], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    res = {}
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            res[m.group(1)] = tuple(int(re.search(k + r":(\d+)", lines[i + 1]).group(1)) for k in ("REG", "STACK", "LOCAL"))
    names = subprocess.run([CUFILT], input="\n".join(res), capture_output=True, text=True, check=True).stdout.splitlines()
    return {_without_params(d): v for d, v in zip(names, res.values())}


def _without_params(demangled: str) -> str:
    """``void name<args>(params)`` -> ``name<args>``, with the template arguments' casts (``(int)128``) dropped."""
    depth = 0
    for i, ch in enumerate(demangled):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0 and i > 0 and demangled[i - 1] == ">":
            demangled = demangled[:i]
            break
    return re.sub(r"\((?:int|bool)\)", "", demangled).replace("void ", "", 1)


def _sibling(name: str) -> str:
    """The wrapped library's kernel of an accumulating kernel: same configuration and K-mode, AccumF32<> unwrapped."""
    m = re.fullmatch(r"b200::hgemm_accum_kernel<b200::AccumF32<(.*)>, (?:\(int\))?(\d)>", name)
    assert m, name
    inner, mode = m.group(1).strip(), m.group(2)
    kernel = "hgemm_block_1d1d_kernel" if "BlockScaled1D1D" in inner else "hgemm_tn_kernel"
    return f"b200::{kernel}<{inner}, {mode}>"


@pytest.mark.skipif(not Path(CUOBJDUMP).exists(), reason="cuobjdump not available")
def test_kernel_count_and_local_memory_against_the_wrapped_kernels(libs):
    """56 K-grouped kernels (28 configurations x fp16 / bf16), 46 rowwise e4m3 ones (libb200_hgemm.so's (configuration,
    K-mode) pairs) and 19 1 x 128 ones (libb200_fp8block_1d1d.so's); none uses more stack or local memory than the
    kernel it wraps, in libb200_grouped_bwd.so, libb200_hgemm.so or libb200_fp8block_1d1d.so."""
    accum = _resources(libs["wgrad_accum"])
    assert len(accum) == 121
    kinds = {"GroupedK": 0, "BlockScaled1D1D": 0}
    for name in accum:
        kind = next((k for k in kinds if k in name), None)
        if kind:
            kinds[kind] += 1
    assert kinds == {"GroupedK": 56, "BlockScaled1D1D": 19}
    siblings = {**_resources(libs["capi"]), **_resources(libs["grouped_bwd"]), **_resources(libs["fp8block_1d1d"])}
    for name, (regs, stack, local) in accum.items():
        sib = siblings[_sibling(name)]
        assert regs <= 168, name
        assert stack <= sib[1] and local <= sib[2], (name, (stack, local), sib)


@pytest.mark.parametrize("cfg", [-1, 1])
def test_grouped_statuses_come_back_before_any_cuda_call(libs, cfg):
    before = capi.wgrad_accum_launch_count()
    for variant in (1, 3, 5, 7, -1):
        assert _grouped(variant, cfg) == KBADCONFIG
    assert _grouped(cfg=cfg, a=None) == KNULL
    assert _grouped(cfg=cfg, b=None) == KNULL
    assert _grouped(cfg=cfg, c=None) == KNULL
    assert _grouped(cfg=cfg, offs=None) == KNULL
    assert _grouped(cfg=cfg, c=C + 8) == KBADALIGN          # C32: 16-byte aligned
    assert _grouped(cfg=cfg, offs=OFFS + 2) == KBADALIGN
    assert _grouped(cfg=cfg, m=60) == KBADALIGN             # 16-byte rows of A [T, M] ...
    assert _grouped(cfg=cfg, n=60) == KBADALIGN             # ... and of B [T, N]
    for g, t, m, n in ((0, 64, 64, 64), (2, -1, 64, 64), (2, 64, 0, 64), (2, 64, 64, 0)):
        assert _grouped(cfg=cfg, g=g, t=t, m=m, n=n) == KBADSHAPE
    # T == 0: nothing to add, no launch, and the operands are never read
    assert _grouped(cfg=cfg, a=None, b=None, t=0) == 0
    assert capi.wgrad_accum_launch_count() == before


def test_grouped_configurations_without_a_kernel(libs):
    for cfg in (12, 13, 14, 31, 100):   # BN = 32 has no row-major B kernel
        assert _grouped(cfg=cfg) == KBADCONFIG


@pytest.mark.parametrize("cfg", [-1, 1])
def test_fp8_statuses_come_back_before_any_cuda_call(libs, cfg):
    for form in (0, 2, 4, -1):   # per tensor and 128 x 128 scales have no accumulating kernel
        assert _fp8(form, cfg) == KBADCONFIG
    for form in (ROWWISE, BLOCK_1D1D):
        assert _fp8(form, cfg, a=None) == KNULL
        assert _fp8(form, cfg, b=None) == KNULL
        assert _fp8(form, cfg, c=None) == KNULL
        assert _fp8(form, cfg, sa=None) == KNULL
        assert _fp8(form, cfg, sb=None) == KNULL
        assert _fp8(form, cfg, c=C + 8) == KBADALIGN
        assert _fp8(form, cfg, k=120) == KBADFP8K
        assert _fp8(form, cfg, n=60) == KBADALIGN
        for m, n, k in ((0, 64, 128), (64, 0, 128), (64, 64, 0)):
            assert _fp8(form, cfg, m=m, n=n, k=k) == KBADSHAPE
    assert _fp8(ROWWISE, cfg, sb=SB + 4) == KBADALIGN        # rowwise vectors: 16-byte aligned
    assert _fp8(BLOCK_1D1D, cfg, ld_a=60) == KBADLD
    assert _fp8(BLOCK_1D1D, cfg, ld_b=62) == KBADLDB
    assert _fp8(BLOCK_1D1D, cfg, sb=SB + 4) == KBADALIGN     # 1 x 128 scales of Bt: bulk copies
    assert _fp8(ROWWISE, 31) == KBADCONFIG
    assert _fp8(BLOCK_1D1D, 0) == KBADCONFIG                  # BN = 256: no block-scaled kernel
    text = capi.wgrad_accum_lib().cuda_l2_b200_wgrad_accum_strerror(KBADLDB).decode()
    assert text.startswith("1 x 128 scales of Bt")


SHAPES = [(4096, 4096, 4096), (11008, 4096, 2048), (4096, 11008, 4096), (768, 3072, 8192), (16, 4096, 4096),
          (64, 64, 64), (200, 328, 1040), (3000, 136, 65536)]


@pytest.mark.parametrize("shape", SHAPES)
def test_dispatched_choices_are_the_wrapped_libraries(libs, shape):
    m, n, k = shape
    assert capi.wgrad_accum_fp8_select("rowwise", m, n, k) == capi.fp8_select(m, n, k)
    assert capi.wgrad_accum_fp8_select("blockwise_1d1d", m, n, k) == capi.fp8_blockwise_1d1d_select(m, n, k)
    for variant in (0, 2):
        for g in (1, 8):
            assert capi.wgrad_accum_grouped_select(variant, g, k, m, n) == capi.grouped_wgrad_select(variant, g, k, m, n)


def _meta(*shape, dtype=torch.bfloat16, grad=True):
    return torch.empty(shape, dtype=dtype, device="meta", requires_grad=grad)


def test_main_grad_rules():
    w = _meta(24, 32, grad=False)
    ok = torch.empty((24, 32), dtype=torch.float32, device="meta")
    capi.check_main_grad(ok, (24, 32), w.device)
    bad = {
        "dtype": ok.to(torch.bfloat16),
        "shape": torch.empty((32, 24), dtype=torch.float32, device="meta"),
        "contiguity": torch.empty((32, 24), dtype=torch.float32, device="meta").t(),
        "device": torch.empty((24, 32), dtype=torch.float32),
        "missing": None,
    }
    for what, t in bad.items():
        with pytest.raises(capi.B200HgemmError, match="main_grad"):
            capi.check_main_grad(t, (24, 32), w.device)
    with pytest.raises(capi.B200HgemmError, match="16-byte aligned"):
        capi.check_main_grad(torch.zeros(25, dtype=torch.float32)[1:].view(1, 24), (1, 24), torch.device("cpu"))


def test_plain_functions_check_their_arguments():
    gy, x = _meta(40, 24, grad=False), _meta(40, 32, grad=False)
    mg = torch.empty((24, 32), dtype=torch.float32, device="meta")
    assert ops.wgrad_accumulate_(mg, gy, x) is mg
    assert ops.wgrad_accumulate_(mg, _meta(0, 24, grad=False), _meta(0, 32, grad=False)) is mg
    with pytest.raises(capi.B200HgemmError):
        ops.wgrad_accumulate_(mg.half(), gy, x)
    with pytest.raises(capi.B200HgemmError):
        ops.wgrad_accumulate_(mg.t(), gy, x)
    with pytest.raises(capi.B200HgemmError):
        ops.wgrad_accumulate_(mg, gy, _meta(41, 32, grad=False))
    offs = torch.empty(3, dtype=torch.int32, device="meta")
    mg3 = torch.empty((3, 24, 32), dtype=torch.float32, device="meta")
    assert ops.grouped_wgrad_accumulate_(mg3, gy, x, offs) is mg3
    with pytest.raises(capi.B200HgemmError):
        ops.grouped_wgrad_accumulate_(mg, gy, x, offs)
    e4m3 = torch.float8_e4m3fn
    a, b = _meta(24, 64, dtype=e4m3, grad=False), _meta(32, 64, dtype=e4m3, grad=False)
    f32 = torch.float32
    rowwise = (torch.empty((24, 1), dtype=f32, device="meta"), torch.empty((1, 32), dtype=f32, device="meta"))
    one_d = (torch.empty((24, 1), dtype=f32, device="meta"), torch.empty((32, 1), dtype=f32, device="meta"))
    assert ops.fp8_gemm_accumulate_(mg, a, b, *rowwise) is mg
    assert ops.fp8_gemm_accumulate_(mg, a, b, *one_d) is mg
    tensor = (torch.empty(1, dtype=f32, device="meta"), torch.empty(1, dtype=f32, device="meta"))
    with pytest.raises(capi.B200HgemmError, match="rowwise or 1 x 128"):
        ops.fp8_gemm_accumulate_(mg, a, b, *tensor)
    with pytest.raises(capi.B200HgemmError, match="c32"):
        ops.fp8_gemm_accumulate_(mg3, a, b, *rowwise)


def _layers(dtype):
    return [
        ops.B200Linear(32, 24, device="meta", dtype=dtype, fuse_wgrad_accumulation=True),
        ops.B200Linear(32, 24, bias=False, device="meta", dtype=dtype, fuse_wgrad_accumulation=True),
        ops.B200Fp8TrainLinear(32, 48, device="meta", dtype=dtype, fuse_wgrad_accumulation=True),
    ]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_fused_layers_need_main_grad(dtype):
    layers = _layers(dtype) + [ops.B200GroupedLinear(3, 32, 24, device="meta", dtype=dtype,
                                                     fuse_wgrad_accumulation=True)]
    for layer in layers:
        args = (_meta(40, 32, dtype=dtype),) if not isinstance(layer, ops.B200GroupedLinear) else \
            (_meta(40, 32, dtype=dtype), torch.empty(3, dtype=torch.int32, device="meta"))
        with pytest.raises(capi.B200HgemmError, match="main_grad"):
            layer(*args)
        layer.weight.main_grad = torch.empty(layer.weight.shape, dtype=torch.bfloat16, device="meta")
        with pytest.raises(capi.B200HgemmError, match="fp32"):
            layer(*args)
        assert "fuse_wgrad_accumulation=True" in repr(layer)
    lin = torch.nn.Linear(32, 48, device="meta", dtype=dtype)
    assert ops.B200Linear.from_linear(lin, fuse_wgrad_accumulation=True).fuse_wgrad_accumulation
    assert ops.B200Fp8TrainLinear.from_linear(lin, fuse_wgrad_accumulation=True).fuse_wgrad_accumulation
    assert ops.B200GroupedLinear.from_weights(_meta(3, 24, 32, dtype=dtype), fuse_wgrad_accumulation=True) \
        .fuse_wgrad_accumulation
    assert not ops.B200Linear.from_linear(lin).fuse_wgrad_accumulation
    with pytest.raises(capi.B200HgemmError, match="main_grad"):
        ops.fp8_linear(_meta(40, 32, dtype=dtype), lin.weight, main_grad=torch.empty((32, 48), device="meta"))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("lead", [(40,), (1,), (3, 13)])
def test_fused_layers_on_meta_give_x_and_bias_gradients_and_no_weight_gradient(dtype, lead):
    for layer in _layers(dtype):
        layer.weight.main_grad = torch.empty(layer.weight.shape, dtype=torch.float32, device="meta")
        x = _meta(*lead, 32, dtype=dtype)
        y = layer(x)
        assert y.shape == (*lead, layer.out_features) and y.dtype == dtype
        y.sum().backward()
        assert x.grad is not None and x.grad.shape == x.shape and x.grad.dtype == dtype
        assert layer.weight.grad is None
        if layer.bias is not None:
            assert layer.bias.grad is not None and layer.bias.grad.shape == (layer.out_features,)


def test_unfused_layers_are_unchanged():
    for layer in (ops.B200Linear(32, 24, device="meta", dtype=torch.bfloat16),
                  ops.B200Fp8TrainLinear(32, 48, device="meta")):
        assert not layer.fuse_wgrad_accumulation
        x = _meta(40, 32)
        layer(x).sum().backward()
        assert layer.weight.grad is not None and layer.weight.grad.shape == layer.weight.shape
