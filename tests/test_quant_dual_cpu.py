"""The dual-orientation rowwise e4m3 quantiser (libb200_quant_dual.so) and FP8 training of linear layers without a GPU:
argument statuses, exports, resources and kernel names; the shared element arithmetic; the operator's schema and fake
results against the torch composition (ragged rows, the ld_t padding); the routing of CPU tensors to that composition;
and the shape and dtype rules of fp8_linear and B200Fp8TrainLinear."""
import re
import subprocess

import pytest
import torch

from conftest import REPO
from cuda_l2_b200 import build, capi, ops

KBADSHAPE, KBADALIGN, KNULL, KBADDTYPE = -1, -2, -5, -6
X, Q, S, QT, ST, W = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000   # fake, never dereferenced addresses
KERNELS = ("b200_quant_dual_amax_kernel", "b200_quant_dual_kernel")


@pytest.fixture(scope="module")
def lib(built_libs):
    return capi.quant_dual_lib()


def _dual(lib, dtype=1, x=X, rows=37, cols=300, q=Q, s=S, qt=QT, st=ST, w=W):
    return lib.cuda_l2_b200_quant_dual_e4m3_rowwise(dtype, x, rows, cols, q, s, qt, st, w, None)


def test_statuses_come_back_before_any_cuda_call(lib):
    """Every refused argument returns its status without a CUDA call: the addresses are never dereferenced, and this
    runs on a machine without a GPU."""
    before = capi.quant_dual_launch_count()
    for dtype in (-1, 3, 7):
        assert _dual(lib, dtype=dtype) == KBADDTYPE
    for name in ("x", "q", "s", "qt", "st", "w"):
        assert _dual(lib, **{name: None}) == KNULL, name
    for rows, cols in ((0, 300), (37, 0), (-1, 300), (37, -4), (2 ** 31 - 15, 16)):
        assert _dual(lib, rows=rows, cols=cols) == KBADSHAPE, (rows, cols)
    assert _dual(lib, rows=2 ** 30, cols=2 ** 30) == KBADSHAPE   # more than INT_MAX tiles of 64 x 64
    for name, off in (("s", 2), ("st", 1), ("w", 2), ("qt", 8)):
        assert _dual(lib, **{name: {"s": S, "st": ST, "w": W, "qt": QT}[name] + off}) == KBADALIGN, name
    for st in (KBADSHAPE, KBADALIGN, KNULL, KBADDTYPE):
        assert lib.cuda_l2_b200_quant_dual_strerror(st).decode() not in ("", "unknown status")
    assert capi.quant_dual_launch_count() == before


def _exports(path) -> list[str]:
    out = subprocess.run(["nm", "-D", "--defined-only", str(path)], capture_output=True, text=True, check=True).stdout
    return [line.split()[-1] for line in out.splitlines() if line.strip()]


def test_exports_and_internal_header(built_libs):
    names = _exports(built_libs["quant_dual"])
    assert not [s for s in names if s.startswith("b200_")]
    assert sorted(s for s in names if s.startswith("cuda_l2_b200_")) == sorted(capi.INTERNAL_ABI[capi.QUANT_DUAL_LIB])
    assert all(s.startswith("cuda_l2_b200_quant_dual_") for s in capi.INTERNAL_ABI[capi.QUANT_DUAL_LIB])
    assert capi.QUANT_DUAL_LIB not in capi.ABI
    assert not any("quant_dual" in h.read_text() for h in (REPO / "include").glob("*.h"))
    header = (build.CSRC / "b200_quant_dual.h").read_text()
    for sym, (args, _) in capi.INTERNAL_ABI[capi.QUANT_DUAL_LIB].items():
        proto = re.search(rf"\b{sym}\(([^)]*)\);", header)
        assert proto, sym
        params = " ".join(proto.group(1).split())
        assert (0 if params in ("", "void") else params.count(",") + 1) == len(args), sym
    assert "#define CUDA_L2_B200_QUANT_DUAL_WORKSPACE(rows, cols) ((long long)(rows) + (long long)(cols))" in header
    assert capi.quant_dual_workspace(37, 300) == 337
    assert build.LIBRARIES["quant_dual"][1] == [(build.CSRC / "b200_quant_dual.cu", [])]


def test_element_arithmetic_is_shared_not_copied():
    """Both quantiser libraries compile the one text of the element arithmetic, so they cannot drift apart."""
    arith = (build.CSRC / "b200_quant_arith.cuh").read_text()
    for src in ("b200_quant.cu", "b200_quant_dual.cu"):
        text = (build.CSRC / src).read_text()
        assert '#include "b200_quant_arith.cuh"' in text, src
        for fn in ("nan_max", "scale_of", "quotient", "e4m3x2", "load_f32", "store_e4m3"):
            assert re.search(rf"\b{fn}\(", arith), fn
            assert not re.search(rf"__device__ __forceinline__ \S+ {fn}\(", text), (src, fn)


def test_kernels_resources_and_build_flags(tmp_path):
    """-Xptxas -v of the library's one object: no spills, no stack, no C7510, the stable kernel names (the benchmark's
    profiler leg finds the kernels by them), and no fast-math or flush-to-zero option or intrinsic."""
    for flag in ("-use_fast_math", "--use_fast_math", "-ftz=true", "--ftz=true", "-prec-div=false"):
        assert flag not in build.COMMON and flag not in build.ARCH_FLAGS
    src = build.CSRC / "b200_quant_dual.cu"
    for text in (src.read_text(), (build.CSRC / "b200_quant_arith.cuh").read_text()):
        assert "__fdividef" not in text and "__expf" not in text
    r = subprocess.run([build.nvcc_path(), *build.ARCH_FLAGS, *build.COMMON, "-Xptxas", "-v", "-c", "-o",
                        str(tmp_path / "qd.o"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    text = r.stdout + r.stderr
    assert "C7510" not in text and "warning" not in text.lower()
    blocks = text.split("ptxas info    : Compiling entry function ")[1:]
    assert len(blocks) == 12   # 3 dtypes x 2 load widths x 2 kernels
    for block in blocks:
        name = block.split("'")[1]
        assert any(k in name for k in KERNELS), name
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, name


def _meta(shape, dtype=torch.bfloat16):
    return torch.empty(shape, dtype=dtype, device="meta")


def test_operator_schema():
    assert str(torch.ops.cuda_l2_b200.quantize_e4m3_rowwise_dual.default._schema) == \
        "cuda_l2_b200::quantize_e4m3_rowwise_dual(Tensor x) -> (Tensor, Tensor, Tensor, Tensor)"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("shape", [(1, 16), (15, 136), (17, 300), (37, 300), (64, 64), (300, 4096)])
def test_fake_results_have_the_reference_shapes_and_strides(dtype, shape):
    got = torch.ops.cuda_l2_b200.quantize_e4m3_rowwise_dual(_meta(shape, dtype))
    want = ops.quantize_e4m3_rowwise_dual_reference(torch.randn(shape).to(dtype))
    assert len(got) == len(want) == 4
    for g, w in zip(got, want):
        assert (g.shape, g.dtype, g.stride()) == (w.shape, w.dtype, w.stride()), shape
    rows, cols = shape
    assert got[2].shape == (cols, capi.dual_ld_t(rows)) and capi.dual_ld_t(rows) % 16 == 0
    assert got[1].shape == (rows,) and got[3].shape == (cols,)


def test_operator_refuses_what_no_kernel_takes():
    for call in (lambda: torch.ops.cuda_l2_b200.quantize_e4m3_rowwise_dual(_meta((8, 8), torch.float64)),
                 lambda: torch.ops.cuda_l2_b200.quantize_e4m3_rowwise_dual(_meta((0, 8))),
                 lambda: torch.ops.cuda_l2_b200.quantize_e4m3_rowwise_dual(_meta((2, 8, 8))),
                 lambda: torch.ops.cuda_l2_b200.quantize_e4m3_rowwise_dual(torch.ones((8, 8)))):
        with pytest.raises(capi.B200HgemmError):
            call()
    q = torch.ops.cuda_l2_b200.quantize_e4m3_rowwise_dual(_meta((8, 256)).requires_grad_())
    with pytest.raises(capi.B200HgemmError, match="inference only"):
        q[3].sum().backward()


def _bits(t):
    return t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t.view(torch.int32)


def test_cpu_tensors_take_the_torch_composition(lib):
    """CPU tensors never reach the library; the composition is the rowwise reference of x and of x^T padded."""
    before = capi.quant_dual_launch_count()
    g = torch.Generator().manual_seed(3)
    for dtype in (torch.float16, torch.bfloat16, torch.float32):
        x = (torch.randn((37, 300), generator=g) * 8).to(dtype)
        x[5, 7] = float("nan")
        got = ops.quantize_e4m3_rowwise_dual(x)
        want = ops.quantize_e4m3_rowwise_dual_reference(x)
        for a, b in zip(got, want):
            assert a.shape == b.shape and a.stride() == b.stride() and torch.equal(_bits(a), _bits(b))
        q, s = ops.quantize_e4m3_rowwise_reference(x)
        assert torch.equal(_bits(got[0]), _bits(q)) and torch.equal(_bits(got[1]), _bits(s.reshape(-1)))
        pad = torch.zeros((300, 48), dtype=dtype)
        pad[:, :37] = x.t()
        qt, st = ops.quantize_e4m3_rowwise_reference(pad)
        assert torch.equal(_bits(got[2]), _bits(qt)) and torch.equal(_bits(got[3]), _bits(st.reshape(-1)))
        # padding bytes are e4m3(0 / s): 0x00, or the NaN code in the NaN row's column
        assert (_bits(got[2][:, 37:])[torch.arange(300) != 7] == 0).all()
        assert (_bits(got[2][7, 37:]) == 0x7F).all() and torch.isnan(got[3][7])
    assert capi.quant_dual_launch_count() == before
    assert not ops._quant_routed(torch.ones(8))


def test_fp8_linear_and_the_module_refuse_what_the_kernels_cannot_take():
    x = torch.ones((4, 64), dtype=torch.bfloat16)
    w = torch.ones((32, 64), dtype=torch.bfloat16)
    bad = [lambda: ops.fp8_linear(x, w.half()),                                      # one dtype
           lambda: ops.fp8_linear(x.float(), w.float()),                             # 16-bit only
           lambda: ops.fp8_linear(x, torch.ones((40, 64), dtype=torch.bfloat16)),    # N % 16
           lambda: ops.fp8_linear(torch.ones((4, 72), dtype=torch.bfloat16),
                                  torch.ones((32, 72), dtype=torch.bfloat16)),       # K % 16
           lambda: ops.fp8_linear(x, torch.ones((32, 48), dtype=torch.bfloat16)),    # K differs
           lambda: ops.fp8_linear(x, w[0]),                                          # 2-D weight
           lambda: ops.B200Fp8TrainLinear(64, 40),
           lambda: ops.B200Fp8TrainLinear(72, 32),
           lambda: ops.B200Fp8TrainLinear(64, 32, dtype=torch.float32),
           lambda: ops.B200Fp8TrainLinear.from_linear(torch.nn.Linear(64, 24, dtype=torch.bfloat16)),
           lambda: ops.B200Fp8TrainLinear.from_linear(torch.nn.Linear(64, 32))]         # fp32
    for call in bad:
        with pytest.raises(capi.B200HgemmError):
            call()


def test_module_shares_the_parameters_of_its_source():
    lin = torch.nn.Linear(64, 32, dtype=torch.bfloat16)
    layer = ops.B200Fp8TrainLinear.from_linear(lin)
    assert layer.weight is lin.weight and layer.bias is lin.bias
    assert {n for n, _ in layer.named_parameters()} == {"weight", "bias"}
    fresh = ops.B200Fp8TrainLinear(64, 32, bias=False, dtype=torch.float16)
    assert fresh.bias is None and fresh.weight.dtype == torch.float16 and fresh.weight.requires_grad
    assert fresh.weight.abs().max() <= 1 / 8 and "in_features=64" in repr(fresh)


def test_fp8_linear_forward_traces_under_fake_tensors():
    """The forward, with and without a gradient to prepare, runs on fake CUDA tensors through the operators' fakes
    (the backward's engine needs a device: tests/test_gpu_fp8_train.py traces it)."""
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        for shape in ((37, 64), (3, 5, 64)):
            for grad in (False, True):
                x = torch.empty(shape, dtype=torch.bfloat16, device="cuda").requires_grad_(grad)
                w = torch.empty((48, 64), dtype=torch.bfloat16, device="cuda").requires_grad_(grad)
                y = ops.fp8_linear(x, w)
                assert y.shape == (*shape[:-1], 48) and y.dtype == torch.bfloat16 and y.requires_grad == grad
