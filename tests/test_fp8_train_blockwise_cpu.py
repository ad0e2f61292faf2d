"""Blockwise FP8 training without a GPU: the GEMM with 1 x 128 scales on both operands (libb200_fp8block_1d1d.so) and the
dual-orientation block quantisers (libb200_quant_block_dual.so): exports against their internal headers, statuses
returned before any CUDA call, resources of both libraries; the new scale form of scale_granularity and fp8_gemm, and
the calls that refuse it; the routing of CPU tensors to the quantisers' torch compositions; and the granularity rules of
fp8_linear and B200Fp8TrainLinear."""
import re
import subprocess

import pytest
import torch

from conftest import REPO
from cuda_l2_b200 import build, capi, ops

KBADSHAPE, KBADALIGN, KNULL, KBADCONFIG, KBADLDA, KBADLDB = -1, -2, -5, -6, -10, -13
A, B, C, SA, SB, Q, S, QT, ST = (0x10000 * i for i in range(1, 10))   # fake, never dereferenced addresses


@pytest.fixture(scope="module")
def gemm_lib(built_libs):
    return capi.fp8block_1d1d_lib()


@pytest.fixture(scope="module")
def quant_lib(built_libs):
    return capi.quant_block_dual_lib()


def _exports(path) -> list[str]:
    out = subprocess.run(["nm", "-D", "--defined-only", str(path)], capture_output=True, text=True, check=True).stdout
    return [line.split()[-1] for line in out.splitlines() if line.strip()]


@pytest.mark.parametrize("key, lib, header, prefix", [
    ("fp8block_1d1d", capi.FP8BLOCK_1D1D_LIB, "b200_fp8_block_1d1d.h", "cuda_l2_b200_fp8block_1d1d_"),
    ("quant_block_dual", capi.QUANT_BLOCK_DUAL_LIB, "b200_quant_block_dual.h", "cuda_l2_b200_quant_block_dual_")])
def test_exports_and_internal_header(built_libs, key, lib, header, prefix):
    names = _exports(built_libs[key])
    assert not [s for s in names if s.startswith("b200_")]
    assert sorted(s for s in names if s.startswith("cuda_l2_b200_")) == sorted(capi.INTERNAL_ABI[lib])
    assert all(s.startswith(prefix) for s in capi.INTERNAL_ABI[lib])
    assert lib not in capi.ABI
    assert not any(prefix in h.read_text() for h in (REPO / "include").glob("*.h"))
    text = (build.CSRC / header).read_text()
    for sym, (args, _) in capi.INTERNAL_ABI[lib].items():
        proto = re.search(rf"\b{sym}\(([^)]*)\);", text)
        assert proto, sym
        params = " ".join(proto.group(1).split())
        assert (0 if params in ("", "void") else params.count(",") + 1) == len(args), sym


def _run(lib, a=A, b=B, c=C, sa=SA, ld_a=64, sb=SB, ld_b=136, out_bf16=1, m=64, n=136, k=256):
    return lib.cuda_l2_b200_fp8block_1d1d_run(a, b, c, sa, ld_a, sb, ld_b, out_bf16, m, n, k, None)


def test_gemm_statuses_come_back_before_any_cuda_call(gemm_lib):
    before = capi.fp8block_1d1d_launch_count()
    for name in ("a", "b", "c", "sa", "sb"):
        assert _run(gemm_lib, **{name: None}) == KNULL, name
    for out in (-1, 2):
        assert _run(gemm_lib, out_bf16=out) == KBADCONFIG
    for m, n, k in ((0, 136, 256), (64, 0, 256), (64, 136, -16)):
        assert _run(gemm_lib, m=m, n=n, k=k) == KBADSHAPE
    assert _run(gemm_lib, k=264) == -9                              # K % 16
    assert _run(gemm_lib, n=132, ld_b=132) == KBADALIGN             # N % 8
    assert _run(gemm_lib, sa=SA + 4) == KBADALIGN and _run(gemm_lib, sb=SB + 4) == KBADALIGN
    assert _run(gemm_lib, ld_a=60) == KBADLDA and _run(gemm_lib, ld_a=66) == KBADLDA
    assert _run(gemm_lib, ld_b=128) == KBADLDB and _run(gemm_lib, ld_b=138) == KBADLDB
    assert gemm_lib.cuda_l2_b200_fp8block_1d1d_run_config(3, 1, A, B, C, SA, 64, SB, 136, 64, 136, 256, 0, 0, 1,
                                                          None) == KBADCONFIG   # BN 256: no block-scaled kernel
    for st in (KBADSHAPE, KBADALIGN, KNULL, KBADCONFIG, KBADLDA, KBADLDB):
        assert gemm_lib.cuda_l2_b200_fp8block_1d1d_strerror(st).decode() not in ("", "unknown error")
    assert "ld_b" in gemm_lib.cuda_l2_b200_fp8block_1d1d_strerror(KBADLDB).decode()
    assert capi.fp8block_1d1d_launch_count() == before


def test_select_is_the_block_scaled_librarys(gemm_lib):
    for mnk in ((1, 8, 16), (512, 4096, 4096), (1024, 768, 16384), (4096, 7168, 2048), (136, 200, 8192)):
        assert capi.fp8_blockwise_1d1d_select(*mnk) == capi.fp8_blockwise_select(*mnk), mnk
    with pytest.raises(capi.B200HgemmError, match="status -1"):
        capi.fp8_blockwise_1d1d_select(0, 8, 16)


def _quant(lib, which="1x128", dtype=1, x=A, rows=37, cols=300, q=Q, s=S, qt=QT, st=ST):
    return getattr(lib, f"cuda_l2_b200_quant_block_dual_e4m3_{which}")(dtype, x, rows, cols, q, s, qt, st, None)


@pytest.mark.parametrize("which", ["1x128", "128x128"])
def test_quantiser_statuses_come_back_before_any_cuda_call(quant_lib, which):
    before = capi.quant_block_dual_launch_count()
    for dtype in (-1, 2, 3):
        assert _quant(quant_lib, which, dtype=dtype) == -6          # fp16 and bf16 only
    for name in ("x", "q", "s", "qt", "st"):
        assert _quant(quant_lib, which, **{name: None}) == KNULL, name
    for rows, cols in ((0, 300), (37, 0), (-1, 300), (2 ** 31 - 15, 16), (2 ** 30, 2 ** 30)):
        assert _quant(quant_lib, which, rows=rows, cols=cols) == KBADSHAPE, (rows, cols)
    for name, off in (("s", 2), ("st", 1), ("qt", 8)):
        assert _quant(quant_lib, which, **{name: {"s": S, "st": ST, "qt": QT}[name] + off}) == KBADALIGN, name
    for st in (KBADSHAPE, KBADALIGN, KNULL, -6):
        assert quant_lib.cuda_l2_b200_quant_block_dual_strerror(st).decode() not in ("", "unknown status")
    assert capi.quant_block_dual_launch_count() == before


def _res_usage(path) -> list[tuple[str, str]]:
    out = subprocess.run(["cuobjdump", "-res-usage", str(path)], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    return [(lines[i].split("Function ")[1].rstrip(":"), lines[i + 1]) for i in range(len(lines) - 1)
            if "Function " in lines[i]]


@pytest.mark.parametrize("key, count, kernel", [("fp8block_1d1d", 38, "hgemm_block_1d1d_kernel"),
                                                ("quant_block_dual", 8, "b200_quant_block_dual_kernel")])
def test_kernels_and_resources(built_libs, key, count, kernel):
    """cuobjdump -res-usage: the kernel count (1D1D: 17 block-scaled configurations plus the cluster split-K kernels of
    configurations 1 and 2, per output type; quantiser: 2 dtypes x 2 load widths x 2 granularities), no stack (no
    spills) and no local memory; and no fast-math or flush-to-zero option in the build."""
    for flag in ("-use_fast_math", "--use_fast_math", "-ftz=true", "--ftz=true", "-prec-div=false"):
        assert flag not in build.COMMON and flag not in build.ARCH_FLAGS
    for src in ("b200_fp8_block_1d1d.cu", "b200_quant_block_dual.cu"):
        text = (build.CSRC / src).read_text()
        assert "__fdividef" not in text and "__expf" not in text
    funcs = _res_usage(built_libs[key])
    assert len(funcs) == count
    for name, usage in funcs:
        assert kernel in name, name
        assert "STACK:0" in usage and "LOCAL:0" in usage, (name, usage)


def test_block_dual_quantiser_shares_the_element_arithmetic():
    text = (build.CSRC / "b200_quant_block_dual.cu").read_text()
    assert '#include "b200_quant_arith.cuh"' in text
    for fn in ("nan_max", "scale_of", "quotient", "e4m3x2", "store_e4m3"):
        assert not re.search(rf"__device__ __forceinline__ \S+ {fn}\(", text), fn
    assert build.LIBRARIES["quant_block_dual"][1] == [(build.CSRC / "b200_quant_block_dual.cu", [])]
    assert build.LIBRARIES["fp8block_1d1d"][1] == [(build.CSRC / "b200_fp8_block_1d1d.cu", ["-DB200_VARIANT=7"]),
                                                  (build.CSRC / "b200_fp8_block_1d1d.cu", ["-DB200_VARIANT=8"])]


# ------------------------------------------------------------------------------------------------ the scale form
def _meta(shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device="meta")


@pytest.mark.parametrize("m, n, k", [(1, 8, 16), (300, 136, 1040), (4096, 1024, 16384), (64, 128, 128)])
def test_scale_granularity_and_fp8_gemm_meta_shapes(m, n, k):
    nkb = capi.num_k_blocks(k)
    sa, sb = _meta((m, nkb)), _meta((n, nkb))
    assert capi.scale_granularity(m, n, sa, sb, k=k) == "blockwise_1d1d"
    assert capi.scale_granularity(m, n, sa, sb) == "blockwise_1d1d"
    if m * nkb > 1:   # two one-element scales are per-tensor ones
        assert capi.scale_granularity(m, n, sa, _meta((-(-n // 128), nkb)), k=k) == "blockwise"
    a, bt = _meta((m, k), torch.float8_e4m3fn), _meta((n, k), torch.float8_e4m3fn)
    for out in (torch.float16, torch.bfloat16):
        y = ops.fp8_gemm(a, bt, sa, sb, out)
        assert (y.shape, y.dtype) == ((m, n), out)
    with pytest.raises(capi.B200HgemmError):
        capi.scale_granularity(m, n, sa, _meta((n, nkb + 1)), k=k)


def test_calls_that_refuse_the_new_form():
    m, n, k = 64, 136, 256
    a, bt = _meta((m, k), torch.float8_e4m3fn), _meta((n, k), torch.float8_e4m3fn)
    sa, sb = _meta((m, 2)), _meta((n, 2))
    with pytest.raises(capi.B200HgemmError, match="blockwise scales have no bias"):
        ops.fp8_gemm_bias_act(a, bt, sa, sb, None, "relu", torch.bfloat16)
    with pytest.raises(capi.B200HgemmError):
        capi.scale_granularity(m, n, sa, sb, k=k, groups=1)
    with pytest.raises(capi.B200HgemmError):
        capi.scale_granularity(m, n, _meta((1, m, 2)), _meta((1, n, 2)), k=k, batches=1)
    with pytest.raises(capi.B200HgemmError):
        ops.fp8_grouped_gemm(a, _meta((2, n, k), torch.float8_e4m3fn), sa, _meta((2, n, 2)),
                             torch.empty(2, dtype=torch.int32, device="meta"))
    with pytest.raises(capi.B200HgemmError):
        ops.fp8_batched_gemm(_meta((2, m, k), torch.float8_e4m3fn), _meta((2, n, k), torch.float8_e4m3fn),
                             _meta((2, m, 2)), _meta((2, n, 2)))


# ------------------------------------------------------------------------------------------------ python functions
def _bits(t):
    return t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t.view(torch.int32)


def test_cpu_tensors_take_the_torch_compositions(quant_lib):
    before = capi.quant_block_dual_launch_count()
    g = torch.Generator().manual_seed(3)
    for dtype in (torch.float16, torch.bfloat16, torch.float32):
        x = (torch.randn((37, 300), generator=g) * 8).to(dtype)
        x[5, 7] = float("nan")
        got = ops.quantize_e4m3_blockwise_dual(x)
        want = ops.quantize_e4m3_blockwise_dual_reference(x)
        for a, b in zip(got, want):
            assert a.shape == b.shape and a.stride() == b.stride() and torch.equal(_bits(a), _bits(b))
        q, s = ops.quantize_e4m3_blockwise_reference(x)
        assert torch.equal(_bits(got[0]), _bits(q)) and torch.equal(_bits(got[1]), _bits(s))
        assert got[2].shape == (300, 48) and got[3].shape == (300, 1) and got[3].stride() == (1, 300)
        assert (_bits(got[2][:, 37:])[torch.arange(300) != 7] == 0).all() and (_bits(got[2][7, 37:]) == 0x7F).all()
        w = (torch.randn((300, 136), generator=g)).to(dtype)
        q, s, q_t, s_t = ops.quantize_e4m3_block128x128_dual(w)
        qw, sw = ops.quantize_e4m3_block128x128(w)
        assert torch.equal(_bits(q), _bits(qw)) and torch.equal(_bits(s), _bits(sw))
        assert torch.equal(_bits(q_t), _bits(qw.t().contiguous())) and torch.equal(_bits(s_t), _bits(sw.t().contiguous()))
        # with 128 x 128 blocks, quantising w^T is transposing the quantisation of w
        qt2, st2 = ops.quantize_e4m3_block128x128(w.t().contiguous())
        assert torch.equal(_bits(q_t), _bits(qt2)) and torch.equal(_bits(s_t), _bits(st2))
    assert capi.quant_block_dual_launch_count() == before
    for bad in (torch.ones(8), torch.ones((2, 8, 8))):
        with pytest.raises(capi.B200HgemmError):
            ops.quantize_e4m3_blockwise_dual(bad)
        with pytest.raises(capi.B200HgemmError):
            ops.quantize_e4m3_block128x128_dual(bad)


def test_fp8_linear_and_the_module_take_a_granularity():
    x = torch.ones((4, 64), dtype=torch.bfloat16)
    w = torch.ones((32, 64), dtype=torch.bfloat16)
    lin = torch.nn.Linear(64, 32, dtype=torch.bfloat16)
    for call in (lambda: ops.fp8_linear(x, w, "tensor"), lambda: ops.fp8_linear(x, w, granularity="block"),
                 lambda: ops.B200Fp8TrainLinear(64, 32, granularity="tensor"),
                 lambda: ops.B200Fp8TrainLinear.from_linear(lin, granularity="blockwise128"),
                 lambda: ops.fp8_linear(x, torch.ones((40, 64), dtype=torch.bfloat16), "blockwise")):
        with pytest.raises(capi.B200HgemmError):
            call()
    assert ops.B200Fp8TrainLinear(64, 32).granularity == "rowwise"             # the default is unchanged
    assert ops.B200Fp8TrainLinear.from_linear(lin).granularity == "rowwise"
    layer = ops.B200Fp8TrainLinear.from_linear(lin, granularity="blockwise")
    assert layer.weight is lin.weight and layer.bias is lin.bias and layer.granularity == "blockwise"
    assert "granularity=blockwise" in repr(layer)
    assert ops.B200Fp8TrainLinear(64, 32, dtype=torch.float16, granularity="blockwise").granularity == "blockwise"
