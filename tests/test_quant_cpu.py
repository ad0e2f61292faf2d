"""The e4m3 quantisers of FP8 activations (libb200_quant.so) without a GPU: argument statuses, exports, resources and
kernel names; the operators' schemas and fake results (shapes and strides, the M-major scale view included); the routing
of CPU tensors to the torch compositions; B200Fp8GroupedMLP's construction checks; and the SASS and resource lines of
the GEMM libraries, which the quantisers leave as they were."""
import json
import re
import subprocess
from pathlib import Path

import pytest
import torch

import sass_digest
from conftest import REPO
from cuda_l2_b200 import build, capi, ops

KBADSHAPE, KBADALIGN, KNULL, KBADDTYPE, KBADLD = -1, -2, -5, -6, -10
X, Q, S, W = 0x10000, 0x20000, 0x30000, 0x40000   # fake, never dereferenced device addresses
KERNELS = ("b200_quant_tensor_amax_kernel", "b200_quant_tensor_kernel", "b200_quant_rowwise_kernel",
           "b200_quant_blockwise_kernel", "b200_quant_silu_mul_blockwise_kernel")


@pytest.fixture(scope="module")
def lib(built_libs):
    return capi.quant_lib()


def _blockwise(lib, silu=False, dtype=1, x=X, b=2, m=37, k=300, q=Q, s=S, ld_a=40, masked=None):
    fn = lib.cuda_l2_b200_quant_silu_mul_e4m3_blockwise if silu else lib.cuda_l2_b200_quant_e4m3_blockwise
    return fn(dtype, x, b, m, k, q, s, ld_a, masked, None)


def test_statuses_come_back_before_any_cuda_call(lib):
    for dtype in (-1, 3, 7):
        assert lib.cuda_l2_b200_quant_e4m3_tensor(dtype, X, 100, Q, S, W, None) == KBADDTYPE
        assert lib.cuda_l2_b200_quant_e4m3_rowwise(dtype, X, 4, 100, Q, S, None) == KBADDTYPE
        assert _blockwise(lib, dtype=dtype) == KBADDTYPE
        assert _blockwise(lib, silu=True, dtype=dtype) == KBADDTYPE
    assert _blockwise(lib, silu=True, dtype=2) == KBADDTYPE   # SwiGLU: fp16 and bf16 only
    for args in ((0, Q, S, W), (X, None, S, W), (X, Q, None, W), (X, Q, S, None)):
        x, q, s, w = args
        assert lib.cuda_l2_b200_quant_e4m3_tensor(2, x or None, 100, q, s, w, None) == KNULL
    assert lib.cuda_l2_b200_quant_e4m3_tensor(0, X, 0, Q, S, W, None) == KBADSHAPE
    assert lib.cuda_l2_b200_quant_e4m3_tensor(0, X, -5, Q, S, W, None) == KBADSHAPE
    assert lib.cuda_l2_b200_quant_e4m3_tensor(0, X, 100, Q, S + 2, W, None) == KBADALIGN
    assert lib.cuda_l2_b200_quant_e4m3_tensor(0, X, 100, Q, S, W + 1, None) == KBADALIGN
    assert lib.cuda_l2_b200_quant_e4m3_rowwise(0, None, 4, 100, Q, S, None) == KNULL
    assert lib.cuda_l2_b200_quant_e4m3_rowwise(0, X, 0, 100, Q, S, None) == KBADSHAPE
    assert lib.cuda_l2_b200_quant_e4m3_rowwise(0, X, 4, 0, Q, S, None) == KBADSHAPE
    assert lib.cuda_l2_b200_quant_e4m3_rowwise(0, X, 4, 100, Q, S + 1, None) == KBADALIGN
    for silu in (False, True):
        assert _blockwise(lib, silu, x=None) == KNULL
        assert _blockwise(lib, silu, q=None) == KNULL
        assert _blockwise(lib, silu, s=None) == KNULL
        for b, m, k in ((0, 37, 300), (2, 0, 300), (2, 37, 0), (-1, 37, 300)):
            assert _blockwise(lib, silu, b=b, m=m, k=k) == KBADSHAPE
        assert _blockwise(lib, silu, b=65536, m=2 ** 30, k=300) == KBADSHAPE   # more than INT_MAX tiles
        assert _blockwise(lib, silu, s=S + 2) == KBADALIGN
        assert _blockwise(lib, silu, ld_a=36) == KBADLD    # < M
        assert _blockwise(lib, silu, ld_a=38) == KBADLD    # % 4
    for st in (KBADSHAPE, KBADALIGN, KNULL, KBADDTYPE, KBADLD):
        assert lib.cuda_l2_b200_quant_strerror(st).decode() not in ("", "unknown status")
    assert lib.cuda_l2_b200_quant_strerror(KBADLD).decode().startswith("ld_a")


def _exports(path) -> list[str]:
    out = subprocess.run(["nm", "-D", "--defined-only", str(path)], capture_output=True, text=True, check=True).stdout
    return [line.split()[-1] for line in out.splitlines() if line.strip()]


def test_exports_and_internal_header(built_libs):
    names = _exports(built_libs["quant"])
    assert not [s for s in names if s.startswith("b200_")]
    assert sorted(s for s in names if s.startswith("cuda_l2_b200_")) == sorted(capi.INTERNAL_ABI[capi.QUANT_LIB])
    assert capi.QUANT_LIB not in capi.ABI
    assert not any("cuda_l2_b200_quant" in h.read_text() for h in (REPO / "include").glob("*.h"))
    header = (build.CSRC / "b200_quant.h").read_text()
    for sym, (args, _) in capi.INTERNAL_ABI[capi.QUANT_LIB].items():
        proto = re.search(rf"\b{sym}\(([^)]*)\);", header)
        assert proto, sym
        params = " ".join(proto.group(1).split())
        assert (0 if params in ("", "void") else params.count(",") + 1) == len(args), sym
    assert f"#define CUDA_L2_B200_QUANT_TENSOR_WORKSPACE {capi.QUANT_TENSOR_WORKSPACE}" in header
    assert build.LIBRARIES["quant"][1] == [(build.CSRC / "b200_quant.cu", [])]


def test_kernels_resources_and_build_flags(tmp_path):
    """-Xptxas -v of the library's one object: no spills, no stack, no C7510, and the stable kernel names (the
    benchmark's profiler leg finds the kernels by them). The build flags carry no fast-math or flush-to-zero option."""
    for flag in ("-use_fast_math", "--use_fast_math", "-ftz=true", "--ftz=true", "-prec-div=false"):
        assert flag not in build.COMMON and flag not in build.ARCH_FLAGS
    src = build.CSRC / "b200_quant.cu"
    assert "__fdividef" not in src.read_text() and "__expf" not in src.read_text()
    r = subprocess.run([build.nvcc_path(), *build.ARCH_FLAGS, *build.COMMON, "-Xptxas", "-v", "-c", "-o",
                        str(tmp_path / "q.o"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    text = r.stdout + r.stderr
    assert "C7510" not in text and "warning" not in text.lower()
    blocks = text.split("ptxas info    : Compiling entry function ")[1:]
    assert len(blocks) == 28   # 3 dtypes x 2 load widths x 4 kernels + 2 x 2 SwiGLU kernels (fp16, bf16)
    for block in blocks:
        name = block.split("'")[1]
        assert any(k in name for k in KERNELS), name
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, name


def test_gemm_libraries_keep_their_sass_and_resources(built_libs):
    """The digest of every GEMM library's per-kernel SASS and resource lines equals the one recorded before the
    quantisers were added: no source of theirs changed, and none was added to their objects."""
    if not Path(sass_digest.CUOBJDUMP).exists():
        pytest.skip("cuobjdump not available")
    want = json.loads(sass_digest.GOLDEN.read_text())
    assert sorted(want) == sorted(built_libs[key].name for key in sass_digest.GEMM_LIBRARIES)
    assert sass_digest.digests(built_libs) == want
    for key in sass_digest.GEMM_LIBRARIES:
        assert all("b200_quant" not in str(src) for src, _ in build.LIBRARIES[key][1]), key


def _meta(shape, dtype=torch.bfloat16):
    return torch.empty(shape, dtype=dtype, device="meta")


def test_operator_schemas():
    want = {"quantize_e4m3": "(Tensor x) -> (Tensor, Tensor)",
            "quantize_e4m3_rowwise": "(Tensor x) -> (Tensor, Tensor)",
            "quantize_e4m3_blockwise": "(Tensor x, Tensor? masked_m=None) -> (Tensor, Tensor)",
            "silu_mul_quantize_e4m3_blockwise": "(Tensor h, Tensor? masked_m=None) -> (Tensor, Tensor)"}
    for name, schema in want.items():
        assert str(getattr(torch.ops.cuda_l2_b200, name).default._schema) == f"cuda_l2_b200::{name}{schema}"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_fake_results_have_the_reference_shapes_and_strides(dtype):
    """Each operator's fake results against the torch composition run on CPU tensors of the same shape: shapes, dtypes
    and strides, the M-major scale view included, and blockwise_ld_a reads that view as the GEMMs do."""
    cases = [("quantize_e4m3", ops.quantize_e4m3_reference, (5, 7, 300)),
             ("quantize_e4m3_rowwise", ops.quantize_e4m3_rowwise_reference, (37, 300)),
             ("quantize_e4m3_blockwise", ops.quantize_e4m3_blockwise_reference, (37, 300)),
             ("quantize_e4m3_blockwise", ops.quantize_e4m3_blockwise_reference, (3, 37, 300)),
             ("quantize_e4m3_blockwise", ops.quantize_e4m3_blockwise_reference, (3, 37, 128)),
             ("quantize_e4m3_blockwise", ops.quantize_e4m3_blockwise_reference, (2, 1, 16)),
             ("quantize_e4m3_blockwise", ops.quantize_e4m3_blockwise_reference, (40, 7168))]
    if dtype != torch.float32:
        cases += [("silu_mul_quantize_e4m3_blockwise", ops.silu_mul_quantize_e4m3_blockwise_reference, (37, 600)),
                  ("silu_mul_quantize_e4m3_blockwise", ops.silu_mul_quantize_e4m3_blockwise_reference, (4, 37, 4096))]
    for name, ref, shape in cases:
        got = getattr(torch.ops.cuda_l2_b200, name)(_meta(shape, dtype))
        want = ref(torch.randn(shape).to(dtype))
        for g, w in zip(got, want):
            assert (g.shape, g.dtype, g.stride()) == (w.shape, w.dtype, w.stride()), (name, shape)
        if "blockwise" in name:
            scale = torch.empty_strided(got[1].shape, got[1].stride(), dtype=torch.float32)
            assert capi.blockwise_ld_a(want[1]) == -(-shape[-2] // 4) * 4
            assert want[1].untyped_storage().nbytes() // 4 == (shape[0] if len(shape) == 3 else 1) * \
                capi.num_k_blocks(got[0].shape[-1]) * -(-shape[-2] // 4) * 4
            assert scale.stride() == want[1].stride()
    masked = torch.empty((3,), dtype=torch.int32, device="meta")
    q, s = torch.ops.cuda_l2_b200.quantize_e4m3_blockwise(_meta((3, 37, 300), dtype), masked)
    assert q.shape == (3, 37, 300) and s.shape == (3, 37, 3) and s.stride() == (120, 1, 40)


def test_operators_refuse_what_no_kernel_takes():
    masked = torch.empty((3,), dtype=torch.int32, device="meta")
    bad = [lambda: torch.ops.cuda_l2_b200.quantize_e4m3(_meta((8, 8), torch.float64)),
           lambda: torch.ops.cuda_l2_b200.quantize_e4m3(_meta((0, 8))),
           lambda: torch.ops.cuda_l2_b200.quantize_e4m3_rowwise(_meta((2, 8, 8))),
           lambda: torch.ops.cuda_l2_b200.quantize_e4m3_blockwise(_meta((8,))),
           lambda: torch.ops.cuda_l2_b200.quantize_e4m3_blockwise(_meta((2, 2, 8, 8))),
           lambda: torch.ops.cuda_l2_b200.quantize_e4m3_blockwise(_meta((2, 8, 8)), masked),      # B differs
           lambda: torch.ops.cuda_l2_b200.quantize_e4m3_blockwise(_meta((3, 8, 8)), masked.long()),
           lambda: torch.ops.cuda_l2_b200.silu_mul_quantize_e4m3_blockwise(_meta((8, 8), torch.float32)),
           lambda: torch.ops.cuda_l2_b200.silu_mul_quantize_e4m3_blockwise(_meta((8, 9)))]
    for call in bad:
        with pytest.raises(capi.B200HgemmError):
            call()
    with pytest.raises(capi.B200HgemmError, match="h must be"):
        ops.silu_mul_quantize_e4m3_blockwise(torch.ones((4, 9), dtype=torch.bfloat16))


def test_operators_have_no_gradient():
    x = _meta((8, 256)).requires_grad_()
    for q, s in (torch.ops.cuda_l2_b200.quantize_e4m3_blockwise(x),
                 torch.ops.cuda_l2_b200.silu_mul_quantize_e4m3_blockwise(x)):
        with pytest.raises(capi.B200HgemmError, match="inference only"):
            s.sum().backward()


def test_cpu_tensors_take_the_torch_composition(lib):
    """CPU tensors never reach the library: the public functions return the reference's results (and launch nothing),
    the operators themselves refuse them."""
    before = capi.quant_launch_count()
    g = torch.Generator().manual_seed(3)
    for dtype in (torch.float16, torch.bfloat16, torch.float32):
        x = (torch.randn((3, 37, 300), generator=g) * 8).to(dtype)
        h = (torch.randn((37, 512), generator=g) * 4).to(dtype)
        pairs = [(ops.quantize_e4m3(x), ops.quantize_e4m3_reference(x)),
                 (ops.quantize_e4m3_rowwise(x[0]), ops.quantize_e4m3_rowwise_reference(x[0])),
                 (ops.quantize_e4m3_blockwise(x), ops.quantize_e4m3_blockwise_reference(x)),
                 (ops.quantize_e4m3_blockwise(x, torch.tensor([1, 0, 5], dtype=torch.int32)),
                  ops.quantize_e4m3_blockwise_reference(x)),
                 (ops.silu_mul_quantize_e4m3_blockwise(h), ops.silu_mul_quantize_e4m3_blockwise_reference(h))]
        for got, want in pairs:
            for a, b in zip(got, want):
                assert a.shape == b.shape and a.stride() == b.stride() and a.dtype == b.dtype
                assert torch.equal(a.view(torch.uint8) if a.dtype == torch.float8_e4m3fn else a.view(torch.int32),
                                   b.view(torch.uint8) if b.dtype == torch.float8_e4m3fn else b.view(torch.int32))
        q, s = ops.silu_mul_quantize_e4m3_blockwise(h)
        manual = ops.quantize_e4m3_blockwise_reference(torch.nn.functional.silu(h[:, :256]) * h[:, 256:])
        assert torch.equal(q.view(torch.uint8), manual[0].view(torch.uint8)) and torch.equal(s, manual[1])
    for call in (lambda: torch.ops.cuda_l2_b200.quantize_e4m3(torch.ones(8)),
                 lambda: torch.ops.cuda_l2_b200.quantize_e4m3_blockwise(torch.ones((8, 8))),
                 lambda: torch.ops.cuda_l2_b200.silu_mul_quantize_e4m3_blockwise(torch.ones((8, 8)).half())):
        with pytest.raises(capi.B200HgemmError, match="no CPU implementation"):
            call()
    assert capi.quant_launch_count() == before
    assert not ops._quant_routed(torch.ones(8)) and not ops._quant_routed(torch.ones(8, dtype=torch.float64))


def test_reference_bits_on_known_values():
    """The composition's rule on values worked by hand: the scale is amax * fp32(1/448) (torch's CUDA division by a
    Python scalar), an all-zero or all -0.0 block gets FLT_MIN and keeps its zeros' signs."""
    x = torch.zeros((4, 128), dtype=torch.bfloat16)
    x[1] = -0.0
    x[2, 5] = 448.0
    x[3, :] = 1.0
    x[3, 7] = -896.0
    q, s = ops.quantize_e4m3_blockwise_reference(x)
    tiny = torch.finfo(torch.float32).tiny
    assert s[0, 0] == tiny and s[1, 0] == tiny
    assert (q[0].view(torch.uint8) == 0).all() and (q[1].view(torch.uint8) == 0x80).all()
    assert s[2, 0] == torch.tensor(448.0) / 448.0 and q[2, 5].view(torch.uint8) == 0x7E   # 448 -> e4m3 max
    assert q[3, 7].view(torch.uint8) == 0xFE and q[3, 0].float() == 0.5


def test_grouped_mlp_construction():
    g, hid, i = 3, 256, 128
    gen = torch.Generator().manual_seed(1)
    w13 = torch.randn((g, 2 * i, hid), generator=gen).bfloat16()
    w2 = torch.randn((g, hid, i), generator=gen).bfloat16()
    mlp = ops.B200Fp8GroupedMLP.from_weights(w13, w2)
    assert (mlp.num_experts, mlp.hidden_size, mlp.intermediate_size, mlp.out_dtype) == (g, hid, i, torch.bfloat16)
    assert mlp.w13_fp8.shape == (g, 2 * i, hid) and mlp.w13_scale.shape == (g, 2, 2)
    assert mlp.w2_fp8.shape == (g, hid, i) and mlp.w2_scale.shape == (g, 2, 1)
    want13 = ops.quantize_e4m3_block128x128(w13)
    assert torch.equal(mlp.w13_fp8.view(torch.uint8), want13[0].view(torch.uint8))
    assert torch.equal(mlp.w13_scale, want13[1])
    assert {n for n, _ in mlp.named_buffers()} == {"w13_fp8", "w13_scale", "w2_fp8", "w2_scale"}
    assert "num_experts=3" in repr(mlp)
    q13, s13, q2, s2 = mlp.w13_fp8, mlp.w13_scale, mlp.w2_fp8, mlp.w2_scale
    assert ops.B200Fp8GroupedMLP.from_fp8(q13, s13, q2, s2, torch.float16).out_dtype == torch.float16
    e = torch.float8_e4m3fn
    bad = [lambda: ops.B200Fp8GroupedMLP.from_weights(w13.float(), w2.float()),               # 16-bit only
           lambda: ops.B200Fp8GroupedMLP.from_weights(w13, w2.half()),                         # one dtype
           lambda: ops.B200Fp8GroupedMLP.from_weights(w13[0], w2),                             # stacks
           lambda: ops.B200Fp8GroupedMLP.from_fp8(q13, s13, q2[:2], s2[:2]),                   # G differs
           lambda: ops.B200Fp8GroupedMLP.from_fp8(q13[:, :200], s13, q2, s2),                  # 2I != 2 * I
           lambda: ops.B200Fp8GroupedMLP.from_fp8(torch.zeros((g, 2 * 120, hid), dtype=e), torch.ones((g, 2, 2)),
                                                  torch.zeros((g, hid, 120), dtype=e), torch.ones((g, 2, 1))),  # I % 16
           lambda: ops.B200Fp8GroupedMLP.from_fp8(torch.zeros((g, 2 * i, 264), dtype=e), torch.ones((g, 2, 3)),
                                                  torch.zeros((g, 264, i), dtype=e), torch.ones((g, 3, 1))),    # H % 16
           lambda: ops.B200Fp8GroupedMLP.from_fp8(q13, s13[:, :1], q2, s2),                    # scale shape
           lambda: ops.B200Fp8GroupedMLP.from_fp8(q13.view(torch.uint8), s13, q2, s2),         # e4m3 weights
           lambda: ops.B200Fp8GroupedMLP.from_fp8(q13, s13.double(), q2, s2),                  # fp32 scales
           lambda: ops.B200Fp8GroupedMLP.from_fp8(q13, s13, q2, s2, torch.float32),            # out dtype
           lambda: ops.B200Fp8GroupedMLP.from_fp8(q13[:0], s13[:0], q2[:0], s2[:0])]           # G >= 1
    for call in bad:
        with pytest.raises(capi.B200HgemmError):
            call()
