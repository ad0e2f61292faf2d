"""How often one FP8 GEMM call classifies its scales (capi.scale_granularity), on the H100.

The classification is Python run on every call of the decode-size FP8 path. An operator classifies once in its shape
check, which the fake path needs too, and hands the granularity to its launch; capi.fp8_gemm and capi.gemm_bias_act
classify once each and pick the entry point and its scale arguments from that one answer. Each call is also
bit-compared with the direct capi call on kernel-ready scales, so the scales that reach the kernel are the same.
"""
import pytest
import torch

from cuda_l2_b200 import capi, ops

pytestmark = pytest.mark.gpu

M, N, K = 64, 256, 512


@pytest.fixture
def calls(monkeypatch):
    """The (M, N) of every capi.scale_granularity call made while the test runs."""
    seen, real = [], capi.scale_granularity

    def counted(*args, **kwargs):
        seen.append(args[:2])
        return real(*args, **kwargs)

    monkeypatch.setattr(capi, "scale_granularity", counted)
    return seen


def operands(granularity: str, m_major: bool):
    """e4m3 a [M,K] and bt [N,K] with scales of ``granularity``; ``m_major=False`` gives 1 x 128 scales as contiguous
    [rows, nkb] tensors, which the operator copies into the M-major layout."""
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn((M, K), device="cuda", generator=gen)
    w = torch.randn((N, K), device="cuda", generator=gen)
    if granularity == "tensor":
        (a, sa), (bt, sb) = ops.quantize_e4m3(x), ops.quantize_e4m3(w)
    elif granularity == "rowwise":
        (a, sa), (bt, sb) = ops.quantize_e4m3_rowwise(x), ops.quantize_e4m3_rowwise(w)
        sb = sb.reshape(1, N)
    elif granularity == "blockwise":
        (a, sa), (bt, sb) = ops.quantize_e4m3_blockwise(x), ops.quantize_e4m3_block128x128(w)
    else:
        (a, sa), (bt, sb) = ops.quantize_e4m3_blockwise(x), ops.quantize_e4m3_blockwise(w)
    if not m_major:
        sa = sa.contiguous()
        sb = sb.contiguous()
        assert capi.blockwise_ld_a(sa) is None
    return a, bt, sa, sb


def kernel_ready(granularity: str, sa, sb):
    """The scales as capi.fp8_gemm takes them, made without classifying."""
    return (capi.m_major(sa) if granularity.startswith("blockwise") else sa,
            capi.m_major(sb) if granularity == "blockwise_1d1d" else sb)


def bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("granularity, m_major", [("tensor", True), ("rowwise", True), ("blockwise", True),
                                                  ("blockwise", False), ("blockwise_1d1d", True),
                                                  ("blockwise_1d1d", False)])
def test_fp8_gemm_classifies_in_its_shape_check_and_in_capi_only(calls, granularity, m_major):
    a, bt, sa, sb = operands(granularity, m_major)
    assert capi.scale_granularity(M, N, sa, sb, k=K) == granularity
    calls.clear()
    y = ops.fp8_gemm(a, bt, sa, sb, torch.bfloat16)
    assert calls == [(M, N)] * 2                     # the operator's shape check, then capi.fp8_gemm
    dsa, dsb = kernel_ready(granularity, sa, sb)
    calls.clear()
    c = torch.empty_like(y)
    capi.fp8_gemm(a, bt, c, dsa, dsb, stream=torch.cuda.current_stream().cuda_stream)
    assert calls == [(M, N)]
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(c))


@pytest.mark.parametrize("granularity", ["tensor", "rowwise"])
def test_fp8_gemm_bias_act_classifies_in_its_shape_check_and_in_capi_only(calls, granularity):
    a, bt, sa, sb = operands(granularity, True)
    bias = torch.randn(N, device="cuda").bfloat16()
    calls.clear()
    y = ops.fp8_gemm_bias_act(a, bt, sa, sb, bias, "relu", torch.bfloat16)
    assert calls == [(M, N)] * 2                     # the operator's shape check, then capi.gemm_bias_act
    calls.clear()
    c = torch.empty_like(y)
    capi.gemm_bias_act(a, bt, c, bias, "relu", sa, sb, stream=torch.cuda.current_stream().cuda_stream)
    assert calls == [(M, N)]
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(c))
