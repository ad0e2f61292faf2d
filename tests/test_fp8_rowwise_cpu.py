"""FP8 (e4m3) GEMM with rowwise scales, without a GPU: the CPU reference against the golden fixtures, the C ABI's
argument checks, the torch operator's shape inference and scale rule, and B200Fp8Linear's buffers."""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

import oracle
from conftest import GOLDEN
from cuda_l2_b200 import capi
from fp8_rowwise_ref import fp8gemm_f32acc_rowwise


def load_rowwise_cases():
    """Operands as uint8 e4m3 codes, scale vectors as fp32, truth as uint16 bits; kind 0 = small integers, 1 = randn."""
    z = np.load(GOLDEN / "fp8_rowwise_cases.npz")
    cases, i = [], 0
    while f"meta{i}" in z:
        m, n, k, kind, out_bf16, seed = (int(x) for x in z[f"meta{i}"])
        cases.append(dict(m=m, n=n, k=k, kind=("int", "randn")[kind], out_bf16=bool(out_bf16), seed=seed,
                          a=z[f"a{i}"], bt=z[f"bt{i}"], sa=z[f"sa{i}"], sb=z[f"sb{i}"], truth=z[f"truth{i}"]))
        i += 1
    return cases


def out_values(bits: np.ndarray, out_bf16: bool) -> np.ndarray:
    return oracle.bf16_bits_to_f32(bits) if out_bf16 else bits.view(np.float16).astype(np.float32)


def test_reference_reproduces_the_rowwise_fixtures():
    cases = load_rowwise_cases()
    assert {c["kind"] for c in cases} == {"int", "randn"} and {c["out_bf16"] for c in cases} == {False, True}
    ints = [c for c in cases if c["kind"] == "int"]
    assert any(np.any(np.log2(c["sa"]) % 1 != 0) and np.any(np.log2(c["sb"]) % 1 != 0) for c in ints)
    assert any(np.all(np.log2(c["sa"]) % 1 == 0) and np.all(np.log2(c["sb"]) % 1 == 0) for c in ints)
    assert any(c["m"] % 128 and c["n"] % 64 and c["k"] % 128 for c in ints)          # ragged in every dimension
    for c in cases:
        assert c["sa"].shape == (c["m"],) and c["sb"].shape == (c["n"],)
        got = fp8gemm_f32acc_rowwise(c["a"], c["bt"], c["sa"], c["sb"], c["out_bf16"])
        if c["kind"] == "int":
            assert np.array_equal(got, c["truth"]), (c["m"], c["n"], c["k"], c["out_bf16"])
        else:
            # torch's fp32 matmul sums in another order: the two may differ by one rounding of the output
            g, t = out_values(got, c["out_bf16"]), out_values(c["truth"], c["out_bf16"])
            ulp = 2.0 ** (-7 if c["out_bf16"] else -10)
            assert np.all(np.abs(g - t) <= ulp * np.abs(t) + 1e-6), (c["m"], c["n"], c["k"])


def test_reference_applies_the_column_scale_before_the_row_scale():
    # acc = 3; 3 * 0.1f and then * 3.0f rounds differently from 3 * 3.0f and then * 0.1f (both fp32)
    one = np.array([[0x38]], dtype=np.uint8)                            # e4m3 1.0
    three = np.array([[0x44]], dtype=np.uint8)                          # e4m3 3.0
    sa, sb = np.float32(3.0), np.float32(0.1)
    got = fp8gemm_f32acc_rowwise(three, one, [sa], [sb], False)
    want = np.float16(np.float32(np.float32(3.0) * sb) * sa)
    assert got[0, 0] == want.view(np.uint16)


def _aligned(buf) -> int:
    return (ctypes.addressof(buf) + 15) & ~15


def test_rowwise_argument_validation_happens_before_any_cuda_call(built_libs):
    lib = capi.hgemm_lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = _aligned(buf)
    s = p + 4096
    assert lib.b200_fp8gemm_rowwise(p, p, p, None, s, 0, 64, 64, 64, None) == -5       # null vector
    assert lib.b200_fp8gemm_rowwise(p, p, p, s, None, 1, 64, 64, 64, None) == -5
    assert lib.b200_fp8gemm_rowwise(p, p, p, s + 4, s, 0, 64, 64, 64, None) == -2      # 4-byte aligned is not enough
    assert lib.b200_fp8gemm_rowwise(p, p, p, s, s + 8, 0, 64, 64, 64, None) == -2
    assert lib.b200_fp8gemm_rowwise(p, p, p, s, s, 0, 64, 64, 72, None) == -9          # K % 16 != 0
    assert lib.b200_fp8gemm_rowwise(p, p, p, s, s, 0, 64, 64, 0, None) == -1
    assert lib.b200_fp8gemm_rowwise(p, p, p, s, s, 2, 64, 64, 64, None) == -6          # bad output selector
    assert lib.b200_fp8gemm_rowwise_run_config(99, 0, p, p, p, s, s, 64, 64, 64, 0, 0, 1, None) == -6   # unknown config
    assert lib.b200_fp8gemm_rowwise_run_config(0, 2, p, p, p, s, s, 64, 64, 64, 0, 0, 1, None) == -6
    assert lib.b200_fp8gemm_rowwise_run_config(0, 1, p, p, p, s + 4, s, 64, 64, 64, 0, 0, 1, None) == -2
    assert lib.b200_fp8gemm_rowwise_run_config(0, 1, p, p, p, s, None, 64, 64, 64, 0, 0, 1, None) == -5
    assert lib.b200_fp8gemm_rowwise_run_config(0, 0, p, p, p, s, s, 64, 64, 40, 0, 0, 1, None) == -9
    assert capi.launch_count() == 0


E4 = torch.float8_e4m3fn


def _meta(*shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device="meta")


def test_rowwise_operator_shapes_on_meta_tensors():
    from cuda_l2_b200 import ops
    a, b = _meta(200, 144, dtype=E4), _meta(328, 144, dtype=E4)
    for dt in (torch.float16, torch.bfloat16):
        y = ops.fp8_gemm(a, b, _meta(200, 1), _meta(1, 328), dt)
        assert y.shape == (200, 328) and y.dtype == dt and y.device.type == "meta"
    assert capi.scale_granularity(200, 328, _meta(200, 1), _meta(1, 328)) == "rowwise"
    assert capi.scale_granularity(200, 328, _meta(1), _meta(1, 1)) == "tensor"
    assert capi.scale_granularity(1, 8, _meta(1, 1), _meta(1, 1)) == "tensor"      # one element each: per tensor


@pytest.mark.parametrize("sa,sb", [
    ((200, 1), (1,)),            # mixed granularity
    ((1,), (1, 328)),            # mixed granularity
    ((199, 1), (1, 328)),        # [M-1, 1]
    ((200, 1), (1, 320)),        # [1, N-8]
    ((200,), (328,)),            # 1-D vectors
    ((1, 200), (328, 1)),        # transposed
    ((200, 1), (328, 1)),
])
def test_rowwise_scale_shapes_that_are_rejected(sa, sb):
    from cuda_l2_b200 import ops
    a, b = _meta(200, 144, dtype=E4), _meta(328, 144, dtype=E4)
    with pytest.raises(capi.B200HgemmError):
        ops.fp8_gemm(a, b, _meta(*sa), _meta(*sb), torch.float16)


def test_rowwise_scales_must_be_fp32():
    from cuda_l2_b200 import ops
    a, b = _meta(200, 144, dtype=E4), _meta(328, 144, dtype=E4)
    for sa, sb in ((_meta(200, 1, dtype=torch.float16), _meta(1, 328)), (_meta(200, 1), _meta(1, 328, dtype=torch.bfloat16))):
        with pytest.raises(capi.B200HgemmError):
            ops.fp8_gemm(a, b, sa, sb, torch.float16)


def test_rowwise_python_binding_checks_before_the_library():
    a = torch.zeros((64, 64), dtype=E4)
    c = torch.zeros((64, 64), dtype=torch.half)
    with pytest.raises(capi.B200HgemmError):
        capi.fp8_gemm(a, a, c, torch.ones(64, 1), torch.ones(1, 64))       # CPU tensors: no fallback


def test_quantize_e4m3_rowwise():
    from cuda_l2_b200 import ops
    x = torch.randn(6, 64, dtype=torch.float16)
    x[2] *= 1000
    x[4] = 0
    q, s = ops.quantize_e4m3_rowwise(x)
    assert q.dtype == E4 and q.shape == x.shape and s.dtype == torch.float32 and s.shape == (6, 1)
    assert torch.equal(s[:, 0], (x.abs().amax(dim=1).float() / 448).clamp_min(torch.finfo(torch.float32).tiny))
    assert torch.equal(q.float()[4], torch.zeros(64))
    assert torch.allclose(q.float() * s, x.float(), rtol=2 ** -4, atol=1e-6)


def test_fp8_linear_granularity_buffers():
    from cuda_l2_b200 import ops
    lin = nn.Linear(64, 32, dtype=torch.float16)
    t = ops.B200Fp8Linear.from_linear(lin)
    assert t.granularity == "tensor" and t.weight_scale.shape == (1,)
    r = ops.B200Fp8Linear.from_linear(lin, granularity="rowwise")
    assert r.granularity == "rowwise" and r.weight_scale.shape == (1, 32) and r.weight_scale.dtype == torch.float32
    assert r.weight_fp8.dtype == E4 and r.weight_fp8.shape == (32, 64)
    assert set(dict(r.named_buffers())) == {"weight_fp8", "weight_scale"} and r.bias is lin.bias
    assert torch.allclose(r.weight_fp8.float() * r.weight_scale.t(), lin.weight.float(), rtol=2 ** -4, atol=1e-6)
    assert "granularity=rowwise" in repr(r) and "granularity=tensor" in repr(t)
    with pytest.raises(capi.B200HgemmError):
        ops.B200Fp8Linear.from_linear(lin, granularity="block")
