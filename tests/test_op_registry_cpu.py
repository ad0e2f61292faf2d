"""What every cuda_l2_b200 operator's registration promises, without a GPU: its schema, the refusal of CPU tensors, the
refusal of a backward through an inference-only operator (with its reason), the shapes and dtypes of the gradients
of the differentiable ones on meta tensors, and an entry point's status decoded by the library that returned it."""
import pytest
import torch

from cuda_l2_b200 import capi, ops  # noqa: F401  (ops registers the operators)

SCHEMAS = {
    "fp8_batched_gemm": "(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, ScalarType out_dtype, "
                        "Tensor? masked_m=None) -> Tensor",
    "fp8_gemm": "(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, ScalarType out_dtype) -> Tensor",
    "fp8_gemm_bias_act": "(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, Tensor? bias, str activation, "
                         "ScalarType out_dtype) -> Tensor",
    "fp8_grouped_gemm": "(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, Tensor offs, "
                        "ScalarType out_dtype) -> Tensor",
    "grouped_linear": '(Tensor x, Tensor w, Tensor offs, str acc="fp32") -> Tensor',
    "hgemm": '(Tensor a, Tensor b_kmajor, str acc="fp32") -> Tensor',
    "hgemm_batched": '(Tensor a, Tensor b_kmajor, str acc="fp32", Tensor? masked_m=None) -> Tensor',
    "hgemm_bias_act": '(Tensor a, Tensor b_kmajor, Tensor? bias, str activation="none") -> Tensor',
    "hgemm_grouped": '(Tensor a, Tensor b_kmajor, Tensor offs, str acc="fp32") -> Tensor',
    "hgemm_grouped_nn": '(Tensor a, Tensor b, Tensor offs, str acc="fp32") -> Tensor',
    "hgemm_grouped_wgrad": '(Tensor a, Tensor b, Tensor offs, str acc="fp32") -> Tensor',
    "hgemm_nn": '(Tensor a, Tensor b, str acc="fp32") -> Tensor',
    "quantize_e4m3": "(Tensor x) -> (Tensor, Tensor)",
    "quantize_e4m3_blockwise": "(Tensor x, Tensor? masked_m=None) -> (Tensor, Tensor)",
    "quantize_e4m3_rowwise": "(Tensor x) -> (Tensor, Tensor)",
    "quantize_e4m3_rowwise_dual": "(Tensor x) -> (Tensor, Tensor, Tensor, Tensor)",
    "silu_mul_quantize_e4m3_blockwise": "(Tensor h, Tensor? masked_m=None) -> (Tensor, Tensor)",
}

_QUANT = " (quantisation is not differentiable: train the 16-bit model and quantise afterwards)"
_BWD_KERNEL = " (it is a backward kernel: train through grouped_linear)"
# The reason each inference-only operator gives for having no gradient.
WHY = {
    "hgemm_grouped": " (train through grouped_linear, the same product with a gradient)",
    "hgemm_grouped_nn": _BWD_KERNEL,
    "hgemm_grouped_wgrad": _BWD_KERNEL,
    "fp8_gemm": " (train with the fp16 / bf16 operator and quantise afterwards)",
    "fp8_gemm_bias_act": " (train with the fp16 / bf16 operator hgemm_bias_act and quantise afterwards)",
    "fp8_grouped_gemm": "",
    "fp8_batched_gemm": "",
    "quantize_e4m3": _QUANT,
    "quantize_e4m3_rowwise": _QUANT,
    "quantize_e4m3_blockwise": _QUANT,
    "silu_mul_quantize_e4m3_blockwise": _QUANT,
    "quantize_e4m3_rowwise_dual": _QUANT,
}


def _args(name: str, device: str) -> tuple:
    """Arguments every check of operator ``name`` accepts (T = M = 16, N = 24, K = 32, three groups, two batches)."""
    h, b, e, f, i = torch.float16, torch.bfloat16, torch.float8_e4m3fn, torch.float32, torch.int32

    def t(*shape, dtype=h):
        return torch.zeros(shape, dtype=dtype, device=device)

    return {
        "hgemm": (t(16, 32), t(24, 32), "fp32"),
        "hgemm_nn": (t(16, 32), t(32, 24), "fp32"),
        "hgemm_batched": (t(2, 16, 32), t(2, 24, 32), "fp32", None),
        "hgemm_grouped": (t(16, 32), t(3, 24, 32), t(3, dtype=i), "fp32"),
        "hgemm_grouped_nn": (t(16, 32), t(3, 32, 24), t(3, dtype=i), "fp32"),
        "hgemm_grouped_wgrad": (t(16, 32), t(16, 24), t(3, dtype=i), "fp32"),
        "grouped_linear": (t(16, 32), t(3, 24, 32), t(3, dtype=i), "fp32"),
        "hgemm_bias_act": (t(16, 32), t(24, 32), t(24), "relu"),
        "fp8_gemm": (t(16, 32, dtype=e), t(24, 32, dtype=e), t(1, dtype=f), t(1, dtype=f), h),
        "fp8_gemm_bias_act": (t(16, 32, dtype=e), t(24, 32, dtype=e), t(16, 1, dtype=f), t(1, 24, dtype=f), t(24),
                              "gelu_tanh", h),
        "fp8_grouped_gemm": (t(16, 32, dtype=e), t(3, 24, 32, dtype=e), t(16, 1, dtype=f), t(3, 1, 1, dtype=f),
                             t(3, dtype=i), b),
        "fp8_batched_gemm": (t(2, 16, 32, dtype=e), t(2, 24, 32, dtype=e), t(2, 16, 1, dtype=f), t(2, 1, 1, dtype=f), b,
                             None),
        "quantize_e4m3": (t(16, 32, dtype=b),),
        "quantize_e4m3_rowwise": (t(16, 32, dtype=b),),
        "quantize_e4m3_blockwise": (t(16, 32, dtype=b), None),
        "silu_mul_quantize_e4m3_blockwise": (t(16, 64, dtype=b), None),
        "quantize_e4m3_rowwise_dual": (t(16, 32, dtype=b),),
    }[name]


def _op(name: str):
    return getattr(torch.ops.cuda_l2_b200, name)


def test_every_schema():
    assert {n for n in dir(torch.ops.cuda_l2_b200) if not n.startswith("_") and n != "name"} == set(SCHEMAS)
    for name, schema in SCHEMAS.items():
        assert str(_op(name).default._schema) == f"cuda_l2_b200::{name}{schema}"


@pytest.mark.parametrize("name", sorted(SCHEMAS))
def test_cpu_tensors_have_no_implementation(name):
    with pytest.raises(capi.B200HgemmError) as err:
        _op(name)(*_args(name, "cpu"))
    assert str(err.value) == (f"cuda_l2_b200::{name} has no CPU implementation (and no fallback): move the tensors to "
                              f"an H100")


@pytest.mark.parametrize("name", sorted(WHY))
def test_a_backward_through_an_inference_only_operator_raises_its_reason(name):
    args = tuple(a.requires_grad_() if isinstance(a, torch.Tensor) and a.is_floating_point() else a
                 for a in _args(name, "meta"))
    out = _op(name)(*args)
    loss = sum(o.float().sum() for o in (out if isinstance(out, tuple) else (out,)))
    with pytest.raises(capi.B200HgemmError) as err:
        loss.backward()
    assert str(err.value) == f"cuda_l2_b200::{name} is inference only: it has no gradient{WHY[name]}"


def test_a_backward_through_the_masked_batched_product_raises():
    a, b_kmajor, acc, _ = _args("hgemm_batched", "meta")
    y = _op("hgemm_batched")(a.requires_grad_(), b_kmajor, acc, torch.zeros(2, dtype=torch.int32, device="meta"))
    with pytest.raises(capi.B200HgemmError) as err:
        y.sum().backward()
    assert str(err.value) == "cuda_l2_b200::hgemm_batched with masked_m is inference only: it has no gradient"


def _grads_match_inputs(y: torch.Tensor, inputs: tuple) -> None:
    grads = torch.autograd.grad(y.sum(), inputs)
    for g, x in zip(grads, inputs, strict=True):
        assert (g.shape, g.dtype, g.device) == (x.shape, x.dtype, x.device)


def _meta(*shape, dtype):
    return torch.empty(shape, dtype=dtype, device="meta", requires_grad=True)


# The token count M is free: the weight gradient reduces over it, at M % 8 != 0 through the K-grouped kernel.
TOKENS = [40, 41, 1, 193]


@pytest.mark.parametrize("m", TOKENS)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_meta_gradients_of_the_products(dtype, m):
    a, b_kmajor, b = _meta(m, 32, dtype=dtype), _meta(24, 32, dtype=dtype), _meta(32, 24, dtype=dtype)
    _grads_match_inputs(ops.hgemm(a, b_kmajor), (a, b_kmajor))
    _grads_match_inputs(ops.hgemm_nn(a, b), (a, b))
    a3, b3 = _meta(3, m, 32, dtype=dtype), _meta(3, 24, 32, dtype=dtype)
    _grads_match_inputs(ops.hgemm_batched(a3, b3), (a3, b3))
    lin = ops.B200Linear(32, 24, device="meta", dtype=dtype)
    x = _meta(3, m, 32, dtype=dtype)
    _grads_match_inputs(lin(x), (x, lin.weight, lin.bias))


@pytest.mark.parametrize("m", TOKENS)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("activation", ["none", "relu", "gelu_tanh"])
@pytest.mark.parametrize("with_bias", [True, False])
def test_meta_gradients_of_bias_act(dtype, activation, with_bias, m):
    a, b_kmajor = _meta(m, 32, dtype=dtype), _meta(24, 32, dtype=dtype)
    bias = _meta(24, dtype=dtype) if with_bias else None
    inputs = (a, b_kmajor, bias) if with_bias else (a, b_kmajor)
    _grads_match_inputs(ops.hgemm_bias_act(a, b_kmajor, bias, activation), inputs)


@pytest.mark.parametrize("select, lib, symbol, strerror, args", [
    (capi.epilogue_select, capi.epilogue_lib, "cuda_l2_b200_epilogue_select", "cuda_l2_b200_epilogue_strerror",
     (1, 64, 64, 64)),
    (capi.grouped_nn_select, capi.grouped_bwd_lib, "cuda_l2_b200_grouped_bwd_nn_select",
     "cuda_l2_b200_grouped_bwd_strerror", (1, 4, 64, 64, 64)),
    (capi.batched_select, capi.batched_lib, "b200_batched_select", "b200_batched_strerror", (7, 4, 64, 64, 64)),
])
def test_a_select_status_is_decoded_by_its_own_library(built_libs, select, lib, symbol, strerror, args):
    """A variant without a kernel: the status comes back before any CUDA call."""
    with pytest.raises(capi.B200HgemmError) as err:
        select(*args)
    assert str(err.value) == f"{symbol} failed: status -6 ({getattr(lib(), strerror)(-6).decode()})"
