"""Deployable face of the kernel: a ``torch.library`` custom op and an ``nn.Linear`` drop-in.

The reference's README lists "easy deployment for open-source LLMs" as to-do and tells users of off-grid shapes to pad
to the nearest larger configuration (README.md:75,83-86). Here nothing is padded — the kernels take any
``M, N, K > 0`` with ``N % 8 == 0`` and ``K % 8 == 0`` and the dispatcher maps an off-grid shape to the tuned entry of
the nearest grid shape — so deployment is a plain operator:

* ``torch.ops.cuda_l2_b200.hgemm(a, b_kmajor, acc)``: ``a`` [M,K] times B given K-major as ``b_kmajor`` [N,K]
  (exactly the layout of an ``nn.Linear`` weight: ``[out_features, in_features]``), returns [M,N]. fp16 or bf16
  operands (bf16 always accumulates in fp32); ``acc`` = "fp32" | "fp16".
* :class:`B200Linear`: ``y = x @ W^T (+ b)`` for any leading dimensions; :func:`replace_linear_modules` swaps the
  eligible ``nn.Linear`` layers of a model in place.

There is no CPU or PyTorch fallback on the forward path: a non-CUDA tensor, a missing library or a non-H100 device
raises. Backward (training is not what the reference targets) is provided through the same kernel on explicitly
transposed copies, so a fine-tuning loop works, at the price of two transposes per layer.
"""
from __future__ import annotations

import torch
from torch import nn

from . import capi

_LIB = "cuda_l2_b200"
_DTYPES = (torch.float16, torch.bfloat16)

torch.library.define(f"{_LIB}::hgemm", "(Tensor a, Tensor b_kmajor, str acc='fp32') -> Tensor")


def _check_operands(a: torch.Tensor, b_kmajor: torch.Tensor, acc: str) -> tuple[int, int, int]:
    if a.dim() != 2 or b_kmajor.dim() != 2:
        raise capi.B200HgemmError(f"hgemm wants 2-D operands, got {tuple(a.shape)} and {tuple(b_kmajor.shape)}")
    if a.dtype not in _DTYPES or b_kmajor.dtype != a.dtype:
        raise capi.B200HgemmError(f"hgemm wants matching fp16 or bf16 operands, got {a.dtype} and {b_kmajor.dtype}")
    if acc not in ("fp32", "fp16"):
        raise capi.B200HgemmError(f"acc must be 'fp32' or 'fp16', got {acc!r}")
    if a.dtype == torch.bfloat16 and acc != "fp32":
        raise capi.B200HgemmError("bf16 operands accumulate in fp32 only (wgmma has no bf16 accumulator)")
    m, k = a.shape
    n, k2 = b_kmajor.shape
    if k2 != k:
        raise capi.B200HgemmError(f"inner dimensions differ: a {tuple(a.shape)}, b_kmajor {tuple(b_kmajor.shape)} (K-major: [N, K])")
    if n % 8 or k % 8:
        raise capi.B200HgemmError(f"N and K must be multiples of 8 (16-byte TMA strides), got N={n}, K={k}")
    return m, n, k


@torch.library.impl(f"{_LIB}::hgemm", "CUDA")
def _hgemm_cuda(a: torch.Tensor, b_kmajor: torch.Tensor, acc: str = "fp32") -> torch.Tensor:
    m, n, k = _check_operands(a, b_kmajor, acc)
    a = a.contiguous()
    b_kmajor = b_kmajor.contiguous()
    c = torch.empty((m, n), dtype=a.dtype, device=a.device)
    if m == 0:
        return c
    with torch.cuda.device(a.device):
        # the kernel is launched on torch's current stream, so it orders with the surrounding torch ops
        capi.gemm_kmajor(a, b_kmajor, c, acc, stream=torch.cuda.current_stream(a.device).cuda_stream)
    return c


@torch.library.impl(f"{_LIB}::hgemm", "CPU")
def _hgemm_cpu(a, b_kmajor, acc="fp32"):
    raise capi.B200HgemmError("cuda_l2_b200::hgemm has no CPU implementation (and no fallback): move the tensors to an H100")


@torch.library.register_fake(f"{_LIB}::hgemm")
def _hgemm_fake(a, b_kmajor, acc="fp32"):
    m, n, _ = _check_operands(a, b_kmajor, acc)
    return a.new_empty((m, n))


def _hgemm_backward(ctx, grad_c):
    a, b_kmajor = ctx.saved_tensors
    grad_a = grad_b = None
    g = grad_c.contiguous()
    # C = A Bt^T  =>  dA = dC Bt  (reduction over N: B operand K-major in N = Bt^T),  dBt = dC^T A  (reduction over M)
    if ctx.needs_input_grad[0]:
        grad_a = torch.ops.cuda_l2_b200.hgemm(g, b_kmajor.t().contiguous(), "fp32")
    if ctx.needs_input_grad[1]:
        grad_b = torch.ops.cuda_l2_b200.hgemm(g.t().contiguous(), a.t().contiguous(), "fp32")
    return grad_a, grad_b, None


def _hgemm_setup_context(ctx, inputs, output):
    a, b_kmajor, _ = inputs
    ctx.save_for_backward(a, b_kmajor)


torch.library.register_autograd(f"{_LIB}::hgemm", _hgemm_backward, setup_context=_hgemm_setup_context)


def hgemm(a: torch.Tensor, b_kmajor: torch.Tensor, acc: str = "fp32") -> torch.Tensor:
    """``a`` [M,K] @ ``b_kmajor`` [N,K]^T -> [M,N] through the H100 kernel (see the module docstring)."""
    return torch.ops.cuda_l2_b200.hgemm(a, b_kmajor, acc)


def linear_supported(in_features: int, out_features: int, dtype: torch.dtype) -> bool:
    return dtype in _DTYPES and in_features % 8 == 0 and out_features % 8 == 0


class B200Linear(nn.Module):
    """``nn.Linear`` whose matmul runs on the H100 HGEMM kernel. The weight keeps ``nn.Linear``'s layout
    ``[out_features, in_features]`` — which IS the kernel's K-major B operand — so swapping a layer copies nothing."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, device=None,
                 dtype: torch.dtype = torch.float16, acc: str = "fp32"):
        super().__init__()
        if not linear_supported(in_features, out_features, dtype):
            raise capi.B200HgemmError(f"B200Linear needs fp16/bf16 and feature counts divisible by 8, got "
                                      f"{in_features}->{out_features} {dtype}")
        self.in_features, self.out_features, self.acc = in_features, out_features, acc
        self.weight = nn.Parameter(torch.empty((out_features, in_features), device=device, dtype=dtype))
        self.bias = nn.Parameter(torch.empty(out_features, device=device, dtype=dtype)) if bias else None
        self.reset_parameters()

    def reset_parameters(self) -> None:
        bound = 1.0 / (self.in_features ** 0.5)
        with torch.no_grad():
            self.weight.uniform_(-bound, bound)
            if self.bias is not None:
                self.bias.uniform_(-bound, bound)

    @classmethod
    def from_linear(cls, lin: nn.Linear, acc: str = "fp32") -> "B200Linear":
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        if not linear_supported(lin.in_features, lin.out_features, lin.weight.dtype):
            raise capi.B200HgemmError(f"cannot convert {lin}: needs fp16/bf16 weights and feature counts divisible by 8")
        new.in_features, new.out_features, new.acc = lin.in_features, lin.out_features, acc
        new.weight, new.bias = lin.weight, lin.bias          # shared storage, no copy
        return new

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        lead = x.shape[:-1]
        y = torch.ops.cuda_l2_b200.hgemm(x.reshape(-1, self.in_features), self.weight, self.acc)
        if self.bias is not None:
            y = y + self.bias
        return y.view(*lead, self.out_features)

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, acc={self.acc}"


def replace_linear_modules(model: nn.Module, acc: str = "fp32", skip: tuple[str, ...] = ()) -> list[str]:
    """Swap every eligible ``nn.Linear`` of ``model`` (fp16/bf16 weights, features divisible by 8) for a
    :class:`B200Linear` sharing its parameters. Returns the qualified names that were replaced."""
    done = []
    for name, mod in list(model.named_modules()):
        for child_name, child in list(mod.named_children()):
            full = f"{name}.{child_name}" if name else child_name
            if type(child) is nn.Linear and full not in skip and \
                    linear_supported(child.in_features, child.out_features, child.weight.dtype):
                setattr(mod, child_name, B200Linear.from_linear(child, acc))
                done.append(full)
    return done


__all__ = ["hgemm", "B200Linear", "replace_linear_modules", "linear_supported"]
