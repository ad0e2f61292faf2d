"""float32 numpy reference of the SwiGLU arithmetic (cuda_l2_b200/csrc/swiglu_arith.cuh), operation for operation.

Every step is one IEEE fp32 operation in numpy's float32; the fused multiply-add is evaluated in float64 (the product of
two floats is exact there) and rounded once to float32. expf is not correctly rounded on the GPU, so the caller passes
the exponential it wants (``exp``): numpy's on the CPU, or CUDA's through ``torch.exp`` on a float32 CUDA tensor, which
compiles the same expf as the kernels."""
from __future__ import annotations

import numpy as np
import torch

F32 = np.float32


def round_to(v: np.ndarray, dtype) -> np.ndarray:
    """RN to ``dtype`` (np.float16, "bfloat16" or np.float32), back as float32."""
    v = np.asarray(v, dtype=F32)
    if dtype is np.float32:
        return v
    if dtype is np.float16:
        return v.astype(np.float16).astype(F32)
    return torch.from_numpy(v.copy()).to(torch.bfloat16).float().numpy()


def _fma(a, b, c) -> np.ndarray:
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def silu_rn(g, dtype, exp=np.exp) -> np.ndarray:
    """RN(g / (1 + expf(-g))): the tensor ``F.silu(g)`` holds."""
    g = np.asarray(g, dtype=F32)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        return round_to(g / (F32(1) + exp(-g).astype(F32)), dtype)


def silu_mul(g, u, dtype, exp=np.exp) -> np.ndarray:
    with np.errstate(over="ignore", invalid="ignore"):
        return round_to(silu_rn(g, dtype, exp) * np.asarray(u, dtype=F32), dtype)


def swiglu_grad_reference(dy, g, u, dtype, exp=np.exp) -> tuple[np.ndarray, np.ndarray]:
    """(dg, du) of y = silu(g) * u for dy, each rounded to ``dtype``:
    du = RN(dy * s), t = RN(dy * u), sig = 1 / (1 + expf(-g)), dg = RN((t * sig) * fmaf(g, 1 - sig, 1))."""
    dy, g, u = (np.asarray(v, dtype=F32) for v in (dy, g, u))
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        du = round_to(dy * silu_rn(g, dtype, exp), dtype)
        t = round_to(dy * u, dtype)
        sig = F32(1) / (F32(1) + exp(-g).astype(F32))
        dg = round_to((t * sig) * _fma(g, F32(1) - sig, np.ones_like(g)), dtype)
    return dg, du


def cuda_exp(v: np.ndarray) -> np.ndarray:
    """CUDA's expf of float32 values, through torch.exp on the current CUDA device."""
    return torch.exp(torch.from_numpy(np.ascontiguousarray(v, dtype=F32)).cuda()).cpu().numpy()
