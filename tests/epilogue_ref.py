"""CPU reference of the fused bias + activation epilogue (libb200_epilogue.so, csrc/b200_epilogue.h), for operands whose
products sum exactly in fp32 (tests/exact_domain.py's domains):

  s  = the float64 sum A @ Bt^T, rounded to fp32 as the kernel's sum is (exact on these domains)
       e4m3 per tensor: fp32(s * fp32(sa * sb));  rowwise: fp32(fp32(s * sb[n]) * sa[m])
  z  = fp32(s + fp32(bias[n]))                   one IEEE fp32 addition (none without a bias)
  y  = round_out(act(z))                         relu: z > 0 ? z : +0.0; gelu_tanh in float64, rounded once

gelu_tanh is 0.5 z (1 + tanh(u)), u = sqrt(2/pi) (z + 0.044715 z^3), in float64. The kernel evaluates the same form in
fp32 with CUDA's tanhf, whose 1 + tanhf(u) carries an absolute error of a few 2^-24: gelu_excess() states what that
allows against this reference (one unit in the last place, plus |z| 2^-22 where 1 + tanh(u) has cancelled)."""
from __future__ import annotations

import numpy as np

import oracle

ACTIVATIONS = ("none", "relu", "gelu_tanh")


def gelu_tanh(z: np.ndarray) -> np.ndarray:
    z = np.asarray(z, dtype=np.float64)
    u = np.sqrt(2.0 / np.pi) * (z + 0.044715 * z ** 3)
    return 0.5 * z * (1.0 + np.tanh(u))


GELU_ABS = 2.0 ** -22   # times |z|: the fp32 form's absolute error bound, 0.5 |z| times 2^-21 for 1 + tanhf(u)


def ulp_at(x: np.ndarray, out: str) -> np.ndarray:
    """The spacing of fp16 / bf16 values at |x| (the subnormal spacing below the smallest normal)."""
    p, emin = (11, -14) if out == "fp16" else (8, -126)
    ax = np.abs(np.asarray(x, dtype=np.float64))
    e = np.where(ax > 0, np.maximum(np.frexp(ax)[1] - 1, emin), emin)
    return np.exp2((e - (p - 1)).astype(np.float64))


def gelu_excess(got_bits: np.ndarray, z: np.ndarray, out: str) -> np.ndarray:
    """How far each gelu_tanh output lies outside what the kernel's fp32 form allows against the float64 reference:
    |got - gelu(z)| - (one unit in the last place at gelu(z) + |z| GELU_ABS). At most 0 everywhere."""
    want = gelu_tanh(z)
    got = bits_to_f64(got_bits, out)
    return np.abs(got - want) - (ulp_at(want, out) + np.abs(np.asarray(z, dtype=np.float64)) * GELU_ABS)


def activate(z: np.ndarray, activation: str) -> np.ndarray:
    """act(z) of fp32 values z: fp32 for none / relu, float64 for gelu_tanh (rounded once by round_out)."""
    if activation == "relu":
        return np.where(z > 0, z, np.float32(0.0)).astype(np.float32)
    if activation == "gelu_tanh":
        return gelu_tanh(z)
    return z


def round_out(x: np.ndarray, out: str) -> np.ndarray:
    """float32 / float64 values -> fp16 or bf16 bits, round to nearest even. fp16: one rounding from the value itself.
    bf16: through fp32, one rounding for fp32 values (none, relu), at most two for gelu_tanh's float64 ones (the tests
    allow it one unit in the last place)."""
    x = np.asarray(x)
    if out == "fp16":
        with np.errstate(over="ignore"):   # values past 65504 round to inf, as they should
            return x.astype(np.float16).view(np.uint16)
    return oracle.f32_to_bf16_bits(x.astype(np.float32))


def fp32_sum(a: np.ndarray, bt: np.ndarray) -> np.ndarray:
    """A @ Bt^T in float64, rounded to fp32."""
    return (np.asarray(a, dtype=np.float64) @ np.asarray(bt, dtype=np.float64).T).astype(np.float32)


def scaled(s: np.ndarray, scale_a=None, scale_b=None, rowwise: bool = False) -> np.ndarray:
    """The e4m3 scale steps on the fp32 sum s (per tensor or rowwise), in fp32."""
    if scale_a is None:
        return s
    sa, sb = np.asarray(scale_a, dtype=np.float32), np.asarray(scale_b, dtype=np.float32)
    if rowwise:
        return (s * sb.reshape(1, -1)) * sa.reshape(-1, 1)
    return s * (sa.reshape(()) * sb.reshape(()))


def pre_activation(a, bt, bias_f32=None, scale_a=None, scale_b=None, rowwise=False) -> np.ndarray:
    """z as fp32 values: the scaled fp32 sum plus the bias (fp32 values of the output-typed bias), one fp32 addition."""
    z = scaled(fp32_sum(a, bt), scale_a, scale_b, rowwise).astype(np.float32)
    if bias_f32 is not None:
        z = z + np.asarray(bias_f32, dtype=np.float32).reshape(1, -1)
    return z


def reference(a, bt, bias_f32, activation: str, out: str, scale_a=None, scale_b=None, rowwise=False) -> np.ndarray:
    """Output bits of the fused product (module docstring)."""
    return round_out(activate(pre_activation(a, bt, bias_f32, scale_a, scale_b, rowwise), activation), out)


def bits_to_f64(bits: np.ndarray, out: str) -> np.ndarray:
    bits = np.asarray(bits, dtype=np.uint16)
    if out == "fp16":
        return bits.view(np.float16).astype(np.float64)
    return oracle.bf16_bits_to_f32(bits).astype(np.float64)


def ulp_distance(got_bits: np.ndarray, want_bits: np.ndarray) -> np.ndarray:
    """Units in the last place between two arrays of 16-bit floats of one type (sign-magnitude order; +0 and -0 are 0
    apart)."""
    def key(b):
        b = np.asarray(b, dtype=np.uint16).astype(np.int32)
        return np.where(b & 0x8000, -(b & 0x7FFF), b)
    return np.abs(key(got_bits) - key(want_bits))
