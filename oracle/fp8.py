"""CPU oracle of the FP8 (e4m3) GEMM — TEST INFRASTRUCTURE, never the product (same rules as the ``oracle`` package).

``fp8_oracle.c`` restates the e4m3 codec and ``C = RN_out(fp32(A @ Bt^T) * fp32(scale_a * scale_b))`` with one
canonical fp32 accumulator; it includes ``hgemm_oracle.c`` for the bit-exact fp16 / bf16 output roundings and is built
into its own library, ``libfp8_oracle.so``. Pinned by ``tests/golden/fp8_cases.npz`` (``tests/golden/make_fp8_golden.py``).
"""
from __future__ import annotations

import ctypes
import shutil
import subprocess
from pathlib import Path

import numpy as np

_DIR = Path(__file__).resolve().parent
_SRCS = (_DIR / "fp8_oracle.c", _DIR / "hgemm_oracle.c")
_LIB = _DIR / "libfp8_oracle.so"
_lib = None


def build(force: bool = False) -> Path:
    """Compile fp8_oracle.c with gcc (generic x86-64 code, like the 16-bit oracle)."""
    if not force and _LIB.exists() and all(_LIB.stat().st_mtime >= s.stat().st_mtime for s in _SRCS):
        return _LIB
    gcc = shutil.which("gcc")
    if gcc is None:
        raise RuntimeError("gcc not found: cannot build the FP8 CPU oracle")
    cmd = [gcc, "-O2", "-fopenmp", "-shared", "-fPIC", "-o", str(_LIB), str(_SRCS[0]), "-lm"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"FP8 oracle build failed:\n{r.stdout}")
    return _LIB


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(str(build()))
        u8p, u16p, i = ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint16), ctypes.c_int
        _lib.oracle_e4m3_to_f32.argtypes = [ctypes.c_uint8]
        _lib.oracle_e4m3_to_f32.restype = ctypes.c_float
        _lib.oracle_f32_to_e4m3.argtypes = [ctypes.c_float]
        _lib.oracle_f32_to_e4m3.restype = ctypes.c_uint8
        _lib.oracle_fp8gemm_f32acc.argtypes = [u8p, u8p, ctypes.c_float, ctypes.c_float, u16p, i, i, i, i]
    return _lib


def e4m3_to_f32(codes: np.ndarray) -> np.ndarray:
    """float8_e4m3fn codes (uint8) -> their exact fp32 values (NaN for 0x7F / 0xFF)."""
    f = lib().oracle_e4m3_to_f32
    return np.array([f(int(c)) for c in np.asarray(codes, dtype=np.uint8).ravel()], dtype=np.float32).reshape(np.shape(codes))


def f32_to_e4m3(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even fp32 -> float8_e4m3fn codes (uint8), for |x| <= 448."""
    f = lib().oracle_f32_to_e4m3
    return np.array([f(float(v)) for v in np.asarray(x, dtype=np.float32).ravel()], dtype=np.uint8).reshape(np.shape(x))


def fp8gemm_f32acc(a_codes: np.ndarray, bt_codes: np.ndarray, scale_a: float, scale_b: float, out_bf16: bool) -> np.ndarray:
    """``a_codes`` [M,K] and ``bt_codes`` [N,K] are uint8 float8_e4m3fn codes, the scales fp32 values. Returns the uint16
    bits of C[M,N] = RN_out(fp32(A @ Bt^T) * fp32(scale_a * scale_b)), fp16 or bf16."""
    (m, k), (n, k2) = a_codes.shape, bt_codes.shape
    assert k == k2 and a_codes.dtype == np.uint8 and bt_codes.dtype == np.uint8
    c = np.empty((m, n), dtype=np.uint16)
    u8p, u16p = ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint16)
    lib().oracle_fp8gemm_f32acc(np.ascontiguousarray(a_codes).ctypes.data_as(u8p), np.ascontiguousarray(bt_codes).ctypes.data_as(u8p),
                                float(np.float32(scale_a)), float(np.float32(scale_b)), c.ctypes.data_as(u16p), m, n, k,
                                int(bool(out_bf16)))
    return c


__all__ = ["build", "lib", "e4m3_to_f32", "f32_to_e4m3", "fp8gemm_f32acc"]
