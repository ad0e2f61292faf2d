"""CPU reference of the block-scaled FP8 GEMM (include/b200_fp8_block.h) for the tests: ``fp8_block_ref.c``, built with
gcc on first use into a per-user temporary directory (the repository tree may be read-only where the tests run)."""
from __future__ import annotations

import ctypes
import hashlib
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

_DIR = Path(__file__).resolve().parent
_SRCS = (_DIR / "fp8_block_ref.c", _DIR.parent / "oracle" / "fp8_oracle.c", _DIR.parent / "oracle" / "hgemm_oracle.c")
_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        digest = hashlib.sha256(b"".join(p.read_bytes() for p in _SRCS)).hexdigest()[:16]
        out = Path(tempfile.gettempdir()) / f"cuda_l2_b200_ref_{os.getuid()}" / f"libfp8_block_ref_{digest}.so"
        if not out.exists():
            gcc = shutil.which("gcc")
            if gcc is None:
                raise RuntimeError("gcc not found: cannot build the block-scaled FP8 reference")
            out.parent.mkdir(parents=True, exist_ok=True)
            tmp = out.with_suffix(f".{os.getpid()}.tmp")
            cmd = [gcc, "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o", str(tmp), str(_SRCS[0]), "-lm"]
            r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"block-scaled FP8 reference build failed:\n{r.stdout}")
            os.replace(tmp, out)
        _lib = ctypes.CDLL(str(out))
        u8p, u16p, fp, i = (ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint16),
                            ctypes.POINTER(ctypes.c_float), ctypes.c_int)
        _lib.ref_fp8gemm_f32acc_block.argtypes = [u8p, u8p, fp, i, fp, u16p, i, i, i, i, i]
        _lib.ref_fp8gemm_f32acc_block.restype = None
    return _lib


def fp8gemm_f32acc_block(a_codes: np.ndarray, bt_codes: np.ndarray, sa: np.ndarray, sb: np.ndarray, out_bf16: bool,
                         splits: int = 1) -> np.ndarray:
    """``a_codes`` [M,K] / ``bt_codes`` [N,K]: uint8 float8_e4m3fn codes; ``sa`` [M, nkb] and ``sb`` [ceil(N/128), nkb]
    fp32 values. Returns the uint16 bits of C[M,N] (fp16 or bf16) by the block-scaled contract; ``splits``: the
    k-blocks divided as cluster split-K with that many splits divides them."""
    (m, k), (n, k2) = a_codes.shape, bt_codes.shape
    nkb = -(-k // 128)
    sa, sb = np.asarray(sa, dtype=np.float32), np.asarray(sb, dtype=np.float32)
    assert k == k2 and sa.shape == (m, nkb) and sb.shape == (-(-n // 128), nkb)
    sa_mmajor = np.ascontiguousarray(sa.T)          # [nkb, M]: ld_a = M
    sb = np.ascontiguousarray(sb)
    c = np.empty((m, n), dtype=np.uint16)
    u8p, u16p, fp = ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint16), ctypes.POINTER(ctypes.c_float)
    lib().ref_fp8gemm_f32acc_block(np.ascontiguousarray(a_codes).ctypes.data_as(u8p),
                                   np.ascontiguousarray(bt_codes).ctypes.data_as(u8p), sa_mmajor.ctypes.data_as(fp), m,
                                   sb.ctypes.data_as(fp), c.ctypes.data_as(u16p), m, n, k, int(bool(out_bf16)), splits)
    return c
