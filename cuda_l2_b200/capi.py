"""ctypes binding of the C-ABI libraries (include/b200_hgemm.h, include/b200_baselines.h).

This is the Python face of the drop-in boundary: the same entry points the torch extension
(``pybind/hgemm_b200_fp32.cc`` / ``hgemm_b200_fp16.cc``) wraps, reachable without a JIT build.  Tensors
are torch CUDA tensors used purely as device-memory handles (``data_ptr()``); all arithmetic happens in
``libb200_hgemm.so``.  There is no CPU or PyTorch fallback: if the library is missing or the device is
not an H100, these functions raise.
"""
from __future__ import annotations

import ctypes
from pathlib import Path
from typing import NamedTuple

LIB_DIR = Path(__file__).resolve().parent / "lib"

ACC_BITS = {"fp32": 32, "fp16": 16, 32: 32, 16: 16}


class B200HgemmError(RuntimeError):
    pass


# The entry points of a tile-list library, b200_<prefix>_<suffix>, with the same signatures in both libraries of a
# pair: suffix -> (argtypes, restype). The 16-bit pair (include/b200_batched.h, include/b200_grouped.h) and the
# block-scaled FP8 pair (include/b200_batched_fp8.h, include/b200_grouped_fp8.h).
_vp, _i, _ip = ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int)
_TILE_LIST_ABI = {
    "gemm": ([_i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp], _i),
    "gemm_run_config": ([_i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp], _i),
    "select": ([_i, _i, _i, _i, _i, _ip, _ip], _i),
    "schedule_units": ([_i, _i, _i, _i, _i, _ip, _i, _i, _ip, _i, _ip], _i),
    "launch_count": ([], ctypes.c_ulonglong),
    "strerror": ([_i], ctypes.c_char_p),
}
_FP8_TILE_LIST_ABI = {
    "gemm": ([_vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _vp], _i),
    "gemm_run_config": ([_i, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp], _i),
    "select": ([_i, _i, _i, _i, _ip, _ip], _i),
    "launch_count": ([], ctypes.c_ulonglong),
    "strerror": ([_i], ctypes.c_char_p),
}


def _prefixed(prefix: str, abi: dict) -> dict:
    return {f"b200_{prefix}_{suffix}": sig for suffix, sig in abi.items()}


# The C ABI of every library, as its header declares it: file name -> {symbol: (argtypes, restype)}. The loaders apply
# it, exported_symbols() lists it, and build() checks each library's exports against it.
_GEMM = ([_vp, _vp, _vp, _vp, _i, _i, _i, _vp], _i)
_FP8GEMM = ([_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp], _i)
_FP8GEMM_RUN_CONFIG = ([_i, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp], _i)
_BASELINE = ([_i, _i, _vp, _vp, _vp, _i, _i, _i], _i)
ABI = {
    "libb200_hgemm.so": {
        "b200_hgemm_f32acc": _GEMM,
        "b200_hgemm_f16acc": _GEMM,
        "b200_bgemm_f32acc": _GEMM,
        "b200_bgemm_run_config": ([_i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp], _i),
        "b200_fp8gemm": _FP8GEMM,
        "b200_fp8gemm_run_config": _FP8GEMM_RUN_CONFIG,
        "b200_fp8gemm_rowwise": _FP8GEMM,
        "b200_fp8gemm_rowwise_run_config": _FP8GEMM_RUN_CONFIG,
        "b200_fp8gemm_select": ([_i, _i, _i, _ip, _ip, _ip], _i),
        "b200_hgemm_num_configs": ([], _i),
        "b200_hgemm_config_info": ([_i, _ip, _ip, _ip], _i),
        "b200_hgemm_config_cluster": ([_i, _ip, _ip], _i),
        "b200_hgemm_config_m_rep": ([_i], _i),
        "b200_hgemm_config_stages_requested": ([_i], _i),
        "b200_hgemm_select_config": ([_i, _i, _i, _i], _i),
        "b200_hgemm_select": ([_i, _i, _i, _i, _ip, _ip, _ip], _i),
        "b200_hgemm_run_config": ([_i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp], _i),
        "b200_hgemm_host": ([_i, _vp, _vp, _vp, _i, _i, _i], _i),
        "b200_hgemm_schedule_units": ([_i, _i, _i, _i, _i, _i, _i, _ip, _i, _ip, _ip, _ip, _ip], _i),
        "b200_hgemm_prewarm": ([_vp], _i),
        "b200_hgemm_release": ([], _i),
        "b200_hgemm_launch_count": ([], ctypes.c_ulonglong),
        "b200_hgemm_strerror": ([_i], ctypes.c_char_p),
    },
    "libb200_fp8block.so": {
        "b200_fp8gemm_blockwise": ([_vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _vp], _i),
        "b200_fp8gemm_blockwise_run_config": ([_i, _i, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp], _i),
        "b200_fp8gemm_blockwise_select": ([_i, _i, _i, _ip, _ip, _ip], _i),
        "b200_fp8block_launch_count": ([], ctypes.c_ulonglong),
        "b200_fp8block_strerror": ([_i], ctypes.c_char_p),
    },
    "libb200_batched.so": _prefixed("batched", _TILE_LIST_ABI),
    "libb200_grouped.so": _prefixed("grouped", _TILE_LIST_ABI),
    "libb200_grouped_fp8.so": _prefixed("grouped_fp8", _FP8_TILE_LIST_ABI),
    "libb200_batched_fp8.so": _prefixed("batched_fp8", _FP8_TILE_LIST_ABI),
    "libb200_baselines.so": {
        "b200_bl_init": ([_i], _i),
        "b200_bl_destroy": ([_i], None),
        "b200_bl_cublas": _BASELINE,
        "b200_bl_lt_heuristic": _BASELINE,
        "b200_bl_lt_autotune_find": ([_i, _i, _i, _i, _i, _i, _i], _i),
        "b200_bl_lt_autotune": _BASELINE,
        "b200_bl_lt_autotune_info": ([_i, _i, _ip, ctypes.POINTER(ctypes.c_float)], _i),
    },
}
# Libraries without a public ABI: their entry points are declared in an internal header under cuda_l2_b200/csrc/ and
# none under include/, so they are kept out of ABI (which mirrors the headers). Same form: {symbol: (argtypes, restype)}.
GROUPED_BWD_LIB = "libb200_grouped_bwd.so"   # csrc/b200_grouped_bwd.h
_BWD_RUN = ([_i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp], _i)
_BWD_SELECT = ([_i, _i, _i, _i, _i, _ip, _ip], _i)
EPILOGUE_LIB = "libb200_epilogue.so"         # csrc/b200_epilogue.h
QUANT_LIB = "libb200_quant.so"               # csrc/b200_quant.h
QUANT_DUAL_LIB = "libb200_quant_dual.so"     # csrc/b200_quant_dual.h
FP8BLOCK_1D1D_LIB = "libb200_fp8block_1d1d.so"       # csrc/b200_fp8_block_1d1d.h
QUANT_BLOCK_DUAL_LIB = "libb200_quant_block_dual.so"  # csrc/b200_quant_block_dual.h
WGRAD_ACCUM_LIB = "libb200_wgrad_accum.so"   # csrc/b200_wgrad_accum.h
SWIGLU_LIB = "libb200_swiglu.so"             # csrc/b200_swiglu.h
GROUPED_SWIGLU_LIB = "libb200_grouped_swiglu.so"   # csrc/b200_grouped_swiglu.h
_QUANT_BLOCK_DUAL = ([_i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp], _i)
_QUANT_BLOCKWISE = ([_i, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp], _i)
INTERNAL_ABI = {
    GROUPED_BWD_LIB: {
        "cuda_l2_b200_grouped_bwd_nn": _BWD_RUN,
        "cuda_l2_b200_grouped_bwd_wgrad": _BWD_RUN,
        "cuda_l2_b200_grouped_bwd_nn_select": _BWD_SELECT,
        "cuda_l2_b200_grouped_bwd_wgrad_select": _BWD_SELECT,
        "cuda_l2_b200_grouped_bwd_wgrad_schedule": ([_i, _i, _i, _i, _i, _ip, _i, _i, _ip, _i, _ip], _i),
        "cuda_l2_b200_grouped_bwd_launch_count": ([], ctypes.c_ulonglong),
        "cuda_l2_b200_grouped_bwd_strerror": ([_i], ctypes.c_char_p),
    },
    EPILOGUE_LIB: {
        "cuda_l2_b200_epilogue_run": ([_i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _vp], _i),
        "cuda_l2_b200_epilogue_run_config": ([_i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i,
                                              _vp], _i),
        "cuda_l2_b200_epilogue_select": ([_i, _i, _i, _i, _ip, _ip, _ip], _i),
        "cuda_l2_b200_epilogue_prewarm": ([_vp], _i),
        "cuda_l2_b200_epilogue_release": ([], _i),
        "cuda_l2_b200_epilogue_launch_count": ([], ctypes.c_ulonglong),
        "cuda_l2_b200_epilogue_strerror": ([_i], ctypes.c_char_p),
    },
    QUANT_LIB: {
        "cuda_l2_b200_quant_e4m3_tensor": ([_i, _vp, ctypes.c_longlong, _vp, _vp, _vp, _vp], _i),
        "cuda_l2_b200_quant_e4m3_rowwise": ([_i, _vp, _i, _i, _vp, _vp, _vp], _i),
        "cuda_l2_b200_quant_e4m3_blockwise": _QUANT_BLOCKWISE,
        "cuda_l2_b200_quant_silu_mul_e4m3_blockwise": _QUANT_BLOCKWISE,
        "cuda_l2_b200_quant_launch_count": ([], ctypes.c_ulonglong),
        "cuda_l2_b200_quant_strerror": ([_i], ctypes.c_char_p),
    },
    QUANT_DUAL_LIB: {
        "cuda_l2_b200_quant_dual_e4m3_rowwise": ([_i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp], _i),
        "cuda_l2_b200_quant_dual_launch_count": ([], ctypes.c_ulonglong),
        "cuda_l2_b200_quant_dual_strerror": ([_i], ctypes.c_char_p),
    },
    FP8BLOCK_1D1D_LIB: {
        "cuda_l2_b200_fp8block_1d1d_run": ([_vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _vp], _i),
        "cuda_l2_b200_fp8block_1d1d_run_config": ([_i, _i, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i,
                                                   _vp], _i),
        "cuda_l2_b200_fp8block_1d1d_select": ([_i, _i, _i, _ip, _ip, _ip], _i),
        "cuda_l2_b200_fp8block_1d1d_launch_count": ([], ctypes.c_ulonglong),
        "cuda_l2_b200_fp8block_1d1d_strerror": ([_i], ctypes.c_char_p),
    },
    QUANT_BLOCK_DUAL_LIB: {
        "cuda_l2_b200_quant_block_dual_e4m3_1x128": _QUANT_BLOCK_DUAL,
        "cuda_l2_b200_quant_block_dual_e4m3_128x128": _QUANT_BLOCK_DUAL,
        "cuda_l2_b200_quant_block_dual_launch_count": ([], ctypes.c_ulonglong),
        "cuda_l2_b200_quant_block_dual_strerror": ([_i], ctypes.c_char_p),
    },
    WGRAD_ACCUM_LIB: {
        "cuda_l2_b200_wgrad_accum_grouped": _BWD_RUN,
        "cuda_l2_b200_wgrad_accum_fp8": ([_i, _i, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _vp], _i),
        "cuda_l2_b200_wgrad_accum_grouped_select": _BWD_SELECT,
        "cuda_l2_b200_wgrad_accum_fp8_select": ([_i, _i, _i, _i, _ip, _ip, _ip], _i),
        "cuda_l2_b200_wgrad_accum_prewarm": ([_vp], _i),
        "cuda_l2_b200_wgrad_accum_release": ([], _i),
        "cuda_l2_b200_wgrad_accum_launch_count": ([], ctypes.c_ulonglong),
        "cuda_l2_b200_wgrad_accum_strerror": ([_i], ctypes.c_char_p),
    },
    SWIGLU_LIB: {
        "cuda_l2_b200_swiglu_run": ([_i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp], _i),
        "cuda_l2_b200_swiglu_run_config": ([_i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp], _i),
        "cuda_l2_b200_swiglu_select": ([_i, _i, _i, _i, _ip, _ip, _ip], _i),
        "cuda_l2_b200_swiglu_backward": ([_i, _vp, _vp, _vp, _i, _i, _vp], _i),
        "cuda_l2_b200_swiglu_launch_count": ([], ctypes.c_ulonglong),
        "cuda_l2_b200_swiglu_strerror": ([_i], ctypes.c_char_p),
    },
    GROUPED_SWIGLU_LIB: {
        "cuda_l2_b200_grouped_swiglu_run": ([_i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp], _i),
        "cuda_l2_b200_grouped_swiglu_run_config": ([_i, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp], _i),
        "cuda_l2_b200_grouped_swiglu_select": ([_i, _i, _i, _i, _i, _ip, _ip], _i),
        "cuda_l2_b200_grouped_swiglu_backward": ([_i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp], _i),
        "cuda_l2_b200_grouped_swiglu_launch_count": ([], ctypes.c_ulonglong),
        "cuda_l2_b200_grouped_swiglu_strerror": ([_i], ctypes.c_char_p),
    },
}
_TABLES = {**ABI, **INTERNAL_ABI}
_LIBRARY_OF = {symbol: name for name, table in _TABLES.items() for symbol in table}   # entry point -> its library
_libs: dict = {}


def load(name: str) -> ctypes.CDLL:
    """The library ``name`` (a key of :data:`ABI` or :data:`INTERNAL_ABI`), loaded once with its table's argtypes and
    restypes applied: a symbol it does not export raises."""
    if name not in _libs:
        path = LIB_DIR / name
        if not path.exists():
            raise B200HgemmError(
                f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `python cuda_l2_b200/build.py`). There is no fallback path.")
        lib = ctypes.CDLL(str(path))
        for sym, (args, res) in _TABLES[name].items():
            fn = getattr(lib, sym)
            fn.argtypes, fn.restype = args, res
        _libs[name] = lib
    return _libs[name]


def hgemm_lib() -> ctypes.CDLL:
    """libb200_hgemm.so: the 16-bit and per-tensor / rowwise e4m3 GEMMs (include/b200_hgemm.h)."""
    return load("libb200_hgemm.so")


def fp8block_lib() -> ctypes.CDLL:
    """libb200_fp8block.so: the block-scaled e4m3 GEMM (include/b200_fp8_block.h)."""
    return load("libb200_fp8block.so")


def batched_lib() -> ctypes.CDLL:
    """libb200_batched.so: the batched fp16 / bf16 GEMM (include/b200_batched.h)."""
    return load("libb200_batched.so")


def grouped_lib() -> ctypes.CDLL:
    """libb200_grouped.so: the grouped fp16 / bf16 GEMM over contiguous row groups (include/b200_grouped.h)."""
    return load("libb200_grouped.so")


def grouped_fp8_lib() -> ctypes.CDLL:
    """libb200_grouped_fp8.so: the block-scaled e4m3 grouped GEMM over contiguous row groups
    (include/b200_grouped_fp8.h)."""
    return load("libb200_grouped_fp8.so")


def batched_fp8_lib() -> ctypes.CDLL:
    """libb200_batched_fp8.so: the block-scaled e4m3 batched GEMM with per-batch row counts on the device
    (include/b200_batched_fp8.h)."""
    return load("libb200_batched_fp8.so")


def baselines_lib() -> ctypes.CDLL:
    """libb200_baselines.so: the cuBLAS / cuBLASLt comparators (include/b200_baselines.h)."""
    return load("libb200_baselines.so")


def exported_symbols() -> dict[str, list[str]]:
    """Symbols each header declares — used by the CPU tests to check the libraries export all of them."""
    return {name: list(symbols) for name, symbols in ABI.items()}


def strerror(status: int) -> str:
    return hgemm_lib().b200_hgemm_strerror(status).decode()


def _check(status: int, fn) -> None:
    """B200HgemmError unless ``status``, what the entry point ``fn`` (a loaded function or its symbol) returned, is 0.
    The message decodes the status with the strerror of the library that exports ``fn``, which knows its own codes."""
    if status != 0:
        symbol = fn if isinstance(fn, str) else fn.__name__
        name = _LIBRARY_OF[symbol]
        text = getattr(load(name), next(s for s in _TABLES[name] if s.endswith("_strerror")))(status).decode()
        raise B200HgemmError(f"{symbol} failed: status {status} ({text})")


def _shape_check(a, b_col_major, c):
    import torch

    for name, t in (("a", a), ("b_col_major", b_col_major), ("c", c)):
        if t.dtype != torch.half:
            raise B200HgemmError(f"{name} must be torch.half, got {t.dtype}")
        if not t.is_cuda:
            raise B200HgemmError(f"{name} must be a CUDA tensor")
        if not t.is_contiguous():
            raise B200HgemmError(f"{name} must be contiguous")
    m, k = a.shape
    # b_col_major is shape-labelled [K,N] but its memory is [N,K] (tools/utils.py:110-115 in the reference)
    kb, n = b_col_major.shape
    if kb != k or tuple(c.shape) != (m, n):
        raise B200HgemmError(f"shape mismatch: a {tuple(a.shape)}, b_col_major {tuple(b_col_major.shape)}, c {tuple(c.shape)}")
    return m, n, k


def hgemm(a, b_col_major, c, acc: str | int = "fp32", stream: int | None = None) -> None:
    """c[M,N] = a[M,K] @ B[K,N] where ``b_col_major`` holds B K-major. Asynchronous on ``stream``
    (``None`` = the legacy default stream, like the reference's launches)."""
    m, n, k = _shape_check(a, b_col_major, c)
    bits = ACC_BITS[acc]
    fn = hgemm_lib().b200_hgemm_f32acc if bits == 32 else hgemm_lib().b200_hgemm_f16acc
    _check(fn(a.data_ptr(), None, b_col_major.data_ptr(), c.data_ptr(), m, n, k, stream), fn)


class GemmType(NamedTuple):
    """A data-type variant of the kernel family (include/b200_hgemm.h)."""
    k_align: int    # K % k_align == 0: 16-byte operand rows
    scale: object   # dtype of the scales the variant takes (e4m3 operands: float32), None if it takes none

    def fits(self, n: int, k: int) -> bool:
        """Whether an [M,K] x [N,K] problem meets the 16-byte row rule (TMA strides) of this variant."""
        return n % 8 == 0 and k % self.k_align == 0


_GEMM_TYPES: dict = {}   # (operand dtype, output dtype, accumulator bits) -> GemmType, filled on first use


def gemm_type(operand, output, acc: str | int = "fp32") -> GemmType | None:
    """The variant with these operand and output dtypes and accumulator, or None: the kernel family has none."""
    if not _GEMM_TYPES:
        import torch
        h, b, e, f = torch.float16, torch.bfloat16, torch.float8_e4m3fn, torch.float32
        _GEMM_TYPES.update({(h, h, 32): GemmType(8, None), (h, h, 16): GemmType(8, None), (b, b, 32): GemmType(8, None),
                            (e, h, 32): GemmType(16, f), (e, b, 32): GemmType(16, f)})
    return _GEMM_TYPES.get((operand, output, ACC_BITS.get(acc)))


BLOCK = 128   # block scales: one per (row of A, 128 k) and one per 128 x 128 block of Bt


def num_k_blocks(k: int) -> int:
    """ceil(K / 128): the scale blocks along K of a block-scaled product."""
    return -(-k // BLOCK)


def scale_granularity(m: int, n: int, scale_a, scale_b, k: int | None = None, groups: int | None = None,
                      batches: int | None = None) -> str:
    """torch._scaled_mm's rule for the scales of an [M,K] x [N,K] e4m3 product: two one-element fp32 tensors are
    ``"tensor"`` scales; ``scale_a`` [M,1] with ``scale_b`` [1,N], both fp32, are ``"rowwise"`` scales (one per row of A,
    one per output column); ``scale_a`` [M, nkb] with ``scale_b`` [ceil(N/128), nkb], nkb = ceil(K/128), both fp32, are
    ``"blockwise"`` scales (one per row of A and 128 k, one per 128 x 128 block of Bt); ``scale_a`` [M, nkb] with
    ``scale_b`` [N, nkb] are ``"blockwise_1d1d"`` scales (one per row and 128 k on both operands: the weight gradient of
    blockwise FP8 training; N % 8 == 0, so N > ceil(N/128) and the two blockwise forms never meet). Without ``k``, any
    nkb the two agree on is accepted. ``groups``: the grouped product of M = T rows by ``groups`` matrices Bt [N,K], whose only
    scales are blockwise, with ``scale_b`` [groups, ceil(N/128), nkb]. ``batches``: the batched product of ``batches``
    matrices [M,K] by as many Bt [N,K], whose only scales are blockwise, with ``scale_a`` [batches, M, nkb] and
    ``scale_b`` [batches, ceil(N/128), nkb]. Anything else, a mix of them included, raises B200HgemmError."""
    import torch

    sa, sb = tuple(scale_a.shape), tuple(scale_b.shape)
    lead_a = () if batches is None else (batches,)
    lead = lead_a if groups is None else (groups,)
    plain = groups is None and batches is None
    if scale_a.dtype == torch.float32 and scale_b.dtype == torch.float32:
        if plain and scale_a.numel() == 1 and scale_b.numel() == 1:
            return "tensor"
        if plain and sa == (m, 1) and sb == (1, n):
            return "rowwise"
        nkb = num_k_blocks(k) if k is not None else (sa[-1] if len(sa) == 2 + len(lead_a) else -1)
        if sa == (*lead_a, m, nkb) and sb == (*lead, -(-n // BLOCK), nkb):
            return "blockwise"
        if plain and sa == (m, nkb) and sb == (n, nkb) and n > -(-n // BLOCK):
            return "blockwise_1d1d"
    if groups is not None:
        raise B200HgemmError(f"grouped scales must be fp32 blockwise scales, scale_a [{m}, ceil(K/128)] with scale_b "
                             f"[{groups}, ceil({n}/128), ceil(K/128)], got {scale_a.dtype} {sa} and {scale_b.dtype} {sb}")
    if batches is not None:
        raise B200HgemmError(f"batched scales must be fp32 blockwise scales, scale_a [{batches}, {m}, ceil(K/128)] with "
                             f"scale_b [{batches}, ceil({n}/128), ceil(K/128)], got {scale_a.dtype} {sa} and "
                             f"{scale_b.dtype} {sb}")
    raise B200HgemmError(f"scales must be fp32 and either both one-element (per tensor), scale_a [{m}, 1] with "
                         f"scale_b [1, {n}] (rowwise), or scale_a [{m}, ceil(K/128)] with scale_b [ceil({n}/128), "
                         f"ceil(K/128)] (blockwise) or [{n}, ceil(K/128)] (blockwise_1d1d), got {scale_a.dtype} {sa} and "
                         f"{scale_b.dtype} {sb}")


def blockwise_ld_a(scale_a) -> int | None:
    """The row stride ld_a with which the kernels can read a blockwise ``scale_a`` [M, nkb] in place: M-major (strides
    (1, ld_a), torch's ``[nkb, ld_a]`` buffer viewed as ``buf[:, :M].t()``), ld_a >= M, ld_a % 4 == 0, 16-byte aligned,
    and nkb * ld_a floats readable in its storage (one k-block: ld_a = M rounded up to 4). A batched ``scale_a``
    [B, M, nkb] holds one such block per matrix, stacked (strides (nkb * ld_a, 1, ld_a), torch's ``[B, nkb, ld_a]``
    buffer viewed as ``buf[:, :, :M].transpose(1, 2)``), B * nkb * ld_a floats readable. Strides of size-1 dimensions
    are never stepped and do not count. None if the tensor is not laid out that way."""
    *lead, m, nkb = scale_a.shape
    bsz, st = (lead[0] if lead else 1), scale_a.stride()
    ld = st[-1] if nkb > 1 else _m_major_ld(m)     # one k-block: the k stride is never stepped
    if nkb == 1 and bsz > 1:   # the batch stride is the only one stepped: it is nkb * ld_a = ld_a
        ld = st[0]
    if (bsz > 1 and st[0] != nkb * ld) or (m > 1 and st[-2] != 1) or ld < m or ld % 4 or scale_a.data_ptr() % 16:
        return None
    readable = scale_a.untyped_storage().nbytes() // 4 - scale_a.storage_offset()
    return ld if bsz * nkb * ld <= readable else None


def _m_major_ld(m: int) -> int:
    """ld_a of the M-major scales the quantisers write and :func:`m_major` copies into: M rounded up to 4."""
    return -(-m // 4) * 4


def empty_m_major(lead: tuple, m: int, nkb: int, device):
    """An empty fp32 blockwise scale [*lead, M, nkb] that the block-scaled kernels read in place: the view
    ``buf[..., :M].transpose(-2, -1)`` of a [*lead, nkb, ld_a] buffer, ld_a = M rounded up to 4."""
    import torch

    buf = torch.empty((*lead, nkb, _m_major_ld(m)), dtype=torch.float32, device=device)
    return buf[..., :m].transpose(-2, -1)


def m_major(scale):
    """A blockwise scale [(B,) M, nkb] as the block-scaled kernels read it: ``scale`` itself where
    :func:`blockwise_ld_a` reads it in place, else a device copy into :func:`empty_m_major`."""
    if blockwise_ld_a(scale) is not None:
        return scale
    *lead, m, nkb = scale.shape
    return empty_m_major(lead, m, nkb, scale.device).copy_(scale)


def _scale_ld_a(scale_a, name: str = "scale_a") -> int:
    """blockwise_ld_a of a ``scale_a`` (or a 1 x 128 ``scale_b``, the same layout) the kernel reads in place;
    B200HgemmError if it cannot (a CPU tensor included)."""
    ld_a = blockwise_ld_a(scale_a) if scale_a.is_cuda else None
    if ld_a is None:
        raise B200HgemmError(f"blockwise {name} must be a CUDA tensor holding one M-major [ceil(K/128), ld_a] block "
                             f"per matrix (strides (1, ld_a), batched (ceil(K/128) * ld_a, 1, ld_a)) with ld_a >= M, "
                             f"ld_a % 4 == 0, 16-byte aligned, every block readable; got strides "
                             f"{tuple(scale_a.stride())} on {scale_a.device}")
    return ld_a


def _scale_args(granularity: str, scale_a, scale_b) -> tuple:
    """The scale arguments of the e4m3 entry points for scales of ``granularity`` (:func:`scale_granularity`):
    ``(scale_a, ld_a, scale_b, ld_b)`` for 1 x 128 scales on both operands, both read in place (:func:`_scale_ld_a`);
    ``(scale_a, ld_a, scale_b)`` for blockwise ones, ``scale_a`` read in place and ``scale_b`` a contiguous CUDA
    tensor; ``(scale_a, scale_b)`` otherwise, both contiguous CUDA tensors. B200HgemmError if a scale is not so."""
    if granularity == "blockwise_1d1d":
        return scale_a.data_ptr(), _scale_ld_a(scale_a), scale_b.data_ptr(), _scale_ld_a(scale_b, "scale_b")
    if granularity == "blockwise":
        _contiguous_cuda(scale_b=scale_b)
        return scale_a.data_ptr(), _scale_ld_a(scale_a), scale_b.data_ptr()
    _contiguous_cuda(scale_a=scale_a, scale_b=scale_b)
    return scale_a.data_ptr(), scale_b.data_ptr()


def check_operands(a, b_kmajor, out_dtype, acc: str | int = "fp32",
                   scales: tuple = ()) -> tuple[int, int, int, str | None]:
    """(M, N, K, granularity) of a[M,K] @ b_kmajor[N,K]^T -> ``out_dtype``, by the rules of the variant the dtypes and
    ``acc`` name: 2-D operands of one dtype, a shared K, 16-byte rows, two scales exactly for a scaled variant, of the
    granularity :func:`scale_granularity` returns (None without scales). Checks shapes and dtypes only (meta tensors
    pass); B200HgemmError otherwise."""
    try:
        (m, k), (n, k2) = a.shape, b_kmajor.shape
    except ValueError:
        raise B200HgemmError(f"2-D operands expected, got {tuple(a.shape)} and {tuple(b_kmajor.shape)}") from None
    t = _operand_type(a, b_kmajor, out_dtype, acc, scales)
    granularity = scale_granularity(m, n, *scales, k=k) if scales else None
    _check_k(a, b_kmajor, t, n, k, k2, "[N, K]")
    return m, n, k, granularity


def _operand_type(a, b_kmajor, out_dtype, acc: str | int, scales: tuple, scaled: bool = True) -> GemmType:
    """The variant of a @ b_kmajor^T -> ``out_dtype`` with ``acc``: operands of one dtype that name one (``scaled=False``:
    a 16-bit one), and two ``scales`` exactly if it is scaled. B200HgemmError otherwise."""
    t = gemm_type(a.dtype, out_dtype, acc) if b_kmajor.dtype == a.dtype else None
    if t is None or (t.scale is not None and not scaled):
        kinds = "fp16 with fp32 or fp16 accumulation, bf16 with fp32"
        if scaled:
            kinds += ", e4m3 -> fp16 / bf16 with fp32"
        raise B200HgemmError(f"no kernel for {a.dtype} x {b_kmajor.dtype} -> {out_dtype} with acc={acc!r} ({kinds})")
    if len(scales) != (0 if t.scale is None else 2):
        raise B200HgemmError(f"{a.dtype} operands take {'no' if t.scale is None else 'two'} scales, got {len(scales)}")
    return t


def _check_k(a, b_kmajor, t: GemmType, n: int, k: int, k2: int, b_layout: str) -> None:
    """The rules every product shares: a's K is b_kmajor's (``b_layout``, K-major), and rows of 16 bytes
    (:meth:`GemmType.fits`). B200HgemmError otherwise."""
    if k2 != k:
        raise B200HgemmError(f"inner dimensions differ: a {tuple(a.shape)}, b_kmajor {tuple(b_kmajor.shape)} "
                             f"(K-major: {b_layout})")
    if not t.fits(n, k):
        raise B200HgemmError(f"{a.dtype} operands need N % 8 == 0 and K % {t.k_align} == 0 (16-byte TMA strides), "
                             f"got N={n}, K={k}")


def _contiguous_cuda(**tensors) -> None:
    """B200HgemmError unless every tensor given (None: not passed) is a contiguous CUDA tensor."""
    for name, x in tensors.items():
        if x is not None and (not x.is_cuda or not x.is_contiguous()):
            raise B200HgemmError(f"{name} must be a contiguous CUDA tensor")


def _kmajor_operands(a, b_kmajor, c, acc: str | int, scales: tuple = ()) -> tuple[int, int, int, str | None]:
    """check_operands for c = a @ b_kmajor^T, the three contiguous CUDA tensors and c of shape [M,N]. The scales are
    checked only by shape and dtype here: how they may be laid out depends on the granularity (:func:`_scale_args`)."""
    _contiguous_cuda(a=a, b_kmajor=b_kmajor, c=c)
    m, n, k, granularity = check_operands(a, b_kmajor, c.dtype, acc, scales)
    if c.shape != (m, n):
        raise B200HgemmError(f"shape mismatch: a {tuple(a.shape)}, b_kmajor {tuple(b_kmajor.shape)}, c {tuple(c.shape)}")
    return m, n, k, granularity


def gemm_kmajor(a, b_kmajor, c, acc: str | int = "fp32", stream: int | None = None, config_id: int | None = None,
                group_m: int = 0, splits: int = 1, max_ctas: int = 0) -> None:
    """c[M,N] = a[M,K] @ b_kmajor[N,K]^T with the operands' dtype deciding the kernel family: fp16 (fp32 or fp16
    accumulation) or bf16 (fp32 accumulation). ``b_kmajor`` is shaped as stored, [N,K] — an ``nn.Linear`` weight.
    ``config_id`` pins one kernel configuration (tests); default is the dispatcher. ``max_ctas`` (with ``config_id``)
    caps the CTAs of the launch, 0 meaning all SMs, so that each worker runs several tiles."""
    import torch

    m, n, k, _ = _kmajor_operands(a, b_kmajor, c, acc)
    lib = hgemm_lib()
    bits = ACC_BITS[acc]
    if config_id is None:
        fn = (lib.b200_bgemm_f32acc if a.dtype == torch.bfloat16 else
              lib.b200_hgemm_f32acc if bits == 32 else lib.b200_hgemm_f16acc)
        st = fn(a.data_ptr(), None, b_kmajor.data_ptr(), c.data_ptr(), m, n, k, stream)
    elif a.dtype == torch.bfloat16:
        fn = lib.b200_bgemm_run_config
        st = fn(config_id, a.data_ptr(), b_kmajor.data_ptr(), c.data_ptr(), m, n, k, group_m, max_ctas, splits, stream)
    else:
        fn = lib.b200_hgemm_run_config
        st = fn(bits, config_id, a.data_ptr(), b_kmajor.data_ptr(), c.data_ptr(), m, n, k, group_m, max_ctas, splits,
                stream)
    _check(st, fn)


def check_rowmajor_operands(a, b, out_dtype=None, acc: str | int = "fp32") -> tuple[int, int, int]:
    """(M, N, K) of a[M,K] @ b[K,N] with ``b`` row-major (``torch.matmul``'s layout), by the rules of the 16-bit variant
    the dtypes and ``acc`` name (fp16 with fp32 or fp16 accumulation, bf16 with fp32; the output dtype is the operands'):
    2-D operands of one dtype, a shared K, N % 8 == 0 and K % 8 == 0 (16-byte rows of A, B and C). Checks shapes and
    dtypes only (meta tensors pass); B200HgemmError otherwise."""
    try:
        (m, k), (k2, n) = a.shape, b.shape
    except ValueError:
        raise B200HgemmError(f"2-D operands expected, got {tuple(a.shape)} and {tuple(b.shape)}") from None
    t = _operand_type(a, b, a.dtype if out_dtype is None else out_dtype, acc, (), scaled=False)
    if k2 != k:
        raise B200HgemmError(f"inner dimensions differ: a {tuple(a.shape)}, b {tuple(b.shape)} (row-major: [K, N])")
    if not t.fits(n, k):
        raise B200HgemmError(f"{a.dtype} operands need N % 8 == 0 and K % {t.k_align} == 0 (16-byte TMA strides), "
                             f"got N={n}, K={k}")
    return m, n, k


def gemm_rowmajor(a, b, c, acc: str | int = "fp32", stream: int | None = None) -> None:
    """c[M,N] = a[M,K] @ b[K,N] with ``b`` row-major (N contiguous, ``torch.matmul(a, b)``'s layout), read in place by
    the row-major B (NN) kernels of libb200_nn.so: the drop-in entry points called with ``B_rowmajor`` and no
    ``B_kmajor`` (include/b200_hgemm.h). fp16 (fp32 or fp16 accumulation) or bf16 (fp32) operands, all three contiguous
    CUDA tensors. The dispatcher's TN choice for the shape runs, BN = 32 configurations mapped to a BN = 64 sibling."""
    import torch

    _contiguous_cuda(a=a, b=b, c=c)
    m, n, k = check_rowmajor_operands(a, b, c.dtype, acc)
    if tuple(c.shape) != (m, n):
        raise B200HgemmError(f"shape mismatch: a {tuple(a.shape)}, b {tuple(b.shape)}, c {tuple(c.shape)}")
    lib = hgemm_lib()
    if a.dtype == torch.bfloat16:
        fn = lib.b200_bgemm_f32acc
    else:
        fn = lib.b200_hgemm_f32acc if ACC_BITS[acc] == 32 else lib.b200_hgemm_f16acc
    _check(fn(a.data_ptr(), b.data_ptr(), None, c.data_ptr(), m, n, k, stream), fn)


def fp8_gemm(a, b_kmajor, c, scale_a, scale_b, stream: int | None = None, config_id: int | None = None,
             group_m: int = 0, splits: int = 1, max_ctas: int = 0) -> None:
    """c[M,N] = (a[M,K] @ b_kmajor[N,K]^T) scaled, with ``float8_e4m3fn`` operands, fp32 accumulation and one rounding
    to ``c``'s dtype (fp16 or bf16). ``scale_a`` / ``scale_b`` are fp32 CUDA tensors, read when the kernel runs: one
    element each (per tensor: ``* scale_a * scale_b``), or ``scale_a`` [M,1] and ``scale_b`` [1,N], 16-byte aligned
    (rowwise: ``* scale_b[n]``, then ``* scale_a[m]``), or blockwise scales (include/b200_fp8_block.h): ``scale_a``
    [M, ceil(K/128)] M-major (strides (1, ld_a), see :func:`blockwise_ld_a`), ``scale_b`` [ceil(N/128), ceil(K/128)]
    contiguous, run by libb200_fp8block.so, or 1 x 128 scales on both operands (csrc/b200_fp8_block_1d1d.h):
    ``scale_a`` as for blockwise, ``scale_b`` [N, ceil(K/128)] N-major in the same layout (strides (1, ld_b)), read in
    place, run by libb200_fp8block_1d1d.so. ``config_id`` pins one kernel configuration (tests; ``splits`` as in
    b200_hgemm_run_config; ``max_ctas`` as in :func:`gemm_kmajor`); default is the dispatcher."""
    import torch

    m, n, k, granularity = _kmajor_operands(a, b_kmajor, c, "fp32", (scale_a, scale_b))
    # granularity -> the dispatched and the pinned entry point; their arguments differ only in the scales (_scale_args)
    dispatched, pinned = {
        "tensor": ("b200_fp8gemm", "b200_fp8gemm_run_config"),
        "rowwise": ("b200_fp8gemm_rowwise", "b200_fp8gemm_rowwise_run_config"),
        "blockwise": ("b200_fp8gemm_blockwise", "b200_fp8gemm_blockwise_run_config"),
        "blockwise_1d1d": ("cuda_l2_b200_fp8block_1d1d_run", "cuda_l2_b200_fp8block_1d1d_run_config"),
    }[granularity]
    ptrs = (a.data_ptr(), b_kmajor.data_ptr(), c.data_ptr(), *_scale_args(granularity, scale_a, scale_b))
    lib = load(_LIBRARY_OF[dispatched])
    out_bf16 = int(c.dtype == torch.bfloat16)
    if config_id is None:
        fn = getattr(lib, dispatched)
        st = fn(*ptrs, out_bf16, m, n, k, stream)
    else:
        fn = getattr(lib, pinned)
        st = fn(config_id, out_bf16, *ptrs, m, n, k, group_m, max_ctas, splits, stream)
    _check(st, fn)


def _select(fn, *args) -> tuple[int, ...]:
    """A *_select entry point's answer: ``fn`` called with ``args``, then one int out-parameter for each of its
    remaining arguments, whose values it returns. B200HgemmError on a non-zero status."""
    outs = [ctypes.c_int() for _ in fn.argtypes[len(args):]]
    _check(fn(*args, *map(ctypes.byref, outs)), fn)
    return tuple(v.value for v in outs)


def fp8_select(m: int, n: int, k: int) -> tuple[int, int, int]:
    """(config id, rasterisation group, split-K factor) the dispatcher uses for an e4m3 problem."""
    return _select(hgemm_lib().b200_fp8gemm_select, m, n, k)


def fp8_blockwise_select(m: int, n: int, k: int) -> tuple[int, int, int]:
    """(config id, rasterisation group, splits code) the block-scaled dispatcher uses (b200_fp8gemm_blockwise_select)."""
    return _select(fp8block_lib().b200_fp8gemm_blockwise_select, m, n, k)


def fp8block_launch_count() -> int:
    return int(fp8block_lib().b200_fp8block_launch_count())


def fp8block_1d1d_lib() -> ctypes.CDLL:
    """libb200_fp8block_1d1d.so: the block-scaled e4m3 GEMM with 1 x 128 scales on both operands
    (csrc/b200_fp8_block_1d1d.h, no public ABI)."""
    return load(FP8BLOCK_1D1D_LIB)


def fp8_blockwise_1d1d_select(m: int, n: int, k: int) -> tuple[int, int, int]:
    """(config id, rasterisation group, splits code) of the dispatched 1 x 128 x 1 x 128 call
    (cuda_l2_b200_fp8block_1d1d_select: b200_fp8gemm_blockwise_select's choice)."""
    return _select(fp8block_1d1d_lib().cuda_l2_b200_fp8block_1d1d_select, m, n, k)


def fp8block_1d1d_launch_count() -> int:
    return int(fp8block_1d1d_lib().cuda_l2_b200_fp8block_1d1d_launch_count())


def _tile_list_schedule(schedule_units, ints: int, *args) -> dict:
    """Every worker's units, ``ints`` values each, from a tile-list library's ``schedule_units`` entry point, called
    with ``args`` (config id, the list's count, rows, N and K, host list, SMs) and then the worker and its buffer."""
    nw = ctypes.c_int()
    cap = 256
    buf = (ctypes.c_int * (ints * cap))()
    _check(min(schedule_units(*args, 0, buf, cap, ctypes.byref(nw)), 0), schedule_units)
    units = []
    for w in range(nw.value):
        cnt = schedule_units(*args, w, buf, cap, None)
        if cnt > cap:
            cap = cnt
            buf = (ctypes.c_int * (ints * cap))()
            cnt = schedule_units(*args, w, buf, cap, None)
        units.append([tuple(buf[ints * j:ints * (j + 1)]) for j in range(cnt)])
    return {"workers": nw.value, "units": units}


def _tile_list_gemm(kind: str, a, b_kmajor, c, lst, acc: str | int, scales: tuple, config_id: int | None,
                    group_m: int, max_ctas: int, stream: int | None) -> None:
    """The call of a tile-list library: ``kind`` "batched" (``lst``: the optional row counts masked_m) or "grouped"
    (``lst``: the group ends offs); with two blockwise ``scales`` the block-scaled FP8 library of that kind, with fp16 /
    bf16 output as ``c``'s dtype. Every tensor is a contiguous CUDA tensor, except that scale_a is read in place
    (:func:`_scale_args`). ``config_id`` pins one kernel configuration; default is the dispatcher."""
    import torch

    list_name = "masked_m" if kind == "batched" else "offs"
    _contiguous_cuda(a=a, b_kmajor=b_kmajor, c=c, **{list_name: lst})
    out_dtype = c.dtype if scales else None
    if kind == "batched":
        count, rows, n, k = check_batched_operands(a, b_kmajor, acc, lst, out_dtype, scales)
        c_shape = (count, rows, n)
    else:
        count, rows, n, k = check_grouped_operands(a, b_kmajor, lst, acc, out_dtype, scales)
        c_shape = (rows, n)
    want = c.dtype if scales else a.dtype
    if c.dtype != want or tuple(c.shape) != c_shape:
        raise B200HgemmError(f"c must be {want} {list(c_shape)}, got {c.dtype} {tuple(c.shape)}")
    ptrs = (a.data_ptr(), b_kmajor.data_ptr(), c.data_ptr())
    if scales:   # the FP8 entry points take the scales after the operands, and the output selector after them
        selector = int(c.dtype == torch.bfloat16)
        ptrs += _scale_args("blockwise", *scales)
    else:        # the 16-bit ones take the variant first
        selector = batched_variant(a.dtype, acc)
    prefix = f"{kind}_fp8" if scales else kind
    lib = load(f"libb200_{prefix}.so")
    problem = (None if lst is None else lst.data_ptr(), count, rows, n, k)
    if config_id is None:
        args = (*ptrs, selector) if scales else (selector, *ptrs)
        fn = getattr(lib, f"b200_{prefix}_gemm")
        st = fn(*args, *problem, stream)
    else:
        head = (config_id, selector) if scales else (selector, config_id)
        fn = getattr(lib, f"b200_{prefix}_gemm_run_config")
        st = fn(*head, *ptrs, *problem, group_m, max_ctas, stream)
    _check(st, fn)


# ------------------------------------------------------------------------------------------ batched (libb200_batched.so)
def batched_variant(dtype, acc: str | int = "fp32") -> int | None:
    """The ``variant`` argument of include/b200_batched.h (the GemmType index): 0 fp16 with fp32 accumulation, 1 fp16
    with fp16 accumulation, 2 bf16; None for any other combination."""
    import torch

    return {(torch.float16, 32): 0, (torch.float16, 16): 1, (torch.bfloat16, 32): 2}.get((dtype, ACC_BITS.get(acc)))


def check_batched_operands(a, b_kmajor, acc: str | int = "fp32", masked_m=None, out_dtype=None,
                           scales: tuple = ()) -> tuple[int, int, int, int]:
    """(B, M, N, K) of a[B,M,K] @ b_kmajor[B,N,K]^T per batch, by the rules of the variant the dtypes and ``acc`` name
    (the 2-D rules per matrix, :meth:`GemmType.fits`): a 16-bit one with the output dtype of the operands, or e4m3
    operands with ``out_dtype`` fp16 / bf16 and two blockwise ``scales`` (:func:`scale_granularity` with ``batches``).
    ``masked_m``, if given, is an int32 tensor of B elements. Checks shapes and dtypes only (meta tensors pass);
    B200HgemmError otherwise."""
    import torch

    try:
        (bsz, m, k), (bsz2, n, k2) = a.shape, b_kmajor.shape
    except ValueError:
        raise B200HgemmError(f"3-D operands expected, got {tuple(a.shape)} and {tuple(b_kmajor.shape)}") from None
    t = _operand_type(a, b_kmajor, a.dtype if out_dtype is None else out_dtype, acc, scales, scaled=bool(scales))
    if bsz2 != bsz:
        raise B200HgemmError(f"batch counts differ: a {tuple(a.shape)}, b_kmajor {tuple(b_kmajor.shape)}")
    if scales:
        scale_granularity(m, n, *scales, k=k, batches=bsz)
    _check_k(a, b_kmajor, t, n, k, k2, "[B, N, K]")
    if masked_m is not None and (masked_m.dtype != torch.int32 or tuple(masked_m.shape) != (bsz,)):
        raise B200HgemmError(f"masked_m must be an int32 tensor of shape [{bsz}], got {masked_m.dtype} "
                             f"{tuple(masked_m.shape)}")
    return bsz, m, n, k


def gemm_batched(a, b_kmajor, c, acc: str | int = "fp32", masked_m=None, stream: int | None = None,
                 config_id: int | None = None, group_m: int = 0, max_ctas: int = 0) -> None:
    """c[b] = a[b] @ b_kmajor[b]^T for every b, fp16 (fp32 or fp16 accumulation) or bf16 operands, all three contiguous
    CUDA tensors ([B,M,K], [B,N,K], [B,M,N]). ``masked_m``: an optional int32 CUDA tensor [B], read by the kernel when
    it runs: only rows [0, clamp(masked_m[b], 0, M)) of c[b] are computed (include/b200_batched.h). ``config_id``
    pins one kernel configuration (tests), ``max_ctas`` caps the CTAs (0: all SMs); default is the dispatcher."""
    _tile_list_gemm("batched", a, b_kmajor, c, masked_m, acc, (), config_id, group_m, max_ctas, stream)


def batched_select(variant: int, b: int, m: int, n: int, k: int) -> tuple[int, int]:
    """(config id, rasterisation group) the batched dispatcher uses (b200_batched_select)."""
    return _select(batched_lib().b200_batched_select, variant, b, m, n, k)


def batched_schedule(config_id: int, b: int, m: int, n: int, k: int, masked_m=None, num_sms: int = 132) -> dict:
    """Host-side view of a batched launch's schedule (no GPU needed; the kernel walks the same code), with the
    launcher's default rasterisation. ``masked_m``: per-batch row counts (a sequence of ints) or None (dense).

    Returns ``{"workers": W, "units": [[(batch, m_block, n_block), ...] per worker]}``; blocks are cluster blocks."""
    counts = None if masked_m is None else (ctypes.c_int * b)(*masked_m)
    return _tile_list_schedule(batched_lib().b200_batched_schedule_units, 3, config_id, b, m, n, k, counts, num_sms)


def batched_launch_count() -> int:
    return int(batched_lib().b200_batched_launch_count())


# ------------------------------------------------------------------------------------------ grouped (libb200_grouped.so)
def check_grouped_operands(a, b_kmajor, offs, acc: str | int = "fp32", out_dtype=None,
                           scales: tuple = ()) -> tuple[int, int, int, int]:
    """(G, T, N, K) of the grouped product a[T,K] by b_kmajor[G,N,K] with the int32 group ends ``offs`` [G]
    (``torch._grouped_mm(a, b_kmajor.transpose(-2, -1), offs=offs)``), by the rules of the variant the dtypes and ``acc``
    name (the 2-D rules, :meth:`GemmType.fits`): a 16-bit one with the output dtype of the operands, or e4m3 operands
    with ``out_dtype`` fp16 / bf16 and two blockwise ``scales`` (:func:`scale_granularity` with ``groups``). Checks
    shapes and dtypes only (meta tensors pass); B200HgemmError otherwise."""
    try:
        (t, k), (g, n, k2) = a.shape, b_kmajor.shape
    except ValueError:
        raise B200HgemmError(f"a [T, K] and b_kmajor [G, N, K] expected, got {tuple(a.shape)} and "
                             f"{tuple(b_kmajor.shape)}") from None
    typ = _operand_type(a, b_kmajor, a.dtype if out_dtype is None else out_dtype, acc, scales, scaled=bool(scales))
    if scales:
        scale_granularity(t, n, *scales, k=k, groups=g)
    _check_k(a, b_kmajor, typ, n, k, k2, "[G, N, K]")
    _check_offs(offs, g)
    return g, t, n, k


def _check_offs(offs, g: int) -> None:
    """The group ends of a grouped product of ``g`` groups: an int32 tensor [g]. B200HgemmError otherwise."""
    import torch

    if offs.dtype != torch.int32 or tuple(offs.shape) != (g,):
        raise B200HgemmError(f"offs must be an int32 tensor of shape [{g}], got {offs.dtype} {tuple(offs.shape)}")


def gemm_grouped(a, b_kmajor, c, offs, acc: str | int = "fp32", config_id: int | None = None, group_m: int = 0,
                 max_ctas: int = 0, stream: int | None = None) -> None:
    """c[start_g:end_g] = a[start_g:end_g] @ b_kmajor[g]^T for every group g, fp16 (fp32 or fp16 accumulation) or bf16
    operands, all contiguous CUDA tensors ([T,K], [G,N,K], [T,N]). ``offs``: an int32 CUDA tensor [G] of cumulative
    group ends, read by the kernel when it runs (clamped as include/b200_grouped.h describes); rows of c at or past the
    last group's end are not written. ``config_id`` pins one kernel configuration (tests), ``max_ctas`` caps the CTAs
    (0: all SMs); default is the dispatcher."""
    _tile_list_gemm("grouped", a, b_kmajor, c, offs, acc, (), config_id, group_m, max_ctas, stream)


def grouped_select(variant: int, g: int, t: int, n: int, k: int) -> tuple[int, int]:
    """(config id, rasterisation group) the grouped dispatcher uses (b200_grouped_select)."""
    return _select(grouped_lib().b200_grouped_select, variant, g, t, n, k)


def grouped_schedule(config_id: int, t: int, n: int, k: int, offs, num_sms: int = 132) -> dict:
    """Host-side view of a grouped launch's schedule (no GPU needed; the kernel walks the same code), with the
    launcher's default rasterisation. ``offs``: the cumulative group ends (a sequence of ints, G of them).

    Returns ``{"workers": W, "units": [[(group, m_block, n_block), ...] per worker]}``; blocks are cluster blocks, and
    m-blocks count from the group's first row."""
    ends = (ctypes.c_int * len(offs))(*offs)
    return _tile_list_schedule(grouped_lib().b200_grouped_schedule_units, 3, config_id, len(offs), t, n, k, ends,
                               num_sms)


def grouped_launch_count() -> int:
    return int(grouped_lib().b200_grouped_launch_count())


# ------------------------------------------------------------------------------------------ grouped backward
#                                                                                            (libb200_grouped_bwd.so)
def grouped_bwd_lib() -> ctypes.CDLL:
    """libb200_grouped_bwd.so: the backward of the grouped fp16 / bf16 GEMM (csrc/b200_grouped_bwd.h, no public ABI)."""
    return load(GROUPED_BWD_LIB)


def _bwd_variant(dtype, acc: str | int) -> int:
    """The ``variant`` of the grouped backward: 0 fp16 or 2 bf16, both with fp32 accumulation; B200HgemmError
    otherwise."""
    v = batched_variant(dtype, acc)
    if v not in (0, 2):
        raise B200HgemmError(f"the grouped backward takes fp16 or bf16 operands with fp32 accumulation, got {dtype} "
                             f"with acc={acc!r}")
    return v


def _bwd_operand_type(a, b, acc: str | int) -> GemmType:
    """The 16-bit variant of the operands (:func:`_operand_type`), one that the grouped backward runs (fp32
    accumulation). B200HgemmError otherwise."""
    t = _operand_type(a, b, a.dtype, acc, (), scaled=False)
    _bwd_variant(a.dtype, acc)
    return t


def check_grouped_nn_operands(a, b, offs, acc: str | int = "fp32") -> tuple[int, int, int, int]:
    """(G, T, N, K) of the grouped row-major B product a[T,K] by b[G,K,N] (rows [start_g, end_g) of the result are
    those rows of ``a`` times ``b[g]``; ``torch._grouped_mm(a, b, offs=offs)``) with the int32 group ends ``offs`` [G]:
    one dtype, fp16 or bf16 with fp32 accumulation, N % 8 == 0 and K % 8 == 0. Checks shapes and dtypes only (meta
    tensors pass); B200HgemmError otherwise."""
    try:
        (t, k), (g, k2, n) = a.shape, b.shape
    except ValueError:
        raise B200HgemmError(f"a [T, K] and b [G, K, N] expected, got {tuple(a.shape)} and {tuple(b.shape)}") from None
    typ = _bwd_operand_type(a, b, acc)
    if k2 != k:
        raise B200HgemmError(f"inner dimensions differ: a {tuple(a.shape)}, b {tuple(b.shape)} (row-major: [G, K, N])")
    if not typ.fits(n, k):
        raise B200HgemmError(f"{a.dtype} operands need N % 8 == 0 and K % 8 == 0 (16-byte TMA strides), got N={n}, K={k}")
    _check_offs(offs, g)
    return g, t, n, k


def check_grouped_wgrad_operands(a, b, offs, acc: str | int = "fp32") -> tuple[int, int, int, int]:
    """(G, T, M, N) of the K-grouped product: for every group g, a[start_g:end_g]^T @ b[start_g:end_g] -> [M, N], with
    a [T,M], b [T,N] and the int32 group ends ``offs`` [G] (``torch._grouped_mm(a.t(), b, offs=offs)``): one dtype, fp16
    or bf16 with fp32 accumulation, M % 8 == 0 and N % 8 == 0. Checks shapes and dtypes only (meta tensors pass);
    B200HgemmError otherwise."""
    try:
        (t, m), (t2, n) = a.shape, b.shape
        (g,) = offs.shape
    except ValueError:
        raise B200HgemmError(f"a [T, M], b [T, N] and offs [G] expected, got {tuple(a.shape)}, {tuple(b.shape)} and "
                             f"{tuple(offs.shape)}") from None
    typ = _bwd_operand_type(a, b, acc)
    if t2 != t:
        raise B200HgemmError(f"row counts differ: a {tuple(a.shape)}, b {tuple(b.shape)}")
    if not typ.fits(n, m):   # M is the K-major product's K: the rows of A hold it
        raise B200HgemmError(f"{a.dtype} operands need M % 8 == 0 and N % 8 == 0 (16-byte TMA strides), got M={m}, N={n}")
    if g < 1:
        raise B200HgemmError("offs must hold at least one group")
    _check_offs(offs, g)
    return g, t, m, n


def _bwd_call(symbol: str, variant: int, ptrs: tuple, problem: tuple, config_id: int | None, group_m: int,
              max_ctas: int, stream: int | None) -> None:
    _check(getattr(grouped_bwd_lib(), symbol)(variant, -1 if config_id is None else config_id, *ptrs, *problem, group_m,
                                              max_ctas, stream), symbol)


def gemm_grouped_nn(a, b, c, offs, acc: str | int = "fp32", config_id: int | None = None, group_m: int = 0,
                    max_ctas: int = 0, stream: int | None = None) -> None:
    """c[start_g:end_g] = a[start_g:end_g] @ b[g] for every group g, with ``b`` [G,K,N] row-major (an expert weight
    stack [G, N_model, K_model] read in place: the input gradient of the grouped product), fp16 or bf16 operands with
    fp32 accumulation, all contiguous CUDA tensors ([T,K], [G,K,N], [T,N]). ``offs``: int32 CUDA tensor [G] of
    cumulative group ends, read by the kernel and clamped as for :func:`gemm_grouped`; rows of c at or past the last
    group's end are not written. ``config_id`` pins one kernel configuration (one with BN >= 64), ``max_ctas`` caps the
    CTAs (0: all SMs); default is the dispatcher."""
    _contiguous_cuda(a=a, b=b, c=c, offs=offs)
    g, t, n, k = check_grouped_nn_operands(a, b, offs, acc)
    if c.dtype != a.dtype or tuple(c.shape) != (t, n):
        raise B200HgemmError(f"c must be {a.dtype} {[t, n]}, got {c.dtype} {tuple(c.shape)}")
    _bwd_call("cuda_l2_b200_grouped_bwd_nn", _bwd_variant(a.dtype, acc), (a.data_ptr(), b.data_ptr(), c.data_ptr(),
              offs.data_ptr()), (g, t, n, k), config_id, group_m, max_ctas, stream)


def gemm_grouped_wgrad(a, b, c, offs, acc: str | int = "fp32", config_id: int | None = None, group_m: int = 0,
                       max_ctas: int = 0, stream: int | None = None) -> None:
    """c[g] = a[start_g:end_g]^T @ b[start_g:end_g] for every group g (the weight gradient of the grouped product), a
    [T,M] and b [T,N] fp16 or bf16 with fp32 accumulation, c [G,M,N], all contiguous CUDA tensors. ``offs``: int32
    CUDA tensor [G] of cumulative group ends, read by the kernel and clamped as for :func:`gemm_grouped`. Every matrix
    of c is written: an empty group's with zeros, and T == 0 zero-fills c without a launch. ``config_id`` pins one
    kernel configuration (one with BN >= 64), ``max_ctas`` caps the CTAs (0: all SMs); default is the dispatcher."""
    _contiguous_cuda(a=a, b=b, c=c, offs=offs)
    g, t, m, n = check_grouped_wgrad_operands(a, b, offs, acc)
    if c.dtype != a.dtype or tuple(c.shape) != (g, m, n):
        raise B200HgemmError(f"c must be {a.dtype} {[g, m, n]}, got {c.dtype} {tuple(c.shape)}")
    _bwd_call("cuda_l2_b200_grouped_bwd_wgrad", _bwd_variant(a.dtype, acc), (a.data_ptr(), b.data_ptr(), c.data_ptr(),
              offs.data_ptr()), (g, t, m, n), config_id, group_m, max_ctas, stream)


def grouped_nn_select(variant: int, g: int, t: int, n: int, k: int) -> tuple[int, int]:
    """(config id, rasterisation group) the dispatcher of :func:`gemm_grouped_nn` uses."""
    return _select(grouped_bwd_lib().cuda_l2_b200_grouped_bwd_nn_select, variant, g, t, n, k)


def grouped_wgrad_select(variant: int, g: int, t: int, m: int, n: int) -> tuple[int, int]:
    """(config id, rasterisation group) the dispatcher of :func:`gemm_grouped_wgrad` uses."""
    return _select(grouped_bwd_lib().cuda_l2_b200_grouped_bwd_wgrad_select, variant, g, t, m, n)


def grouped_wgrad_schedule(config_id: int, t: int, m: int, n: int, offs, num_sms: int = 132) -> dict:
    """Host-side view of a K-grouped launch's schedule (no GPU needed; the kernel walks the same code), with the
    launcher's default rasterisation. ``offs``: the cumulative group ends (a sequence of ints, G of them).

    Returns ``{"workers": W, "units": [[(group, m_block, n_block, k_blocks), ...] per worker]}``; blocks are cluster
    blocks, k_blocks the tile's 64-row k-blocks of its group (0 for an empty group)."""
    ends = (ctypes.c_int * len(offs))(*offs)
    return _tile_list_schedule(grouped_bwd_lib().cuda_l2_b200_grouped_bwd_wgrad_schedule, 4, config_id, len(offs), t,
                               m, n, ends, num_sms)


def grouped_bwd_launch_count() -> int:
    return int(grouped_bwd_lib().cuda_l2_b200_grouped_bwd_launch_count())


def fp8_grouped_gemm(a, b_kmajor, c, scale_a, scale_b, offs, config_id: int | None = None, group_m: int = 0,
                     max_ctas: int = 0, stream: int | None = None) -> None:
    """c[start_g:end_g] = the block-scaled product of a[start_g:end_g] and b_kmajor[g]^T for every group g, with
    ``float8_e4m3fn`` operands a [T,K] and b_kmajor [G,N,K] (contiguous CUDA tensors), c [T,N] fp16 or bf16, and block
    scales read by the kernel when it runs (include/b200_grouped_fp8.h): ``scale_a`` [T, ceil(K/128)] M-major (strides
    (1, ld_a), see :func:`blockwise_ld_a`: what ``ops.quantize_e4m3_blockwise`` returns), ``scale_b``
    [G, ceil(N/128), ceil(K/128)] contiguous. ``offs``: an int32 CUDA tensor [G] of cumulative group ends, clamped as
    for :func:`gemm_grouped`; rows of c at or past the last group's end are not written. ``config_id`` pins one kernel
    configuration (tests), ``max_ctas`` caps the CTAs (0: all SMs); default is the dispatcher."""
    _tile_list_gemm("grouped", a, b_kmajor, c, offs, "fp32", (scale_a, scale_b), config_id, group_m, max_ctas, stream)


def fp8_grouped_select(g: int, t: int, n: int, k: int) -> tuple[int, int]:
    """(config id, rasterisation group) the block-scaled grouped dispatcher uses (b200_grouped_fp8_select)."""
    return _select(grouped_fp8_lib().b200_grouped_fp8_select, g, t, n, k)


def fp8_grouped_launch_count() -> int:
    return int(grouped_fp8_lib().b200_grouped_fp8_launch_count())


def fp8_batched_gemm(a, b_kmajor, c, scale_a, scale_b, masked_m=None, config_id: int | None = None, group_m: int = 0,
                     max_ctas: int = 0, stream: int | None = None) -> None:
    """c[b] = the block-scaled product of a[b] and b_kmajor[b]^T for every b, with ``float8_e4m3fn`` operands a [B,M,K]
    and b_kmajor [B,N,K] (contiguous CUDA tensors), c [B,M,N] fp16 or bf16, and block scales read by the kernel when
    it runs (include/b200_batched_fp8.h): ``scale_a`` [B, M, ceil(K/128)] with one M-major block per matrix (strides
    (nkb * ld_a, 1, ld_a), see :func:`blockwise_ld_a`: what ``ops.quantize_e4m3_blockwise`` of a [B,M,K]
    tensor returns), ``scale_b`` [B, ceil(N/128), ceil(K/128)] contiguous. ``masked_m``: an optional int32 CUDA tensor
    [B], read by the kernel: only rows [0, clamp(masked_m[b], 0, M)) of c[b] are computed, as for
    :func:`gemm_batched`. ``config_id`` pins one kernel configuration (tests), ``max_ctas`` caps the CTAs (0: all SMs);
    default is the dispatcher."""
    _tile_list_gemm("batched", a, b_kmajor, c, masked_m, "fp32", (scale_a, scale_b), config_id, group_m, max_ctas,
                    stream)


def fp8_batched_select(b: int, m: int, n: int, k: int) -> tuple[int, int]:
    """(config id, rasterisation group) the block-scaled batched dispatcher uses (b200_batched_fp8_select)."""
    return _select(batched_fp8_lib().b200_batched_fp8_select, b, m, n, k)


def fp8_batched_launch_count() -> int:
    return int(batched_fp8_lib().b200_batched_fp8_launch_count())


def hgemm_config(a, b_col_major, c, config_id: int, acc: str | int = "fp32", group_m: int = 0, max_ctas: int = 0,
                 splits: int = 1, stream: int | None = None) -> None:
    m, n, k = _shape_check(a, b_col_major, c)
    _check(hgemm_lib().b200_hgemm_run_config(ACC_BITS[acc], config_id, a.data_ptr(), b_col_major.data_ptr(),
                                            c.data_ptr(), m, n, k, group_m, max_ctas, splits, stream), "b200_hgemm_run_config")


def hgemm_host(a_host, b_col_major_host, c_host, acc: str | int = "fp32") -> None:
    """End-to-end call on HOST tensors (H2D + GEMM + D2H, synchronous) — what bench.py's e2e leg times."""
    m, k = a_host.shape
    kb, n = b_col_major_host.shape
    assert kb == k and tuple(c_host.shape) == (m, n)
    for t in (a_host, b_col_major_host, c_host):
        assert (not t.is_cuda) and t.is_contiguous()
    _check(hgemm_lib().b200_hgemm_host(ACC_BITS[acc], a_host.data_ptr(), b_col_major_host.data_ptr(),
                                       c_host.data_ptr(), m, n, k), "b200_hgemm_host")


def configs() -> list[dict]:
    lib = hgemm_lib()
    out = []
    for cid in range(lib.b200_hgemm_num_configs()):
        bn, st, cg = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        lib.b200_hgemm_config_info(cid, ctypes.byref(bn), ctypes.byref(st), ctypes.byref(cg))
        cm, cn = ctypes.c_int(), ctypes.c_int()
        lib.b200_hgemm_config_cluster(cid, ctypes.byref(cm), ctypes.byref(cn))
        out.append({"id": cid, "bn": bn.value, "stages": st.value, "cta_group": cg.value,
                    "stages_requested": lib.b200_hgemm_config_stages_requested(cid),
                    "cluster_m": cm.value, "cluster_n": cn.value, "m_rep": lib.b200_hgemm_config_m_rep(cid)})
    return out


def select_config(acc: str | int, m: int, n: int, k: int) -> int:
    return hgemm_lib().b200_hgemm_select_config(ACC_BITS[acc], m, n, k)


def select(acc: str | int, m: int, n: int, k: int) -> tuple[int, int, int]:
    """(config id, rasterisation group, split-K factor) the dispatcher uses for this problem."""
    return _select(hgemm_lib().b200_hgemm_select, ACC_BITS[acc], m, n, k)


STREAMK_TAIL, STREAMK_TAIL_PLUS_WAVE = 100, 101      # `splits` codes of b200_hgemm_run_config
KMODES = ("plain", "split-k", "cluster-split-k", "stream-k")   # the K-modes b200_hgemm_schedule_units reports, in order


def schedule(config_id: int, m: int, n: int, k: int, splits: int = 1, num_sms: int = 132) -> dict:
    """Host-side view of the kernel's schedule (no GPU needed; the kernel walks the same code).

    Returns ``{"workers": W, "sk_tiles": S, "mode": one of KMODES,
    "units": [[(tile, kb0, kb1, contributors), ...] per worker]}``."""
    lib = hgemm_lib()
    nw, sk, mode = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    cap = 64
    buf, contrib = (ctypes.c_int * (3 * cap))(), (ctypes.c_int * cap)()
    st = lib.b200_hgemm_schedule_units(config_id, m, n, k, splits, num_sms, 0, buf, cap, ctypes.byref(nw),
                                       ctypes.byref(sk), ctypes.byref(mode), contrib)
    _check(min(st, 0), "b200_hgemm_schedule_units")
    units = []
    for w in range(nw.value):
        cnt = lib.b200_hgemm_schedule_units(config_id, m, n, k, splits, num_sms, w, buf, cap, None, None, None, contrib)
        _check(min(cnt, 0), "b200_hgemm_schedule_units")
        if cnt > cap:
            cap = cnt
            buf, contrib = (ctypes.c_int * (3 * cap))(), (ctypes.c_int * cap)()
            cnt = lib.b200_hgemm_schedule_units(config_id, m, n, k, splits, num_sms, w, buf, cap, None, None, None, contrib)
        units.append([(buf[3 * j], buf[3 * j + 1], buf[3 * j + 2], contrib[j]) for j in range(cnt)])
    return {"workers": nw.value, "sk_tiles": sk.value, "mode": KMODES[mode.value], "units": units}


def prewarm(stream: int | None = None) -> None:
    """Allocate the split-K / stream-K scratch of (current device, stream) now — needed before a CUDA-graph capture."""
    _check(hgemm_lib().b200_hgemm_prewarm(stream), "b200_hgemm_prewarm")


def release() -> None:
    """Free every device allocation the library holds (scratch, host-entry staging). Nothing may be in flight."""
    _check(hgemm_lib().b200_hgemm_release(), "b200_hgemm_release")


def gpu_local_cpus(device_index: int = 0) -> set[int] | None:
    """The CPUs NVML reports as local to the GPU (same NUMA node / PCIe root), intersected with the CPUs this process
    may use; None when NVML or the answer is unavailable."""
    import os

    try:
        import pynvml as nv
        nv.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        phys = device_index
        if vis:
            try:
                phys = int(vis.split(",")[device_index])
            except (ValueError, IndexError):
                pass
        h = nv.nvmlDeviceGetHandleByIndex(phys)
        words = nv.nvmlDeviceGetCpuAffinity(h, ((os.cpu_count() or 64) + 63) // 64)
        cpus = {64 * w + b for w, word in enumerate(words) for b in range(64) if (int(word) >> b) & 1}
        cpus &= os.sched_getaffinity(0)
        return cpus or None
    except Exception:
        return None


class host_near_gpu:
    """Context manager: run the calling thread on the CPUs local to ``device_index`` while HOST buffers for
    b200_hgemm_host are allocated (and, ideally, while the calls are made). Pinned memory lands on the NUMA node of the
    allocating thread; a buffer on the far socket costs the PCIe copies a cross-socket hop — in round 1 the same
    end-to-end call measured 55.7 TFLOP/s per GPU from a far node against 71.4 from the near one. Equivalent to
    launching under ``numactl --cpunodebind``; a no-op when NVML cannot tell."""

    def __init__(self, device_index: int = 0):
        self.device_index, self.saved, self.cpus = device_index, None, None

    def __enter__(self):
        import os
        self.cpus = gpu_local_cpus(self.device_index)
        if self.cpus:
            self.saved = os.sched_getaffinity(0)
            try:
                os.sched_setaffinity(0, self.cpus)
            except OSError:
                self.saved, self.cpus = None, None
        return self

    def __exit__(self, *exc):
        import os
        if self.saved is not None:
            os.sched_setaffinity(0, self.saved)
        return False


def launch_count() -> int:
    return int(hgemm_lib().b200_hgemm_launch_count())


# ------------------------------------------------------------------------------------------ comparators
class Baselines:
    """cuBLAS / cuBLASLt comparators (library calls; never part of the product path)."""

    NN, TN = 0, 1

    def __init__(self, acc: str | int = "fp32"):
        self.bits = ACC_BITS[acc]
        self.lib = baselines_lib()
        if self.lib.b200_bl_init(self.bits) != 0:
            raise B200HgemmError("cuBLAS/cuBLASLt handle creation failed")

    def close(self):
        self.lib.b200_bl_destroy(self.bits)

    def _call(self, fn, layout, a, b, c):
        m, k = a.shape
        n = c.shape[1]
        st = fn(self.bits, layout, a.data_ptr(), b.data_ptr(), c.data_ptr(), m, n, k)
        if st != 0:
            raise B200HgemmError(f"baseline call failed with status {st}")

    def cublas(self, layout, a, b, c):
        self._call(self.lib.b200_bl_cublas, layout, a, b, c)

    def lt_heuristic(self, layout, a, b, c):
        self._call(self.lib.b200_bl_lt_heuristic, layout, a, b, c)

    def lt_autotune_find(self, layout, m, n, k, warm_rounds=0, bench_rounds=0):
        st = self.lib.b200_bl_lt_autotune_find(self.bits, layout, m, n, k, warm_rounds, bench_rounds)
        if st != 0:
            raise B200HgemmError(f"cuBLASLt auto-tuning failed with status {st}")
        cand, ms = ctypes.c_int(), ctypes.c_float()
        self.lib.b200_bl_lt_autotune_info(self.bits, layout, ctypes.byref(cand), ctypes.byref(ms))
        return cand.value, ms.value

    def lt_autotune(self, layout, a, b, c):
        self._call(self.lib.b200_bl_lt_autotune, layout, a, b, c)


# ------------------------------------------------------------------------------- bias + activation (libb200_epilogue.so)
ACTIVATIONS = {"none": 0, "relu": 1, "gelu_tanh": 2}   # the activation codes of csrc/b200_epilogue.h


def epilogue_lib() -> ctypes.CDLL:
    """libb200_epilogue.so: the 2-D GEMM with a fused bias + activation epilogue (csrc/b200_epilogue.h, no public ABI)."""
    return load(EPILOGUE_LIB)


def epilogue_variant(operand, out_dtype) -> int:
    """The GemmType index of the bias + activation kernels for these dtypes: 0 fp16, 2 bf16, 3 / 4 e4m3 with fp16 / bf16
    output (fp32 accumulation). B200HgemmError for any other pair."""
    import torch

    variants = {(torch.float16, torch.float16): 0, (torch.bfloat16, torch.bfloat16): 2,
                (torch.float8_e4m3fn, torch.float16): 3, (torch.float8_e4m3fn, torch.bfloat16): 4}
    if (operand, out_dtype) not in variants:
        raise B200HgemmError(f"no bias + activation kernel for {operand} -> {out_dtype} (fp16, bf16 with fp32 accumulation; "
                             f"e4m3 -> fp16 / bf16 with per-tensor or rowwise scales)")
    return variants[(operand, out_dtype)]


def activation_code(activation: str) -> int:
    if activation not in ACTIVATIONS:
        raise B200HgemmError(f"unknown activation {activation!r}: one of {', '.join(ACTIVATIONS)}")
    return ACTIVATIONS[activation]


def check_bias(bias, n: int, out_dtype) -> None:
    """B200HgemmError unless ``bias`` is None or a 1-D tensor of ``n`` elements of ``out_dtype`` (shape and dtype only:
    meta tensors pass)."""
    if bias is not None and (bias.dim() != 1 or bias.shape[0] != n or bias.dtype != out_dtype):
        raise B200HgemmError(f"bias must be 1-D with N = {n} elements of {out_dtype}, got {bias.dtype} "
                             f"{tuple(bias.shape)}")


def _aligned(t):
    """``t`` as the kernels read a bias or a vector of scales: contiguous and 16-byte aligned (a fresh copy if it is
    not). None stays None."""
    if t is None:
        return None
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def gemm_bias_act(a, b_kmajor, c, bias=None, activation: str = "none", scale_a=None, scale_b=None,
                  stream: int | None = None, config_id: int | None = None, group_m: int = 0, splits: int = 1,
                  max_ctas: int = 0) -> None:
    """c[M,N] = act(a[M,K] @ b_kmajor[N,K]^T (scaled) + bias), fp32 throughout and one rounding to ``c``'s dtype
    (csrc/b200_epilogue.h). fp16 or bf16 operands with fp32 accumulation (no scales), or ``float8_e4m3fn`` operands with
    per-tensor or rowwise scales as for :func:`fp8_gemm` (blockwise scales have no bias kernel). ``bias``: None or a 1-D
    CUDA tensor of N elements of ``c``'s dtype; a misaligned one is copied. ``activation``: "none", "relu" or
    "gelu_tanh". ``config_id`` pins one kernel configuration (tests; ``group_m``, ``splits`` and ``max_ctas`` as for
    :func:`gemm_kmajor`); default is the dispatcher's choice for the same variant."""
    scales = () if scale_a is None and scale_b is None else (scale_a, scale_b)
    m, n, k, granularity = _kmajor_operands(a, b_kmajor, c, "fp32", scales)
    variant = epilogue_variant(a.dtype, c.dtype)
    act = activation_code(activation)
    _contiguous_cuda(bias=bias)
    check_bias(bias, n, c.dtype)
    if granularity in ("blockwise", "blockwise_1d1d"):
        raise B200HgemmError("blockwise e4m3 scales have no bias + activation kernel (per-tensor or rowwise only)")
    scale_args = _scale_args(granularity, *scales) if scales else (None, None)
    bias = _aligned(bias)
    args = (a.data_ptr(), b_kmajor.data_ptr(), c.data_ptr(), *scale_args, int(granularity == "rowwise"),
            None if bias is None else bias.data_ptr(), act, m, n, k)
    lib = epilogue_lib()
    if config_id is None:
        fn = lib.cuda_l2_b200_epilogue_run
        st = fn(variant, *args, stream)
    else:
        fn = lib.cuda_l2_b200_epilogue_run_config
        st = fn(variant, config_id, *args, group_m, max_ctas, splits, stream)
    _check(st, fn)


def epilogue_select(variant: int, m: int, n: int, k: int) -> tuple[int, int, int]:
    """(config_id, group_m, splits): the dispatched bias + activation call's choice for variant ``variant``."""
    return _select(epilogue_lib().cuda_l2_b200_epilogue_select, variant, m, n, k)


def epilogue_prewarm(stream: int | None = None) -> None:
    """Allocate libb200_epilogue.so's split-K scratch for ``stream`` ahead of a CUDA-graph capture (a first split-K or
    stream-K call inside a capture runs undivided without it)."""
    _check(epilogue_lib().cuda_l2_b200_epilogue_prewarm(stream), "cuda_l2_b200_epilogue_prewarm")


def epilogue_release() -> None:
    """Free libb200_epilogue.so's split-K scratch (no launch of it may be in flight)."""
    _check(epilogue_lib().cuda_l2_b200_epilogue_release(), "cuda_l2_b200_epilogue_release")


def epilogue_launch_count() -> int:
    return int(epilogue_lib().cuda_l2_b200_epilogue_launch_count())


# ------------------------------------------------------------------------------------ SwiGLU (libb200_swiglu.so)
SWIGLU_BLOCK = 64   # gate and up rows of w_gu interleave in blocks of this many (csrc/b200_swiglu.h)


def swiglu_lib() -> ctypes.CDLL:
    """libb200_swiglu.so: the gate / up GEMM with silu(g) * u fused into its epilogue, and the one-pass SwiGLU backward
    (csrc/b200_swiglu.h, no public ABI)."""
    return load(SWIGLU_LIB)


def swiglu_variant(dtype) -> int:
    """The GemmType index of the SwiGLU kernels for ``dtype``: 0 fp16, 2 bf16 (fp32 accumulation). B200HgemmError for
    any other dtype."""
    import torch

    if dtype not in (torch.float16, torch.bfloat16):
        raise B200HgemmError(f"SwiGLU kernels take fp16 or bf16 tensors, got {dtype}")
    return 0 if dtype == torch.float16 else 2


def check_swiglu_operands(x, w_gu) -> tuple[int, int, int]:
    """(M, I, K) of y = swiglu(x [M, K] @ w_gu [2I, K]^T): 2-D operands of one 16-bit dtype, a shared K with K % 8 == 0,
    and 2I rows with I % 64 == 0 (whole 64-row gate / up blocks). Shapes and dtypes only (meta tensors pass);
    B200HgemmError otherwise."""
    try:
        (m, k), (n, k2) = x.shape, w_gu.shape
    except ValueError:
        raise B200HgemmError(f"2-D operands expected, got {tuple(x.shape)} and {tuple(w_gu.shape)}") from None
    swiglu_variant(x.dtype)
    if w_gu.dtype != x.dtype:
        raise B200HgemmError(f"x and w_gu must share a dtype, got {x.dtype} and {w_gu.dtype}")
    if k2 != k:
        raise B200HgemmError(f"inner dimensions differ: x {tuple(x.shape)}, w_gu {tuple(w_gu.shape)} ([2I, K])")
    if n % (2 * SWIGLU_BLOCK) or k % 8:
        raise B200HgemmError(f"w_gu [2I, K] needs I % {SWIGLU_BLOCK} == 0 and K % 8 == 0, got 2I={n}, K={k}")
    return m, n // 2, k


def swiglu(x, w_gu, y, h=None, stream: int | None = None, config_id: int | None = None, group_m: int = 0,
           splits: int = 1, max_ctas: int = 0) -> None:
    """y [M, I] = silu(g) * u of h = x [M, K] @ w_gu [2I, K]^T, whose gate and up columns interleave in blocks of 64
    (csrc/b200_swiglu.h), with fp32 accumulation: torch's ``F.silu(g) * u`` on the 16-bit h, bit for bit. ``h``
    [M, 2I] (optional) receives h itself, the bits :func:`gemm_kmajor` writes with the same configuration. All
    contiguous CUDA tensors of one dtype (fp16 or bf16). ``config_id`` pins one configuration (BN = 128 or 256; tests;
    ``group_m``, ``max_ctas`` as for :func:`gemm_kmajor`, every ``splits`` runs the plain schedule); default is the
    dispatcher's TN choice for (M, 2I, K) mapped to its gated sibling."""
    _contiguous_cuda(x=x, w_gu=w_gu, y=y, h=h)
    m, i, k = check_swiglu_operands(x, w_gu)
    if tuple(y.shape) != (m, i) or y.dtype != x.dtype or (h is not None and (tuple(h.shape) != (m, 2 * i) or
                                                                             h.dtype != x.dtype)):
        raise B200HgemmError(f"y must be [{m}, {i}] and h [{m}, {2 * i}] of {x.dtype}, got y {y.dtype} "
                             f"{tuple(y.shape)}" + ("" if h is None else f", h {h.dtype} {tuple(h.shape)}"))
    args = (x.data_ptr(), w_gu.data_ptr(), None if h is None else h.data_ptr(), y.data_ptr(), m, i, k)
    lib = swiglu_lib()
    if config_id is None:
        fn = lib.cuda_l2_b200_swiglu_run
        st = fn(swiglu_variant(x.dtype), *args, stream)
    else:
        fn = lib.cuda_l2_b200_swiglu_run_config
        st = fn(swiglu_variant(x.dtype), config_id, *args, group_m, splits, max_ctas, stream)
    _check(st, fn)


def swiglu_backward(dy, h, dh, stream: int | None = None) -> None:
    """dh [M, 2I] = the gradient of y = silu(g) * u at h [M, 2I] for dy [M, I], in h's interleaved layout: the steps
    torch's autograd takes through ``F.silu(g) * u`` (csrc/b200_swiglu.h). Contiguous CUDA tensors of one dtype."""
    _contiguous_cuda(dy=dy, h=h, dh=dh)
    if dy.dim() != 2 or h.dim() != 2 or tuple(h.shape) != (dy.shape[0], 2 * dy.shape[1]) or dh.shape != h.shape or \
            not dy.dtype == h.dtype == dh.dtype:
        raise B200HgemmError(f"dy [M, I], h and dh [M, 2I] of one dtype expected, got dy {dy.dtype} {tuple(dy.shape)}, "
                             f"h {h.dtype} {tuple(h.shape)}, dh {dh.dtype} {tuple(dh.shape)}")
    fn = swiglu_lib().cuda_l2_b200_swiglu_backward
    _check(fn(swiglu_variant(dy.dtype), dy.data_ptr(), h.data_ptr(), dh.data_ptr(), dy.shape[0], dy.shape[1], stream),
           fn)


def swiglu_select(variant: int, m: int, i: int, k: int) -> tuple[int, int, int]:
    """(config_id, group_m, splits): the dispatched SwiGLU call's choice for variant ``variant`` (0 fp16, 2 bf16)."""
    return _select(swiglu_lib().cuda_l2_b200_swiglu_select, variant, m, i, k)


def swiglu_launch_count() -> int:
    return int(swiglu_lib().cuda_l2_b200_swiglu_launch_count())


# ------------------------------------------------------------------ grouped SwiGLU (libb200_grouped_swiglu.so)
def grouped_swiglu_lib() -> ctypes.CDLL:
    """libb200_grouped_swiglu.so: the gate / up GEMM of SwiGLU experts over contiguous row groups with silu(g) * u fused
    into its epilogue, and the SwiGLU backward over the groups' rows (csrc/b200_grouped_swiglu.h, no public ABI)."""
    return load(GROUPED_SWIGLU_LIB)


def check_grouped_swiglu_operands(x, w_gu, offs) -> tuple[int, int, int, int]:
    """(G, T, I, H) of y = swiglu(h) with h[start_g:end_g] = x[start_g:end_g] @ w_gu[g]^T: x [T, H] and the expert stack
    w_gu [G, 2I, H] of one 16-bit dtype, H % 8 == 0, I % 64 == 0 (whole 64-row gate / up blocks), and the int32 group
    ends ``offs`` [G]. Shapes and dtypes only (meta tensors pass); B200HgemmError otherwise."""
    try:
        (t, k), (g, n, k2) = x.shape, w_gu.shape
    except ValueError:
        raise B200HgemmError(f"x [T, H] and w_gu [G, 2I, H] expected, got {tuple(x.shape)} and "
                             f"{tuple(w_gu.shape)}") from None
    swiglu_variant(x.dtype)
    if w_gu.dtype != x.dtype:
        raise B200HgemmError(f"x and w_gu must share a dtype, got {x.dtype} and {w_gu.dtype}")
    if k2 != k:
        raise B200HgemmError(f"inner dimensions differ: x {tuple(x.shape)}, w_gu {tuple(w_gu.shape)} ([G, 2I, H])")
    if g < 1:
        raise B200HgemmError("w_gu must hold at least one expert")
    if n == 0 or n % (2 * SWIGLU_BLOCK) or k % 8:
        raise B200HgemmError(f"w_gu [G, 2I, H] needs I % {SWIGLU_BLOCK} == 0 (I > 0) and H % 8 == 0, got 2I={n}, H={k}")
    _check_offs(offs, g)
    return g, t, n // 2, k


def grouped_swiglu(x, w_gu, offs, y, h=None, stream: int | None = None, config_id: int | None = None,
                   group_m: int = 0, max_ctas: int = 0) -> None:
    """y [T, I] = silu(g) * u of the grouped product h[start_g:end_g] = x[start_g:end_g] @ w_gu[g]^T, each expert's
    gate and up rows interleaved in blocks of 64 (csrc/b200_grouped_swiglu.h), fp32 accumulation: torch's
    ``F.silu(g) * u`` on the 16-bit h, bit for bit. ``offs``: int32 CUDA tensor [G] of cumulative group ends, read by
    the kernel and clamped as for :func:`gemm_grouped`. ``h`` [T, 2I] (optional) receives h itself, the bits
    :func:`gemm_grouped` writes with the same configuration. Rows of y and h at or past the last group's end are not
    written. Contiguous CUDA tensors of one dtype (fp16 or bf16). ``config_id`` pins one configuration (BN = 128 or
    256; tests; ``group_m``, ``max_ctas`` as for :func:`gemm_grouped`); default is the grouped dispatcher's choice for
    (G, T, 2I, H) mapped to its gated sibling."""
    _contiguous_cuda(x=x, w_gu=w_gu, y=y, h=h, offs=offs)
    g, t, i, k = check_grouped_swiglu_operands(x, w_gu, offs)
    if tuple(y.shape) != (t, i) or y.dtype != x.dtype or (h is not None and (tuple(h.shape) != (t, 2 * i) or
                                                                             h.dtype != x.dtype)):
        raise B200HgemmError(f"y must be [{t}, {i}] and h [{t}, {2 * i}] of {x.dtype}, got y {y.dtype} "
                             f"{tuple(y.shape)}" + ("" if h is None else f", h {h.dtype} {tuple(h.shape)}"))
    args = (x.data_ptr(), w_gu.data_ptr(), None if h is None else h.data_ptr(), y.data_ptr(), offs.data_ptr(), g, t, i,
            k)
    lib = grouped_swiglu_lib()
    if config_id is None:
        fn = lib.cuda_l2_b200_grouped_swiglu_run
        st = fn(swiglu_variant(x.dtype), *args, stream)
    else:
        fn = lib.cuda_l2_b200_grouped_swiglu_run_config
        st = fn(swiglu_variant(x.dtype), config_id, *args, group_m, max_ctas, stream)
    _check(st, fn)


def grouped_swiglu_backward(dy, h, dh, offs, stream: int | None = None) -> None:
    """dh [T, 2I] = the gradient of y = silu(g) * u at h [T, 2I] for dy [T, I], in h's interleaved layout, for the rows
    below the groups' last end (read on the device from the int32 CUDA tensor ``offs`` [G]): the steps torch's
    autograd takes through ``F.silu(g) * u`` (csrc/b200_grouped_swiglu.h). Rows of dy and h at or past that end are
    never read, and rows of dh there never written. Contiguous CUDA tensors of one dtype."""
    _contiguous_cuda(dy=dy, h=h, dh=dh, offs=offs)
    if dy.dim() != 2 or h.dim() != 2 or tuple(h.shape) != (dy.shape[0], 2 * dy.shape[1]) or dh.shape != h.shape or \
            not dy.dtype == h.dtype == dh.dtype:
        raise B200HgemmError(f"dy [T, I], h and dh [T, 2I] of one dtype expected, got dy {dy.dtype} {tuple(dy.shape)}, "
                             f"h {h.dtype} {tuple(h.shape)}, dh {dh.dtype} {tuple(dh.shape)}")
    if offs.dim() != 1:
        raise B200HgemmError(f"offs must be an int32 tensor [G], got {tuple(offs.shape)}")
    _check_offs(offs, offs.shape[0])
    fn = grouped_swiglu_lib().cuda_l2_b200_grouped_swiglu_backward
    _check(fn(swiglu_variant(dy.dtype), dy.data_ptr(), h.data_ptr(), dh.data_ptr(), offs.data_ptr(), offs.shape[0],
              dy.shape[0], dy.shape[1], stream), fn)


def grouped_swiglu_select(variant: int, g: int, t: int, i: int, h: int) -> tuple[int, int]:
    """(config_id, group_m): the dispatched grouped SwiGLU call's choice for variant ``variant`` (0 fp16, 2 bf16)."""
    return _select(grouped_swiglu_lib().cuda_l2_b200_grouped_swiglu_select, variant, g, t, i, h)


def grouped_swiglu_launch_count() -> int:
    return int(grouped_swiglu_lib().cuda_l2_b200_grouped_swiglu_launch_count())


# ---------------------------------------------------------------- fp32 weight-gradient accumulation
#                                                                  (libb200_wgrad_accum.so)
WGRAD_ACCUM_FORMS = {"rowwise": 1, "blockwise_1d1d": 3}   # the scale forms of cuda_l2_b200_wgrad_accum_fp8


def wgrad_accum_lib() -> ctypes.CDLL:
    """libb200_wgrad_accum.so: weight gradients added into fp32 buffers by the GEMM epilogue (csrc/b200_wgrad_accum.h,
    no public ABI)."""
    return load(WGRAD_ACCUM_LIB)


def check_main_grad(main_grad, shape: tuple, device, what: str = "main_grad") -> None:
    """B200HgemmError unless ``main_grad`` is what the accumulating kernels add into: an fp32 tensor of ``shape``,
    contiguous, on ``device`` (shape, dtype and layout only on the meta device; 16-byte aligned on a real one)."""
    import torch

    if main_grad is None:
        raise B200HgemmError(f"{what} is missing: an fp32 tensor of shape {list(shape)} on {device} is needed")
    if (main_grad.dtype != torch.float32 or tuple(main_grad.shape) != tuple(shape) or main_grad.device != device
            or not main_grad.is_contiguous()):
        raise B200HgemmError(f"{what} must be a contiguous fp32 tensor of shape {list(shape)} on {device}, got "
                             f"{main_grad.dtype} {list(main_grad.shape)} on {main_grad.device}"
                             f"{'' if main_grad.is_contiguous() else ', not contiguous'}")
    if main_grad.device.type != "meta" and main_grad.data_ptr() % 16:
        raise B200HgemmError(f"{what} must be 16-byte aligned")


def wgrad_accum_grouped(a, b, c32, offs, config_id: int | None = None, group_m: int = 0, max_ctas: int = 0,
                        stream: int | None = None) -> None:
    """c32[g] += a[start_g:end_g]^T @ b[start_g:end_g] for every group g, in fp32 with one rounding per element after
    the whole sum (csrc/b200_wgrad_accum.h): :func:`gemm_grouped_wgrad`'s product, a [T,M] and b [T,N] fp16 or bf16,
    offs the int32 group ends [G], c32 [G,M,N] fp32, all contiguous CUDA tensors. An empty group's matrix and, with
    T == 0, all of c32 stay as they are, and T == 0 launches nothing. ``config_id`` pins one kernel configuration (one
    with BN >= 64); default is :func:`gemm_grouped_wgrad`'s dispatcher."""
    _contiguous_cuda(a=a, b=b, offs=offs)
    g, t, m, n = check_grouped_wgrad_operands(a, b, offs)
    check_main_grad(c32, (g, m, n), a.device, "c32")
    fn = wgrad_accum_lib().cuda_l2_b200_wgrad_accum_grouped
    _check(fn(_bwd_variant(a.dtype, "fp32"), -1 if config_id is None else config_id, a.data_ptr(), b.data_ptr(),
              c32.data_ptr(), offs.data_ptr(), g, t, m, n, group_m, max_ctas, stream), fn)


def wgrad_accum_fp8(a, b_kmajor, c32, scale_a, scale_b, stream: int | None = None, config_id: int | None = None,
                    group_m: int = 0, splits: int = 1, max_ctas: int = 0) -> None:
    """c32[M,N] += the e4m3 product of :func:`fp8_gemm` for ``a`` [M,K] and ``b_kmajor`` [N,K], in fp32 with one
    rounding per element after the whole sum (csrc/b200_wgrad_accum.h): exactly the value fp8_gemm rounds to its output
    is added. The scales are rowwise (``scale_a`` [M,1], ``scale_b`` [1,N], contiguous) or 1 x 128 on both operands
    (``scale_a`` [M, ceil(K/128)], ``scale_b`` [N, ceil(K/128)], read in place as for :func:`fp8_gemm`); per-tensor and
    128 x 128 scales have no accumulating kernel. ``config_id`` pins one kernel configuration (``splits``, ``group_m``
    and ``max_ctas`` as for :func:`fp8_gemm`); default is :func:`fp8_gemm`'s dispatcher for those scales."""
    import torch

    _contiguous_cuda(a=a, b_kmajor=b_kmajor)
    m, n, k, granularity = check_operands(a, b_kmajor, torch.bfloat16, "fp32", (scale_a, scale_b))
    if granularity not in WGRAD_ACCUM_FORMS:
        raise B200HgemmError(f"fp32 accumulation takes rowwise or 1 x 128 x 1 x 128 (blockwise_1d1d) scales, got "
                             f"{granularity} scales")
    check_main_grad(c32, (m, n), a.device, "c32")
    args = _scale_args(granularity, scale_a, scale_b)
    if granularity == "rowwise":
        args = (args[0], 0, args[1], 0)
    fn = wgrad_accum_lib().cuda_l2_b200_wgrad_accum_fp8
    _check(fn(WGRAD_ACCUM_FORMS[granularity], -1 if config_id is None else config_id, a.data_ptr(),
              b_kmajor.data_ptr(), c32.data_ptr(), *args, m, n, k, group_m, max_ctas, splits, stream), fn)


def wgrad_accum_grouped_select(variant: int, g: int, t: int, m: int, n: int) -> tuple[int, int]:
    """(config id, rasterisation group) of the dispatched :func:`wgrad_accum_grouped` call."""
    return _select(wgrad_accum_lib().cuda_l2_b200_wgrad_accum_grouped_select, variant, g, t, m, n)


def wgrad_accum_fp8_select(granularity: str, m: int, n: int, k: int) -> tuple[int, int, int]:
    """(config id, rasterisation group, splits code) of the dispatched :func:`wgrad_accum_fp8` call."""
    return _select(wgrad_accum_lib().cuda_l2_b200_wgrad_accum_fp8_select, WGRAD_ACCUM_FORMS[granularity], m, n, k)


def wgrad_accum_prewarm(stream: int | None = None) -> None:
    """Allocate libb200_wgrad_accum.so's split-K scratch for ``stream`` ahead of a CUDA-graph capture (a first split-K
    or stream-K call inside a capture runs undivided without it)."""
    _check(wgrad_accum_lib().cuda_l2_b200_wgrad_accum_prewarm(stream), "cuda_l2_b200_wgrad_accum_prewarm")


def wgrad_accum_release() -> None:
    """Free libb200_wgrad_accum.so's split-K scratch (no launch of it may be in flight)."""
    _check(wgrad_accum_lib().cuda_l2_b200_wgrad_accum_release(), "cuda_l2_b200_wgrad_accum_release")


def wgrad_accum_launch_count() -> int:
    return int(wgrad_accum_lib().cuda_l2_b200_wgrad_accum_launch_count())


# ------------------------------------------------------------------------------------------ e4m3 quantisers
#                                                                                            (libb200_quant.so)
QUANT_TENSOR_WORKSPACE = 1024   # floats of the per-tensor quantiser's workspace (csrc/b200_quant.h)


def quant_lib() -> ctypes.CDLL:
    """libb200_quant.so: the one-pass e4m3 quantisers of FP8 activations (csrc/b200_quant.h, no public ABI)."""
    return load(QUANT_LIB)


def quant_dtype(dtype, silu_mul: bool = False) -> int | None:
    """The ``dtype`` code of csrc/b200_quant.h for an input of this torch dtype: 0 fp16, 1 bf16, 2 fp32 (the SwiGLU
    kernel takes fp16 and bf16 only); None if no kernel takes it."""
    import torch

    codes = {torch.float16: 0, torch.bfloat16: 1} if silu_mul else {torch.float16: 0, torch.bfloat16: 1,
                                                                     torch.float32: 2}
    return codes.get(dtype)


def _quant_input(x, silu_mul: bool = False) -> int:
    """The dtype code of ``x``, a contiguous CUDA tensor of a dtype a quantiser takes; B200HgemmError otherwise."""
    code = quant_dtype(x.dtype, silu_mul)
    if code is None:
        raise B200HgemmError(f"no e4m3 quantiser for {x.dtype} input (fp16, bf16{'' if silu_mul else ', fp32'})")
    _contiguous_cuda(x=x)
    return code


def _quant_output(q, shape, x) -> None:
    import torch

    if q.dtype != torch.float8_e4m3fn or tuple(q.shape) != tuple(shape) or not q.is_contiguous() or \
            q.device != x.device:
        raise B200HgemmError(f"q must be a contiguous float8_e4m3fn tensor {list(shape)} on {x.device}, got {q.dtype} "
                             f"{tuple(q.shape)} on {q.device}")


def _fp32_on(t, x, name: str, shape) -> None:
    import torch

    if t.dtype != torch.float32 or tuple(t.shape) != tuple(shape) or t.device != x.device:
        raise B200HgemmError(f"{name} must be an fp32 tensor {list(shape)} on {x.device}, got {t.dtype} "
                             f"{tuple(t.shape)} on {t.device}")


def quantize_e4m3(x, q, scale, workspace, stream: int | None = None) -> None:
    """Per-tensor quantisation of ``x`` (fp16, bf16 or fp32, contiguous, at least one element) into ``q`` (e4m3,
    x's shape) and ``scale`` (one fp32 element), in two launches; ``workspace``: QUANT_TENSOR_WORKSPACE fp32 elements
    of device memory that no other call uses until this one has run (csrc/b200_quant.h)."""
    code = _quant_input(x)
    _quant_output(q, x.shape, x)
    _fp32_on(scale, x, "scale", (1,))
    _fp32_on(workspace, x, "workspace", (QUANT_TENSOR_WORKSPACE,))
    _contiguous_cuda(workspace=workspace)
    _check(quant_lib().cuda_l2_b200_quant_e4m3_tensor(code, x.data_ptr(), x.numel(), q.data_ptr(), scale.data_ptr(),
                                                      workspace.data_ptr(), stream), "cuda_l2_b200_quant_e4m3_tensor")


def quantize_e4m3_rowwise(x, q, scale, stream: int | None = None) -> None:
    """Rowwise quantisation of a 2-D ``x`` [rows, cols] (fp16, bf16 or fp32, contiguous) into ``q`` (e4m3 [rows, cols])
    and ``scale`` (fp32 [rows, 1], contiguous), in one launch."""
    code = _quant_input(x)
    if x.dim() != 2:
        raise B200HgemmError(f"the rowwise quantiser takes a 2-D [rows, cols] tensor, got {list(x.shape)}")
    rows, cols = x.shape
    _quant_output(q, x.shape, x)
    _fp32_on(scale, x, "scale", (rows, 1))
    _contiguous_cuda(scale=scale)
    _check(quant_lib().cuda_l2_b200_quant_e4m3_rowwise(code, x.data_ptr(), rows, cols, q.data_ptr(), scale.data_ptr(),
                                                       stream), "cuda_l2_b200_quant_e4m3_rowwise")


def _blockwise_call(symbol: str, x, q, scale, masked_m, k: int, silu_mul: bool, stream) -> None:
    """The 1 x 128 quantisers: ``x`` [(B,) M, K] (or SwiGLU's h [(B,) M, 2K]) into ``q`` [(B,) M, K] and ``scale``
    [(B,) M, ceil(K/128)] in the M-major layout of :func:`blockwise_ld_a`, with optional int32 ``masked_m`` [B]."""
    import torch

    code = _quant_input(x, silu_mul)
    if x.dim() not in (2, 3):
        raise B200HgemmError(f"the 1 x 128 quantisers take [M, K] or [B, M, K] inputs, got {list(x.shape)}")
    *lead, m, _ = x.shape
    bsz = lead[0] if lead else 1
    _quant_output(q, (*lead, m, k), x)
    _fp32_on(scale, x, "scale", (*lead, m, num_k_blocks(k)))
    ld_a = _scale_ld_a(scale)
    if masked_m is not None:
        _contiguous_cuda(masked_m=masked_m)
        if masked_m.dtype != torch.int32 or tuple(masked_m.shape) != (bsz,) or masked_m.device != x.device:
            raise B200HgemmError(f"masked_m must be an int32 tensor of shape [{bsz}] on {x.device}, got "
                                 f"{masked_m.dtype} {tuple(masked_m.shape)} on {masked_m.device}")
    _check(getattr(quant_lib(), symbol)(code, x.data_ptr(), bsz, m, k, q.data_ptr(), scale.data_ptr(), ld_a,
                                        None if masked_m is None else masked_m.data_ptr(), stream), symbol)


def quantize_e4m3_blockwise(x, q, scale, masked_m=None, stream: int | None = None) -> None:
    """1 x 128 quantisation of ``x`` [(B,) M, K] (fp16, bf16 or fp32, contiguous) into ``q`` (e4m3, x's shape) and
    ``scale`` [(B,) M, ceil(K/128)], written in place in its M-major layout (:func:`blockwise_ld_a`: a view of a
    [(B,) ceil(K/128), ld_a] buffer), in one launch. ``masked_m``: an optional int32 CUDA tensor [B]; only rows
    [0, clamp(masked_m[b], 0, M)) of matrix b are read and written, in q and in scale."""
    _blockwise_call("cuda_l2_b200_quant_e4m3_blockwise", x, q, scale, masked_m, x.shape[-1], False, stream)


def silu_mul_quantize_e4m3_blockwise(h, q, scale, masked_m=None, stream: int | None = None) -> None:
    """1 x 128 quantisation of silu(g) * u, with g = h[..., :I] and u = h[..., I:] of ``h`` [(B,) M, 2I] (fp16 or
    bf16, contiguous), into ``q`` [(B,) M, I] and ``scale`` [(B,) M, ceil(I/128)] as for
    :func:`quantize_e4m3_blockwise`, ``masked_m`` likewise, in one launch."""
    if h.shape[-1] % 2:
        raise B200HgemmError(f"h must be [(B,) M, 2I], got {list(h.shape)}")
    _blockwise_call("cuda_l2_b200_quant_silu_mul_e4m3_blockwise", h, q, scale, masked_m, h.shape[-1] // 2, True,
                    stream)


def quant_launch_count() -> int:
    return int(quant_lib().cuda_l2_b200_quant_launch_count())


# ------------------------------------------------------------------------------------------ dual-orientation rowwise
#                                                                                            e4m3 (libb200_quant_dual.so)
def quant_dual_lib() -> ctypes.CDLL:
    """libb200_quant_dual.so: x and x^T quantised rowwise to e4m3 from one tensor (csrc/b200_quant_dual.h, no public
    ABI)."""
    return load(QUANT_DUAL_LIB)


def dual_ld_t(rows: int) -> int:
    """The row length of the transposed e4m3 copy of an x with ``rows`` rows: rows rounded up to 16, so that it is a
    K-major FP8 GEMM operand (K % 16 == 0)."""
    return -(-rows // 16) * 16


def quant_dual_workspace(rows: int, cols: int) -> int:
    """Floats of the workspace of :func:`quantize_e4m3_rowwise_dual` (CUDA_L2_B200_QUANT_DUAL_WORKSPACE)."""
    return rows + cols


def quantize_e4m3_rowwise_dual(x, q, scale, q_t, scale_t, workspace, stream: int | None = None) -> None:
    """Both rowwise quantisations of a 2-D ``x`` [rows, cols] (fp16, bf16 or fp32, contiguous): ``q`` (e4m3
    [rows, cols]) with ``scale`` (fp32 [rows]), and ``q_t`` (e4m3 [cols, dual_ld_t(rows)], x^T zero-padded) with
    ``scale_t`` (fp32 [cols]), in one memset and two launches; ``workspace``: quant_dual_workspace(rows, cols) fp32
    elements of device memory that no other call uses until this one has run (csrc/b200_quant_dual.h)."""
    code = _quant_input(x)
    if x.dim() != 2:
        raise B200HgemmError(f"the dual rowwise quantiser takes a 2-D [rows, cols] tensor, got {list(x.shape)}")
    rows, cols = x.shape
    _quant_output(q, x.shape, x)
    _quant_output(q_t, (cols, dual_ld_t(rows)), x)
    _fp32_on(scale, x, "scale", (rows,))
    _fp32_on(scale_t, x, "scale_t", (cols,))
    _fp32_on(workspace, x, "workspace", (quant_dual_workspace(rows, cols),))
    _contiguous_cuda(scale=scale, scale_t=scale_t, workspace=workspace)
    fn = quant_dual_lib().cuda_l2_b200_quant_dual_e4m3_rowwise
    _check(fn(code, x.data_ptr(), rows, cols, q.data_ptr(), scale.data_ptr(), q_t.data_ptr(), scale_t.data_ptr(),
              workspace.data_ptr(), stream), fn)


def quant_dual_launch_count() -> int:
    return int(quant_dual_lib().cuda_l2_b200_quant_dual_launch_count())


# ------------------------------------------------------------------------------------------ dual-orientation block
#                                                                                            e4m3 (libb200_quant_block_dual.so)
def quant_block_dual_lib() -> ctypes.CDLL:
    """libb200_quant_block_dual.so: x and x^T quantised per 1 x 128 group, or w and w^T per 128 x 128 block, from one
    read of the tensor (csrc/b200_quant_block_dual.h, no public ABI)."""
    return load(QUANT_BLOCK_DUAL_LIB)


def _block_dual_input(x) -> tuple[int, int, int]:
    """(dtype code, rows, cols) of a 2-D contiguous fp16 / bf16 CUDA ``x``; B200HgemmError otherwise."""
    code = quant_dtype(x.dtype, silu_mul=True)   # fp16 and bf16 only, as for the SwiGLU kernel
    if code is None or x.dim() != 2:
        raise B200HgemmError(f"the dual block quantisers take a 2-D fp16 / bf16 [rows, cols] tensor, got {x.dtype} "
                             f"{list(x.shape)}")
    _contiguous_cuda(x=x)
    return code, *x.shape


def quantize_e4m3_blockwise_dual(x, q, scale, q_t, scale_t, stream: int | None = None) -> None:
    """Both 1 x 128 quantisations of a 2-D ``x`` [rows, cols] (fp16 or bf16, contiguous) in one launch: ``q`` (e4m3
    [rows, cols]) with ``scale`` [rows, ceil(cols/128)], and ``q_t`` (e4m3 [cols, dual_ld_t(rows)], x^T zero-padded)
    with ``scale_t`` [cols, ceil(rows/128)], both scales written in place in the M-major layout of
    :func:`blockwise_ld_a` with ld = rows (cols) rounded up to 4, as :func:`empty_m_major` allocates them
    (csrc/b200_quant_block_dual.h)."""
    code, rows, cols = _block_dual_input(x)
    _quant_output(q, x.shape, x)
    _quant_output(q_t, (cols, dual_ld_t(rows)), x)
    for name, s, (m, nkb) in (("scale", scale, (rows, num_k_blocks(cols))),
                              ("scale_t", scale_t, (cols, num_k_blocks(rows)))):
        _fp32_on(s, x, name, (m, nkb))
        if blockwise_ld_a(s) != _m_major_ld(m):
            raise B200HgemmError(f"{name} must be the M-major view of a [{nkb}, {_m_major_ld(m)}] buffer")
    fn = quant_block_dual_lib().cuda_l2_b200_quant_block_dual_e4m3_1x128
    _check(fn(code, x.data_ptr(), rows, cols, q.data_ptr(), scale.data_ptr(), q_t.data_ptr(), scale_t.data_ptr(),
              stream), fn)


def quantize_e4m3_block128x128_dual(w, q, scale, q_t, scale_t, stream: int | None = None) -> None:
    """Both 128 x 128 block quantisations of a 2-D ``w`` [rows, cols] (fp16 or bf16, contiguous) in one launch: ``q``
    (e4m3 [rows, cols]) with ``scale`` (fp32 [ceil(rows/128), ceil(cols/128)], contiguous), and ``q_t`` = q^T (e4m3
    [cols, rows]) with ``scale_t`` = scale^T (csrc/b200_quant_block_dual.h)."""
    code, rows, cols = _block_dual_input(w)
    _quant_output(q, w.shape, w)
    _quant_output(q_t, (cols, rows), w)
    _fp32_on(scale, w, "scale", (-(-rows // BLOCK), num_k_blocks(cols)))
    _fp32_on(scale_t, w, "scale_t", (num_k_blocks(cols), -(-rows // BLOCK)))
    _contiguous_cuda(scale=scale, scale_t=scale_t)
    fn = quant_block_dual_lib().cuda_l2_b200_quant_block_dual_e4m3_128x128
    _check(fn(code, w.data_ptr(), rows, cols, q.data_ptr(), scale.data_ptr(), q_t.data_ptr(), scale_t.data_ptr(),
              stream), fn)


def quant_block_dual_launch_count() -> int:
    return int(quant_block_dual_lib().cuda_l2_b200_quant_block_dual_launch_count())
