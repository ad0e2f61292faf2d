"""JIT-build glue of the harness — same public surface as the reference's ``tools/utils.py``
(``extract_bm_bk_bn``, ``get_build_sources``, ``get_build_cuda_cflags``, ``build_from_sources``,
``as_col_major``; reference tools/utils.py:8-115), written for ``--device_type b200`` (the H100 kernel family's name in the harness).

Differences that matter here:

* the five sources of one ``hgemm_lib`` build are torch-free ``.cu`` files plus ONE ``.cc`` that holds every
  ``torch::Tensor`` wrapper, so a per-shape rebuild is a few seconds of nvcc instead of minutes;
* ``CUTLASS_DIR`` is not needed (the b200 kernels are hand-written PTX, not CuTe templates);
* the arch flag is pinned to ``-gencode arch=compute_90a,code=sm_90a`` (plain ``sm_90`` rejects wgmma and setmaxnreg);
* nothing here touches the GPU, so ``compile.py`` can pre-build on a machine without one.
"""
from __future__ import annotations

import os
import re
from pathlib import Path

import torch

PROJECT_DIR = Path(__file__).resolve().parent.parent

DEVICE_TYPES = ("b200",)
ACC_DIRS = {"fp16": "F16F16F16F16", "fp32": "F32F16F16F32"}
SM90A_GENCODE = "-gencode=arch=compute_90a,code=sm_90a"

_TILE_TOKEN = re.compile(r"(BM|BN|BK)=Int<(\d+)>")


def extract_bm_bk_bn(text: str) -> tuple[int, int, int]:
    """Tile sizes a kernel source declares as ``BM = Int<..>`` / ``BK`` / ``BN`` (reference tools/utils.py:8-36).

    The harness pads operands up to multiples of these. All three must be present, otherwise
    ``(-1, -1, -1)`` (= no padding). The b200 kernels declare none on purpose: TMA handles the edges.
    When a name is declared several times the last declaration wins, as in the reference.
    """
    found = {"BM": -1, "BK": -1, "BN": -1}
    for line in text.splitlines():
        hit = _TILE_TOKEN.search(line.replace(" ", ""))   # first declaration on a line, blanks ignored
        if hit:
            found[hit.group(1)] = int(hit.group(2))
    if min(found.values()) > 0:
        return found["BM"], found["BK"], found["BN"]
    return -1, -1, -1


def acc_dir_name(acc_precise: str) -> str:
    try:
        return ACC_DIRS[acc_precise]
    except KeyError:
        raise ValueError(f"acc_precise must be 'fp16' or 'fp32', got {acc_precise!r}") from None


def kernel_source_path(mnk: str, acc_precise: str, device_type: str) -> str:
    return f"kernels/{device_type}_{acc_dir_name(acc_precise)}/{mnk}.cu"


def get_build_sources(mnk, acc_precise, device_type):
    """The five translation units of one ``hgemm_lib`` (reference tools/utils.py:39-54), repo-relative."""
    acc_dir_name(acc_precise)
    return [
        f"cublas/{acc_precise}/hgemm_cublas.cu",
        f"cublas/{acc_precise}/hgemm_cublaslt_heuristic.cu",
        f"cublas/{acc_precise}/hgemm_cublaslt_auto_tuning.cu",
        kernel_source_path(mnk, acc_precise, device_type),
        f"pybind/hgemm_{device_type}_{acc_precise}.cc",
    ]


def get_build_cuda_cflags(build_pkg: bool = False):
    """nvcc flags (reference tools/utils.py:57-92 minus the CUTLASS include paths, plus the sm_90a target)."""
    flags = [
        "-O3",
        "-std=c++17",
        "-lineinfo",
        SM90A_GENCODE,
        "-U__CUDA_NO_HALF_OPERATORS__",
        "-U__CUDA_NO_HALF_CONVERSIONS__",
        "-U__CUDA_NO_HALF2_OPERATORS__",
        "--expt-relaxed-constexpr",
        "--use_fast_math",
        "-Xcompiler=-fno-gnu-unique",   # template statics stay private to this .so (libb200_hgemm.so has its own copies)
        f"-I{PROJECT_DIR}",
        f"-I{PROJECT_DIR}/pybind",
    ]
    flags += ["--ptxas-options=-v", "--ptxas-options=-O3"] if build_pkg else ["-diag-suppress=177", "-Xptxas=-v"]
    cutlass_dir = os.environ.get("CUTLASS_DIR")  # optional: only reference (non-b200) kernels need it
    if cutlass_dir:
        flags += [f"-I{cutlass_dir}/include", f"-I{cutlass_dir}/tools/util/include"]
    return flags


def build_from_sources(mnk, acc_precise, device_type, base_dir: str, verbose: bool):
    """JIT-build (or reuse) ``hgemm_lib`` for one shape in ``base_dir`` and import it
    (reference tools/utils.py:95-107). Ninja reuses every object whose source did not change, so a
    persistent ``base_dir`` recompiles only ``kernels/.../<mnk>.cu`` when the shape changes."""
    from torch.utils.cpp_extension import load

    if device_type not in DEVICE_TYPES:
        raise ValueError(f"device_type must be one of {DEVICE_TYPES}, got {device_type!r}")
    sources = [str(PROJECT_DIR / s) for s in get_build_sources(mnk, acc_precise, device_type)]
    missing = [s for s in sources if not os.path.exists(s)]
    if missing:
        raise FileNotFoundError(f"no kernel for this configuration: {missing}")
    if torch.cuda.is_available():
        dev = torch.cuda.current_device()
        print(f"Loading hgemm lib on device: {torch.cuda.get_device_name(dev)} :: "
              f"{torch.cuda.get_device_capability(dev)} :: sm_90a")
    os.makedirs(base_dir, exist_ok=True)
    # torch appends its own -gencode flags from TORCH_CUDA_ARCH_LIST; make that exactly sm_90a too
    prev = os.environ.get("TORCH_CUDA_ARCH_LIST")
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    try:
        return load(
            name="hgemm_lib",
            sources=sources,
            extra_cuda_cflags=get_build_cuda_cflags(),
            extra_cflags=["-std=c++17", "-O2", "-fno-gnu-unique"],
            extra_ldflags=["-lcublas", "-lcublasLt"],
            verbose=verbose,
            build_directory=base_dir,
        )
    finally:
        if prev is None:
            os.environ.pop("TORCH_CUDA_ARCH_LIST", None)
        else:
            os.environ["TORCH_CUDA_ARCH_LIST"] = prev


@torch.no_grad()
def as_col_major(x: torch.Tensor):
    """Row-major [K,N] -> a tensor still *labelled* [K,N] whose storage is the transpose [N,K], contiguous
    (reference tools/utils.py:110-115). Kernels read it as the K-major B operand."""
    return x.t().reshape(x.shape).contiguous()
