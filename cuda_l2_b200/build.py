"""In-tree builds of the native pieces (nvcc cross-compiles sm_90a without a GPU).

Artifacts land in ``cuda_l2_b200/lib/`` (git-ignored build products):

* ``libb200_hgemm.so``  — the C-ABI product library (include/b200_hgemm.h)
* ``libb200_fp8block.so`` — the block-scaled FP8 GEMM (include/b200_fp8_block.h)
* ``libb200_fp8block_1d1d.so`` — the block-scaled FP8 GEMM with 1 x 128 scales on both operands, the weight gradient of
  blockwise FP8 training (csrc/b200_fp8_block_1d1d.h; no public symbol)
* ``libb200_batched.so`` — the batched fp16 / bf16 GEMM (include/b200_batched.h)
* ``libb200_grouped.so`` — the grouped fp16 / bf16 GEMM over contiguous row groups (include/b200_grouped.h)
* ``libb200_grouped_fp8.so`` — the block-scaled FP8 grouped GEMM over contiguous row groups (include/b200_grouped_fp8.h)
* ``libb200_batched_fp8.so`` — the block-scaled FP8 batched GEMM with per-batch row counts (include/b200_batched_fp8.h)
* ``libb200_nn.so``     — the row-major B (NN) fp16 / bf16 kernels, loaded by libb200_hgemm.so on its first call with
  ``B_rowmajor`` (csrc/b200_nn.h; no public symbol)
* ``libb200_grouped_bwd.so`` — the backward of the grouped fp16 / bf16 GEMM: the grouped row-major B (NN) kernels of
  the input gradient and the K-grouped kernels of the weight gradient (csrc/b200_grouped_bwd.h; no public symbol)
* ``libb200_epilogue.so`` — the 2-D fp16 / bf16 / e4m3 GEMM with a fused bias + ReLU / tanh-GELU epilogue
  (csrc/b200_epilogue.h; no public symbol)
* ``libb200_wgrad_accum.so`` — weight gradients added into fp32 main-grad buffers by the GEMM epilogue: the 16-bit
  K-grouped, e4m3 rowwise and e4m3 1 x 128 kernels (csrc/b200_wgrad_accum.h; no public symbol)
* ``libb200_swiglu.so`` — the gate / up projection of a SwiGLU MLP with silu(g) * u fused into the GEMM epilogue, and
  the one-pass SwiGLU backward (csrc/b200_swiglu.h; no public symbol)
* ``libb200_grouped_swiglu.so`` — the gate / up projection of SwiGLU experts over contiguous row groups with
  silu(g) * u fused into the GEMM epilogue, and the SwiGLU backward over the groups' rows (csrc/b200_grouped_swiglu.h;
  no public symbol)
* ``libb200_quant.so``  — the one-pass e4m3 quantisers of FP8 activations: per tensor, rowwise, 1 x 128 blocks and
  SwiGLU + 1 x 128 blocks (csrc/b200_quant.h; no public symbol)
* ``libb200_quant_dual.so`` — the dual-orientation rowwise e4m3 quantiser of FP8 training: x and x^T quantised from
  one tensor (csrc/b200_quant_dual.h; no public symbol)
* ``libb200_quant_block_dual.so`` — the dual-orientation 1 x 128 and 128 x 128 e4m3 quantisers of blockwise FP8
  training: both orientations of a tensor from one read of it (csrc/b200_quant_block_dual.h; no public symbol)
* ``libb200_baselines.so`` — cuBLAS / cuBLASLt comparators behind a C ABI (include/b200_baselines.h)
* ``dev_check``         — standalone bring-up / tuning binary (developer tool)

Every step is skipped when the artifact is newer than all of its inputs.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
REPO = PKG_DIR.parent
CSRC = PKG_DIR / "csrc"
LIB_DIR = PKG_DIR / "lib"

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-std=c++17", "-O3", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fno-gnu-unique"]


def nvcc_path() -> str:
    cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(cand).exists():
        raise RuntimeError("nvcc not found: the HGEMM library cannot be built")
    return cand


def _stale(out: Path, inputs: list[Path]) -> bool:
    if not out.exists():
        return True
    t = out.stat().st_mtime
    return any(p.stat().st_mtime > t for p in inputs if p.exists())


def _run(cmd: list[str], verbose: bool) -> None:
    if verbose:
        print("+", " ".join(cmd), flush=True)
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError(f"build step failed ({r.returncode}): {' '.join(cmd)}")
    if verbose and r.stdout.strip():
        print(r.stdout)
    elif "warning" in r.stdout.lower():
        sys.stderr.write(r.stdout)   # compiler warnings are always shown
    # C7510: ptxas serialised the wgmma pipeline (a function call or a non-inlined boundary inside the MMA loop). The
    # kernels are still correct but lose the overlap of consecutive wgmma groups, so such a build is refused.
    if "C7510" in r.stdout:
        raise RuntimeError(f"ptxas serialised wgmma (warning C7510) in: {' '.join(cmd)}")


def _headers() -> list[Path]:
    return (sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.inc")) + sorted(CSRC.glob("*.h")) +
            sorted((REPO / "include").glob("*.h")))


def _compile_and_link(out: Path, objects: list[tuple[Path, list[str]]], link_flags: list[str], verbose: bool,
                      force: bool) -> Path:
    """Compiles each (source, defines) object in parallel, then links them into the shared library ``out``."""
    LIB_DIR.mkdir(exist_ok=True)
    if force or _stale(out, [src for src, _ in objects] + _headers()):
        objs = [LIB_DIR / f"{out.stem}_{i}.o" for i in range(len(objects))]
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(len(objects)) as pool:
            for f in [pool.submit(_run, [nvcc_path(), *ARCH_FLAGS, *COMMON, *defines, "-c", "-o", str(obj), str(src)],
                                  verbose)
                      for (src, defines), obj in zip(objects, objs)]:
                f.result()
        _run([nvcc_path(), *ARCH_FLAGS, *COMMON, "--shared", "-o", str(out), *map(str, objs), *link_flags], verbose)
        for obj in objs:
            obj.unlink()
    return out


VARIANTS = (0, 1, 2)   # fp16 with fp32 accumulation, fp16 with fp16 accumulation, bf16 (the GemmType index)
BLOCK_VARIANTS = (5, 6)   # block-scaled e4m3 with fp16 / bf16 output (the GemmType index)
BWD_VARIANTS = (0, 2)     # the grouped backward: fp16 and bf16, both with fp32 accumulation (the GemmType index)
EPILOGUE_VARIANTS = (0, 2, 3, 4)   # bias + activation: fp16, bf16, e4m3 to fp16, e4m3 to bf16 (the GemmType index)
BLOCK_1D1D_VARIANTS = (7, 8)      # 1 x 128 scales on both operands: e4m3 to fp16 / bf16 (the GemmType index)
# fp32 weight-gradient accumulation: K-grouped fp16 and bf16, e4m3 rowwise, e4m3 1 x 128 (the GemmType index; one
# object per e4m3 family, whose fp32 output does not depend on the 16-bit flavour)
WGRAD_ACCUM_VARIANTS = (0, 2, 3, 7)
SWIGLU_VARIANTS = (0, 2)   # the SwiGLU epilogue: fp16 and bf16, both with fp32 accumulation (the GemmType index)
GROUPED_SWIGLU_VARIANTS = (0, 2)   # the grouped SwiGLU epilogue: the same two variants


def _per_variant(source: str, variants: tuple[int, ...]) -> list[tuple[Path, list[str]]]:
    """One object of ``source`` per variant: each instantiates only that variant's kernels."""
    return [(CSRC / source, [f"-DB200_VARIANT={v}"]) for v in variants]


# Every library: key -> (file name, its (source, defines) objects, extra link flags). The libraries other than
# libb200_hgemm.so hold kernels of their own, so that the device code of the others stays as it is. libb200_hgemm.so
# compiles its 16-bit kernels (b200_hgemm_capi.cu) and its e4m3 ones (b200_fp8_capi.cu) in parallel; the tile-list
# libraries compile one source per variant (31 kernels each for the 16-bit variants, 17 for the block-scaled ones), and
# so does libb200_nn.so (43 kernels per 16-bit variant), libb200_grouped_bwd.so (56 per variant: 28 configurations
# times two kinds), libb200_epilogue.so (46 per variant: libb200_hgemm.so's (configuration, K-mode) pairs),
# libb200_fp8block_1d1d.so (19 per output type, libb200_fp8block.so's configurations and K-modes) and
# libb200_wgrad_accum.so (28 K-grouped kernels per 16-bit variant, 46 rowwise e4m3 ones and 19 1 x 128 ones) and
# libb200_swiglu.so (18 gated kernels per variant, the BN = 128 and 256 configurations on the plain schedule, and the
# backward kernel of each variant in the object of variant 0), and so does libb200_grouped_swiglu.so (the same 18
# configurations per variant over row groups, and its two backward kernels in the object of variant 0).
LIBRARIES = {
    "capi": ("libb200_hgemm.so", [(CSRC / "b200_hgemm_capi.cu", []), (CSRC / "b200_fp8_capi.cu", [])], []),
    "fp8block": ("libb200_fp8block.so", [(CSRC / "b200_fp8_block_capi.cu", [])], []),
    "fp8block_1d1d": ("libb200_fp8block_1d1d.so", _per_variant("b200_fp8_block_1d1d.cu", BLOCK_1D1D_VARIANTS), []),
    "batched": ("libb200_batched.so", _per_variant("b200_batched_capi.cu", VARIANTS), []),
    "grouped": ("libb200_grouped.so", _per_variant("b200_grouped_capi.cu", VARIANTS), []),
    "grouped_fp8": ("libb200_grouped_fp8.so", _per_variant("b200_grouped_fp8_capi.cu", BLOCK_VARIANTS), []),
    "batched_fp8": ("libb200_batched_fp8.so", _per_variant("b200_batched_fp8_capi.cu", BLOCK_VARIANTS), []),
    "nn": ("libb200_nn.so", _per_variant("b200_nn.cu", VARIANTS), []),
    "grouped_bwd": ("libb200_grouped_bwd.so", _per_variant("b200_grouped_bwd.cu", BWD_VARIANTS), []),
    "epilogue": ("libb200_epilogue.so", _per_variant("b200_epilogue.cu", EPILOGUE_VARIANTS), []),
    "wgrad_accum": ("libb200_wgrad_accum.so", _per_variant("b200_wgrad_accum.cu", WGRAD_ACCUM_VARIANTS), []),
    "swiglu": ("libb200_swiglu.so", _per_variant("b200_swiglu.cu", SWIGLU_VARIANTS), []),
    "grouped_swiglu": ("libb200_grouped_swiglu.so", _per_variant("b200_grouped_swiglu.cu", GROUPED_SWIGLU_VARIANTS), []),
    "quant": ("libb200_quant.so", [(CSRC / "b200_quant.cu", [])], []),
    "quant_dual": ("libb200_quant_dual.so", [(CSRC / "b200_quant_dual.cu", [])], []),
    "quant_block_dual": ("libb200_quant_block_dual.so", [(CSRC / "b200_quant_block_dual.cu", [])], []),
    "baselines": ("libb200_baselines.so", [(CSRC / "b200_baselines_capi.cu", [])], ["-lcublas", "-lcublasLt"]),
}


def build_library(key: str, verbose: bool = False, force: bool = False) -> Path:
    name, objects, link_flags = LIBRARIES[key]
    return _compile_and_link(LIB_DIR / name, objects, link_flags, verbose, force)


def build_dev_check(verbose: bool = False, force: bool = False) -> Path:
    lib = build_library("capi", verbose, force)
    build_library("baselines", verbose, force)
    out = LIB_DIR / "dev_check"
    src = CSRC / "dev_check.cu"
    if force or _stale(out, [src, lib] + _headers()):
        _run([nvcc_path(), *ARCH_FLAGS, "-std=c++17", "-O3", "-lineinfo", "-o", str(out), str(src),
              f"-L{LIB_DIR}", "-lb200_hgemm", "-lb200_baselines", "-lcublas", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN"], verbose)
    return out


def build_all(verbose: bool = False, force: bool = False) -> dict[str, Path]:
    """Every library of LIBRARIES, compiled next to each other, then dev_check."""
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(len(LIBRARIES)) as pool:
        futures = {key: pool.submit(build_library, key, verbose, force) for key in LIBRARIES}
        out = {key: f.result() for key, f in futures.items()}
    out["dev_check"] = build_dev_check(verbose, force)
    return out


if __name__ == "__main__":
    for k, v in build_all(verbose=True, force="--force" in sys.argv).items():
        print(f"{k}: {v}")
