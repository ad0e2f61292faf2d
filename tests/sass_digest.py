"""Digests of the device code of the GEMM libraries: per library, a SHA-256 over its kernels' SASS (`cuobjdump -sass`)
and over their resource lines (`cuobjdump -res-usage`: registers, stack, shared memory), each kernel's text taken
separately and sorted by name, so the link order of the objects does not count. The object identifier lines, which name
the build directory, are left out.

`python tests/sass_digest.py` (after a build) rewrites tests/golden/gemm_sass_digest.json; run it only when a change is
meant to alter those kernels."""
from __future__ import annotations

import hashlib
import json
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
GOLDEN = REPO / "tests" / "golden" / "gemm_sass_digest.json"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
# every library of cuda_l2_b200/build.py that holds GEMM kernels (the quantisers of libb200_quant.so are not among them)
GEMM_LIBRARIES = ("capi", "fp8block", "fp8block_1d1d", "batched", "grouped", "grouped_fp8", "batched_fp8", "nn",
                  "grouped_bwd", "epilogue", "wgrad_accum", "swiglu", "grouped_swiglu", "baselines")


def _digest(text: str, marker: str) -> str:
    """SHA-256 of the sections of a cuobjdump listing that start at lines containing ``marker``, sorted."""
    sections, cur = [], []
    for line in text.splitlines():
        if line.strip().startswith("identifier"):
            continue
        if marker in line and cur:
            sections.append("\n".join(cur))
            cur = []
        cur.append(line)
    if cur:
        sections.append("\n".join(cur))
    h = hashlib.sha256()
    for s in sorted(sections):
        h.update(s.encode())
        h.update(b"\0")
    return h.hexdigest()


def library_digest(path: Path) -> dict:
    sass = subprocess.run([CUOBJDUMP, "-sass", str(path)], capture_output=True, text=True, check=True).stdout
    res = subprocess.run([CUOBJDUMP, "-res-usage", str(path)], capture_output=True, text=True, check=True).stdout
    return {"sass": _digest(sass, "Function :"), "resources": _digest(res, "Function ")}


def digests(libs: dict) -> dict:
    """{library file name: {"sass": ..., "resources": ...}} of the GEMM libraries among the built ``libs``
    (build.build_all()'s answer)."""
    with ThreadPoolExecutor(len(GEMM_LIBRARIES)) as pool:
        out = dict(zip(GEMM_LIBRARIES, pool.map(lambda key: library_digest(libs[key]), GEMM_LIBRARIES)))
    return {libs[key].name: out[key] for key in GEMM_LIBRARIES}


if __name__ == "__main__":
    sys.path.insert(0, str(REPO))
    from cuda_l2_b200 import build

    GOLDEN.write_text(json.dumps(digests(build.build_all()), indent=1, sort_keys=True) + "\n")
    print(f"wrote {GOLDEN}")
