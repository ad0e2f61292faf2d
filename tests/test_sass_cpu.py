"""SASS of the library kernels without a GPU: what the consumer k-loop must not contain."""
import shutil
import subprocess
import sys
from pathlib import Path

import pytest

from conftest import REPO

sys.path.insert(0, str(REPO / "tools"))
import sass_summary  # noqa: E402


def test_no_gpu_scope_fence_in_any_consumer_k_loop(built_libs):
    """A consumer's stage release reports finished wgmma reads and publishes no data, so it needs no GPU-scope fence.
    A `.release.cluster` arrive compiles to MEMBAR.ALL.GPU before the release, on every k-block of every consumer warp
    of every CTA-pair and cluster kernel, right where only one wgmma group is in flight to cover it."""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(built_libs["capi"])], capture_output=True, text=True, check=True).stdout
    kernels = sass_summary.sass_by_kernel(sass)
    assert len(kernels) == 5 * 46
    for name, insns in kernels.items():
        loop = sass_summary.k_loop(insns)
        assert any(op == "WARPGROUP.ARRIVE" for _, op, _ in loop), name
        assert any(op.startswith("SYNCS.ARRIVE") for _, op, _ in loop), name   # the stage release is inside
        assert sass_summary.k_loop_gpu_membars(insns) == 0, name
