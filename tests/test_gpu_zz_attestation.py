"""The reference's defense.py properties on the real kernel (SURVEY §8(f) item 2). Runs after the parity tests: it is
the newest GPU test."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_kernel_passes_the_timing_integrity_attestation():
    """The five defense.py properties on the real kernel: its work is on the stream the harness times."""
    from cuda_l2_b200 import capi
    from cuda_l2_b200.harness.attestation import attest
    from tools.utils import as_col_major

    def kernel(a, b, b_col_major, c):
        capi.hgemm(a, b_col_major, c, "fp32")
    m, n, k = 8192, 8192, 8192      # ~0.85 ms of kernel: the host-sync latency inside the fenced measurement is a few percent of it
    a = torch.randn((m, k), device="cuda").half()
    b = torch.randn((k, n), device="cuda").half()
    v = attest(kernel, a, b, as_col_major(b), torch.empty((m, n), dtype=torch.half, device="cuda"))
    assert v.passed, v.checks
