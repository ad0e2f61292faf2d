import sys
from pathlib import Path

import numpy as np
import pytest

REPO = Path(__file__).resolve().parent.parent
if str(REPO) not in sys.path:
    sys.path.insert(0, str(REPO))
GOLDEN = REPO / "tests" / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine with one)")


def load_zero_one_cases():
    z = np.load(GOLDEN / "zero_one_cases.npz")
    cases = []
    i = 0
    while f"meta{i}" in z:
        m, n, k, levels, seed = (int(x) for x in z[f"meta{i}"])
        a = np.unpackbits(z[f"a{i}"])[: m * k].reshape(m, k).astype(np.float16)
        b = np.unpackbits(z[f"b{i}"])[: k * n].reshape(k, n).astype(np.float16)
        cases.append(dict(m=m, n=n, k=k, levels=levels, seed=seed, a=a, b=b, truth=z[f"truth{i}"]))
        i += 1
    return cases


def load_randn_cases():
    z = np.load(GOLDEN / "randn_cases.npz")
    cases = []
    i = 0
    while f"meta{i}" in z:
        m, n, k, seed = (int(x) for x in z[f"meta{i}"])
        cases.append(dict(m=m, n=n, k=k, seed=seed, a=z[f"a{i}"], b=z[f"b{i}"], truth=z[f"truth{i}"]))
        i += 1
    return cases


def load_bf16_cases():
    """bf16 fixtures: operands and truth as uint16 bit patterns; kind 0 = 0/1, 1 = small integers (both exact), 2 = randn."""
    z = np.load(GOLDEN / "bf16_cases.npz")
    cases = []
    i = 0
    while f"meta{i}" in z:
        m, n, k, kind, seed = (int(x) for x in z[f"meta{i}"])
        cases.append(dict(m=m, n=n, k=k, kind=("01", "int", "randn")[kind], seed=seed, a=z[f"a{i}"], b=z[f"b{i}"], truth=z[f"truth{i}"]))
        i += 1
    return cases


@pytest.fixture(scope="session")
def bf16_cases():
    return load_bf16_cases()


@pytest.fixture(scope="session")
def zero_one_cases():
    return load_zero_one_cases()


@pytest.fixture(scope="session")
def randn_cases():
    return load_randn_cases()


@pytest.fixture(scope="session")
def built_libs():
    """The C-ABI libraries, built in-tree if they are not there yet (nvcc cross-compiles without a GPU)."""
    from cuda_l2_b200 import build

    return build.build_all()
