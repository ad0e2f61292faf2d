"""Row-major B (NN) GEMM without a GPU: the drop-in entry points' statuses with B_rowmajor, the unchanged C ABI, the
hgemm_nn operator's schema, meta shapes and CPU refusal, and the SASS and resource usage of libb200_nn.so's kernels."""
import re
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import pytest
import torch

from conftest import REPO
from cuda_l2_b200 import build, capi, ops

sys.path.insert(0, str(REPO / "tools"))
import sass_summary  # noqa: E402

ENTRY_POINTS = ("b200_hgemm_f32acc", "b200_hgemm_f16acc", "b200_bgemm_f32acc")
KNULL, KBADSHAPE, KBADALIGN, KNONN = -5, -1, -2, -11
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def libs(built_libs):
    return built_libs


@pytest.mark.parametrize("entry", ENTRY_POINTS)
def test_statuses_come_back_before_any_cuda_call(libs, entry):
    """Fake, never dereferenced device addresses: every refusal happens in the argument checks."""
    fn = getattr(capi.hgemm_lib(), entry)
    a, b, c = 0x10000, 0x20000, 0x30000
    assert fn(a, None, None, c, 64, 64, 64, None) == KNULL            # both B pointers NULL
    assert fn(a, b + 8, None, c, 64, 64, 64, None) == KBADALIGN       # misaligned B_rowmajor
    assert fn(a, b, None, c, 64, 64, 60, None) == KBADALIGN           # K % 8
    assert fn(a, b, None, c, 64, 60, 64, None) == KBADALIGN           # N % 8
    for m, n, k in ((0, 64, 64), (64, 0, 64), (64, 64, 0), (-1, 64, 64)):
        assert fn(a, b, None, c, m, n, k, None) == KBADSHAPE
    assert fn(None, b, None, c, 64, 64, 64, None) == KNULL
    assert fn(a, b, None, None, 64, 64, 64, None) == KNULL


def test_missing_nn_library_has_a_status_text():
    assert "libb200_nn.so" in capi.strerror(KNONN)


def test_c_abi_is_unchanged_and_the_nn_library_exports_nothing_public(libs):
    # the headers and the table still hold the same 57 prototypes (test_abi_table_cpu.py pins the count); no header
    # declares the NN library's entry point
    assert not any("nn_run_config" in h.read_text() for h in (REPO / "include").glob("*.h"))
    assert "libb200_nn.so" not in capi.ABI
    out = subprocess.run(["nm", "-D", "--defined-only", str(libs["nn"])], capture_output=True, text=True,
                         check=True).stdout
    names = [line.split()[-1] for line in out.splitlines() if line.strip()]
    assert not [s for s in names if s.startswith("b200_")]
    assert "cuda_l2_b200_nn_run_config" in names


def test_operator_schema_and_meta_shapes():
    schema = str(torch.ops.cuda_l2_b200.hgemm_nn.default._schema)
    assert schema == 'cuda_l2_b200::hgemm_nn(Tensor a, Tensor b, str acc="fp32") -> Tensor'
    for dtype, acc in ((torch.float16, "fp32"), (torch.float16, "fp16"), (torch.bfloat16, "fp32")):
        a = torch.empty((77, 136), dtype=dtype, device="meta")
        b = torch.empty((136, 520), dtype=dtype, device="meta")
        out = ops.hgemm_nn(a, b, acc)
        assert out.shape == (77, 520) and out.dtype == dtype and out.device.type == "meta"
    for a, b, acc in [((64, 128), (64, 128), "fp32"),   # K differs ([K, N] expected)
                      ((64, 128), (128, 60), "fp32"),   # N % 8
                      ((64, 60), (60, 64), "fp32")]:    # K % 8
        with pytest.raises(capi.B200HgemmError):
            ops.hgemm_nn(torch.empty(a, dtype=torch.half, device="meta"), torch.empty(b, dtype=torch.half, device="meta"),
                         acc)
    with pytest.raises(capi.B200HgemmError):   # bf16 accumulates in fp32 only
        ops.hgemm_nn(torch.empty((8, 8), dtype=torch.bfloat16, device="meta"),
                     torch.empty((8, 8), dtype=torch.bfloat16, device="meta"), "fp16")
    with pytest.raises(capi.B200HgemmError):   # no e4m3 NN kernel
        ops.hgemm_nn(torch.empty((8, 16), dtype=torch.float8_e4m3fn, device="meta"),
                     torch.empty((16, 8), dtype=torch.float8_e4m3fn, device="meta"))


def test_cpu_path_raises():
    with pytest.raises(capi.B200HgemmError, match="no CPU implementation"):
        ops.hgemm_nn(torch.ones((8, 8), dtype=torch.half), torch.ones((8, 8), dtype=torch.half))


def _configs_with_nn_kernel_and_modes():
    """(config id, number of K-modes its kernels carry) for every configuration with an NN kernel (BN % 64 == 0)."""
    out = []
    for c in capi.configs():
        if c["bn"] % 64:
            continue
        stream_k = c["cluster_m"] * c["cluster_n"] == 1 and c["m_rep"] == 1
        out.append((c["id"], 1 + stream_k + 2 * (stream_k and c["cta_group"] == 1)))
    return out


def test_sass_of_every_nn_kernel(libs):
    if not Path(CUOBJDUMP).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([CUOBJDUMP, "-sass", str(libs["nn"])], capture_output=True, text=True, check=True).stdout
    kernels = sass_summary.sass_by_kernel(sass)
    assert len(kernels) == 3 * sum(modes for _, modes in _configs_with_nn_kernel_and_modes()) == 129
    for name, insns in kernels.items():
        assert "RowMajorB" in name, name
        loop = sass_summary.k_loop(insns)
        assert any(op == "WARPGROUP.ARRIVE" for _, op, _ in loop), name
        assert any(op.startswith("SYNCS.ARRIVE") for _, op, _ in loop), name   # the stage release
        assert sass_summary.k_loop_gpu_membars(insns) == 0, name


PTXAS = re.compile(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                   r"(\d+) bytes spill loads", re.S)


def _ptxas_spills(source: Path, defines: list[str], tmp: Path) -> tuple[dict, str]:
    """{demangled kernel: spill store bytes} of one object compiled with -Xptxas -v, and the compiler's output."""
    r = subprocess.run([build.nvcc_path(), *build.ARCH_FLAGS, *build.COMMON, "-Xptxas", "-v", *defines, "-c", "-o",
                        str(tmp / f"{source.stem}_{len(defines)}_{abs(hash(tuple(defines)))}.o"), str(source)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    text = r.stdout + r.stderr
    out = {}
    for block in text.split("ptxas info    : Compiling entry function ")[1:]:
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        name = block.split("'")[1]
        out[name] = int(m.group(2)) if m else 0
    return out, text


def _demangle(names) -> dict:
    names = list(names)
    r = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True, check=True)
    return dict(zip(names, r.stdout.splitlines()))


def test_no_nn_kernel_spills_more_than_its_tn_kernel(tmp_path):
    """-Xptxas -v of libb200_nn.so's objects and of the 16-bit TN object of libb200_hgemm.so: an NN kernel may spill
    no more than the TN kernel of the same configuration, mode and type, and no object triggers C7510."""
    csrc = build.CSRC
    jobs = [(csrc / "b200_nn.cu", [f"-DB200_VARIANT={v}"]) for v in build.VARIANTS] + [(csrc / "b200_hgemm_capi.cu", [])]
    with ThreadPoolExecutor(len(jobs)) as pool:
        results = list(pool.map(lambda j: _ptxas_spills(*j, tmp_path), jobs))
    for _, text in results:
        assert "C7510" not in text
    nn, tn = {}, {}
    for spills, _ in results[:-1]:
        nn.update(spills)
    tn.update(results[-1][0])
    nn_names, tn_names = _demangle(nn), _demangle(tn)
    tn_by_name = {tn_names[k]: v for k, v in tn.items()}
    assert len(nn) == 129
    for mangled, spill in nn.items():
        name = nn_names[mangled]
        twin = re.sub(r"b200::RowMajorB<(b200::Config<[^>]*>) ?>", r"\1", name)
        assert twin != name and twin in tn_by_name, name
        assert spill <= tn_by_name[twin], (name, spill, tn_by_name[twin])
