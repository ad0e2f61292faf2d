"""The grouped backward (libb200_grouped_bwd.so) without a GPU: argument statuses, the unchanged public ABI, the
operators' schemas, meta shapes and CPU refusal, the K-grouped schedule view, and the SASS and resource usage of the
library's kernels."""
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

KNULL, KBADSHAPE, KBADALIGN, KBADCONFIG = -5, -1, -2, -6
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
NN_CONFIGS = [c for c in range(31) if c not in (12, 13, 14)]
A, B, C, O = 0x10000, 0x20000, 0x30000, 0x40000   # fake, never dereferenced device addresses


@pytest.fixture(scope="module")
def libs(built_libs):
    return built_libs


@pytest.mark.parametrize("variant", [0, 2])
def test_statuses_come_back_before_any_cuda_call(libs, variant):
    lib = capi.grouped_bwd_lib()
    nn, wg = lib.cuda_l2_b200_grouped_bwd_nn, lib.cuda_l2_b200_grouped_bwd_wgrad
    for cfg in (-1, 1):
        # grouped NN: A [T, K], B [G, K, N], C [T, N]
        assert nn(variant, cfg, None, B, C, O, 2, 64, 64, 64, 0, 0, None) == KNULL
        assert nn(variant, cfg, A, B, C, None, 2, 64, 64, 64, 0, 0, None) == KNULL
        assert nn(variant, cfg, A, B + 8, C, O, 2, 64, 64, 64, 0, 0, None) == KBADALIGN
        assert nn(variant, cfg, A, B, C, O + 2, 2, 64, 64, 64, 0, 0, None) == KBADALIGN
        assert nn(variant, cfg, A, B, C, O, 2, 64, 60, 64, 0, 0, None) == KBADALIGN   # N % 8
        assert nn(variant, cfg, A, B, C, O, 2, 64, 64, 60, 0, 0, None) == KBADALIGN   # K % 8
        for g, t, n, k in ((0, 64, 64, 64), (2, -1, 64, 64), (2, 64, 0, 64), (2, 64, 64, 0)):
            assert nn(variant, cfg, A, B, C, O, g, t, n, k, 0, 0, None) == KBADSHAPE
        # K-grouped: A [T, M], B [T, N], C [G, M, N]
        assert wg(variant, cfg, A, B, None, O, 2, 64, 64, 64, 0, 0, None) == KNULL
        assert wg(variant, cfg, None, B, C, O, 2, 64, 64, 64, 0, 0, None) == KNULL
        assert wg(variant, cfg, A, B, C, None, 2, 64, 64, 64, 0, 0, None) == KNULL
        assert wg(variant, cfg, A + 8, B, C, O, 2, 64, 64, 64, 0, 0, None) == KBADALIGN
        assert wg(variant, cfg, A, B, C, O, 2, 64, 60, 64, 0, 0, None) == KBADALIGN   # M % 8
        assert wg(variant, cfg, A, B, C, O, 2, 64, 64, 60, 0, 0, None) == KBADALIGN   # N % 8
        for g, t, m, n in ((0, 64, 64, 64), (2, -1, 64, 64), (2, 64, 0, 64), (2, 64, 64, 0)):
            assert wg(variant, cfg, A, B, C, O, g, t, m, n, 0, 0, None) == KBADSHAPE
    # the worst-case tile list must fit an int: G dense matrices of M x N tiles
    assert wg(variant, 1, A, B, C, O, 1 << 20, 64, 1 << 16, 1 << 16, 0, 0, None) == KBADSHAPE
    # a configuration without a row-major B kernel (BN = 32), an unknown one
    assert nn(variant, 12, A, B, C, O, 2, 64, 64, 64, 0, 0, None) == KBADCONFIG
    assert wg(variant, 31, A, B, C, O, 2, 64, 64, 64, 0, 0, None) == KBADCONFIG


def test_unknown_variants_are_refused(libs):
    lib = capi.grouped_bwd_lib()
    for v in (1, 3, -1):   # fp16 accumulation has no backward kernel
        assert lib.cuda_l2_b200_grouped_bwd_nn(v, -1, A, B, C, O, 2, 64, 64, 64, 0, 0, None) == KBADCONFIG
        assert lib.cuda_l2_b200_grouped_bwd_wgrad(v, 1, A, B, C, O, 2, 64, 64, 64, 0, 0, None) == KBADCONFIG


def test_no_public_symbol_and_no_header(libs):
    assert not any("grouped_bwd" in h.read_text() for h in (REPO / "include").glob("*.h"))
    assert capi.GROUPED_BWD_LIB not in capi.ABI
    out = subprocess.run(["nm", "-D", "--defined-only", str(libs["grouped_bwd"])], capture_output=True, text=True,
                         check=True).stdout
    names = [line.split()[-1] for line in out.splitlines() if line.strip()]
    assert not [s for s in names if s.startswith("b200_")]
    assert sorted(s for s in names if s.startswith("cuda_l2_b200_")) == sorted(capi.INTERNAL_ABI[capi.GROUPED_BWD_LIB])


def test_selects_map_to_row_major_b_configurations(libs):
    for variant in (0, 2):
        for g, t, n, k in ((8, 8192, 4096, 14336), (64, 16384, 7168, 2048), (4, 100, 64, 64), (1, 1, 8, 8)):
            cfg, _ = capi.grouped_nn_select(variant, g, t, n, k)
            assert cfg in NN_CONFIGS
            cfg, _ = capi.grouped_wgrad_select(variant, g, t, k, n)
            assert cfg in NN_CONFIGS
    cfg, _ = capi.grouped_wgrad_select(2, 4, 0, 64, 64)   # T == 0 is a valid (empty) reduction
    assert cfg in NN_CONFIGS


def test_operator_schemas_and_meta_shapes():
    assert str(torch.ops.cuda_l2_b200.hgemm_grouped_nn.default._schema) == \
        'cuda_l2_b200::hgemm_grouped_nn(Tensor a, Tensor b, Tensor offs, str acc="fp32") -> Tensor'
    assert str(torch.ops.cuda_l2_b200.hgemm_grouped_wgrad.default._schema) == \
        'cuda_l2_b200::hgemm_grouped_wgrad(Tensor a, Tensor b, Tensor offs, str acc="fp32") -> Tensor'
    assert str(torch.ops.cuda_l2_b200.grouped_linear.default._schema) == \
        'cuda_l2_b200::grouped_linear(Tensor x, Tensor w, Tensor offs, str acc="fp32") -> Tensor'

    def meta(shape, dtype=torch.bfloat16):
        return torch.empty(shape, dtype=dtype, device="meta")

    offs = meta((5,), torch.int32)
    for dtype in (torch.float16, torch.bfloat16):
        assert ops.hgemm_grouped_nn(meta((77, 136), dtype), meta((5, 136, 520), dtype), offs).shape == (77, 520)
        assert ops.hgemm_grouped_wgrad(meta((77, 136), dtype), meta((77, 64), dtype), offs).shape == (5, 136, 64)
        y = ops.grouped_linear(meta((77, 520), dtype), meta((5, 136, 520), dtype), offs)
        assert y.shape == (77, 136) and y.dtype == dtype
    bad = [lambda: ops.hgemm_grouped_nn(meta((8, 64)), meta((5, 72, 64)), offs),            # K differs ([G, K, N])
           lambda: ops.hgemm_grouped_nn(meta((8, 64)), meta((5, 64, 60)), offs),            # N % 8
           lambda: ops.hgemm_grouped_nn(meta((8, 64)), meta((4, 64, 64)), offs),            # offs is not [G]
           lambda: ops.hgemm_grouped_wgrad(meta((8, 64)), meta((9, 64)), offs),             # T differs
           lambda: ops.hgemm_grouped_wgrad(meta((8, 60)), meta((8, 64)), offs),             # M % 8
           lambda: ops.hgemm_grouped_wgrad(meta((8, 64)), meta((8, 64)), meta((5,), torch.int64)),
           lambda: ops.hgemm_grouped_wgrad(meta((8, 64), torch.float16), meta((8, 64), torch.float16), offs, "fp16"),
           lambda: ops.grouped_linear(meta((8, 64), torch.float16), meta((5, 64, 64), torch.float16), offs, "fp16")]
    for call in bad:
        with pytest.raises(capi.B200HgemmError):
            call()


def test_cpu_paths_raise():
    a, offs = torch.ones((8, 8), dtype=torch.half), torch.tensor([8], dtype=torch.int32)
    for call in (lambda: ops.hgemm_grouped_nn(a, torch.ones((1, 8, 8), dtype=torch.half), offs),
                 lambda: ops.hgemm_grouped_wgrad(a, a, offs),
                 lambda: ops.grouped_linear(a, torch.ones((1, 8, 8), dtype=torch.half), offs),
                 lambda: ops.B200GroupedLinear.from_weights(torch.ones((1, 8, 8), dtype=torch.half))(a, offs)):
        with pytest.raises(capi.B200HgemmError, match="no CPU implementation"):
            call()


def test_module_shares_the_weight_storage():
    w = torch.nn.Parameter(torch.zeros((3, 16, 8), dtype=torch.bfloat16))
    layer = ops.B200GroupedLinear.from_weights(w)
    assert layer.weight is w and (layer.num_groups, layer.in_features, layer.out_features) == (3, 8, 16)
    t = torch.zeros((3, 16, 8), dtype=torch.float16)
    assert ops.B200GroupedLinear.from_weights(t).weight.data_ptr() == t.data_ptr()
    with pytest.raises(capi.B200HgemmError):
        ops.B200GroupedLinear.from_weights(torch.zeros((3, 16, 12), dtype=torch.float16))   # K % 8


def clamped_groups(offs, t):
    out, s = [], 0
    for o in offs:
        e = min(max(o, s), t)
        out.append((s, e))
        s = e
    return out


@pytest.mark.parametrize("offs", [[37, 37, 137, 300, 250],     # an empty group, a decreasing offset
                                  [-4, 100, 90, 700, 1000],     # negative, decreasing, past T
                                  [0, 0, 0],                    # every group empty
                                  [300]])                       # one group of all rows
@pytest.mark.parametrize("config_id", [1, 4, 9, 27, 29])
def test_schedule_view_clamps_offsets_and_counts_k_blocks(libs, offs, config_id):
    t, m, n = 300, 136, 264
    cfg = capi.configs()[config_id]
    block_m = 128 * cfg["m_rep"] * cfg["cta_group"] * cfg["cluster_m"]
    block_n = cfg["bn"] * cfg["cluster_n"]
    per = -(-m // block_m) * -(-n // block_n)
    sched = capi.grouped_wgrad_schedule(config_id, t, m, n, offs, num_sms=132)
    tiles = [u for w in sched["units"] for u in w]
    assert len(tiles) == len(offs) * per and sched["workers"] == min(132 // (cfg["cta_group"] * cfg["cluster_m"] *
                                                                             cfg["cluster_n"]), len(offs) * per)
    seen = set()
    groups = clamped_groups(offs, t)
    for g, mb, nb, kbs in tiles:
        s, e = groups[g]
        assert kbs == -(-(e - s) // 64), (g, kbs)
        seen.add((g, mb, nb))
    assert len(seen) == len(tiles)   # every tile once
    small = capi.grouped_wgrad_schedule(config_id, t, m, n, offs, num_sms=2 * cfg["cta_group"] * cfg["cluster_m"] *
                                        cfg["cluster_n"])
    assert small["workers"] == min(2, len(tiles)) and sorted(u for w in small["units"] for u in w) == sorted(tiles)


def test_kernel_count_and_the_k_loop_of_every_kernel(libs):
    if not Path(CUOBJDUMP).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([CUOBJDUMP, "-sass", str(libs["grouped_bwd"])], capture_output=True, text=True,
                          check=True).stdout
    kernels = sass_summary.sass_by_kernel(sass)
    assert len(kernels) == 2 * 28 * 2 == 112
    kinds = {"GroupedK": 0, "Grouped": 0}
    for name, insns in kernels.items():
        assert "RowMajorB" in name, name
        kinds["GroupedK" if "GroupedK" in name else "Grouped"] += 1
        loop = sass_summary.k_loop(insns)
        assert any(op == "WARPGROUP.ARRIVE" for _, op, _ in loop), name
        assert any(op.startswith("SYNCS.ARRIVE") for _, op, _ in loop), name   # the stage release
        assert sass_summary.k_loop_gpu_membars(insns) == 0, name
    assert kinds == {"GroupedK": 56, "Grouped": 56}


def _ptxas_spills(source: Path, defines: list[str], tmp: Path) -> tuple[dict, str]:
    """{kernel: spill store bytes} of one object compiled with -Xptxas -v, and the compiler's output."""
    r = subprocess.run([build.nvcc_path(), *build.ARCH_FLAGS, *build.COMMON, "-Xptxas", "-v", *defines, "-c", "-o",
                        str(tmp / f"{source.stem}_{'_'.join(defines)}.o"), str(source)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    text = r.stdout + r.stderr
    out = {}
    for block in text.split("ptxas info    : Compiling entry function ")[1:]:
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        out[block.split("'")[1]] = int(m.group(2)) if m else 0
    return out, text


def _demangle(names) -> dict:
    names = list(names)
    r = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True, check=True)
    return dict(zip(names, r.stdout.splitlines()))


def test_no_kernel_spills_more_than_its_nn_twin(tmp_path):
    """-Xptxas -v of libb200_grouped_bwd.so's objects and of libb200_nn.so's: a backward kernel may spill no more than
    the plain-schedule NN kernel of the same configuration and type, and no object triggers C7510."""
    csrc = build.CSRC
    jobs = [(csrc / "b200_grouped_bwd.cu", [f"-DB200_VARIANT={v}"]) for v in build.BWD_VARIANTS] + \
           [(csrc / "b200_nn.cu", [f"-DB200_VARIANT={v}"]) for v in build.BWD_VARIANTS]
    with ThreadPoolExecutor(len(jobs)) as pool:
        results = list(pool.map(lambda j: _ptxas_spills(*j, tmp_path), jobs))
    for _, text in results:
        assert "C7510" not in text
    bwd, nn = {}, {}
    for spills, _ in results[:2]:
        bwd.update(spills)
    for spills, _ in results[2:]:
        nn.update(spills)
    bwd_names, nn_names = _demangle(bwd), _demangle(nn)
    nn_by_name = {nn_names[k]: v for k, v in nn.items()}
    assert len(bwd) == 112
    for mangled, spill in bwd.items():
        name = bwd_names[mangled]
        twin = re.sub(r"b200::Grouped(K)?<(b200::RowMajorB<b200::Config<[^>]*> ?>) ?>", r"\2", name)
        assert twin != name and twin in nn_by_name, name
        assert spill <= nn_by_name[twin], (name, spill, nn_by_name[twin])
