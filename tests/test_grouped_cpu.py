"""Grouped fp16 / bf16 GEMM over contiguous row groups without a GPU: the C ABI of libb200_grouped.so (exports,
statuses before any CUDA call, the dispatcher), the operator's schema and shape inference, the host view of the
schedule the kernels walk, and the SASS of the grouped kernels."""
import ctypes
import random
import re
import shutil
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from conftest import REPO
from cuda_l2_b200 import capi

DECL = re.compile(r"^\s*(?:const\s+)?(?:unsigned\s+long\s+long|int|void|char\s*\*|const\s+char\s*\*)\s*\*?\s*(b200_\w+)\s*\(", re.M)
NUM_CONFIGS = 31


def test_header_binding_and_library_exports_agree(built_libs):
    declared = sorted(set(DECL.findall((REPO / "include" / "b200_grouped.h").read_text())))
    assert declared == sorted(capi.exported_symbols()["libb200_grouped.so"])
    assert built_libs["grouped"].name == "libb200_grouped.so"
    lib = ctypes.CDLL(str(built_libs["grouped"]))
    for sym in declared:
        assert hasattr(lib, sym), sym
    for other in (capi.hgemm_lib(), capi.batched_lib()):   # neither of the other libraries carries them
        assert not any(hasattr(other, sym) for sym in declared)


def _aligned(buf) -> int:
    return (ctypes.addressof(buf) + 15) & ~15


def test_argument_validation_happens_before_any_cuda_call(built_libs):
    lib = capi.grouped_lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = _aligned(buf)
    offs = p + 4096
    g, r = lib.b200_grouped_gemm, lib.b200_grouped_gemm_run_config
    for v in (0, 1, 2):
        assert g(v, None, p, p, offs, 4, 64, 64, 64, None) == -5                       # null operands
        assert g(v, p, None, p, offs, 4, 64, 64, 64, None) == -5
        assert g(v, p, p, None, offs, 4, 64, 64, 64, None) == -5
        assert g(v, p, p, p, None, 4, 64, 64, 64, None) == -5                          # null offs
        assert g(v, p, p, p, offs, 0, 64, 64, 64, None) == -1                          # G <= 0
        assert g(v, p, p, p, offs, -3, 64, 64, 64, None) == -1
        assert g(v, p, p, p, offs, 4, -1, 64, 64, None) == -1                          # T < 0
        assert g(v, p, p, p, offs, 4, 64, 0, 64, None) == -1                           # N, K <= 0
        assert g(v, p, p, p, offs, 4, 64, 64, 0, None) == -1
        assert g(v, p, p, p, offs, 4, 64, 64, 60, None) == -2                          # K % 8
        assert g(v, p, p, p, offs, 4, 64, 60, 64, None) == -2                          # N % 8
        assert g(v, p + 8, p, p, offs, 4, 64, 64, 64, None) == -2                      # 16-byte A, Bt, C
        assert g(v, p, p + 8, p, offs, 4, 64, 64, 64, None) == -2
        assert g(v, p, p, p + 8, offs, 4, 64, 64, 64, None) == -2
        assert g(v, p, p, p, offs + 2, 4, 64, 64, 64, None) == -2                      # offs: 4-byte aligned
        for cfg in range(NUM_CONFIGS):
            assert r(v, cfg, None, p, p, offs, 4, 64, 64, 64, 0, 0, None) == -5, cfg
            assert r(v, cfg, p, p, p, None, 4, 64, 64, 64, 0, 0, None) == -5, cfg
            assert r(v, cfg, p, p, p, offs, 0, 64, 64, 64, 0, 0, None) == -1, cfg
            assert r(v, cfg, p, p, p, offs + 1, 4, 64, 64, 64, 0, 0, None) == -2, cfg
            assert r(v, cfg, p, p, p, offs, 4, 64, 64, 64 + 4, 0, 0, None) == -2, cfg
            # worst-case tile count (ceil(T / block rows) + G) * column blocks past INT_MAX
            assert r(v, cfg, p, p, p, offs, 2**31 - 1, 2**31 - 1, 8, 64, 0, 0, None) == -1, cfg
        assert r(v, NUM_CONFIGS, p, p, p, offs, 4, 64, 64, 64, 0, 0, None) == -6      # unknown configuration
        assert r(v, -1, p, p, p, offs, 4, 64, 64, 64, 0, 0, None) == -6
        # T == 0: nothing to compute, no launch (and no CUDA call)
        assert g(v, p, p, p, offs, 4, 0, 64, 64, None) == 0
        assert r(v, 0, p, p, p, offs, 4, 0, 64, 64, 0, 0, None) == 0
    # past the bound only through the groups' extra row blocks (configuration 12: 128 x 32 tiles, N = 32: one column
    # block; 2^24 row blocks of T and 2^31 - 2^24 groups)
    assert r(0, 12, p, p, p, offs, 2**31 - 2**24, 2**31 - 1, 32, 64, 0, 0, None) == -1
    for v in (3, -1, 5):                                                                 # unknown variant
        assert g(v, p, p, p, offs, 4, 64, 64, 64, None) == -6
        assert r(v, 0, p, p, p, offs, 4, 64, 64, 64, 0, 0, None) == -6
        assert lib.b200_grouped_select(v, 4, 64, 64, 64, None, None) == -6
    assert lib.b200_grouped_select(0, 0, 64, 64, 64, None, None) == -1
    assert lib.b200_grouped_select(0, 4, 0, 64, 64, None, None) == -1
    assert "aligned" in lib.b200_grouped_strerror(-2).decode()
    assert lib.b200_grouped_launch_count() == 0 and capi.grouped_launch_count() == 0


def test_dispatch_is_the_batched_rule_on_the_average_group(built_libs):
    rng = random.Random(20261016)
    shapes = [(8, 8192, 14336, 4096), (64, 16384, 2048, 7168), (1, 4096, 4096, 4096), (128, 100, 512, 64)]
    shapes += [(rng.randrange(1, 300), rng.randrange(1, 50000), 8 * rng.randrange(1, 1500), 8 * rng.randrange(1, 1500))
               for _ in range(300)]
    for g, t, n, k in shapes:
        for variant in (0, 1, 2):
            assert capi.grouped_select(variant, g, t, n, k) == capi.batched_select(variant, g, -(-t // g), n, k), \
                (variant, g, t, n, k)


def test_operator_schema_and_meta_shapes():
    from cuda_l2_b200 import ops
    schema = str(torch.ops.cuda_l2_b200.hgemm_grouped.default._schema)
    assert schema == "cuda_l2_b200::hgemm_grouped(Tensor a, Tensor b_kmajor, Tensor offs, str acc=\"fp32\") -> Tensor"
    assert "hgemm_grouped" in ops.__all__
    meta = lambda *s, dtype=torch.float16: torch.empty(s, dtype=dtype, device="meta")   # noqa: E731
    offs = meta(6, dtype=torch.int32)
    for dt, acc in ((torch.float16, "fp32"), (torch.float16, "fp16"), (torch.bfloat16, "fp32")):
        y = ops.hgemm_grouped(meta(1000, 72, dtype=dt), meta(6, 328, 72, dtype=dt), offs, acc)
        assert y.shape == (1000, 328) and y.dtype == dt and y.device.type == "meta"
    assert ops.hgemm_grouped(meta(0, 8), meta(3, 16, 8), meta(3, dtype=torch.int32)).shape == (0, 16)
    assert ops.hgemm_grouped(meta(5, 8), meta(0, 16, 8), meta(0, dtype=torch.int32)).shape == (5, 16)
    bad = [
        ((1000, 72), (6, 328, 64), offs),                                   # K
        ((1000, 68), (6, 328, 68), offs),                                   # K % 8
        ((1000, 72), (6, 324, 72), offs),                                   # N % 8
        ((2, 1000, 72), (6, 328, 72), offs),                                # 3-D a
        ((1000, 72), (328, 72), offs),                                      # 2-D b
        ((1000, 72), (6, 328, 72), meta(5, dtype=torch.int32)),            # G
        ((1000, 72), (6, 328, 72), meta(6, dtype=torch.int64)),            # int32 offsets
        ((1000, 72), (6, 328, 72), meta(6, 1, dtype=torch.int32)),
    ]
    for sa, sb, o in bad:
        with pytest.raises(capi.B200HgemmError):
            ops.hgemm_grouped(meta(*sa), meta(*sb), o)
    for a, b, acc in ((meta(8, 16, dtype=torch.bfloat16), meta(2, 8, 16, dtype=torch.bfloat16), "fp16"),
                      (meta(8, 16), meta(2, 8, 16, dtype=torch.bfloat16), "fp32"),
                      (meta(8, 16, dtype=torch.float8_e4m3fn), meta(2, 8, 16, dtype=torch.float8_e4m3fn), "fp32"),
                      (meta(8, 16, dtype=torch.float32), meta(2, 8, 16, dtype=torch.float32), "fp32")):
        with pytest.raises(capi.B200HgemmError):
            ops.hgemm_grouped(a, b, meta(2, dtype=torch.int32), acc)


def test_operator_has_no_cpu_path():
    from cuda_l2_b200 import ops
    a, b = torch.zeros((32, 16), dtype=torch.float16), torch.zeros((2, 16, 16), dtype=torch.float16)
    offs = torch.tensor([10, 32], dtype=torch.int32)
    with pytest.raises(capi.B200HgemmError):
        ops.hgemm_grouped(a, b, offs)
    with pytest.raises(capi.B200HgemmError):
        capi.gemm_grouped(a, b, torch.zeros((32, 16), dtype=torch.float16), offs)


def clamped_groups(offs, t):
    """(start, end) of every group: end_g = clamp(offs[g], start_g, T), start_g = end_{g-1}."""
    out, s = [], 0
    for o in offs:
        e = min(max(o, s), t)
        out.append((s, e))
        s = e
    return out


def _check_schedule(cfg: dict, t: int, n: int, k: int, offs, num_sms: int) -> None:
    block_rows = 128 * cfg["m_rep"] * cfg["cta_group"] * cfg["cluster_m"]
    block_cols = cfg["bn"] * cfg["cluster_n"]
    groups = clamped_groups(offs, t)
    want = {(g, mb, nb) for g, (s, e) in enumerate(groups) for mb in range(-(-(e - s) // block_rows))
            for nb in range(-(-n // block_cols))}
    s = capi.grouped_schedule(cfg["id"], t, n, k, offs, num_sms)
    worst = (-(-t // block_rows) + len(offs)) * -(-n // block_cols)
    assert s["workers"] == min(max(num_sms // (cfg["cta_group"] * cfg["cluster_m"] * cfg["cluster_n"]), 1), worst)
    got = [u for units in s["units"] for u in units]
    assert len(got) == len(set(got)) and set(got) == want, (cfg["id"], t, n, offs)
    # nothing past a group's clamped rows: every m-block starts below the group's row count
    assert all(mb * block_rows < groups[g][1] - groups[g][0] for g, mb, _ in got)
    sizes = [len(units) for units in s["units"]]
    assert max(sizes) - min(sizes) <= 1
    for units in s["units"]:      # each worker's groups never go backwards (the cursor only moves forward)
        assert [u[0] for u in units] == sorted(u[0] for u in units)


def random_offsets(rng, g, t):
    """Cumulative ends with empty groups, one-row groups, non-multiples of 16, and (sometimes) offs[-1] < T."""
    sizes = [rng.choice([0, 0, 1, 15, 17, 128, 129, 255, 300, rng.randrange(0, 700)]) for _ in range(g)]
    ends, acc = [], 0
    for sz in sizes:
        acc += sz
        ends.append(acc)
    return ends


@pytest.mark.parametrize("config_id", range(NUM_CONFIGS))
def test_schedule_covers_every_valid_tile_once(built_libs, config_id):
    cfg = capi.configs()[config_id]
    rng = random.Random(2000 + config_id)
    for trial in range(12):
        g = rng.choice([1, 2, 3, 8, 16, 64])
        ends = random_offsets(rng, g, 0)
        t = max(1, ends[-1] + rng.choice([0, 0, 5, 100, -3]))      # offs[-1] == T, < T (rows past it), > T (clamped)
        n = 8 * rng.randrange(1, 200)
        _check_schedule(cfg, t, n, 64, ends, rng.choice([132, 16, 5]))
    # malformed offsets: decreasing, negative, past T; a single group; every group empty
    _check_schedule(cfg, 1000, 256, 64, [300, 100, -5, 700, 5000, 900], 132)
    _check_schedule(cfg, 1000, 256, 64, [-1, -1, 1000], 132)
    _check_schedule(cfg, 777, 264, 64, [777], 132)
    _check_schedule(cfg, 777, 264, 64, [1], 16)
    _check_schedule(cfg, 500, 256, 64, [0] * 7, 132)


def test_schedule_rejects_bad_arguments(built_libs):
    lib = capi.grouped_lib()
    nw = ctypes.c_int()
    offs = (ctypes.c_int * 2)(64, 128)
    assert lib.b200_grouped_schedule_units(NUM_CONFIGS, 2, 128, 64, 64, offs, 132, 0, None, 0, None) == -6
    assert lib.b200_grouped_schedule_units(0, 0, 128, 64, 64, offs, 132, 0, None, 0, None) == -1
    assert lib.b200_grouped_schedule_units(0, 2, 128, 64, 64, None, 132, 0, None, 0, None) == -1
    assert lib.b200_grouped_schedule_units(0, 2, 128, 64, 64, offs, 0, 0, None, 0, None) == -1
    assert lib.b200_grouped_schedule_units(0, 2, 128, 64, 64, offs, 132, 5, None, 0, ctypes.byref(nw)) == -1
    assert nw.value == 3                      # the worst case: one row block of T plus one per group


def test_grouped_sass(built_libs):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sys.path.insert(0, str(REPO / "tools"))
    import sass_summary
    sass = subprocess.run([cuobjdump, "-sass", str(built_libs["grouped"])], capture_output=True, text=True,
                          check=True).stdout
    kernels = sass_summary.sass_by_kernel(sass)
    assert len(kernels) == NUM_CONFIGS * 3                                  # plain only, three data types
    assert all(re.search(r"GroupedINS_6ConfigI.*ELi0EEEv14CUtensorMap", name) for name in kernels)   # K-mode 0: plain
    for name, insns in kernels.items():
        ops_ = {op for _, op, _ in insns}
        assert any(op.startswith("HGMMA") for op in ops_), name
        assert not any(op.startswith(("QGMMA", "HMMA", "UTMASTG.3D")) for op in ops_), name
        assert any(op.startswith("UTMALDG.2D") for op in ops_), name        # A [T, K]
        assert any(op.startswith("UTMALDG.3D") for op in ops_), name        # Bt [G, N, K]
        assert "UTMASTG.2D" in ops_, name                                   # whole boxes of C [T, N]
        assert "STG.E.128" in ops_, name                                    # the rows of a box that straddles a group end
        loop = sass_summary.k_loop(insns)
        assert any(op == "WARPGROUP.ARRIVE" for _, op, _ in loop), name
        assert any(op.startswith("SYNCS.ARRIVE") for _, op, _ in loop), name   # the stage release is inside
        assert sass_summary.k_loop_gpu_membars(insns) == 0, name
