"""Batched fp16 / bf16 GEMM without a GPU: the C ABI of libb200_batched.so (exports, statuses before any CUDA call, the
dispatcher), the operator's schema and shape inference, the host view of the schedule the kernels walk, and the SASS
of the batched kernels."""
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
    declared = sorted(set(DECL.findall((REPO / "include" / "b200_batched.h").read_text())))
    assert declared == sorted(capi.exported_symbols()["libb200_batched.so"])
    assert built_libs["batched"].name == "libb200_batched.so"
    lib = ctypes.CDLL(str(built_libs["batched"]))
    for sym in declared:
        assert hasattr(lib, sym), sym
    assert not any(hasattr(capi.hgemm_lib(), sym) for sym in declared)     # the product library does not carry them


def _aligned(buf) -> int:
    return (ctypes.addressof(buf) + 15) & ~15


def test_argument_validation_happens_before_any_cuda_call(built_libs):
    lib = capi.batched_lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = _aligned(buf)
    mm = p + 4096
    g, r = lib.b200_batched_gemm, lib.b200_batched_gemm_run_config
    for v in (0, 1, 2):
        assert g(v, None, p, p, None, 4, 64, 64, 64, None) == -5                       # null operands
        assert g(v, p, None, p, mm, 4, 64, 64, 64, None) == -5
        assert g(v, p, p, None, None, 4, 64, 64, 64, None) == -5
        assert g(v, p, p, p, None, 0, 64, 64, 64, None) == -1                          # B <= 0
        assert g(v, p, p, p, None, -3, 64, 64, 64, None) == -1
        assert g(v, p, p, p, None, 4, 0, 64, 64, None) == -1
        assert g(v, p, p, p, None, 4, 64, 64, 60, None) == -2                          # K % 8
        assert g(v, p, p, p, None, 4, 64, 60, 64, None) == -2                          # N % 8
        assert g(v, p + 8, p, p, None, 4, 64, 64, 64, None) == -2                      # 16-byte operands
        assert g(v, p, p, p, mm + 2, 4, 64, 64, 64, None) == -2                        # masked_m: 4-byte aligned
        for cfg in range(NUM_CONFIGS):
            assert r(v, cfg, None, p, p, None, 4, 64, 64, 64, 0, 0, None) == -5, cfg
            assert r(v, cfg, p, p, p, None, 0, 64, 64, 64, 0, 0, None) == -1, cfg
            assert r(v, cfg, p, p, p, mm + 1, 4, 64, 64, 64, 0, 0, None) == -2, cfg
        assert r(v, NUM_CONFIGS, p, p, p, None, 4, 64, 64, 64, 0, 0, None) == -6      # unknown configuration
        assert r(v, -1, p, p, p, None, 4, 64, 64, 64, 0, 0, None) == -6
    # more than INT_MAX tiles in all (configuration 0: 128 x 256 tiles, two per 256 x 256 matrix)
    assert r(0, 0, p, p, p, None, 1 << 30, 256, 256, 64, 0, 0, None) == -1
    for v in (3, -1, 5):                                                                 # unknown variant
        assert g(v, p, p, p, None, 4, 64, 64, 64, None) == -6
        assert r(v, 0, p, p, p, None, 4, 64, 64, 64, 0, 0, None) == -6
        assert lib.b200_batched_select(v, 4, 64, 64, 64, None, None) == -6
    assert lib.b200_batched_select(0, 0, 64, 64, 64, None, None) == -1
    assert "aligned" in lib.b200_batched_strerror(-2).decode()
    assert lib.b200_batched_launch_count() == 0 and capi.batched_launch_count() == 0


def _usable(cfg: dict, m: int, n: int) -> bool:
    return (m + 127) // 128 >= cfg["cta_group"] * cfg["cluster_m"] * cfg["m_rep"] and -(-n // cfg["bn"]) >= cfg["cluster_n"]


def test_dispatch_takes_the_stacked_entry_where_it_fits_one_matrix(built_libs):
    cfgs = capi.configs()
    rng = random.Random(20261015)
    shapes = [(64, 1024, 1024, 128), (64, 1024, 128, 1024), (8, 512, 14336, 4096), (32, 256, 4096, 7168), (1, 4096, 4096, 4096)]
    shapes += [(rng.randrange(1, 300), rng.randrange(1, 5000), 8 * rng.randrange(1, 1500), 8 * rng.randrange(1, 1500))
               for _ in range(400)]
    for b, m, n, k in shapes:
        for variant, acc in ((0, "fp32"), (1, "fp16"), (2, "fp32")):
            stacked = capi.select(acc, min(b * m, 2**31 - 1), n, k)
            want = stacked if _usable(cfgs[stacked[0]], m, n) else capi.select(acc, m, n, k)
            assert capi.batched_select(variant, b, m, n, k) == want[:2], (variant, b, m, n, k)


def test_operator_schema_and_meta_shapes():
    from cuda_l2_b200 import ops
    schema = str(torch.ops.cuda_l2_b200.hgemm_batched.default._schema)
    assert schema == ("cuda_l2_b200::hgemm_batched(Tensor a, Tensor b_kmajor, str acc=\"fp32\", Tensor? masked_m=None) "
                      "-> Tensor")
    assert "hgemm_batched" in ops.__all__
    meta = lambda *s, dtype=torch.float16: torch.empty(s, dtype=dtype, device="meta")   # noqa: E731
    for dt, acc in ((torch.float16, "fp32"), (torch.float16, "fp16"), (torch.bfloat16, "fp32")):
        y = ops.hgemm_batched(meta(6, 200, 72, dtype=dt), meta(6, 328, 72, dtype=dt), acc)
        assert y.shape == (6, 200, 328) and y.dtype == dt and y.device.type == "meta"
        y = ops.hgemm_batched(meta(6, 200, 72, dtype=dt), meta(6, 328, 72, dtype=dt), acc, meta(6, dtype=torch.int32))
        assert y.shape == (6, 200, 328)
    assert ops.hgemm_batched(meta(0, 5, 8), meta(0, 8, 8)).shape == (0, 5, 8)
    bad = [
        ((6, 200, 72), (5, 328, 72), {}),                                  # batch counts
        ((6, 200, 72), (6, 328, 64), {}),                                  # K
        ((6, 200, 68), (6, 328, 68), {}),                                  # K % 8
        ((6, 200, 72), (6, 324, 72), {}),                                  # N % 8
        ((200, 72), (328, 72), {}),                                        # 2-D
        ((6, 200, 72), (6, 328, 72), {"masked_m": meta(5, dtype=torch.int32)}),
        ((6, 200, 72), (6, 328, 72), {"masked_m": meta(6, dtype=torch.int64)}),
        ((6, 200, 72), (6, 328, 72), {"masked_m": meta(6, 1, dtype=torch.int32)}),
    ]
    for sa, sb, kw in bad:
        with pytest.raises(capi.B200HgemmError):
            ops.hgemm_batched(meta(*sa), meta(*sb), "fp32", kw.get("masked_m"))
    for a, b, acc in ((meta(2, 8, 16, dtype=torch.bfloat16), meta(2, 8, 16, dtype=torch.bfloat16), "fp16"),
                      (meta(2, 8, 16), meta(2, 8, 16, dtype=torch.bfloat16), "fp32"),
                      (meta(2, 8, 16, dtype=torch.float8_e4m3fn), meta(2, 8, 16, dtype=torch.float8_e4m3fn), "fp32"),
                      (meta(2, 8, 16, dtype=torch.float32), meta(2, 8, 16, dtype=torch.float32), "fp32")):
        with pytest.raises(capi.B200HgemmError):
            ops.hgemm_batched(a, b, acc)


def test_operator_has_no_cpu_path():
    from cuda_l2_b200 import ops
    a = torch.zeros((2, 16, 16), dtype=torch.float16)
    with pytest.raises(capi.B200HgemmError):
        ops.hgemm_batched(a, a)
    with pytest.raises(capi.B200HgemmError):
        capi.gemm_batched(a, a, torch.zeros((2, 16, 16), dtype=torch.float16))


def _check_schedule(cfg: dict, b: int, m: int, n: int, k: int, counts, num_sms: int) -> None:
    block_rows = 128 * cfg["m_rep"] * cfg["cta_group"] * cfg["cluster_m"]
    block_cols = cfg["bn"] * cfg["cluster_n"]
    rows = [m] * b if counts is None else [min(max(c, 0), m) for c in counts]
    want = {(bi, mb, nb) for bi in range(b) for mb in range(-(-rows[bi] // block_rows)) for nb in range(-(-n // block_cols))}
    s = capi.batched_schedule(cfg["id"], b, m, n, k, counts, num_sms)
    dense_tiles = b * -(-m // block_rows) * -(-n // block_cols)
    assert s["workers"] == min(max(num_sms // (cfg["cta_group"] * cfg["cluster_m"] * cfg["cluster_n"]), 1), dense_tiles)
    got = [t for units in s["units"] for t in units]
    assert len(got) == len(set(got)) and set(got) == want, (cfg["id"], b, m, n, counts)
    assert all(mb * block_rows < rows[bi] for bi, mb, _ in got)
    sizes = [len(units) for units in s["units"]]
    assert max(sizes) - min(sizes) <= 1
    for units in s["units"]:      # each worker's tiles come batch after batch (the cursor only moves forward)
        assert [t[0] for t in units] == sorted(t[0] for t in units)


@pytest.mark.parametrize("config_id", range(NUM_CONFIGS))
def test_schedule_covers_every_valid_tile_once(built_libs, config_id):
    cfg = capi.configs()[config_id]
    rng = random.Random(1000 + config_id)
    for trial in range(12):
        b = rng.choice([1, 2, 3, 7, 16, 33])
        m = rng.choice([1, 100, 128, 257, 512, 777, 1024])
        n = 8 * rng.randrange(1, 200)
        counts = None if trial % 4 == 0 else \
            [rng.choice([0, m, m + rng.randrange(1, 99), -rng.randrange(1, 99), rng.randrange(0, m + 1)]) for _ in range(b)]
        _check_schedule(cfg, b, m, n, 64, counts, rng.choice([132, 16, 5]))
    _check_schedule(cfg, 5, 300, 256, 64, [0] * 5, 132)                    # nothing to do: no tiles at all
    _check_schedule(cfg, 4, 300, 256, 64, [-5, 0, 400, 1], 132)


def test_schedule_rejects_bad_arguments(built_libs):
    lib = capi.batched_lib()
    nw = ctypes.c_int()
    assert lib.b200_batched_schedule_units(NUM_CONFIGS, 2, 64, 64, 64, None, 132, 0, None, 0, None) == -6
    assert lib.b200_batched_schedule_units(0, 0, 64, 64, 64, None, 132, 0, None, 0, None) == -1
    assert lib.b200_batched_schedule_units(0, 2, 64, 64, 64, None, 0, 0, None, 0, None) == -1
    assert lib.b200_batched_schedule_units(0, 2, 64, 64, 64, None, 132, 5, None, 0, ctypes.byref(nw)) == -1
    assert nw.value == 2                                                     # one tile per matrix: two workers
    with pytest.raises(capi.B200HgemmError) as err:                          # the status, with its text
        capi.batched_schedule(NUM_CONFIGS, 2, 64, 64, 64)
    assert str(err.value) == f"b200_batched_schedule_units failed: status -6 ({lib.b200_batched_strerror(-6).decode()})"


def test_batched_sass(built_libs):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sys.path.insert(0, str(REPO / "tools"))
    import sass_summary
    sass = subprocess.run([cuobjdump, "-sass", str(built_libs["batched"])], capture_output=True, text=True,
                          check=True).stdout
    kernels = sass_summary.sass_by_kernel(sass)
    assert len(kernels) == NUM_CONFIGS * 3                                  # plain only, three data types
    assert all(re.search(r"BatchedINS_6ConfigI.*ELi0EEEv14CUtensorMap", name) for name in kernels)   # K-mode 0: plain
    for name, insns in kernels.items():
        ops_ = {op for _, op, _ in insns}
        assert any(op.startswith("HGMMA") for op in ops_), name
        assert not any(op.startswith(("QGMMA", "HMMA", "UTMALDG.2D", "UTMASTG.2D")) for op in ops_), name
        assert any(op.startswith("UTMALDG.3D") for op in ops_) and "UTMASTG.3D" in ops_, name
        loop = sass_summary.k_loop(insns)
        assert any(op == "WARPGROUP.ARRIVE" for _, op, _ in loop), name
        assert any(op.startswith("SYNCS.ARRIVE") for _, op, _ in loop), name   # the stage release is inside
        assert sass_summary.k_loop_gpu_membars(insns) == 0, name
