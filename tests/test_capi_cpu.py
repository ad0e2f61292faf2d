"""The C-ABI libraries load and export every symbol include/*.h declares (no compute without a GPU)."""
import ctypes
import re

import pytest

from conftest import REPO
from cuda_l2_b200 import capi

DECL = re.compile(r"^\s*(?:const\s+)?(?:unsigned\s+long\s+long|int|void|char\s*\*|const\s+char\s*\*)\s*\*?\s*(b200_\w+)\s*\(", re.M)


def declared(header: str) -> list[str]:
    return sorted(set(DECL.findall((REPO / "include" / header).read_text())))


def test_headers_and_python_binding_agree():
    assert declared("b200_hgemm.h") == sorted(capi.exported_symbols()["libb200_hgemm.so"])
    assert declared("b200_baselines.h") == sorted(capi.exported_symbols()["libb200_baselines.so"])


def test_libraries_export_every_declared_symbol(built_libs):
    for header, path in (("b200_hgemm.h", built_libs["capi"]), ("b200_baselines.h", built_libs["baselines"])):
        lib = ctypes.CDLL(str(path))
        for sym in declared(header):
            assert hasattr(lib, sym), f"{path.name} does not export {sym}"


def test_config_table_and_dispatch(built_libs):
    cfgs = capi.configs()
    assert len(cfgs) >= 5
    for c in cfgs:
        assert (c["bn"] == 32 or c["bn"] % 64 == 0) and c["bn"] <= 256 and c["cta_group"] in (1, 2) and c["stages"] >= 2
        assert c["cta_group"] * c["cluster_m"] * c["cluster_n"] <= 8
        assert c["m_rep"] in (1, 2)
        smem = 1024 + c["stages"] * (128 * c["m_rep"] * 64 * 2 + (c["bn"] // c["cta_group"]) * 64 * 2) + 32768 + 256
        assert smem + 256 <= 232448
    ids = {c["id"] for c in cfgs}
    for acc in ("fp32", "fp16"):
        for mnk in ((64, 4096, 64), (4096, 4096, 4096), (8192, 8192, 8192), (2048, 11008, 4096), (64, 64, 64),
                    (16384, 16384, 16384), (200, 328, 72)):
            cid, gm, sp = capi.select(acc, *mnk)
            assert cid in ids and gm >= 0 and (sp >= 1 or sp in (-2, -4, -8))
            if mnk[0] <= 128:
                assert cfgs[cid]["cta_group"] == 1     # a CTA pair would waste its second half on padding


def test_argument_validation_happens_before_any_cuda_call(built_libs):
    lib = capi.hgemm_lib()
    assert lib.b200_hgemm_f32acc(None, None, None, None, 64, 64, 64, None) == -5       # null pointers
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    p = (p + 15) & ~15
    assert lib.b200_hgemm_f32acc(p, None, p, p, 0, 64, 64, None) == -1                  # bad shape
    assert lib.b200_hgemm_f16acc(p, None, p, p, 64, 64, 60, None) == -2                 # K % 8 != 0
    assert lib.b200_hgemm_f16acc(p, None, p, p, 64, 60, 64, None) == -2                 # N % 8 != 0
    assert lib.b200_hgemm_f32acc(p + 2, None, p, p, 64, 64, 64, None) == -2             # misaligned A
    assert lib.b200_hgemm_run_config(32, 99, p, p, p, 64, 64, 64, 0, 0, 1, None) == -6     # unknown config
    assert lib.b200_hgemm_run_config(8, 0, p, p, p, 64, 64, 64, 0, 0, 1, None) == -6       # unknown accumulator
    assert "16-byte" in capi.strerror(-2)
    assert capi.launch_count() == 0


def test_python_binding_rejects_cpu_tensors(built_libs):
    import torch
    a = torch.zeros(64, 64, dtype=torch.half)
    with pytest.raises(capi.B200HgemmError):
        capi.hgemm(a, a, a)          # CPU tensors: there is no CPU fallback
    with pytest.raises(capi.B200HgemmError):
        capi.hgemm(a.float(), a, a)


def test_library_keeps_its_template_statics_private(built_libs):
    """libb200_hgemm.so and a JIT-built hgemm_lib.so instantiate the same templates; a process-wide (STB_GNU_UNIQUE)
    static would let one library skip the per-kernel setup of the other (seen on the GPU as `invalid argument` on the
    first launch after the harness ran). The build uses -fno-gnu-unique: no 'u' symbols may remain."""
    import shutil
    import subprocess
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not available")
    out = subprocess.run([nm, "-D", str(built_libs["capi"])], capture_output=True, text=True, check=True).stdout
    assert not [ln for ln in out.splitlines() if " u " in ln]


def test_tuned_table_entries_are_launchable_for_every_grid_shape(built_libs):
    """Every tuned entry must name an existing configuration whose cluster is not wider than the problem, and
    split-K (either flavour) only on plain single-CTA configurations with tiles of at least 64 columns."""
    from cuda_l2_b200 import farm
    cfgs = {c["id"]: c for c in capi.configs()}
    seen_cluster_split = seen_mcast = 0
    for (m, n, k) in farm.grid_shapes():
        for acc in ("fp32", "fp16"):
            cid, gm, sp = capi.select(acc, m, n, k)
            c = cfgs[cid]
            assert 0 <= gm <= 64
            assert -(-m // 128) >= c["cta_group"] * c["cluster_m"] * c["m_rep"], (m, n, k, acc, c)
            assert -(-n // c["bn"]) >= c["cluster_n"], (m, n, k, acc, c)
            if sp in (capi.STREAMK_TAIL, capi.STREAMK_TAIL_PLUS_WAVE):   # stream-K: single CTAs and CTA pairs
                assert c["cluster_m"] * c["cluster_n"] == 1 and c["bn"] >= 64 and c["m_rep"] == 1, (m, n, k, acc, sp, c)
            elif sp != 1:
                assert sp in (-2, -4, -8) or 2 <= sp <= 64
                assert c["cta_group"] == 1 and c["cluster_m"] * c["cluster_n"] == 1 and c["bn"] >= 64, (m, n, k, acc, sp, c)
                seen_cluster_split += sp < 0
            seen_mcast += c["cluster_m"] * c["cluster_n"] > 1
    assert seen_cluster_split > 50 and seen_mcast > 20          # the table really uses both mechanisms


def test_off_grid_shapes_borrow_the_nearest_tuned_entry(built_libs):
    assert capi.select("fp32", 2048, 11008, 4096) == capi.select("fp32", 2048, 11008, 4096)
    assert capi.select("fp32", 4000, 4100, 4090) == capi.select("fp32", 4096, 4096, 4096)
    assert capi.select("fp16", 70, 60 * 8, 16000) == capi.select("fp16", 64, 512, 16384)
    cid, _, _ = capi.select("fp32", 8, 16, 8192)               # far off the grid in M and N: still a valid choice
    cfg = capi.configs()[cid]
    assert cfg["cta_group"] == 1 and cfg["cluster_m"] * cfg["cluster_n"] == 1


def _check_schedule(cfg, m, n, k, splits, num_sms=132):
    """Every k-block of every tile is run exactly once, and the stream-K fix-up protocol cannot wait forever."""
    tile_m = 128 * cfg["cta_group"] * cfg["cluster_m"] * cfg["m_rep"]
    tile_n = cfg["bn"] * cfg["cluster_n"]
    tiles = -(-m // tile_m) * -(-n // tile_n)
    nkb = -(-k // 64)
    s = capi.schedule(cfg["id"], m, n, k, splits, num_sms)
    seen = {}
    for w, units in enumerate(s["units"]):
        for pos, (t, kb0, kb1, contrib) in enumerate(units):
            assert 0 <= t < tiles and 0 <= kb0 < kb1 <= nkb, (w, units)
            for kb in range(kb0, kb1):
                assert (t, kb) not in seen, f"k-block {kb} of tile {t} is run by workers {seen[(t, kb)]} and {w}"
                seen[(t, kb)] = w
            if s["sk_tiles"] and kb0 > 0:
                assert pos == 0, "a contributor unit must be its worker's first unit (it may not wait behind an owner)"
            if s["sk_tiles"] and kb0 == 0 and kb1 < nkb:
                # the owner's contributors are the first units of the next workers, contiguous in k up to the tile end
                assert contrib >= 1
                at = kb1
                for p in range(1, contrib + 1):
                    ft, fk0, fk1, _ = s["units"][w + p][0]
                    assert (ft, fk0) == (t, at), (w, p, units, s["units"][w + p])
                    at = fk1
                assert at == nkb
            else:
                assert contrib == 0
    assert len(seen) == tiles * nkb, f"{tiles * nkb - len(seen)} k-blocks are never run"
    return s


def test_schedule_covers_every_k_block_once_in_every_mode(built_libs):
    cfgs = capi.configs()
    shapes = [(512, 8192, 8192), (4096, 4096, 4096), (1024, 1024, 4096), (2048, 11008, 4096), (200, 328, 72),
              (12288, 2048, 4096), (64, 64, 16384), (16384, 512, 1024), (8192, 8192, 512), (256, 256, 256)]
    for cfg in cfgs:
        for m, n, k in shapes:
            for splits in (1, 4, 32, -2, -8, capi.STREAMK_TAIL, capi.STREAMK_TAIL_PLUS_WAVE):
                _check_schedule(cfg, m, n, k, splits)
    # a device with fewer SMs (e.g. under max_ctas) changes the decomposition, not its correctness
    for num_sms in (16, 100, 132):
        for splits in (1, capi.STREAMK_TAIL, capi.STREAMK_TAIL_PLUS_WAVE):
            _check_schedule(cfgs[3], 4096, 4096, 4096, splits, num_sms)


def test_stream_k_fills_the_partial_wave_and_balances_the_workers(built_libs):
    cfgs = capi.configs()
    # 512 x 8192 with 256 x 256 pair tiles: 64 tiles on 66 CTA pairs — the plain schedule leaves 2 pairs idle
    plain = _check_schedule(cfgs[3], 512, 8192, 8192, 1)
    assert plain["workers"] == 64 and plain["sk_tiles"] == 0
    sk = _check_schedule(cfgs[3], 512, 8192, 8192, capi.STREAMK_TAIL)
    assert sk["workers"] == 66 and sk["sk_tiles"] == 64
    work = [sum(kb1 - kb0 for _, kb0, kb1, _ in u) for u in sk["units"]]
    assert max(work) - min(work) <= 1 and sum(work) == 64 * 128
    # 4096^3 with 256 x 192 pair tiles: 352 tiles = 5 full waves + 22; the tail mode splits the 22, the other 22 + 66
    assert _check_schedule(cfgs[6], 4096, 4096, 4096, capi.STREAMK_TAIL)["sk_tiles"] == 22
    assert _check_schedule(cfgs[6], 4096, 4096, 4096, capi.STREAMK_TAIL_PLUS_WAVE)["sk_tiles"] == 88
    # full waves need no stream-K; multicast clusters and 32-wide tiles are not wired for it; tiny K is not worth it
    assert _check_schedule(cfgs[3], 256 * 66, 256, 4096, capi.STREAMK_TAIL)["sk_tiles"] == 0
    assert _check_schedule(cfgs[18], 512, 8192, 8192, capi.STREAMK_TAIL)["sk_tiles"] == 0
    assert _check_schedule(cfgs[12], 512, 8192, 8192, capi.STREAMK_TAIL)["sk_tiles"] == 0
    assert _check_schedule(cfgs[3], 512, 8192, 128, capi.STREAMK_TAIL)["sk_tiles"] == 0


def test_schedule_is_a_partition_for_random_problems(built_libs):
    """Randomised version of the coverage test: odd sizes, short and long K, restricted SM counts, every mode."""
    import random
    rng = random.Random(20260923)
    cfgs = capi.configs()
    modes = (1, 2, 3, 7, 32, -2, -4, -8, capi.STREAMK_TAIL, capi.STREAMK_TAIL_PLUS_WAVE)
    for _ in range(400):
        cfg = rng.choice(cfgs)
        m = rng.choice((8, 64, 72, 128, 200, 256, 520, 1024, 3000, 4096, 10000))
        n = rng.choice((8, 64, 136, 256, 328, 1000, 2048, 5000, 8192))
        k = rng.choice((8, 64, 72, 256, 512, 1096, 4096, 16384, 30000))
        num_sms = rng.choice((8, 36, 100, 132, 148, 160))
        _check_schedule(cfg, m, n, k, rng.choice(modes), num_sms)
