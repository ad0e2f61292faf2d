"""FP8 (e4m3) GEMM without a GPU: the oracle's e4m3 codec and GEMM against torch and the golden fixtures, the C ABI's
argument checks and dispatcher, the torch operator's schema and shape inference, the host planner's k-blocks, and the
SASS of the e4m3 kernels."""
import ctypes
import random
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
from oracle import fp8 as fp8_oracle
from conftest import GOLDEN, REPO
from cuda_l2_b200 import capi


def load_fp8_cases():
    """Operands as uint8 e4m3 codes, scales as fp32, truth as uint16 bits; kind 0 = small integers, 1 = randn."""
    z = np.load(GOLDEN / "fp8_cases.npz")
    cases, i = [], 0
    while f"meta{i}" in z:
        m, n, k, kind, out_bf16, seed = (int(x) for x in z[f"meta{i}"])
        sa, sb = (float(x) for x in z[f"scales{i}"])
        cases.append(dict(m=m, n=n, k=k, kind=("int", "randn")[kind], out_bf16=bool(out_bf16), seed=seed,
                          a=z[f"a{i}"], bt=z[f"bt{i}"], sa=sa, sb=sb, truth=z[f"truth{i}"]))
        i += 1
    return cases


def out_values(bits: np.ndarray, out_bf16: bool) -> np.ndarray:
    return oracle.bf16_bits_to_f32(bits) if out_bf16 else bits.view(np.float16).astype(np.float32)


def test_e4m3_decode_matches_torch_for_all_256_codes():
    codes = np.arange(256, dtype=np.uint8)
    want = torch.from_numpy(codes).view(torch.float8_e4m3fn).float().numpy()
    got = fp8_oracle.e4m3_to_f32(codes)
    assert np.array_equal(got, want, equal_nan=True)
    assert np.isnan(got[0x7F]) and np.isnan(got[0xFF]) and np.isfinite(got[:0x7F]).all()
    assert got[0x7E] == 448.0 and got[1] == 2.0 ** -9


def test_e4m3_encode_matches_torch_on_in_range_values():
    finite = fp8_oracle.e4m3_to_f32(np.arange(0x7F, dtype=np.uint8))
    rng = np.random.default_rng(7)
    x = np.concatenate([finite, -finite, (finite[:-1] + finite[1:]) / 2,            # every tie
                        rng.normal(0, 40, 4000), rng.uniform(-448, 448, 4000), rng.normal(0, 0.01, 2000)]).astype(np.float32)
    x = x[np.abs(x) <= 448]
    want = torch.from_numpy(x).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    assert np.array_equal(fp8_oracle.f32_to_e4m3(x), want)


def test_oracle_reproduces_the_fp8_fixtures():
    cases = load_fp8_cases()
    assert {c["kind"] for c in cases} == {"int", "randn"} and {c["out_bf16"] for c in cases} == {False, True}
    assert any(c["kind"] == "int" and np.log2(c["sa"] * c["sb"]) % 1 != 0 for c in cases)   # a non-power-of-two pair
    for c in cases:
        got = fp8_oracle.fp8gemm_f32acc(c["a"], c["bt"], c["sa"], c["sb"], c["out_bf16"])
        if c["kind"] == "int":
            assert np.array_equal(got, c["truth"]), (c["m"], c["n"], c["k"], c["out_bf16"])
        else:
            # torch's fp32 matmul sums in another order: the two may differ by one rounding of the output
            g, t = out_values(got, c["out_bf16"]), out_values(c["truth"], c["out_bf16"])
            ulp = 2.0 ** (-7 if c["out_bf16"] else -10)
            assert np.all(np.abs(g - t) <= ulp * np.abs(t) + 1e-6), (c["m"], c["n"], c["k"])


def _aligned(buf) -> int:
    return (ctypes.addressof(buf) + 15) & ~15


def test_fp8_argument_validation_happens_before_any_cuda_call(built_libs):
    lib = capi.hgemm_lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = _aligned(buf)
    s = p + 4096
    assert lib.b200_fp8gemm(p, p, p, None, s, 0, 64, 64, 64, None) == -5             # null scale
    assert lib.b200_fp8gemm(p, p, p, s, None, 0, 64, 64, 64, None) == -5
    assert lib.b200_fp8gemm(None, p, p, s, s, 0, 64, 64, 64, None) == -5             # null operand
    assert lib.b200_fp8gemm(p, p, p, s, s, 0, 64, 64, 0, None) == -1                 # bad shape
    assert lib.b200_fp8gemm(p, p, p, s, s, 0, 64, 64, 72, None) == -9                # K % 16 != 0 (K % 8 == 0)
    assert lib.b200_fp8gemm(p, p, p, s, s, 0, 64, 60, 64, None) == -2                # N % 8 != 0
    assert lib.b200_fp8gemm(p + 8, p, p, s, s, 0, 64, 64, 64, None) == -2            # misaligned A
    assert lib.b200_fp8gemm(p, p + 8, p, s, s, 0, 64, 64, 64, None) == -2            # misaligned Bt
    assert lib.b200_fp8gemm(p, p, p + 8, s, s, 0, 64, 64, 64, None) == -2            # misaligned C
    assert lib.b200_fp8gemm(p, p, p, s + 2, s, 0, 64, 64, 64, None) == -2            # misaligned scale
    assert lib.b200_fp8gemm(p, p, p, s, s, 2, 64, 64, 64, None) == -6                # bad output selector
    assert lib.b200_fp8gemm_run_config(99, 0, p, p, p, s, s, 64, 64, 64, 0, 0, 1, None) == -6   # unknown config
    assert lib.b200_fp8gemm_run_config(0, -1, p, p, p, s, s, 64, 64, 64, 0, 0, 1, None) == -6   # bad output selector
    assert lib.b200_fp8gemm_run_config(0, 1, p, p, p, s, s, 64, 64, 40, 0, 0, 1, None) == -9
    assert lib.b200_fp8gemm_run_config(0, 1, p, p, p, None, s, 64, 64, 64, 0, 0, 1, None) == -5
    assert "K % 16" in capi.strerror(-9)
    assert "16-byte" in capi.strerror(-2)                                              # the 16-bit message is unchanged
    assert capi.launch_count() == 0


def test_fp8_dispatch_is_the_fp32_table_at_half_k(built_libs):
    from cuda_l2_b200 import farm
    shapes = list(farm.grid_shapes())
    assert len(shapes) == 1001
    rng = random.Random(20261015)
    shapes += [(rng.randrange(1, 20000), 8 * rng.randrange(1, 2500), 16 * rng.randrange(1, 2000)) for _ in range(2000)]
    for m, n, k in shapes:
        assert capi.fp8_select(m, n, k) == capi.select("fp32", m, n, k // 2), (m, n, k)


def test_fp8_operator_schema_shapes_and_checks():
    from cuda_l2_b200 import ops
    schema = str(torch.ops.cuda_l2_b200.fp8_gemm.default._schema)
    assert schema == ("cuda_l2_b200::fp8_gemm(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, "
                      "ScalarType out_dtype) -> Tensor")
    e4 = torch.float8_e4m3fn
    a = torch.empty((200, 144), dtype=e4, device="meta")
    b = torch.empty((328, 144), dtype=e4, device="meta")
    s = torch.empty(1, dtype=torch.float32, device="meta")
    for dt in (torch.float16, torch.bfloat16):
        y = ops.fp8_gemm(a, b, s, s, dt)
        assert y.shape == (200, 328) and y.dtype == dt and y.device.type == "meta"
    bad = [
        (a.to(torch.float16), b, s, s, torch.float16),                                   # operand dtype
        (a, b, s, s, torch.float32),                                                     # output dtype
        (a, torch.empty((328, 160), dtype=e4, device="meta"), s, s, torch.float16),       # K mismatch
        (torch.empty((8, 72), dtype=e4, device="meta"), torch.empty((8, 72), dtype=e4, device="meta"), s, s, torch.float16),
        (a, torch.empty((324, 144), dtype=e4, device="meta"), s, s, torch.float16),       # N % 8
        (a, b, torch.empty(2, device="meta"), s, torch.float16),                          # scale shape
        (a, b, s, torch.empty(1, dtype=torch.float16, device="meta"), torch.float16),     # scale dtype
        (a[0], b, s, s, torch.float16),                                                  # 1-D operand
    ]
    for args in bad:
        with pytest.raises(capi.B200HgemmError):
            ops.fp8_gemm(*args)
    with pytest.raises(capi.B200HgemmError, match="no CPU implementation"):
        ops.fp8_gemm(torch.zeros((8, 16), dtype=e4), torch.zeros((8, 16), dtype=e4), torch.ones(1), torch.ones(1))


def test_fp8_python_binding_checks_before_the_library():
    e4 = torch.float8_e4m3fn
    a = torch.zeros((64, 64), dtype=e4)
    c = torch.zeros((64, 64), dtype=torch.half)
    one = torch.ones(1)
    with pytest.raises(capi.B200HgemmError):
        capi.fp8_gemm(a, a, c, one, one)                     # CPU tensors: no fallback
    with pytest.raises(capi.B200HgemmError):
        capi.fp8_gemm(a.half(), a, c, one, one)
    with pytest.raises(capi.B200HgemmError):
        capi.fp8_gemm(a, a, c.float(), one, one)


def test_fp8_linear_conversion_rules():
    from torch import nn

    from cuda_l2_b200 import ops
    lin = nn.Linear(64, 32, dtype=torch.float16)
    m = ops.B200Fp8Linear.from_linear(lin)
    assert m.weight_fp8.dtype == torch.float8_e4m3fn and m.weight_fp8.shape == (32, 64)
    assert m.weight_scale.dtype == torch.float32 and m.weight_scale.shape == (1,)
    assert m.bias is lin.bias and m.out_dtype == torch.float16
    assert torch.allclose(m.weight_fp8.float() * m.weight_scale, lin.weight.float(), rtol=2 ** -4, atol=1e-6)
    assert set(dict(m.named_buffers())) == {"weight_fp8", "weight_scale"}
    with pytest.raises(capi.B200HgemmError):
        ops.B200Fp8Linear.from_linear(nn.Linear(72, 32, dtype=torch.float16))   # in_features % 16
    with pytest.raises(capi.B200HgemmError):
        ops.B200Fp8Linear.from_linear(lin, out_dtype=torch.float32)


HOST_PLANS = r"""
#include <cstdio>
#include "cuda_l2_b200/csrc/hgemm_host.cuh"
using namespace b200;
using host::Plan;
static int bad = 0;
template <class F16, class F8>
static void check(int code) {
  static_assert(F8::STAGE_BYTES == F16::STAGE_BYTES && F8::STAGES == F16::STAGES && F8::SMEM_BYTES == F16::SMEM_BYTES, "smem");
  static_assert(F16::BLOCK_K == 64 && F8::BLOCK_K == 128 && F8::OP_BYTES == 1, "k-block");
  for (int m : {64, 200, 4096}) for (int n : {64, 328, 8192}) for (int k : {16, 144, 4096, 16384}) {
    auto all = [] { return 132; };
    const Plan a = host::plan<F8>(m, n, k, code, 132 / F8::CLUSTER_CTAS, all);
    const Plan b = host::plan<F16>(m, n, k / 2, code, 132 / F16::CLUSTER_CTAS, all);
    if (a.mode != b.mode || a.nkb != b.nkb || a.workers != b.workers || a.splits != b.splits || a.sk_tiles != b.sk_tiles) {
      ++bad; std::printf("plan %d %d %d %d\n", code, m, n, k);
    }
  }
}
int main() {
  check<Config<128, 6, 1, true>, Config<128, 6, 1, true, 1, 1, 1, false, true>>(1);
  check<Config<128, 6, 1, true>, Config<128, 6, 1, true, 1, 1, 1, true, true>>(4);
  check<Config<128, 6, 1, true>, Config<128, 6, 1, true, 1, 1, 1, false, true>>(-4);
  check<Config<256, 6, 2, true>, Config<256, 6, 2, true, 1, 1, 1, true, true>>(100);
  check<Config<128, 4, 2, true, 1, 1, 2>, Config<128, 4, 2, true, 1, 1, 2, false, true>>(1);
  // a map of the same pointer and dimensions is another map for another element type
  int x = 0;
  const host::MapKey f16{&x, 64, 64, 64, 64, host::Elem::kF16}, e4{&x, 64, 64, 64, 64, host::Elem::kE4M3};
  if (f16 == e4 || !(f16 == f16)) { ++bad; std::printf("map key\n"); }
  return bad != 0;
}
"""


def test_e4m3_plans_match_fp16_plans_at_half_k(tmp_path):
    """An e4m3 k-block is 128 elements: the planner gives an e4m3 problem (M, N, K) the plan of the fp16 one
    (M, N, K / 2), with the same ring and stage sizes; the tensor-map cache keys on the element type."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("nvcc not available")
    src, exe = tmp_path / "plans.cu", tmp_path / "plans"
    src.write_text(HOST_PLANS)
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O1", f"-I{REPO}", str(src),
                        "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-1500:]
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-1500:]


def _sass_by_kernel(cuobjdump: str, lib: Path) -> dict[str, list[str]]:
    out = subprocess.run([cuobjdump, "-sass", str(lib)], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n\s+Function : (\S+)\n", out)
    return {name: re.findall(r"^\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)", body, re.M)
            for name, body in zip(parts[1::2], parts[2::2])}


def test_e4m3_kernels_use_qgmma_and_keep_the_fp16_wait_structure(built_libs):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sass = _sass_by_kernel(cuobjdump, built_libs["capi"])
    # Config<BN, STAGES, CTA_GROUP, ACC_F32, CLUSTER_M, CLUSTER_N, M_REP, BF16, E4M3>, then the K-mode
    key = re.compile(r"ConfigI(.*?)ELb([01])ELb([01])EEELi(\d)EEEv")
    fp16, fp8 = {}, {}
    for name, ops_ in sass.items():
        m = key.search(name)
        assert m, name
        cfg, bf16, e4m3, mode = m.groups()
        if e4m3 == "1":
            fp8[(cfg, bf16, mode)] = ops_
        elif bf16 == "0" and cfg.split("E")[3] == "Lb1":            # fp16 operands, fp32 accumulation
            fp16[(cfg, mode)] = ops_
    assert len(fp8) == 2 * 46 and len(fp16) == 46
    for (cfg, bf16, mode), ops_ in fp8.items():
        q = [o for o in ops_ if o.startswith("QGMMA")]
        assert q and all(o.endswith("E4M3.E4M3") or ".E4M3.E4M3" in o for o in q), (cfg, bf16, mode, set(q))
        assert not any(o.startswith(("HMMA", "HGMMA")) for o in ops_), (cfg, mode)
        ref = fp16[(cfg, mode)]
        assert sum(o.startswith("WARPGROUP.DEPBAR") for o in ops_) == sum(o.startswith("WARPGROUP.DEPBAR") for o in ref), (cfg, mode)
        assert len(q) == sum(o.startswith("HGMMA") for o in ref), (cfg, mode)
