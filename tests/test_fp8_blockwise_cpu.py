"""FP8 (e4m3) GEMM with block scales, without a GPU: the C reference against the golden fixtures and the promotion's
rounding rules, the C ABI of libb200_fp8block.so (statuses, exports, dispatcher), the scale rule, the operator's shape
inference, the quantisers, B200Fp8Linear's blockwise buffers, and the SASS of the block-scaled kernels."""
import ctypes
import random
import re
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from torch import nn

import oracle
from conftest import GOLDEN, REPO
from cuda_l2_b200 import capi
from fp8_block_ref import fp8gemm_f32acc_block

E4 = torch.float8_e4m3fn
ELIGIBLE = (1, 2, 4, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 22, 23, 30)
ONE, THREE = 0x38, 0x44          # e4m3 codes of 1.0 and 3.0


def load_block_cases():
    """Operands as uint8 e4m3 codes, scales as fp32, truth as uint16 bits; kind 0 = small integers, 1 = randn."""
    z = np.load(GOLDEN / "fp8_block_cases.npz")
    cases, i = [], 0
    while f"meta{i}" in z:
        m, n, k, kind, out_bf16, seed = (int(x) for x in z[f"meta{i}"])
        cases.append(dict(m=m, n=n, k=k, kind=("int", "randn")[kind], out_bf16=bool(out_bf16), seed=seed,
                          a=z[f"a{i}"], bt=z[f"bt{i}"], sa=z[f"sa{i}"], sb=z[f"sb{i}"], truth=z[f"truth{i}"]))
        i += 1
    return cases


def out_values(bits: np.ndarray, out_bf16: bool) -> np.ndarray:
    return oracle.bf16_bits_to_f32(bits) if out_bf16 else bits.view(np.float16).astype(np.float32)


def test_reference_reproduces_the_block_fixtures():
    cases = load_block_cases()
    assert {c["kind"] for c in cases} == {"int", "randn"} and {c["out_bf16"] for c in cases} == {False, True}
    ints = [c for c in cases if c["kind"] == "int"]
    assert any(c["m"] % 4 and c["n"] % 128 and c["k"] % 128 for c in ints)          # ragged in every dimension
    for c in cases:
        nkb = -(-c["k"] // 128)
        assert c["sa"].shape == (c["m"], nkb) and c["sb"].shape == (-(-c["n"] // 128), nkb)
        got = fp8gemm_f32acc_block(c["a"], c["bt"], c["sa"], c["sb"], c["out_bf16"])
        if c["kind"] == "int":
            assert np.array_equal(got, c["truth"]), (c["m"], c["n"], c["k"], c["out_bf16"])
        else:
            # torch sums each block in its own order and rounds p * s before adding: one output rounding apart at most
            g, t = out_values(got, c["out_bf16"]), out_values(c["truth"], c["out_bf16"])
            ulp = 2.0 ** (-7 if c["out_bf16"] else -10)
            assert np.all(np.abs(g - t) <= ulp * np.abs(t) + 1e-6), (c["m"], c["n"], c["k"])


def test_reference_promotes_with_one_fused_multiply_add():
    # block 0 sums to -3 with scale 1, block 1 to 3 with scale s1 = 1 + 2^-23. fmaf(3, s1, -3) = 3 * 2^-23 exactly;
    # rounding 3 * s1 to fp32 first gives 3 + 2^-21 (a tie, to even) and then 2^-21. Both are fp16 subnormals:
    # 6 and 8 units of 2^-24.
    s1 = np.float32(1.0) + np.float32(2.0 ** -23)
    assert np.float32(np.float32(3.0) * s1) - np.float32(3.0) == np.float32(2.0 ** -21)        # mul, then add
    a = np.zeros((1, 256), dtype=np.uint8)
    a[0, 0], a[0, 128] = 0xC4, THREE                                                           # -3.0, 3.0
    bt = np.full((8, 256), ONE, dtype=np.uint8)
    got = fp8gemm_f32acc_block(a, bt, np.array([[1.0, s1]], dtype=np.float32), np.ones((1, 2)), False)
    assert np.all(got == 0x0006), got                                                           # 3 * 2^-23
    # the order is k-block ascending: swapping the blocks' scales rounds 3 * 1 exactly and fuses -3 * s1 instead
    got = fp8gemm_f32acc_block(a, bt, np.array([[s1, 1.0]], dtype=np.float32), np.ones((1, 2)), False)
    assert np.all(got == np.float16(np.float32(-3.0) * s1 + np.float32(3.0)).view(np.uint16)), got


def test_reference_first_block_is_a_multiply_that_keeps_the_sign_of_zero():
    # one k-block whose sum is +0 with a negative scale: fp32(0 * -1) = -0; an fma onto +0 would give +0
    a = np.zeros((1, 16), dtype=np.uint8)
    bt = np.full((8, 16), ONE, dtype=np.uint8)
    for out_bf16 in (False, True):
        got = fp8gemm_f32acc_block(a, bt, np.array([[-1.0]]), np.array([[1.0]]), out_bf16)
        assert np.all(got == 0x8000), got
    # the same problem in the per-tensor oracle gives the same bits: the ambiguous shape (M = 1, K, N <= 128)
    from oracle import fp8 as fp8_oracle
    assert np.array_equal(fp8_oracle.fp8gemm_f32acc(a, bt, -1.0, 1.0, False),
                          fp8gemm_f32acc_block(a, bt, np.array([[-1.0]]), np.array([[1.0]]), False))


def test_reference_split_sums_start_from_positive_zero():
    a = np.zeros((1, 256), dtype=np.uint8)
    bt = np.full((8, 256), ONE, dtype=np.uint8)
    sa = np.array([[-1.0, -1.0]], dtype=np.float32)
    assert np.all(fp8gemm_f32acc_block(a, bt, sa, np.ones((1, 2)), False, 1) == 0x8000)
    assert np.all(fp8gemm_f32acc_block(a, bt, sa, np.ones((1, 2)), False, 2) == 0)      # +0 + -0 + -0 = +0


def _aligned(buf) -> int:
    return (ctypes.addressof(buf) + 15) & ~15


def test_blockwise_argument_validation_happens_before_any_cuda_call(built_libs):
    lib = capi.fp8block_lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = _aligned(buf)
    s = p + 4096
    f = lib.b200_fp8gemm_blockwise
    assert f(p, p, p, None, 64, s, 0, 64, 64, 64, None) == -5                       # null scales
    assert f(p, p, p, s, 64, None, 1, 64, 64, 64, None) == -5
    assert f(p, p, p, s + 4, 64, s, 0, 64, 64, 64, None) == -2                      # scale_a: 16-byte aligned
    assert f(p, p, p, s, 64, s + 2, 0, 64, 64, 64, None) == -2                      # scale_b: 4-byte aligned
    assert f(p, p, p, s, 60, s, 0, 64, 64, 64, None) == -10                         # ld_a < M
    assert f(p, p, p, s, 66, s, 0, 64, 64, 64, None) == -10                         # ld_a % 4
    assert f(p, p, p, s, 64, s, 0, 64, 64, 72, None) == -9                          # K % 16
    assert f(p, p, p, s, 64, s, 0, 64, 60, 64, None) == -2                          # N % 8
    assert f(p, p, p, s, 64, s, 0, 64, 64, 0, None) == -1
    assert f(p, p, p, s, 64, s, 2, 64, 64, 64, None) == -6                          # bad output selector
    r = lib.b200_fp8gemm_blockwise_run_config
    assert r(99, 0, p, p, p, s, 64, s, 64, 64, 64, 0, 0, 1, None) == -6              # unknown config
    for cfg in sorted(set(range(31)) - set(ELIGIBLE)):
        assert r(cfg, 0, p, p, p, s, 64, s, 64, 64, 64, 0, 0, 1, None) == -6, cfg   # no block-scaled kernel
    assert r(1, 2, p, p, p, s, 64, s, 64, 64, 64, 0, 0, 1, None) == -6
    assert r(1, 1, p, p, p, s + 4, 64, s, 64, 64, 64, 0, 0, 1, None) == -2
    assert r(1, 1, p, p, p, s, 64, None, 64, 64, 64, 0, 0, 1, None) == -5
    assert r(4, 0, p, p, p, s, 63, s, 64, 64, 64, 0, 0, 1, None) == -10
    assert r(4, 0, p, p, p, s, 64, s, 64, 64, 40, 0, 0, 1, None) == -9
    assert "ld_a" in lib.b200_fp8block_strerror(-10).decode()
    assert lib.b200_fp8block_launch_count() == 0 and capi.fp8block_launch_count() == 0
    assert capi.launch_count() == 0


DECL = re.compile(r"^\s*(?:const\s+)?(?:unsigned\s+long\s+long|int|void|char\s*\*|const\s+char\s*\*)\s*\*?\s*(b200_\w+)\s*\(", re.M)


def test_header_binding_and_library_exports_agree(built_libs):
    declared = sorted(set(DECL.findall((REPO / "include" / "b200_fp8_block.h").read_text())))
    assert declared == sorted(capi.exported_symbols()["libb200_fp8block.so"])
    assert built_libs["fp8block"].name == "libb200_fp8block.so"
    lib = ctypes.CDLL(str(built_libs["fp8block"]))
    for sym in declared:
        assert hasattr(lib, sym), sym
    # the product library does not carry them
    assert not any(hasattr(capi.hgemm_lib(), sym) for sym in declared)


def block_choice(cfg, gm, sp):
    """The mapping rule, restated from the configuration table: same CTA group and cluster, M_REP 1, BN min(BN, 128);
    workspace split-K s -> cluster split-K of the largest of 8/4/2 <= s where the configuration has split-K kernels,
    stream-K -> plain."""
    cfgs = capi.configs()
    c = cfgs[cfg]
    sib = [d["id"] for d in cfgs if (d["cta_group"], d["cluster_m"], d["cluster_n"], d["m_rep"], d["bn"]) ==
           (c["cta_group"], c["cluster_m"], c["cluster_n"], 1, min(c["bn"], 128))]
    assert len(sib) == 1
    s = sib[0]
    d = cfgs[s]
    split_k = d["cta_group"] == 1 and d["cluster_m"] * d["cluster_n"] == 1 and d["bn"] >= 64 and d["m_rep"] == 1
    if not split_k or sp in (capi.STREAMK_TAIL, capi.STREAMK_TAIL_PLUS_WAVE) or -1 <= sp <= 1:
        return s, gm, 1
    if sp > 1:
        return s, gm, -8 if sp >= 8 else -4 if sp >= 4 else -2
    return s, gm, sp


def test_eligible_set_and_mapping_rule(built_libs):
    cfgs = capi.configs()
    assert tuple(d["id"] for d in cfgs if d["m_rep"] * d["bn"] <= 128) == ELIGIBLE
    want = {3: 4, 6: 4, 26: 4, 0: 1, 29: 30, 20: 22, 24: 22, 28: 22}
    for cfg, sib in want.items():
        assert block_choice(cfg, 0, 1)[0] == sib
    for cfg in range(31):
        assert block_choice(cfg, 0, 1)[0] in ELIGIBLE
        if cfg in ELIGIBLE:
            assert block_choice(cfg, 0, 1)[0] == cfg


def test_dispatch_maps_the_e4m3_choice(built_libs):
    from cuda_l2_b200 import farm
    shapes = list(farm.grid_shapes())
    assert len(shapes) == 1001
    rng = random.Random(20261016)
    shapes += [(rng.randrange(1, 20000), 8 * rng.randrange(1, 2500), 16 * rng.randrange(1, 2000)) for _ in range(2000)]
    seen = set()
    for m, n, k in shapes:
        got = capi.fp8_blockwise_select(m, n, k)
        assert got == block_choice(*capi.fp8_select(m, n, k)), (m, n, k)
        assert got[0] in ELIGIBLE and got[2] in (1, -2, -4, -8)
        seen.add(got[2])
    assert seen >= {1, -2, -4, -8}


def _meta(*shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device="meta")


def test_blockwise_scale_rule_and_operator_shapes_on_meta_tensors():
    from cuda_l2_b200 import ops
    a, b = _meta(200, 400, dtype=E4), _meta(328, 400, dtype=E4)         # nkb = 4, ceil(328 / 128) = 3
    assert capi.scale_granularity(200, 328, _meta(200, 4), _meta(3, 4), k=400) == "blockwise"
    assert capi.scale_granularity(200, 328, _meta(200, 4), _meta(3, 4)) == "blockwise"
    assert capi.scale_granularity(1, 128, _meta(1, 1), _meta(1, 1), k=128) == "tensor"   # the shapes coincide
    assert capi.scale_granularity(200, 328, _meta(200, 1), _meta(1, 328), k=400) == "rowwise"
    for dt in (torch.float16, torch.bfloat16):
        y = ops.fp8_gemm(a, b, _meta(200, 4), _meta(3, 4), dt)
        assert y.shape == (200, 328) and y.dtype == dt and y.device.type == "meta"
        y = ops.fp8_gemm(a, b, _meta(4, 200).t(), _meta(3, 4), dt)      # the M-major view
        assert y.shape == (200, 328)


@pytest.mark.parametrize("sa,sb", [
    ((200, 3), (3, 4)),          # nkb of scale_a
    ((200, 4), (3, 3)),          # nkb of scale_b
    ((200, 4), (2, 4)),          # ceil(N / 128)
    ((200, 4), (4, 4)),
    ((199, 4), (3, 4)),          # M
    ((4, 200), (3, 4)),          # transposed
    ((200, 4), (4, 3)),          # scale_b transposed
    ((200, 4), (1, 328)),        # mixed with rowwise
    ((200, 1), (3, 4)),
    ((200, 4), (1,)),            # mixed with per tensor
])
def test_blockwise_scale_shapes_that_are_rejected(sa, sb):
    from cuda_l2_b200 import ops
    a, b = _meta(200, 400, dtype=E4), _meta(328, 400, dtype=E4)
    with pytest.raises(capi.B200HgemmError):
        ops.fp8_gemm(a, b, _meta(*sa), _meta(*sb), torch.float16)
    with pytest.raises(capi.B200HgemmError):
        ops.fp8_gemm(a, b, _meta(200, 4, dtype=torch.float16), _meta(3, 4), torch.float16)


def test_blockwise_ld_a_reads_the_layout():
    s = torch.zeros((3, 200))                       # [nkb, ld_a] buffer
    assert capi.blockwise_ld_a(s[:, :197].t()) == 200
    assert capi.blockwise_ld_a(s.t()) == 200
    assert capi.blockwise_ld_a(torch.zeros((197, 3))) is None                 # contiguous [M, nkb]: not M-major
    assert capi.blockwise_ld_a(torch.zeros((3, 198))[:, :197].t()) is None    # ld_a % 4
    assert capi.blockwise_ld_a(torch.zeros(3 * 200 + 1)[1:].view(3, 200)[:, :197].t()) is None   # 16-byte alignment
    short = torch.zeros(2 * 200 + 197)                                        # the last row is not ld_a long
    assert capi.blockwise_ld_a(short.as_strided((197, 3), (1, 200))) is None
    assert capi.blockwise_ld_a(torch.zeros((1, 5))[:, :3].t()) == 4                # nkb = 1: ld_a = M rounded up to 4


def test_blockwise_python_binding_checks_before_the_library():
    a = torch.zeros((64, 256), dtype=E4)
    c = torch.zeros((64, 64), dtype=torch.half)
    with pytest.raises(capi.B200HgemmError):
        capi.fp8_gemm(a, a[:64], c, torch.ones(64, 2), torch.ones(1, 2))       # CPU tensors: no fallback


def test_quantize_e4m3_blockwise():
    from cuda_l2_b200 import ops
    x = torch.randn(6, 300, dtype=torch.float16)
    x[2, 130:140] *= 1000
    x[4] = 0
    q, s = ops.quantize_e4m3_blockwise(x)
    assert q.dtype == E4 and q.shape == x.shape and q.is_contiguous()
    assert s.dtype == torch.float32 and s.shape == (6, 3) and s.stride() == (1, 8)    # ld_a = 6 rounded up to 4
    assert capi.blockwise_ld_a(s) == 8
    xp = torch.nn.functional.pad(x.float(), (0, 84)).view(6, 3, 128)
    assert torch.equal(s, (xp.abs().amax(dim=2) / 448).clamp_min(torch.finfo(torch.float32).tiny))
    assert torch.equal(q.float()[4], torch.zeros(300))
    s_el = s.repeat_interleave(128, dim=1)[:, :300]
    # e4m3 keeps 3 mantissa bits (half an ulp: 2^-4 relative); its subnormals are 2^-9 apart, times the block's scale
    assert bool(((q.float() * s_el - x.float()).abs() <= 2 ** -4 * x.float().abs() + 2 ** -10 * s_el).all())
    assert float(s[2, 1]) > 100 * float(s[2, 0])                              # the outlier stays in its block


def test_quantize_e4m3_block128x128():
    from cuda_l2_b200 import ops
    w = torch.randn(200, 300)
    w[130:140, 10:20] *= 1000
    q, s = ops.quantize_e4m3_block128x128(w)
    assert q.dtype == E4 and q.shape == w.shape and s.shape == (2, 3) and s.is_contiguous()
    wp = torch.nn.functional.pad(w, (0, 84, 0, 56)).view(2, 128, 3, 128)
    assert torch.equal(s, (wp.abs().amax(dim=(1, 3)) / 448).clamp_min(torch.finfo(torch.float32).tiny))
    s_el = s.repeat_interleave(128, dim=0)[:200].repeat_interleave(128, dim=1)[:, :300]
    assert bool(((q.float() * s_el - w).abs() <= 2 ** -4 * w.abs() + 2 ** -10 * s_el).all())
    assert float(s[1, 0]) > 100 * float(s[0, 0])


def test_fp8_linear_blockwise_buffers():
    from cuda_l2_b200 import ops
    assert ops.FP8_GRANULARITIES == ("tensor", "rowwise", "blockwise")
    lin = nn.Linear(272, 200, dtype=torch.bfloat16)
    m = ops.B200Fp8Linear.from_linear(lin, granularity="blockwise")
    assert m.granularity == "blockwise" and m.weight_scale.shape == (2, 3) and m.weight_scale.dtype == torch.float32
    assert m.weight_fp8.dtype == E4 and m.weight_fp8.shape == (200, 272) and m.bias is lin.bias
    assert set(dict(m.named_buffers())) == {"weight_fp8", "weight_scale"} and "granularity=blockwise" in repr(m)
    with pytest.raises(capi.B200HgemmError):
        ops.B200Fp8Linear.from_linear(lin, granularity="block")


def test_fp8_linear_from_fp8_takes_the_checkpoint_as_it_is():
    from cuda_l2_b200 import ops
    w = torch.randn(200, 272).to(E4)
    s = torch.rand(2, 3) + 0.5
    bias = torch.randn(200, dtype=torch.bfloat16)
    m = ops.B200Fp8Linear.from_fp8(w, s, bias)
    assert m.granularity == "blockwise" and m.out_dtype == torch.bfloat16
    assert (m.in_features, m.out_features) == (272, 200) and m.bias is bias
    assert torch.equal(m.weight_fp8.view(torch.uint8), w.view(torch.uint8)) and torch.equal(m.weight_scale, s)
    assert ops.B200Fp8Linear.from_fp8(w, s, out_dtype=torch.float16).out_dtype == torch.float16
    for bad_w, bad_s in ((w, torch.rand(3, 2)), (w, s.double()), (w.float(), s), (w[:, :264], s[:, :2]),
                         (torch.randn(196, 272).to(E4), s)):
        with pytest.raises(capi.B200HgemmError):
            ops.B200Fp8Linear.from_fp8(bad_w, bad_s)


def test_block_scaled_sass(built_libs):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sys.path.insert(0, str(REPO / "tools"))
    import sass_summary
    sass = subprocess.run([cuobjdump, "-sass", str(built_libs["fp8block"])], capture_output=True, text=True,
                          check=True).stdout
    kernels = sass_summary.sass_by_kernel(sass)
    # 17 configurations x 2 output types plain, and configurations 1 and 2 with cluster split-K
    assert len(kernels) == 2 * (17 + 2)
    assert all("BlockScaled" in name for name in kernels)
    for name, insns in kernels.items():
        assert any(op.startswith("QGMMA") for _, op, _ in insns), name
        assert not any(op.startswith(("HGMMA", "HMMA")) for _, op, _ in insns), name
        loop = sass_summary.k_loop(insns)
        assert any(op == "WARPGROUP.ARRIVE" for _, op, _ in loop), name
        assert any(op.startswith("SYNCS.ARRIVE") for _, op, _ in loop), name
        assert any(op == "FFMA" for _, op, _ in loop), name                  # the promotion is inside the k-loop
        assert sass_summary.k_loop_gpu_membars(insns) == 0, name
