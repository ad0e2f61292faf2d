"""Block-scaled FP8 batched GEMM with per-batch row counts (the MoE decode layout) without a GPU: the C ABI of
libb200_batched_fp8.so (exports, statuses before any CUDA call, the dispatcher rule, also on extreme shapes), the
operator's schema, shape inference and scale-shape errors, the quantiser's batched form, B200Fp8GroupedLinear's masked
forward on meta tensors, and the SASS of the kernels."""
import ctypes
import json
import os
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

E4 = torch.float8_e4m3fn
ELIGIBLE = (1, 2, 4, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 22, 23, 30)
NUM_CONFIGS = 31
INT_MAX = 2 ** 31 - 1
DECL = re.compile(r"^\s*(?:const\s+)?(?:unsigned\s+long\s+long|int|void|char\s*\*|const\s+char\s*\*)\s*\*?\s*(b200_\w+)\s*\(", re.M)


def test_header_binding_and_library_exports_agree(built_libs):
    declared = sorted(set(DECL.findall((REPO / "include" / "b200_batched_fp8.h").read_text())))
    assert declared == sorted(capi.exported_symbols()["libb200_batched_fp8.so"])
    assert built_libs["batched_fp8"].name == "libb200_batched_fp8.so"
    lib = ctypes.CDLL(str(built_libs["batched_fp8"]))
    for sym in declared:
        assert hasattr(lib, sym), sym
    for other in (capi.hgemm_lib(), capi.fp8block_lib(), capi.batched_lib(), capi.grouped_fp8_lib()):
        assert not any(hasattr(other, sym) for sym in declared)   # none of the others carries them


def _aligned(buf) -> int:
    return (ctypes.addressof(buf) + 15) & ~15


def test_argument_validation_happens_before_any_cuda_call(built_libs):
    lib = capi.batched_fp8_lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = _aligned(buf)
    s, mm = p + 4096, p + 8192
    M = 64

    def g(a=p, b=p, c=p, sa=s, ld=M, sb=s, out=0, mask=mm, B=4, m=M, n=64, k=64):
        return lib.b200_batched_fp8_gemm(a, b, c, sa, ld, sb, out, mask, B, m, n, k, None)

    def r(cfg=1, out=0, a=p, b=p, c=p, sa=s, ld=M, sb=s, mask=mm, B=4, m=M, n=64, k=64):
        return lib.b200_batched_fp8_gemm_run_config(cfg, out, a, b, c, sa, ld, sb, mask, B, m, n, k, 0, 0, None)

    for f in (g, lambda **kw: r(cfg=1, **kw), lambda **kw: r(cfg=30, **kw)):
        for out in (0, 1):
            for mask in (mm, None):                                              # masked and dense
                assert f(out=out, mask=mask, a=None) == -5 and f(out=out, mask=mask, b=None) == -5
                assert f(out=out, mask=mask, c=None) == -5                       # operands
                assert f(out=out, mask=mask, sa=None) == -5 and f(out=out, mask=mask, sb=None) == -5   # scales
                assert f(out=out, mask=mask, sa=s + 4) == -2                     # scale_a: 16-byte aligned
                assert f(out=out, mask=mask, sb=s + 2) == -2                     # scale_b: 4-byte aligned
                assert f(out=out, mask=mask, a=p + 8) == -2 and f(out=out, mask=mask, b=p + 8) == -2
                assert f(out=out, mask=mask, c=p + 8) == -2
                assert f(out=out, mask=mask, ld=M - 4) == -10 and f(out=out, mask=mask, ld=M + 2) == -10
                assert f(out=out, mask=mask, k=72) == -9                         # K % 16
                assert f(out=out, mask=mask, n=60) == -2                         # N % 8
                assert f(out=out, mask=mask, B=0) == -1 and f(out=out, mask=mask, B=-3) == -1   # B <= 0
                assert f(out=out, mask=mask, m=0) == -1 and f(out=out, mask=mask, m=-1) == -1   # M <= 0
                assert f(out=out, mask=mask, n=0) == -1 and f(out=out, mask=mask, k=0) == -1
            assert f(out=out, mask=mm + 2) == -2                                 # masked_m: 4-byte aligned
    for out in (2, -1):                                                          # bad output selector
        assert g(out=out) == -6 and r(out=out) == -6
    for cfg in sorted(set(range(-1, NUM_CONFIGS + 1)) - set(ELIGIBLE)):         # no block-scaled kernel
        assert r(cfg=cfg) == -6 and r(cfg=cfg, out=1) == -6, cfg
    for cfg in ELIGIBLE:
        # tile count B * ceil(M / block rows) * column blocks past INT_MAX
        assert r(cfg=cfg, B=4, m=INT_MAX - 3, ld=INT_MAX - 3, n=INT_MAX - 7) == -1, cfg
    assert g(B=2 * 10 ** 9, m=2 * 10 ** 9, ld=2 * 10 ** 9, n=1024) == -1        # every configuration past the bound
    assert lib.b200_batched_fp8_select(0, 64, 64, 64, None, None) == -1
    assert lib.b200_batched_fp8_select(4, 0, 64, 64, None, None) == -1
    assert "ld_a" in lib.b200_batched_fp8_strerror(-10).decode()
    assert lib.b200_batched_fp8_launch_count() == 0 and capi.fp8_batched_launch_count() == 0
    # M <= 0: the status of the 16-bit batched call
    assert capi.batched_lib().b200_batched_gemm(0, p, p, p, None, 4, 0, 64, 64, None) == g(m=0) == -1


def sibling(cfg: int) -> int:
    """The block-scaled stand-in of a configuration, restated from the table: the same CTA group and cluster, M_REP 1,
    BN min(BN, 128)."""
    cfgs = capi.configs()
    c = cfgs[cfg]
    sib = [d["id"] for d in cfgs if (d["cta_group"], d["cluster_m"], d["cluster_n"], d["m_rep"], d["bn"]) ==
           (c["cta_group"], c["cluster_m"], c["cluster_n"], 1, min(c["bn"], 128))]
    assert len(sib) == 1 and sib[0] in ELIGIBLE
    return sib[0]


def rule(b, m, n, k):
    """The batched 16-bit rule (fp32 accumulation) for e4m3 operands, which read the tuned table at K / 2, mapped to
    the block-scaled sibling."""
    cfg, gm = capi.batched_select(0, b, m, n, max(k // 2, 1))
    return sibling(cfg), gm


def test_dispatch_is_the_block_scaled_sibling_of_the_batched_rule(built_libs):
    rng = random.Random(20261017)
    shapes = [(32, 128, 4096, 7168), (32, 512, 7168, 2048), (256, 64, 2048, 7168), (1, 100, 8, 16),
              (128, 1, 512, 64), (8, 4096, 4096, 4096)]
    shapes += [(rng.randrange(1, 300), rng.randrange(1, 5000), 8 * rng.randrange(1, 1500), 16 * rng.randrange(1, 800))
               for _ in range(300)]
    seen = set()
    for b, m, n, k in shapes:
        got = capi.fp8_batched_select(b, m, n, k)
        assert got == rule(b, m, n, k), (b, m, n, k)
        seen.add(got[0])
    assert len(seen) >= 3


_EXTREMES = r"""
import ctypes, json, sys
sys.path.insert(0, {repo!r})
from cuda_l2_b200 import capi
INT_MAX = 2 ** 31 - 1
i = ctypes.c_int
out = {{"select": [], "gemm": []}}
bl, fl = capi.batched_lib(), capi.batched_fp8_lib()
bm = [(1, 1), (1, INT_MAX), (2, INT_MAX), (INT_MAX, 1), (INT_MAX, INT_MAX), (2 * 10 ** 9, 2 * 10 ** 9),
      (256, 10 ** 7), (3, 10 ** 9), (10 ** 6, 4096)]
for b, m in bm:
    for n in (8, 64, 4096, INT_MAX - 7):
        for k in (16, 4096, INT_MAX - 15):
            c, gm, c16, gm16 = i(-99), i(-99), i(-99), i(-99)
            st = fl.b200_batched_fp8_select(b, m, n, k, ctypes.byref(c), ctypes.byref(gm))
            st16 = bl.b200_batched_select(0, b, m, n, k // 2, ctypes.byref(c16), ctypes.byref(gm16))
            out["select"].append([b, m, n, k, st, c.value, gm.value, st16, c16.value, gm16.value])
buf = ctypes.create_string_buffer(1 << 12)
p = (ctypes.addressof(buf) + 15) & ~15
# shapes whose every block-scaled configuration's tile list passes INT_MAX: refused before any device call
# (M is a multiple of 4, so that ld_a = M is valid)
for b, m, n in ((2 * 10 ** 9, 2 * 10 ** 9, 1024), (INT_MAX, INT_MAX - 3, 4096), (2, INT_MAX - 3, INT_MAX - 7)):
    for out_bf16 in (0, 1):
        for mask in (p, None):
            st = fl.b200_batched_fp8_gemm(p, p, p, p, m, p, out_bf16, mask, b, m, n, 64, None)
            out["gemm"].append([b, m, n, out_bf16, st])
print(json.dumps(out))
"""


def test_selector_is_total_and_refuses_before_the_device_on_extreme_shapes(built_libs):
    r = subprocess.run([sys.executable, "-c", _EXTREMES.format(repo=str(REPO))], capture_output=True, text=True,
                       timeout=600, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, f"the selector process died (status {r.returncode}):\n{r.stderr[-2000:]}"
    out = json.loads(r.stdout)
    assert len(out["select"]) == 9 * 4 * 3
    for b, m, n, k, st, cfg, gm, st16, cfg16, gm16 in out["select"]:
        assert st == 0 and st16 == 0 and gm >= 0, (b, m, n, k, st, cfg)
        assert (cfg, gm) == (sibling(cfg16), gm16), (b, m, n, k, cfg, cfg16)
    assert len(out["gemm"]) == 12
    for b, m, n, out_bf16, st in out["gemm"]:
        assert st == -1, (b, m, n, out_bf16, st)             # kBadShape


def _meta(*shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device="meta")


def test_operator_schema_and_meta_shapes():
    from cuda_l2_b200 import ops
    schema = str(torch.ops.cuda_l2_b200.fp8_batched_gemm.default._schema)
    assert schema == ("cuda_l2_b200::fp8_batched_gemm(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, "
                      "ScalarType out_dtype, Tensor? masked_m=None) -> Tensor")
    assert {"fp8_batched_gemm", "B200Fp8GroupedLinear"} <= set(ops.__all__)
    a, b = _meta(6, 90, 400, dtype=E4), _meta(6, 328, 400, dtype=E4)        # nkb = 4, ceil(328 / 128) = 3
    mm = _meta(6, dtype=torch.int32)
    for dt in (torch.float16, torch.bfloat16):
        for mask in (mm, None):
            y = ops.fp8_batched_gemm(a, b, _meta(6, 90, 4), _meta(6, 3, 4), dt, mask)
            assert y.shape == (6, 90, 328) and y.dtype == dt and y.device.type == "meta"
        y = ops.fp8_batched_gemm(a, b, _meta(6, 4, 92)[:, :, :90].transpose(1, 2), _meta(6, 3, 4), dt, mm)   # in place
        assert y.shape == (6, 90, 328)
    assert ops.fp8_batched_gemm(_meta(6, 0, 400, dtype=E4), b, _meta(6, 0, 4), _meta(6, 3, 4)).shape == (6, 0, 328)
    assert ops.fp8_batched_gemm(_meta(0, 90, 400, dtype=E4), _meta(0, 328, 400, dtype=E4), _meta(0, 90, 4),
                                _meta(0, 3, 4)).shape == (0, 90, 328)
    assert capi.check_batched_operands(a, b, "fp32", mm, torch.float16, (_meta(6, 90, 4), _meta(6, 3, 4))) == \
        (6, 90, 328, 400)
    # the 16-bit form is unchanged
    assert capi.check_batched_operands(_meta(6, 90, 400, dtype=torch.half), _meta(6, 328, 400, dtype=torch.half)) == \
        (6, 90, 328, 400)


@pytest.mark.parametrize("sa,sb", [
    ((6, 90, 3), (6, 3, 4)),         # nkb of scale_a
    ((6, 90, 4), (6, 3, 3)),         # nkb of scale_b
    ((6, 90, 4), (6, 2, 4)),         # ceil(N / 128)
    ((6, 90, 4), (5, 3, 4)),         # B of scale_b
    ((5, 90, 4), (6, 3, 4)),         # B of scale_a
    ((90, 4), (6, 3, 4)),            # the 2-D blockwise scale_a
    ((6, 90, 4), (3, 4)),            # the 2-D blockwise scale_b
    ((6, 89, 4), (6, 3, 4)),         # M
    ((6, 4, 90), (6, 3, 4)),         # transposed
    ((6, 90, 1), (6, 1, 328)),       # rowwise
    ((1,), (1,)),                    # per tensor
])
def test_scale_shapes_that_are_rejected(sa, sb):
    from cuda_l2_b200 import ops
    a, b = _meta(6, 90, 400, dtype=E4), _meta(6, 328, 400, dtype=E4)
    with pytest.raises(capi.B200HgemmError):
        ops.fp8_batched_gemm(a, b, _meta(*sa), _meta(*sb), torch.bfloat16, _meta(6, dtype=torch.int32))


def test_operand_errors():
    from cuda_l2_b200 import ops
    sa, sb, mm = _meta(6, 90, 4), _meta(6, 3, 4), _meta(6, dtype=torch.int32)
    a, b = _meta(6, 90, 400, dtype=E4), _meta(6, 328, 400, dtype=E4)
    bad = [
        (a, _meta(6, 328, 384, dtype=E4), sa, sb, torch.bfloat16, mm),                              # K
        (_meta(6, 90, 408, dtype=E4), _meta(6, 328, 408, dtype=E4), sa, sb, torch.bfloat16, mm),   # K % 16
        (a, _meta(6, 324, 400, dtype=E4), sa, sb, torch.bfloat16, mm),                              # N % 8
        (a, _meta(328, 400, dtype=E4), sa, sb, torch.bfloat16, mm),                                 # 2-D b
        (a, _meta(5, 328, 400, dtype=E4), sa, sb, torch.bfloat16, mm),                              # batch counts
        (a, b, sa, sb, torch.bfloat16, _meta(5, dtype=torch.int32)),                                # B of masked_m
        (a, b, sa, sb, torch.bfloat16, _meta(6, dtype=torch.int64)),                                # int32 counts
        (a, b, sa, sb, torch.float32, mm),                                                          # output type
        (_meta(6, 90, 400, dtype=torch.bfloat16), _meta(6, 328, 400, dtype=torch.bfloat16), sa, sb, torch.bfloat16,
         mm),                                                                                       # 16-bit operands
        (a, b, sa.half(), sb, torch.bfloat16, mm),                                                  # fp32 scales
    ]
    for args in bad:
        with pytest.raises(capi.B200HgemmError):
            ops.fp8_batched_gemm(*args)


def test_operator_has_no_cpu_path():
    from cuda_l2_b200 import ops
    a, b = torch.zeros((2, 32, 128), dtype=E4), torch.zeros((2, 16, 128), dtype=E4)
    sa, sb, mm = torch.ones(2, 32, 1), torch.ones(2, 1, 1), torch.tensor([10, 32], dtype=torch.int32)
    with pytest.raises(capi.B200HgemmError, match="no CPU implementation"):
        ops.fp8_batched_gemm(a, b, sa, sb, torch.bfloat16, mm)
    with pytest.raises(capi.B200HgemmError):
        capi.fp8_batched_gemm(a, b, torch.zeros((2, 32, 16), dtype=torch.bfloat16), sa, sb, mm)


def test_backward_raises_inference_only():
    from cuda_l2_b200 import ops
    a, b = _meta(2, 32, 128, dtype=E4), _meta(2, 16, 128, dtype=E4)
    sa = _meta(2, 32, 1).requires_grad_()
    y = ops.fp8_batched_gemm(a, b, sa, _meta(2, 1, 1), torch.bfloat16, _meta(2, dtype=torch.int32))
    assert y.requires_grad
    with pytest.raises(capi.B200HgemmError, match="inference only"):
        y.sum().backward()


def test_batched_quantiser_is_the_2d_quantiser_on_each_matrix_with_in_place_strides():
    from cuda_l2_b200 import ops
    g = torch.Generator().manual_seed(4)
    for shape in ((3, 90, 272), (1, 128, 128), (4, 37, 1040), (2, 8, 16), (5, 1, 300), (2, 6, 128)):
        x = torch.randn(shape, generator=g)
        x[0, :3, :7] *= 1000
        q, s = ops.quantize_e4m3_blockwise(x)
        bsz, m, k = shape
        nkb, ld = -(-k // 128), -(-m // 4) * 4
        assert q.dtype == E4 and q.shape == x.shape and q.is_contiguous()
        assert s.shape == (bsz, m, nkb) and s.dtype == torch.float32
        assert s.stride() == (nkb * ld, 1, ld) and s.untyped_storage().nbytes() == 4 * bsz * nkb * ld
        assert capi.blockwise_ld_a(s) == ld
        for b in range(bsz):
            q2, s2 = ops.quantize_e4m3_blockwise(x[b])
            assert torch.equal(q[b].view(torch.uint8), q2.view(torch.uint8)) and torch.equal(s[b], s2), (shape, b)
            assert capi.blockwise_ld_a(s2) == ld
    with pytest.raises(capi.B200HgemmError):
        ops.quantize_e4m3_blockwise(torch.randn(2, 2, 8, 128))


def test_batched_ld_a_rules():
    buf = torch.zeros(3, 4, 100)                     # [B, nkb, ld_a] with ld_a = 100
    s = buf[:, :, :90].transpose(1, 2)
    assert capi.blockwise_ld_a(s) == 100
    assert capi.blockwise_ld_a(torch.zeros(3, 90, 4)) is None                          # row-major
    assert capi.blockwise_ld_a(torch.zeros(3, 4, 90).transpose(1, 2)) is None          # ld_a = 90: % 4
    assert capi.blockwise_ld_a(torch.zeros(4, 3, 100)[:, :, :90].transpose(0, 2).transpose(0, 1)) is None
    gap = torch.zeros(3, 5, 100)                     # batch stride 500 != nkb * ld_a = 400
    assert capi.blockwise_ld_a(gap[:, :4, :90].transpose(1, 2)) is None
    assert capi.blockwise_ld_a(torch.zeros(3, 4, 100)[:2, :, :90].transpose(1, 2)) == 100   # fewer batches
    short = torch.zeros(1190).as_strided((3, 90, 4), (400, 1, 100))   # B * nkb * ld_a = 1200 floats not readable
    assert capi.blockwise_ld_a(short) is None
    assert capi.blockwise_ld_a(torch.zeros(1200).as_strided((3, 90, 4), (400, 1, 100))) == 100
    one = torch.zeros(3, 1, 92)                      # one k-block: the batch stride is ld_a
    assert capi.blockwise_ld_a(one[:, :, :90].transpose(1, 2)) == 92


def test_masked_forward_on_meta_tensors():
    from cuda_l2_b200 import ops
    w = torch.empty((4, 200, 272), dtype=E4, device="meta")
    s = torch.empty((4, 2, 3), dtype=torch.float32, device="meta")
    m = ops.B200Fp8GroupedLinear.from_fp8(w, s)
    mm = torch.empty((4,), dtype=torch.int32, device="meta")
    for x_dtype in (torch.bfloat16, torch.float16):
        y = m.forward_masked(torch.empty((4, 90, 272), dtype=x_dtype, device="meta"), mm)
        assert y.shape == (4, 90, 200) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    with pytest.raises(capi.B200HgemmError):
        m.forward_masked(torch.empty((3, 90, 272), device="meta"), torch.empty((3,), dtype=torch.int32, device="meta"))
    with pytest.raises(capi.B200HgemmError):
        m.forward_masked(torch.empty((4, 90, 272), device="meta"), torch.empty((5,), dtype=torch.int32, device="meta"))


def test_batched_fp8_sass(built_libs):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sys.path.insert(0, str(REPO / "tools"))
    import sass_summary
    sass = subprocess.run([cuobjdump, "-sass", str(built_libs["batched_fp8"])], capture_output=True, text=True,
                          check=True).stdout
    kernels = sass_summary.sass_by_kernel(sass)
    assert len(kernels) == 2 * len(ELIGIBLE)                                 # plain only, two output types
    assert all(re.search(r"BatchedINS_11BlockScaledINS_6ConfigI.*ELi0EEEv14CUtensorMap", name) for name in kernels)
    for name, insns in kernels.items():
        ops_ = {op for _, op, _ in insns}
        assert any(op.startswith("QGMMA") for op in ops_), name              # FP8 wgmma
        assert not any(op.startswith(("HGMMA", "HMMA")) for op in ops_), name
        assert any(op.startswith("UTMALDG.3D") for op in ops_), name        # A [B, M, K] and Bt [B, N, K]
        assert not any(op.startswith("UTMALDG.2D") for op in ops_), name    # both operands through 3-D maps
        assert any(op.startswith("UBLKCP") for op in ops_), name            # the bulk copy of A's scales
        assert "UTMASTG.3D" in ops_, name                                   # boxes of C [B, M, N]
        loop = sass_summary.k_loop(insns)
        assert any(op == "WARPGROUP.ARRIVE" for _, op, _ in loop), name
        assert any(op.startswith("SYNCS.ARRIVE") for _, op, _ in loop), name   # the stage release is inside
        assert any(op == "FFMA" for _, op, _ in loop), name                  # the promotion is inside the k-loop
        assert sass_summary.k_loop_gpu_membars(insns) == 0, name
