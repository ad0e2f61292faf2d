"""Block-scaled FP8 grouped GEMM over contiguous row groups without a GPU: the C ABI of libb200_grouped_fp8.so (exports,
statuses before any CUDA call, the dispatcher rule, also on extreme shapes), the operator's schema, shape inference and
scale-shape errors, the quantiser's per-expert form, B200Fp8GroupedLinear's buffers, and the SASS of the kernels."""
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
    declared = sorted(set(DECL.findall((REPO / "include" / "b200_grouped_fp8.h").read_text())))
    assert declared == sorted(capi.exported_symbols()["libb200_grouped_fp8.so"])
    assert built_libs["grouped_fp8"].name == "libb200_grouped_fp8.so"
    lib = ctypes.CDLL(str(built_libs["grouped_fp8"]))
    for sym in declared:
        assert hasattr(lib, sym), sym
    for other in (capi.hgemm_lib(), capi.fp8block_lib(), capi.grouped_lib()):   # none of the others carries them
        assert not any(hasattr(other, sym) for sym in declared)


def _aligned(buf) -> int:
    return (ctypes.addressof(buf) + 15) & ~15


def test_argument_validation_happens_before_any_cuda_call(built_libs):
    lib = capi.grouped_fp8_lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = _aligned(buf)
    s, offs = p + 4096, p + 8192
    T = 64

    def g(a=p, b=p, c=p, sa=s, ld=T, sb=s, out=0, o=offs, G=4, t=T, n=64, k=64):
        return lib.b200_grouped_fp8_gemm(a, b, c, sa, ld, sb, out, o, G, t, n, k, None)

    def r(cfg=1, out=0, a=p, b=p, c=p, sa=s, ld=T, sb=s, o=offs, G=4, t=T, n=64, k=64):
        return lib.b200_grouped_fp8_gemm_run_config(cfg, out, a, b, c, sa, ld, sb, o, G, t, n, k, 0, 0, None)

    for f in (g, lambda **kw: r(cfg=1, **kw), lambda **kw: r(cfg=30, **kw)):
        for out in (0, 1):
            assert f(out=out, a=None) == -5 and f(out=out, b=None) == -5 and f(out=out, c=None) == -5   # operands
            assert f(out=out, sa=None) == -5 and f(out=out, sb=None) == -5                             # scales
            assert f(out=out, o=None) == -5                                                            # offsets
            assert f(out=out, sa=s + 4) == -2                                    # scale_a: 16-byte aligned
            assert f(out=out, sb=s + 2) == -2                                    # scale_b: 4-byte aligned
            assert f(out=out, o=offs + 2) == -2                                  # offs: 4-byte aligned
            assert f(out=out, a=p + 8) == -2 and f(out=out, b=p + 8) == -2 and f(out=out, c=p + 8) == -2
            assert f(out=out, ld=T - 4) == -10 and f(out=out, ld=T + 2) == -10  # ld_a >= T, ld_a % 4 == 0
            assert f(out=out, t=0, ld=0) == -10                                 # ld_a >= max(T, 1)
            assert f(out=out, k=72) == -9                                        # K % 16
            assert f(out=out, n=60) == -2                                        # N % 8
            assert f(out=out, G=0) == -1 and f(out=out, G=-3) == -1              # G <= 0
            assert f(out=out, t=-1) == -1                                        # T < 0
            assert f(out=out, n=0) == -1 and f(out=out, k=0) == -1
            assert f(out=out, t=0, ld=4) == 0                                    # T == 0: no launch, no CUDA call
    for out in (2, -1):                                                          # bad output selector
        assert g(out=out) == -6 and r(out=out) == -6
    for cfg in sorted(set(range(-1, NUM_CONFIGS + 1)) - set(ELIGIBLE)):         # no block-scaled kernel
        assert r(cfg=cfg) == -6 and r(cfg=cfg, out=1) == -6, cfg
    for cfg in ELIGIBLE:
        # worst-case tile count (ceil(T / block rows) + G) * column blocks past INT_MAX
        assert r(cfg=cfg, G=4, t=INT_MAX - 3, ld=INT_MAX - 3, n=INT_MAX - 7) == -1, cfg
    assert g(G=2 * 10 ** 9, t=2 * 10 ** 9, ld=2 * 10 ** 9, n=1024) == -1        # every configuration past the bound
    assert lib.b200_grouped_fp8_select(0, 64, 64, 64, None, None) == -1
    assert lib.b200_grouped_fp8_select(4, 0, 64, 64, None, None) == -1
    assert "ld_a" in lib.b200_grouped_fp8_strerror(-10).decode()
    assert lib.b200_grouped_fp8_launch_count() == 0 and capi.fp8_grouped_launch_count() == 0


def sibling(cfg: int) -> int:
    """The block-scaled stand-in of a configuration, restated from the table: the same CTA group and cluster, M_REP 1,
    BN min(BN, 128)."""
    cfgs = capi.configs()
    c = cfgs[cfg]
    sib = [d["id"] for d in cfgs if (d["cta_group"], d["cluster_m"], d["cluster_n"], d["m_rep"], d["bn"]) ==
           (c["cta_group"], c["cluster_m"], c["cluster_n"], 1, min(c["bn"], 128))]
    assert len(sib) == 1 and sib[0] in ELIGIBLE
    return sib[0]


def rule(g, t, n, k):
    """The grouped 16-bit rule (fp32 accumulation) for e4m3 operands, which read the tuned table at K / 2, mapped to
    the block-scaled sibling."""
    cfg, gm = capi.grouped_select(0, g, t, n, max(k // 2, 1))
    return sibling(cfg), gm


def test_dispatch_is_the_block_scaled_sibling_of_the_grouped_rule(built_libs):
    rng = random.Random(20261016)
    shapes = [(8, 8192, 4096, 7168), (32, 32768, 7168, 2048), (256, 4096, 2048, 7168), (1, 100, 8, 16),
              (128, 100, 512, 64)]
    shapes += [(rng.randrange(1, 300), rng.randrange(1, 50000), 8 * rng.randrange(1, 1500), 16 * rng.randrange(1, 800))
               for _ in range(300)]
    seen = set()
    for g, t, n, k in shapes:
        got = capi.fp8_grouped_select(g, t, n, k)
        assert got == rule(g, t, n, k), (g, t, n, k)
        seen.add(got[0])
    assert len(seen) >= 3


_EXTREMES = r"""
import ctypes, json, sys
sys.path.insert(0, {repo!r})
from cuda_l2_b200 import capi
INT_MAX = 2 ** 31 - 1
i = ctypes.c_int
out = {{"select": [], "gemm": []}}
gl, fl = capi.grouped_lib(), capi.grouped_fp8_lib()
tl = [(1, 1), (1, INT_MAX), (2, INT_MAX), (INT_MAX, 1), (INT_MAX, INT_MAX), (2 * 10 ** 9, 2 * 10 ** 9),
      (256, 10 ** 9), (3, 10 ** 9), (10 ** 6, 4096)]
for g, t in tl:
    for n in (8, 64, 4096, INT_MAX - 7):
        for k in (16, 4096, INT_MAX - 15):
            c, gm, c16, gm16 = i(-99), i(-99), i(-99), i(-99)
            st = fl.b200_grouped_fp8_select(g, t, n, k, ctypes.byref(c), ctypes.byref(gm))
            st16 = gl.b200_grouped_select(0, g, t, n, k // 2, ctypes.byref(c16), ctypes.byref(gm16))
            out["select"].append([g, t, n, k, st, c.value, gm.value, st16, c16.value, gm16.value])
buf = ctypes.create_string_buffer(1 << 12)
p = (ctypes.addressof(buf) + 15) & ~15
# shapes whose every block-scaled configuration's tile list passes INT_MAX: refused before any device call
# (T is a multiple of 4, so that ld_a = T is valid)
for g, t, n in ((2 * 10 ** 9, 2 * 10 ** 9, 1024), (INT_MAX, INT_MAX - 3, 4096), (2, INT_MAX - 3, INT_MAX - 7)):
    for out_bf16 in (0, 1):
        st = fl.b200_grouped_fp8_gemm(p, p, p, p, t, p, out_bf16, p, g, t, n, 64, None)
        out["gemm"].append([g, t, n, out_bf16, st])
print(json.dumps(out))
"""


def test_selector_is_total_and_refuses_before_the_device_on_extreme_shapes(built_libs):
    r = subprocess.run([sys.executable, "-c", _EXTREMES.format(repo=str(REPO))], capture_output=True, text=True,
                       timeout=600, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, f"the selector process died (status {r.returncode}):\n{r.stderr[-2000:]}"
    out = json.loads(r.stdout)
    assert len(out["select"]) == 9 * 4 * 3
    for g, t, n, k, st, cfg, gm, st16, cfg16, gm16 in out["select"]:
        assert st == 0 and st16 == 0 and gm >= 0, (g, t, n, k, st, cfg)
        assert (cfg, gm) == (sibling(cfg16), gm16), (g, t, n, k, cfg, cfg16)
    assert len(out["gemm"]) == 6
    for g, t, n, out_bf16, st in out["gemm"]:
        assert st == -1, (g, t, n, out_bf16, st)             # kBadShape


def _meta(*shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device="meta")


def test_operator_schema_and_meta_shapes():
    from cuda_l2_b200 import ops
    schema = str(torch.ops.cuda_l2_b200.fp8_grouped_gemm.default._schema)
    assert schema == ("cuda_l2_b200::fp8_grouped_gemm(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, "
                      "Tensor offs, ScalarType out_dtype) -> Tensor")
    assert {"fp8_grouped_gemm", "B200Fp8GroupedLinear"} <= set(ops.__all__)
    a, b = _meta(1000, 400, dtype=E4), _meta(6, 328, 400, dtype=E4)        # nkb = 4, ceil(328 / 128) = 3
    offs = _meta(6, dtype=torch.int32)
    for dt in (torch.float16, torch.bfloat16):
        y = ops.fp8_grouped_gemm(a, b, _meta(1000, 4), _meta(6, 3, 4), offs, dt)
        assert y.shape == (1000, 328) and y.dtype == dt and y.device.type == "meta"
        y = ops.fp8_grouped_gemm(a, b, _meta(4, 1000).t(), _meta(6, 3, 4), offs, dt)   # the M-major view
        assert y.shape == (1000, 328)
    assert ops.fp8_grouped_gemm(_meta(0, 400, dtype=E4), b, _meta(0, 4), _meta(6, 3, 4), offs).shape == (0, 328)
    assert capi.check_grouped_operands(a, b, offs, "fp32", torch.float16, (_meta(1000, 4), _meta(6, 3, 4))) == \
        (6, 1000, 328, 400)


@pytest.mark.parametrize("sa,sb", [
    ((1000, 3), (6, 3, 4)),          # nkb of scale_a
    ((1000, 4), (6, 3, 3)),          # nkb of scale_b
    ((1000, 4), (6, 2, 4)),          # ceil(N / 128)
    ((1000, 4), (5, 3, 4)),          # G
    ((1000, 4), (3, 4)),             # the 2-D blockwise scale_b
    ((999, 4), (6, 3, 4)),           # T
    ((4, 1000), (6, 3, 4)),          # transposed
    ((1000, 1), (1, 328)),           # rowwise
    ((1,), (1,)),                    # per tensor
])
def test_scale_shapes_that_are_rejected(sa, sb):
    from cuda_l2_b200 import ops
    a, b, offs = _meta(1000, 400, dtype=E4), _meta(6, 328, 400, dtype=E4), _meta(6, dtype=torch.int32)
    with pytest.raises(capi.B200HgemmError):
        ops.fp8_grouped_gemm(a, b, _meta(*sa), _meta(*sb), offs, torch.bfloat16)


def test_operand_errors():
    from cuda_l2_b200 import ops
    sa, sb, offs = _meta(1000, 4), _meta(6, 3, 4), _meta(6, dtype=torch.int32)
    bad = [
        (_meta(1000, 400, dtype=E4), _meta(6, 328, 384, dtype=E4), sa, sb, offs, torch.bfloat16),   # K
        (_meta(1000, 408, dtype=E4), _meta(6, 328, 408, dtype=E4), sa, sb, offs, torch.bfloat16),   # K % 16
        (_meta(1000, 400, dtype=E4), _meta(6, 324, 400, dtype=E4), sa, sb, offs, torch.bfloat16),   # N % 8
        (_meta(1000, 400, dtype=E4), _meta(328, 400, dtype=E4), sa, sb, offs, torch.bfloat16),      # 2-D b
        (_meta(1000, 400, dtype=E4), _meta(6, 328, 400, dtype=E4), sa, sb, _meta(5, dtype=torch.int32),
         torch.bfloat16),                                                                           # G of offs
        (_meta(1000, 400, dtype=E4), _meta(6, 328, 400, dtype=E4), sa, sb, _meta(6, dtype=torch.int64),
         torch.bfloat16),                                                                           # int32 offsets
        (_meta(1000, 400, dtype=E4), _meta(6, 328, 400, dtype=E4), sa, sb, offs, torch.float32),    # output type
        (_meta(1000, 400, dtype=torch.bfloat16), _meta(6, 328, 400, dtype=torch.bfloat16), sa, sb, offs,
         torch.bfloat16),                                                                           # 16-bit operands
        (_meta(1000, 400, dtype=E4), _meta(6, 328, 400, dtype=E4), sa.half(), sb, offs, torch.bfloat16),   # fp32
    ]
    for args in bad:
        with pytest.raises(capi.B200HgemmError):
            ops.fp8_grouped_gemm(*args)


def test_operator_has_no_cpu_path():
    from cuda_l2_b200 import ops
    a, b = torch.zeros((32, 128), dtype=E4), torch.zeros((2, 16, 128), dtype=E4)
    sa, sb, offs = torch.ones(32, 1), torch.ones(2, 1, 1), torch.tensor([10, 32], dtype=torch.int32)
    with pytest.raises(capi.B200HgemmError, match="no CPU implementation"):
        ops.fp8_grouped_gemm(a, b, sa, sb, offs)
    with pytest.raises(capi.B200HgemmError):
        capi.fp8_grouped_gemm(a, b, torch.zeros((32, 16), dtype=torch.bfloat16), sa, sb, offs)


def test_quantiser_per_expert_is_the_2d_quantiser_on_each_expert():
    from cuda_l2_b200 import ops
    g = torch.Generator().manual_seed(3)
    for shape in ((3, 200, 300), (1, 128, 128), (4, 1000, 1040), (2, 8, 16)):
        w = torch.randn(shape, generator=g)
        w[0, :5, :7] *= 1000
        q, s = ops.quantize_e4m3_block128x128(w)
        assert q.dtype == E4 and q.shape == w.shape and q.is_contiguous()
        assert s.shape == (shape[0], -(-shape[1] // 128), -(-shape[2] // 128)) and s.is_contiguous()
        for e in range(shape[0]):
            q2, s2 = ops.quantize_e4m3_block128x128(w[e])
            assert torch.equal(q[e].view(torch.uint8), q2.view(torch.uint8)) and torch.equal(s[e], s2), (shape, e)
    # the 2-D form is unchanged: its scales are the amax of each 128 x 128 block over 448
    w = torch.randn(200, 300, generator=g, dtype=torch.float32).to(torch.bfloat16)
    q, s = ops.quantize_e4m3_block128x128(w)
    wp = torch.nn.functional.pad(w.float(), (0, 84, 0, 56)).view(2, 128, 3, 128)
    assert torch.equal(s, (wp.abs().amax(dim=(1, 3)) / 448).clamp_min(torch.finfo(torch.float32).tiny))
    assert torch.equal(q.view(torch.uint8), (wp / s[:, None, :, None]).clamp(-448, 448).to(E4).view(256, 384)[:200, :300]
                       .contiguous().view(torch.uint8))


def test_grouped_linear_buffers():
    from cuda_l2_b200 import ops
    w = torch.randn(4, 200, 272).to(E4)
    s = torch.rand(4, 2, 3) + 0.5
    m = ops.B200Fp8GroupedLinear.from_fp8(w, s)
    assert (m.num_groups, m.in_features, m.out_features, m.out_dtype) == (4, 272, 200, torch.bfloat16)
    assert set(dict(m.named_buffers())) == {"weight_fp8", "weight_scale"} and not list(m.parameters())
    assert torch.equal(m.weight_fp8.view(torch.uint8), w.view(torch.uint8)) and torch.equal(m.weight_scale, s)
    assert "num_groups=4" in repr(m)
    assert ops.B200Fp8GroupedLinear.from_fp8(w, s, torch.float16).out_dtype == torch.float16
    for bad_w, bad_s in ((w, torch.rand(4, 3, 2)), (w, s[:3]), (w, s.double()), (w.float(), s), (w[0], s[0]),
                         (w[:, :, :264], s[:, :, :2]), (torch.randn(4, 196, 272).to(E4), s)):
        with pytest.raises(capi.B200HgemmError):
            ops.B200Fp8GroupedLinear.from_fp8(bad_w, bad_s)
    hw = torch.randn(3, 256, 128, dtype=torch.float16)
    m = ops.B200Fp8GroupedLinear.from_weights(hw)
    q, qs = ops.quantize_e4m3_block128x128(hw)
    assert m.out_dtype == torch.float16 and torch.equal(m.weight_scale, qs)
    assert torch.equal(m.weight_fp8.view(torch.uint8), q.view(torch.uint8))
    for bad in (hw.float(), hw[0]):
        with pytest.raises(capi.B200HgemmError):
            ops.B200Fp8GroupedLinear.from_weights(bad)


def test_grouped_fp8_sass(built_libs):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sys.path.insert(0, str(REPO / "tools"))
    import sass_summary
    sass = subprocess.run([cuobjdump, "-sass", str(built_libs["grouped_fp8"])], capture_output=True, text=True,
                          check=True).stdout
    kernels = sass_summary.sass_by_kernel(sass)
    assert len(kernels) == 2 * len(ELIGIBLE)                                 # plain only, two output types
    assert all(re.search(r"GroupedINS_11BlockScaledINS_6ConfigI.*ELi0EEEv14CUtensorMap", name) for name in kernels)
    for name, insns in kernels.items():
        ops_ = {op for _, op, _ in insns}
        assert any(op.startswith("QGMMA") for op in ops_), name              # FP8 wgmma
        assert not any(op.startswith(("HGMMA", "HMMA")) for op in ops_), name
        assert any(op.startswith("UTMALDG.2D") for op in ops_), name        # A [T, K]
        assert any(op.startswith("UTMALDG.3D") for op in ops_), name        # Bt [G, N, K]
        assert any(op.startswith("UBLKCP") for op in ops_), name            # the bulk copy of A's scale window
        assert "UTMASTG.2D" in ops_, name                                   # whole boxes of C [T, N]
        assert "STG.E.128" in ops_, name                                    # the rows of a box that straddles a group end
        loop = sass_summary.k_loop(insns)
        assert any(op == "WARPGROUP.ARRIVE" for _, op, _ in loop), name
        assert any(op.startswith("SYNCS.ARRIVE") for _, op, _ in loop), name   # the stage release is inside
        assert any(op == "FFMA" for _, op, _ in loop), name                  # the promotion is inside the k-loop
        assert sass_summary.k_loop_gpu_membars(insns) == 0, name
