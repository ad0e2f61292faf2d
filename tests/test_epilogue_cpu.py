"""The fused bias + activation epilogue (libb200_epilogue.so) without a GPU: argument statuses, exports, the dispatcher's
choice, the kernels' SASS and resource usage against their TN twins, the operators' schemas, meta shapes and refusals,
and the CPU reference against an independent numpy evaluation."""
import re
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import pytest
import torch

import epilogue_ref
from conftest import REPO
from cuda_l2_b200 import build, capi, ops

sys.path.insert(0, str(REPO / "tools"))
import sass_summary  # noqa: E402

KNULL, KBADSHAPE, KBADALIGN, KBADCONFIG, KBADACT, KBADFP8K = -5, -1, -2, -6, -12, -9
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
A, B, C, S, BIAS = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000   # fake, never dereferenced device addresses
VARIANTS = (0, 2, 3, 4)
MODES_PER_VARIANT = 46   # libb200_hgemm.so's (configuration, K-mode) pairs


@pytest.fixture(scope="module")
def libs(built_libs):
    return built_libs


def _run(variant, cfg, a=A, b=B, c=C, sa=S, sb=S, rowwise=0, bias=BIAS, act=0, m=64, n=64, k=64):
    lib = capi.epilogue_lib()
    if cfg is None:
        return lib.cuda_l2_b200_epilogue_run(variant, a, b, c, sa, sb, rowwise, bias, act, m, n, k, None)
    return lib.cuda_l2_b200_epilogue_run_config(variant, cfg, a, b, c, sa, sb, rowwise, bias, act, m, n, k, 0, 0, 1, None)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("cfg", [None, 1, 12])
def test_statuses_come_back_before_any_cuda_call(libs, variant, cfg):
    e4m3 = variant in (3, 4)
    assert _run(variant, cfg, a=None) == KNULL
    assert _run(variant, cfg, b=None) == KNULL
    assert _run(variant, cfg, c=None) == KNULL
    if e4m3:
        assert _run(variant, cfg, sa=None) == KNULL
        assert _run(variant, cfg, sb=S + 4, rowwise=1) == KBADALIGN   # rowwise vectors: 16-byte aligned
        assert _run(variant, cfg, k=8) == KBADFP8K                     # K % 16
    else:
        assert _run(variant, cfg, k=60) == KBADALIGN                   # K % 8
    for m, n, k in ((0, 64, 64), (64, 0, 64), (64, 64, 0), (-1, 64, 64)):
        assert _run(variant, cfg, m=m, n=n, k=k) == KBADSHAPE
    assert _run(variant, cfg, n=60) == KBADALIGN                             # N % 8
    assert _run(variant, cfg, a=A + 8) == KBADALIGN
    assert _run(variant, cfg, bias=BIAS + 2) == KBADALIGN                    # the bias: 16-byte aligned ...
    assert _run(variant, cfg, bias=BIAS + 8) == KBADALIGN
    for act in (3, -1, 100):                                                # ... and a known activation code
        assert _run(variant, cfg, act=act) == KBADACT
    assert _run(variant, cfg, act=3, bias=BIAS + 8) == KBADACT
    assert capi.epilogue_lib().cuda_l2_b200_epilogue_strerror(KBADACT).decode().startswith("unknown activation")


@pytest.mark.parametrize("variant", [1, 5, 6, 7, -1])
def test_fp16_accumulation_and_block_scales_have_no_bias_kernel(libs, variant):
    assert _run(variant, None) == KBADCONFIG
    assert _run(variant, 1) == KBADCONFIG
    assert capi.epilogue_lib().cuda_l2_b200_epilogue_select(variant, 64, 64, 64, None, None, None) == KBADCONFIG


def test_unknown_configuration(libs):
    assert _run(0, 31) == KBADCONFIG and _run(3, -1) == KBADCONFIG


def _exports(path) -> list[str]:
    out = subprocess.run(["nm", "-D", "--defined-only", str(path)], capture_output=True, text=True, check=True).stdout
    return [line.split()[-1] for line in out.splitlines() if line.strip()]


def test_exports_and_no_header(libs):
    names = _exports(libs["epilogue"])
    assert not [s for s in names if s.startswith("b200_")]
    assert sorted(s for s in names if s.startswith("cuda_l2_b200_")) == sorted(capi.INTERNAL_ABI[capi.EPILOGUE_LIB])
    assert all(s.startswith("cuda_l2_b200_epilogue_") for s in capi.INTERNAL_ABI[capi.EPILOGUE_LIB])
    assert capi.EPILOGUE_LIB not in capi.ABI
    assert not any("cuda_l2_b200_epilogue" in h.read_text() for h in (REPO / "include").glob("*.h"))
    hgemm = sorted(s for s in _exports(libs["capi"]) if s.startswith("b200_"))
    assert hgemm == sorted(capi.ABI["libb200_hgemm.so"])


SHAPES = [(4096, 4096, 4096), (8192, 3072, 768), (8192, 768, 3072), (2048, 11008, 4096), (16, 4096, 4096),
          (64, 64, 64), (16384, 16384, 16384), (1, 8, 16), (200, 328, 1040), (77, 1000, 4112), (3000, 136, 65536)]


@pytest.mark.parametrize("shape", SHAPES)
def test_select_is_the_tn_choice(libs, shape):
    m, n, k = shape
    for variant in VARIANTS:
        got = capi.epilogue_select(variant, m, n, k)
        if variant in (3, 4):
            want = capi.fp8_select(m, n, k)
        else:
            want = capi._select(capi.hgemm_lib().b200_hgemm_select, 32, m, n, k)
        assert got == want, (variant, shape, got, want)


def test_kernel_count_and_the_k_loop_of_every_kernel(libs):
    if not Path(CUOBJDUMP).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([CUOBJDUMP, "-sass", str(libs["epilogue"])], capture_output=True, text=True,
                          check=True).stdout
    kernels = sass_summary.sass_by_kernel(sass)
    assert len(kernels) == len(VARIANTS) * MODES_PER_VARIANT == 184
    for name, insns in kernels.items():
        assert "hgemm_bias_act_kernel" in name and "BiasAct" in name, name
        loop = sass_summary.k_loop(insns)
        assert any(op == "WARPGROUP.ARRIVE" for _, op, _ in loop), name
        assert any(op.startswith("SYNCS.ARRIVE") for _, op, _ in loop), name   # the stage release
        assert any(op.startswith("WARPGROUP.DEPBAR") for _, op, _ in loop), name
        assert sass_summary.k_loop_gpu_membars(insns) == 0, name


def _ptxas(source: Path, defines: list[str], tmp: Path) -> tuple[dict, str]:
    """{kernel: (registers, spill store bytes, stack frame bytes)} of one object compiled with -Xptxas -v, and the
    compiler's output."""
    r = subprocess.run([build.nvcc_path(), *build.ARCH_FLAGS, *build.COMMON, "-Xptxas", "-v", *defines, "-c", "-o",
                        str(tmp / f"{source.stem}_{'_'.join(defines)}.o"), str(source)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    text = r.stdout + r.stderr
    out = {}
    for block in text.split("ptxas info    : Compiling entry function ")[1:]:
        spill = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        regs = re.search(r"Used (\d+) registers", block)
        out[block.split("'")[1]] = (int(regs.group(1)) if regs else 0, int(spill.group(2)) if spill else 0,
                                    int(spill.group(1)) if spill else 0)
    return out, text


def _demangle(names) -> dict:
    names = list(names)
    r = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True, check=True)
    return dict(zip(names, r.stdout.splitlines()))


def _twin_key(name: str):
    """(Config<...>, K-mode) of a demangled kernel name, BiasAct<> unwrapped."""
    m = re.search(r"(?:hgemm_tn_kernel|hgemm_bias_act_kernel)<(?:b200::BiasAct<)?(b200::Config<[^>]*>) ?>?, ?(?:\(int\))?(\d+)>",
                  name)
    assert m, name
    return m.group(1), int(m.group(2))


def test_resources_against_the_tn_twins(tmp_path):
    """-Xptxas -v of libb200_epilogue.so's objects and of libb200_hgemm.so's: 168 registers, no C7510; the plain and
    split-K kernels spill no more than the TN kernel of the same configuration, K-mode and type, and hold no more other
    local memory (stack beyond the spills is an array in local memory, such as accumulators indexed by a loop left
    rolled); the stream-K kernels' spills are listed (DESIGN.md section 5), not bounded."""
    csrc = build.CSRC
    jobs = [(csrc / "b200_epilogue.cu", [f"-DB200_VARIANT={v}"]) for v in build.EPILOGUE_VARIANTS] + \
           [(csrc / "b200_hgemm_capi.cu", []), (csrc / "b200_fp8_capi.cu", [])]
    with ThreadPoolExecutor(len(jobs)) as pool:
        results = list(pool.map(lambda j: _ptxas(*j, tmp_path), jobs))
    for _, text in results:
        assert "C7510" not in text
    epi, tn = {}, {}
    for res, _ in results[:4]:
        epi.update(res)
    for res, _ in results[4:]:
        tn.update(res)
    assert len(epi) == 184
    tn_names = _demangle(tn)
    tn_by_key = {_twin_key(tn_names[k]): v for k, v in tn.items() if "hgemm_tn_kernel" in tn_names[k]}
    rows = []
    names = _demangle(epi)
    for mangled, (regs, spill, stack) in epi.items():
        key = _twin_key(names[mangled])
        assert key in tn_by_key, names[mangled]
        assert regs <= 168, (names[mangled], regs)
        _, twin_spill, twin_stack = tn_by_key[key]
        if key[1] == 3:   # stream-K
            rows.append((key, spill, twin_spill))
        else:
            assert spill <= twin_spill, (names[mangled], spill, twin_spill)
            # local arrays besides the spill area: none the twin does not have
            assert stack - spill <= max(twin_stack - twin_spill, 0), (names[mangled], stack, spill, twin_stack)
    print("stream-K spill stores (bias + activation, TN twin):")
    for key, spill, twin in sorted(rows):
        print(f"  {key[0]}: {spill} B, {twin} B")


def test_operator_schemas_and_meta_shapes():
    assert str(torch.ops.cuda_l2_b200.hgemm_bias_act.default._schema) == \
        'cuda_l2_b200::hgemm_bias_act(Tensor a, Tensor b_kmajor, Tensor? bias, str activation="none") -> Tensor'
    assert str(torch.ops.cuda_l2_b200.fp8_gemm_bias_act.default._schema) == \
        ("cuda_l2_b200::fp8_gemm_bias_act(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, Tensor? bias, "
         "str activation, ScalarType out_dtype) -> Tensor")

    def meta(shape, dtype=torch.float16):
        return torch.empty(shape, dtype=dtype, device="meta")

    for dtype in (torch.float16, torch.bfloat16):
        for act in epilogue_ref.ACTIVATIONS:
            y = ops.hgemm_bias_act(meta((77, 136), dtype), meta((520, 136), dtype), meta((520,), dtype), act)
            assert y.shape == (77, 520) and y.dtype == dtype
        assert ops.hgemm_bias_act(meta((77, 136), dtype), meta((520, 136), dtype)).shape == (77, 520)
        y = ops.linear(meta((3, 5, 136), dtype), meta((520, 136), dtype), meta((520,), dtype), "relu")
        assert y.shape == (3, 5, 520) and y.dtype == dtype
        assert ops.linear(meta((136,), dtype), meta((520, 136), dtype)).shape == (520,)
        assert ops.linear(meta((2, 0, 136), dtype), meta((520, 136), dtype), None, "gelu_tanh").shape == (2, 0, 520)
    e = torch.float8_e4m3fn
    for out in (torch.float16, torch.bfloat16):
        y = ops.fp8_gemm_bias_act(meta((77, 144), e), meta((520, 144), e), meta((1,), torch.float32),
                                  meta((1,), torch.float32), meta((520,), out), "gelu_tanh", out)
        assert y.shape == (77, 520) and y.dtype == out
        y = ops.fp8_gemm_bias_act(meta((77, 144), e), meta((520, 144), e), meta((77, 1), torch.float32),
                                  meta((1, 520), torch.float32), None, "relu", out)
        assert y.shape == (77, 520)
    bad = [lambda: ops.hgemm_bias_act(meta((8, 64)), meta((64, 64)), meta((72,))),                # bias length
           lambda: ops.hgemm_bias_act(meta((8, 64)), meta((64, 64)), meta((64,), torch.bfloat16)),  # bias dtype
           lambda: ops.hgemm_bias_act(meta((8, 64)), meta((64, 64)), meta((1, 64))),                # bias not 1-D
           lambda: ops.hgemm_bias_act(meta((8, 64)), meta((64, 64)), None, "gelu"),                 # activation
           lambda: ops.hgemm_bias_act(meta((8, 64)), meta((60, 64))),                               # N % 8
           lambda: ops.hgemm_bias_act(meta((8, 64)), meta((64, 72))),                               # K differs
           lambda: ops.hgemm_bias_act(meta((8, 64), e), meta((64, 64), e)),                         # e4m3: fp8 op
           lambda: ops.fp8_gemm_bias_act(meta((8, 128), e), meta((64, 128), e), meta((8, 1), torch.float32),
                                         meta((1, 1), torch.float32), None, "none", torch.float16),  # blockwise
           lambda: ops.linear(meta((8, 64)), meta((64, 72)))]
    for call in bad:
        with pytest.raises(capi.B200HgemmError):
            call()
    with pytest.raises(capi.B200HgemmError, match="blockwise scales have no bias"):
        ops.fp8_gemm_bias_act(meta((8, 128), e), meta((64, 128), e), meta((8, 1), torch.float32),
                              meta((1, 1), torch.float32), None, "none", torch.float16)


def test_cpu_paths_raise():
    a = torch.ones((8, 8), dtype=torch.half)
    for call in (lambda: ops.hgemm_bias_act(a, a, torch.ones(8, dtype=torch.half), "relu"),
                 lambda: ops.linear(a, a),
                 lambda: ops.fp8_gemm_bias_act(torch.ones((8, 16)).to(torch.float8_e4m3fn),
                                               torch.ones((8, 16)).to(torch.float8_e4m3fn), torch.ones(1), torch.ones(1),
                                               None, "none", torch.float16)):
        with pytest.raises(capi.B200HgemmError, match="no CPU implementation"):
            call()


def test_fp8_operator_has_no_backward():
    e = torch.float8_e4m3fn

    def meta(shape, dtype):
        return torch.empty(shape, dtype=dtype, device="meta")

    bias = meta((64,), torch.float16).requires_grad_()
    y = ops.fp8_gemm_bias_act(meta((8, 64), e), meta((64, 64), e), meta((1,), torch.float32), meta((1,), torch.float32),
                              bias, "relu", torch.float16)
    with pytest.raises(capi.B200HgemmError, match="inference only"):
        y.sum().backward()


def _numpy_fp16(a, bt, bias, act):
    """An independent evaluation: the exact sum (integers here), fp32 add, activation written out, fp16 rounding."""
    s = np.einsum("mk,nk->mn", a, bt).astype(np.float32)
    z = s + bias.astype(np.float32)[None, :]
    if act == "relu":
        z = np.maximum(z, np.float32(0))
        z[z == 0] = np.float32(0.0)
        return z.astype(np.float16).view(np.uint16)
    if act == "gelu_tanh":
        zz = z.astype(np.float64)
        return (0.5 * zz * (1 + np.tanh(np.sqrt(2 / np.pi) * (zz + 0.044715 * zz ** 3)))).astype(np.float16).view(np.uint16)
    return z.astype(np.float16).view(np.uint16)


@pytest.mark.parametrize("act", epilogue_ref.ACTIVATIONS)
def test_reference_against_numpy(act):
    rng = np.random.default_rng(7)
    m, n, k = 24, 40, 48
    a = rng.integers(-3, 4, size=(m, k)).astype(np.float64) / 8
    bt = rng.integers(-3, 4, size=(n, k)).astype(np.float64) / 8
    bias16 = rng.uniform(-3, 8, size=n).astype(np.float16)
    got = epilogue_ref.reference(a, bt, bias16.astype(np.float32), act, "fp16")
    want = _numpy_fp16(a, bt, bias16, act)
    if act == "gelu_tanh":   # z > -3 here: the two gelu forms agree to the fp16 rounding
        assert epilogue_ref.ulp_distance(got, want).max() <= 1
    else:
        assert np.array_equal(got, want)
    # bias -0.0 and no activation: the plain GEMM's rounding, -0.0 sums included
    neg0 = np.full(n, -0.0, dtype=np.float32)
    assert np.array_equal(epilogue_ref.reference(a, bt, neg0, "none", "fp16"),
                          epilogue_ref.fp32_sum(a, bt).astype(np.float16).view(np.uint16))


def test_reference_gelu_tail_and_scales():
    z = np.array([-8.0, -5.0, -3.0, -1.0, 0.0, 1.0, 8.0])
    g = epilogue_ref.gelu_tanh(z)
    assert g[0] == 0 and g[4] == 0 and g[-1] == 8.0 and -1e-5 < g[1] < 0
    # the fp32 form's allowance: an exact result passes, one off by two units in the last place does not
    want = epilogue_ref.round_out(g, "fp16")
    assert (epilogue_ref.gelu_excess(want, z, "fp16") <= 0).all()
    off = (want.astype(np.int32) + 2).astype(np.uint16)
    assert (epilogue_ref.gelu_excess(off[2:], z[2:], "fp16") > 0).all()
    s = np.array([[3.0, -5.0]], dtype=np.float32)
    assert np.array_equal(epilogue_ref.scaled(s, np.float32(0.5), np.float32(4.0)), s * np.float32(2.0))
    assert np.array_equal(epilogue_ref.scaled(s, np.array([2.0]), np.array([0.5, 0.25]), rowwise=True),
                          np.array([[3.0, -2.5]], dtype=np.float32))
    assert epilogue_ref.ulp_distance(np.array([0x8000]), np.array([0x0000]))[0] == 0
    assert epilogue_ref.ulp_distance(np.array([0x8001]), np.array([0x0001]))[0] == 2
