#!/usr/bin/env python
"""The one-pass e4m3 quantisers of libb200_quant.so on the H100, against the torch compositions they replace, and the
FP8 layers before and after.

    python tools/bench_quant.py [--rounds R] [--ms MS] [--out FILE] [--no-profile]

Quantiser legs, bf16 input, timed with CUDA events on one stream, the kernel and the torch leg alternating within
every round (median and range over the rounds):
  per tensor, rowwise and 1 x 128 at T x 7168 for T in 128, 4096, 16384, and at 2048 x 4096;
  SwiGLU + 1 x 128 at T x 2I = 4096 x 4096 and 16384 x 4096 (the torch leg: F.silu(g) * u, then the 1 x 128 one);
  masked 1 x 128 over 32 experts x 512-row slots x 7168, a quarter of each slot filled.
A second pass of every kernel leg under torch.profiler sums the device time of the library's kernels (found by name,
b200_quant_*_kernel) per call: that kernel time, not the event time per call, gives the achieved bandwidth, the
algorithmic bytes (input read once, e4m3 written once, scales written once; the rows counted by masked_m only) over
kernel time, against the H100 SXM data-sheet 3.35 TB/s.
Layer legs, before (the same chain with the torch quantisers and F.silu(g) * u) against after:
  B200Fp8Linear, blockwise, 2048 x 11008 x 4096 (bf16);
  B200Fp8GroupedMLP.forward at DeepSeek-V3 expert shapes, H = 7168, I = 2048, 8 and 32 experts, 4096 routed tokens
  spread evenly. Both legs' outputs are checked bit for bit first.
The card and its power limit are recorded with the results. Needs an H100; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench_nn import alternate, card  # noqa: E402
from cuda_l2_b200 import capi, ops  # noqa: E402

HBM_TBPS = 3.35   # H100 SXM data sheet
T_SHAPES = [(128, 7168), (4096, 7168), (16384, 7168), (2048, 4096)]
SWIGLU_SHAPES = [(4096, 4096), (16384, 4096)]   # T x 2I
MASKED = (32, 512, 7168, 128)                    # experts, slot rows, K, filled rows per slot


def quant_bytes(rows: int, k: int, in_bytes: int, scales: int) -> int:
    """Algorithmic bytes of one quantisation of [rows, k]: the input once, e4m3 once, fp32 scales once."""
    return rows * k * (in_bytes + 1) + 4 * scales


def quantiser_legs(seed: int) -> list[tuple[str, dict, int]]:
    """(name, {"kernel": fn, "torch": fn}, algorithmic bytes) of every quantiser leg."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for t, k in T_SHAPES:
        x = torch.randn((t, k), device="cuda", generator=g).bfloat16()
        nkb = capi.num_k_blocks(k)
        for name, fn, ref, scales in (("tensor", ops.quantize_e4m3, ops.quantize_e4m3_reference, 1),
                                      ("rowwise", ops.quantize_e4m3_rowwise, ops.quantize_e4m3_rowwise_reference, t),
                                      ("1x128", ops.quantize_e4m3_blockwise, ops.quantize_e4m3_blockwise_reference,
                                       t * nkb)):
            out.append((f"{name}_{t}x{k}", {"kernel": (lambda f=fn, a=x: f(a)), "torch": (lambda f=ref, a=x: f(a))},
                        quant_bytes(t, k, 2, scales)))
    for t, two_i in SWIGLU_SHAPES:
        h = torch.randn((t, two_i), device="cuda", generator=g).bfloat16()
        i = two_i // 2
        out.append((f"swiglu_1x128_{t}x{two_i}",
                    {"kernel": lambda a=h: ops.silu_mul_quantize_e4m3_blockwise(a),
                     "torch": lambda a=h: ops.silu_mul_quantize_e4m3_blockwise_reference(a)},
                    t * two_i * 2 + t * i + 4 * t * capi.num_k_blocks(i)))
    e, m, k, filled = MASKED
    x = torch.randn((e, m, k), device="cuda", generator=g).bfloat16()
    counts = torch.full((e,), filled, dtype=torch.int32, device="cuda")
    out.append((f"masked_1x128_{e}x{m}x{k}_quarter",
                {"kernel": lambda: ops.quantize_e4m3_blockwise(x, counts),
                 "torch": lambda: ops.quantize_e4m3_blockwise_reference(x, counts)},
                quant_bytes(e * filled, k, 2, e * filled * capi.num_k_blocks(k))))
    return out


def kernel_us(fn, calls: int) -> float:
    """Device time of libb200_quant.so's kernels per call of ``fn``, from a torch.profiler trace of ``calls`` calls."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    total = sum(ev.device_time_total for ev in prof.key_averages() if "b200_quant_" in ev.key)
    return total / calls


def layer_legs(seed: int) -> list[tuple[str, dict]]:
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    lin = torch.nn.Linear(4096, 11008, device="cuda", dtype=torch.bfloat16)
    layer = ops.B200Fp8Linear.from_linear(lin, granularity="blockwise")
    x = torch.randn((2048, 4096), device="cuda", generator=g).bfloat16()

    def linear_before():
        xq, xs = ops.quantize_e4m3_blockwise_reference(x)
        return torch.ops.cuda_l2_b200.fp8_gemm(xq, layer.weight_fp8, xs, layer.weight_scale, layer.out_dtype) + lin.bias

    def linear_after():
        return layer(x)

    assert torch.equal(linear_before().view(torch.int16), linear_after().view(torch.int16))
    out.append(("B200Fp8Linear_blockwise_2048x11008x4096", {"after": linear_after, "before": linear_before}))
    hid, inter, tokens = 7168, 2048, 4096
    for experts in (8, 32):
        w13 = (torch.randn((experts, 2 * inter, hid), device="cuda", generator=g) / 32).bfloat16()
        w2 = (torch.randn((experts, hid, inter), device="cuda", generator=g) / 32).bfloat16()
        mlp = ops.B200Fp8GroupedMLP.from_weights(w13, w2)
        del w13, w2
        offs = torch.tensor([tokens * (i + 1) // experts for i in range(experts)], dtype=torch.int32, device="cuda")
        xt = torch.randn((tokens, hid), device="cuda", generator=g).bfloat16()

        def mlp_before(m=mlp, a=xt, o=offs):
            xq, xs = ops.quantize_e4m3_blockwise_reference(a)
            h = ops.fp8_grouped_gemm(xq, m.w13_fp8, xs, m.w13_scale, o, m.out_dtype)
            i = h.shape[1] // 2
            pq, ps = ops.quantize_e4m3_blockwise_reference(F.silu(h[:, :i]) * h[:, i:])
            return ops.fp8_grouped_gemm(pq, m.w2_fp8, ps, m.w2_scale, o, m.out_dtype)

        def mlp_after(m=mlp, a=xt, o=offs):
            return m(a, o)

        assert torch.equal(mlp_before().view(torch.int16), mlp_after().view(torch.int16))
        out.append((f"B200Fp8GroupedMLP_H{hid}_I{inter}_G{experts}_T{tokens}", {"after": mlp_after,
                                                                                "before": mlp_before}))
        torch.cuda.empty_cache()
    return out


def main() -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=7)
    p.add_argument("--ms", type=float, default=100.0, help="length of one timing of one leg")
    p.add_argument("--out", type=str, default=None, help="also write the JSON result here")
    p.add_argument("--no-profile", action="store_true", help="skip the torch.profiler pass (no kernel times)")
    args = p.parse_args()
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        raise SystemExit("bench_quant.py needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)
    result = {"card": card(), "rounds": args.rounds, "hbm_tbps_datasheet": HBM_TBPS, "quantisers": {}, "layers": {}}
    legs = quantiser_legs(1)
    for name, fns, nbytes in legs:
        # the kernel and the composition compute the same bits on these inputs (tests/test_gpu_quant.py); checked here
        for got, want in zip(fns["kernel"](), fns["torch"]()):
            if "masked" not in name:
                dt = torch.uint8 if got.dtype == torch.float8_e4m3fn else torch.int32
                assert torch.equal(got.view(dt), want.view(dt)), name
        times = alternate(fns, args.rounds, args.ms)
        for v in times.values():
            v["us"] = v["ms"] * 1e3
            v["event_gbps"] = nbytes / (v["ms"] * 1e-3) / 1e9
        times["bytes"] = nbytes
        result["quantisers"][name] = times
    if not args.no_profile:   # a pass of its own: tracing slows the host
        for name, fns, nbytes in legs:
            us = kernel_us(fns["kernel"], 50)
            result["quantisers"][name]["kernel_us"] = us
            result["quantisers"][name]["kernel_gbps"] = nbytes / (us * 1e-6) / 1e9
            result["quantisers"][name]["share_of_hbm"] = nbytes / (us * 1e-6) / (HBM_TBPS * 1e12)
    del legs
    torch.cuda.empty_cache()
    for name, fns in layer_legs(2):
        times = alternate(fns, args.rounds, args.ms)
        for v in times.values():
            v["us"] = v["ms"] * 1e3
        times["speedup"] = times["before"]["ms"] / times["after"]["ms"]
        result["layers"][name] = times
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
