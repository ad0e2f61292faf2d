#!/usr/bin/env python
"""The fused bias + activation epilogue on the H100: what one launch saves over a GEMM followed by separate passes.

    python tools/bench_epilogue.py [--rounds R] [--ms MS] [--out FILE]

Legs, timed with CUDA events on one stream, alternating within every round (median and range over the rounds):
  fused      hgemm_bias_act: act(x W^T + b) in one launch (libb200_epilogue.so);
  separate   hgemm, then `+ bias` (then relu / F.gelu(approximate="tanh")) as torch ops: B200Linear's path today;
  torch      torch._addmm_activation (relu / gelu_tanh) or F.linear (bias only): cuBLASLt's bias epilogues;
  hgemm      hgemm alone, without bias or activation: the floor, so that fused - hgemm is the epilogue's cost.
Shapes M x N x K, fp16 and bf16: 8192 x 3072 x 768 with gelu_tanh (a BERT / GPT-2 FFN up projection), 8192 x 768 x 3072
bias only, 2048 x 11008 x 4096 bias and relu, 4096^3 bias, 16 x 4096 x 4096 bias (decode, split-K territory). One e4m3
leg at 2048 x 11008 x 4096 with rowwise scales and a bias (bf16 out): fp8_gemm_bias_act against fp8_gemm + bias and
torch._scaled_mm(..., bias=...); a leg torch refuses is reported as skipped. The card and its power limit are recorded
with the results. Needs an H100; there is no CPU path.
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
from cuda_l2_b200 import ops  # noqa: E402

SHAPES = {   # name -> (M, N, K, activation)
    "8192_3072_768_gelu_tanh": (8192, 3072, 768, "gelu_tanh"),
    "8192_768_3072_bias": (8192, 768, 3072, "none"),
    "2048_11008_4096_relu": (2048, 11008, 4096, "relu"),
    "4096_4096_4096_bias": (4096, 4096, 4096, "none"),
    "16_4096_4096_bias": (16, 4096, 4096, "none"),
}


def act_op(y: torch.Tensor, activation: str) -> torch.Tensor:
    if activation == "relu":
        return torch.relu(y)
    if activation == "gelu_tanh":
        return F.gelu(y, approximate="tanh")
    return y


def legs16(m: int, n: int, k: int, activation: str, dtype, seed: int) -> dict:
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((m, k), device="cuda", generator=g).to(dtype)
    w = torch.randn((n, k), device="cuda", generator=g).to(dtype)
    b = torch.randn((n,), device="cuda", generator=g).to(dtype)

    def fused():
        ops.hgemm_bias_act(x, w, b, activation)

    def separate():
        act_op(ops.hgemm(x, w) + b, activation)

    def cublaslt():
        if activation == "none":
            F.linear(x, w, b)
        else:
            torch._addmm_activation(b, x, w.t(), use_gelu=activation == "gelu_tanh")

    def hgemm():
        ops.hgemm(x, w)

    return {"fused": fused, "separate": separate, "torch": cublaslt, "hgemm": hgemm}


def legs_e4m3(m: int, n: int, k: int, seed: int) -> tuple[dict, dict]:
    g = torch.Generator(device="cuda").manual_seed(seed)
    xq, sa = ops.quantize_e4m3_rowwise(torch.randn((m, k), device="cuda", generator=g))
    wq, sw = ops.quantize_e4m3_rowwise(torch.randn((n, k), device="cuda", generator=g))
    sb = sw.view(1, n)
    b = torch.randn((n,), device="cuda", generator=g).to(torch.bfloat16)
    out = torch.bfloat16

    def fused():
        ops.fp8_gemm_bias_act(xq, wq, sa, sb, b, "none", out)

    def separate():
        ops.fp8_gemm(xq, wq, sa, sb, out) + b

    def scaled_mm():
        torch._scaled_mm(xq, wq.t(), scale_a=sa, scale_b=sb, bias=b, out_dtype=out)

    def plain():
        ops.fp8_gemm(xq, wq, sa, sb, out)

    legs, skipped = {"fused": fused, "separate": separate}, {}
    try:
        scaled_mm()
        torch.cuda.synchronize()
        legs["torch"] = scaled_mm
    except Exception as e:   # noqa: BLE001 - torch refuses the combination on this build: reported, not timed
        skipped["torch"] = f"{type(e).__name__}: {str(e).splitlines()[0] if str(e) else ''}"
    legs["fp8_gemm"] = plain
    return legs, skipped


def main() -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=7)
    p.add_argument("--ms", type=float, default=100.0, help="length of one timing of one leg")
    p.add_argument("--out", type=str, default=None, help="also write the JSON result here")
    args = p.parse_args()
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        raise SystemExit("bench_epilogue.py needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)
    result = {"card": card(), "rounds": args.rounds, "results": {}}
    seed = 0
    for name, (m, n, k, activation) in SHAPES.items():
        for dtype in (torch.float16, torch.bfloat16):
            seed += 1
            times = alternate(legs16(m, n, k, activation, dtype, seed), args.rounds, args.ms)
            flops = 2.0 * m * n * k
            for v in times.values():
                v["tflops"] = flops / (v["ms"] * 1e-3) / 1e12
            result["results"][f"{name}_{str(dtype).split('.')[-1]}"] = times
            torch.cuda.empty_cache()
    legs, skipped = legs_e4m3(2048, 11008, 4096, 99)
    times = alternate(legs, args.rounds, args.ms)
    for v in times.values():
        v["tflops"] = 2.0 * 2048 * 11008 * 4096 / (v["ms"] * 1e-3) / 1e12
    times.update({leg: {"skipped": why} for leg, why in skipped.items()})
    result["results"]["2048_11008_4096_bias_e4m3_rowwise_bf16"] = times
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
