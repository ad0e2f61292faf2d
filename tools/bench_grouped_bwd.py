#!/usr/bin/env python
"""Time the backward of the grouped fp16 / bf16 GEMM (libb200_grouped_bwd.so) on an H100.

    python tools/bench_grouped_bwd.py [--steps K] [--warmup W] [--repeats R]

Cases: tools/bench_grouped.py's two, with its seeded uneven groups (two empty, the last group ending before T), each in
bf16 and fp16 (fp32 accumulation): 8 experts of T = 8192, N = 14336, K = 4096, and 64 experts of T = 16384, N = 2048,
K = 7168. The forward is Y [T, N] = X [T, K] W[g]^T per group, W [G, N, K]; dY is [T, N].

Legs, each group of legs timed R times alternating, reported as the median and the range:
* ``dw``: the weight gradient dW [G, N, K]. ``ours`` (the K-grouped kernel), ``torch_grouped_mm``
  (``torch._grouped_mm(dy.t(), x, offs=offs)``, bf16 only) and ``loop_of_hgemm_nn`` (a Python loop of ops.hgemm_nn
  per expert on ``dy_g.t()``, each copy zero-padded along the group's rows to a multiple of 8, as hgemm_nn needs, with
  the offsets known on the host);
* ``dx``: the input gradient dX [T, K]. ``ours`` (the grouped row-major B kernel on W in place),
  ``torch_grouped_mm`` (``torch._grouped_mm(dy, w, offs=offs)``, bf16 only) and ``hgemm_grouped_on_copy``
  (ops.hgemm_grouped on ``w.transpose(1, 2).contiguous()``, the copy included);
* ``layer``: a B200GroupedLinear forward and backward (dX and dW) against the same through torch._grouped_mm's
  autograd (bf16 only).
Each timing: warm-up, then K back-to-back calls between two CUDA events, rotating over seeded operand sets whose
footprint exceeds the 50 MB L2 four times (at least two). TFLOP/s count valid rows only: 2 * T_valid * N * K per
product, three products for a layer step. Prints one JSON line with the card's name and enforced power limit. Writes
nothing.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_batched import time_legs  # noqa: E402
from bench_fp8 import L2_BYTES, card_info  # noqa: E402
from bench_grouped import group_sizes  # noqa: E402


def operand_sets(g, t, n, k, dtype, gen):
    set_bytes = 2 * (2 * t * k + 2 * g * n * k + 2 * t * n)
    nsets = max(2, min(8, -(-4 * L2_BYTES // set_bytes)))
    sets = []
    for _ in range(nsets):
        sets.append(dict(x=torch.randn((t, k), device="cuda", generator=gen).to(dtype),
                         w=torch.randn((g, n, k), device="cuda", generator=gen).to(dtype),
                         dy=torch.randn((t, n), device="cuda", generator=gen).to(dtype),
                         dw=torch.empty((g, n, k), dtype=dtype, device="cuda"),
                         dx=torch.empty((t, k), dtype=dtype, device="cuda")))
    return sets


def bwd_case(g, t, n, k, dtype, args, gen, seed):
    from cuda_l2_b200 import capi, ops

    sizes = group_sizes(g, t, seed)
    ends = [int(x) for x in np.cumsum(sizes)]
    starts = [0] + ends[:-1]
    offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
    sets = operand_sets(g, t, n, k, dtype, gen)
    stream = lambda: torch.cuda.current_stream().cuda_stream   # noqa: E731
    flops = 2.0 * ends[-1] * n * k
    bf16 = dtype == torch.bfloat16

    def pad8(x, dim):
        r = x.shape[dim]
        pad = (0, 0, 0, -r % 8) if dim == 0 else (0, -r % 8)
        return torch.nn.functional.pad(x, pad)

    def dw_loop(s):
        for e, (r0, r1) in enumerate(zip(starts, ends)):
            if r1 > r0:
                s["dw"][e] = ops.hgemm_nn(pad8(s["dy"][r0:r1].t(), 1), pad8(s["x"][r0:r1], 0))
            else:
                s["dw"][e].zero_()

    dw = {"ours": lambda s: capi.gemm_grouped_wgrad(s["dy"], s["x"], s["dw"], offs, stream=stream())}
    if bf16:
        dw["torch_grouped_mm"] = lambda s: torch._grouped_mm(s["dy"].t(), s["x"], offs=offs)
    dw["loop_of_hgemm_nn"] = dw_loop
    dx = {"ours": lambda s: capi.gemm_grouped_nn(s["dy"], s["w"], s["dx"], offs, stream=stream())}
    if bf16:
        dx["torch_grouped_mm"] = lambda s: torch._grouped_mm(s["dy"], s["w"], offs=offs)
    dx["hgemm_grouped_on_copy"] = lambda s: ops.hgemm_grouped(s["dy"], s["w"].transpose(1, 2).contiguous(), offs)

    layers = [dict(x=s["x"].clone().requires_grad_(), w=torch.nn.Parameter(s["w"].clone()), dy=s["dy"]) for s in sets]
    for s in layers:
        s["mod"] = ops.B200GroupedLinear.from_weights(s["w"])

    def ours_layer(s):
        s["x"].grad = s["w"].grad = None
        s["mod"](s["x"], offs).backward(s["dy"])

    def torch_layer(s):
        s["x"].grad = s["w"].grad = None
        torch._grouped_mm(s["x"], s["w"].transpose(-2, -1), offs=offs).backward(s["dy"])

    layer = {"ours": ours_layer}
    if bf16:
        layer["torch_grouped_mm"] = torch_layer

    row = {"dw": time_legs(dw, sets, flops, args.steps, args.warmup, args.repeats),
           "dx": time_legs(dx, sets, flops, args.steps, args.warmup, args.repeats),
           "layer": time_legs(layer, layers, 3 * flops, args.steps, args.warmup, args.repeats)}
    variant = capi.batched_variant(dtype)
    row["dw"]["ours"]["dispatch"] = dict(zip(("config", "group_m"), capi.grouped_wgrad_select(variant, g, t, n, k)))
    row["dx"]["ours"]["dispatch"] = dict(zip(("config", "group_m"), capi.grouped_nn_select(variant, g, t, k, n)))
    row["group_sizes"] = sizes
    row["t_valid"] = ends[-1]
    return row


def main() -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--repeats", type=int, default=5)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_grouped_bwd.py needs an H100: the grouped backward has no CPU fallback")
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    cases = {}
    for i, (g, t, n, k) in enumerate(((8, 8192, 14336, 4096), (64, 16384, 2048, 7168))):
        for dtype in (torch.bfloat16, torch.float16):
            cases[f"{str(dtype)[6:]}_{g}x_{t}_{n}_{k}"] = bwd_case(g, t, n, k, dtype, args, gen, seed=20261016 + i)
            torch.cuda.empty_cache()
    head = cases["bfloat16_8x_8192_14336_4096"]["dw"]["ours"]
    print(json.dumps({
        "metric": "grouped weight-gradient TFLOP/s (2 * valid rows * N * K per call), median of repeats",
        "value": head["tflops"], "unit": "TFLOP/s", "steps": args.steps, "warmup": args.warmup,
        "repeats": args.repeats, "data": "synthetic N(0,1)", "card": card_info(), "cases": cases,
    }))
    return 0


if __name__ == "__main__":
    sys.exit(main())
