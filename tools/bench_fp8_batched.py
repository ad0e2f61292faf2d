#!/usr/bin/env python
"""Time the masked block-scaled FP8 batched GEMM (libb200_batched_fp8.so), the MoE decode layout, on an H100.

    python tools/bench_fp8_batched.py [--steps K] [--warmup W] [--repeats R]

Cases, the routed experts of a DeepSeek-V3-style FP8 MoE layer at decode: G = 32 local experts, each with a fixed
[M, K] slot of tokens and its real count on the device, one e4m3 [N, K] weight with 128 x 128 block scales per
expert, activations with 1 x 128 block scales. Gate/up projections N = 4096, K = 7168 and down projections
N = 7168, K = 2048, for M in {128, 512} and seeded counts drawn uniformly from [0, M/2] (averaging a quarter of M) or
from [0, M] (averaging half of M). bf16 output.

Legs, each case timed R times with its legs alternating, reported as the median and the range:
* ``ours``: the dispatched masked batched FP8 call, counts and scales on the device;
* ``bf16_hgemm_batched``: the masked bf16 batched call (libb200_batched.so) on the dequantised operands;
* ``fp8_grouped_packed``: the grouped FP8 call (libb200_grouped_fp8.so) on the same valid tokens packed contiguously
  (the packing, and unpacking the result, are not timed);
* ``loop_fp8_blockwise``: a Python loop of the 2-D block-scaled call (libb200_fp8block.so) over each expert's valid
  rows, the counts known on the host and each expert's scale rows copied out beforehand (neither is timed).
Each timing: warm-up, then K back-to-back calls between two CUDA events on the current stream, rotating over seeded
operand sets whose footprint exceeds the 50 MB L2 four times (at least two sets). TFLOP/s count valid rows only,
2 * sum(counts) * N * K per call. Prints one JSON line with the card's name and enforced power limit. Writes nothing.
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

G = 32
CASES = [(G, m, n, k, fill) for (n, k) in ((4096, 7168), (7168, 2048)) for m in (128, 512) for fill in (0.5, 1.0)]


def operand_sets(g, m, n, k, counts, gen):
    from cuda_l2_b200 import capi, ops

    set_bytes = g * m * k + g * n * k + 2 * g * m * n + 2 * (g * m * k + g * n * k)
    nsets = max(2, min(8, -(-4 * L2_BYTES // set_bytes)))
    ends = [int(x) for x in np.cumsum(counts)]
    starts = [0] + ends[:-1]
    sets = []
    for _ in range(nsets):
        a, sa = ops.quantize_e4m3_blockwise(torch.randn((g, m, k), device="cuda", generator=gen))
        bt, sb = ops.quantize_e4m3_block128x128(torch.randn((g, n, k), device="cuda", generator=gen))
        # the bf16 leg's operands: the dequantised values, rounded once to bf16
        a16 = (a.float() * sa.repeat_interleave(128, dim=2)[:, :, :k]).bfloat16()
        bt16 = torch.empty((g, n, k), dtype=torch.bfloat16, device="cuda")
        for e in range(g):
            bt16[e] = (bt[e].float() * sb[e].repeat_interleave(128, dim=0)[:n].repeat_interleave(128, dim=1)[:, :k]
                       ).bfloat16()
        # the grouped leg's operands: the valid tokens packed by expert, with their own quantisation's scales
        packed = torch.cat([a[e, :r] for e, r in enumerate(counts)])
        packed_sa = capi.m_major(torch.cat([sa[e, :r] for e, r in enumerate(counts)]))
        per_expert = [capi.m_major(sa[e, :r]) if r > 0 else None for e, r in enumerate(counts)]
        sets.append(dict(a=a, sa=sa, bt=bt, sb=sb, a16=a16, bt16=bt16, pa=packed, psa=packed_sa, sa_e=per_expert,
                         c=torch.empty((g, m, n), dtype=torch.bfloat16, device="cuda"),
                         pc=torch.empty((max(ends[-1], 1), n), dtype=torch.bfloat16, device="cuda"),
                         starts=starts))
    return sets


def fp8_batched_case(g, m, n, k, fill, args, gen, seed):
    from cuda_l2_b200 import capi

    counts = [int(x) for x in np.random.default_rng(seed).integers(0, int(m * fill) + 1, size=g)]
    masked_m = torch.tensor(counts, dtype=torch.int32, device="cuda")
    offs = torch.tensor(np.cumsum(counts).tolist(), dtype=torch.int32, device="cuda")
    sets = operand_sets(g, m, n, k, counts, gen)
    stream = lambda: torch.cuda.current_stream().cuda_stream   # noqa: E731
    experts = [(e, r) for e, r in enumerate(counts) if r > 0]

    def loop_blockwise(s):
        for e, r in experts:
            capi.fp8_gemm(s["a"][e, :r], s["bt"][e], s["c"][e, :r], s["sa_e"][e], s["sb"][e], stream=stream())

    legs = {
        "ours": lambda s: capi.fp8_batched_gemm(s["a"], s["bt"], s["c"], s["sa"], s["sb"], masked_m, stream=stream()),
        "bf16_hgemm_batched": lambda s: capi.gemm_batched(s["a16"], s["bt16"], s["c"], "fp32", masked_m=masked_m,
                                                          stream=stream()),
        "fp8_grouped_packed": lambda s: capi.fp8_grouped_gemm(s["pa"], s["bt"], s["pc"][:s["pa"].shape[0]], s["psa"],
                                                              s["sb"], offs, stream=stream()),
        "loop_fp8_blockwise": loop_blockwise,
    }
    row = time_legs(legs, sets, 2.0 * sum(counts) * n * k, args.steps, args.warmup, args.repeats)
    row["ours"]["dispatch"] = dict(zip(("config", "group_m"), capi.fp8_batched_select(g, m, n, k)))
    row["bf16_hgemm_batched"]["dispatch"] = dict(zip(("config", "group_m"), capi.batched_select(2, g, m, n, k)))
    row["fp8_grouped_packed"]["dispatch"] = dict(zip(("config", "group_m"),
                                                     capi.fp8_grouped_select(g, sum(counts), n, k)))
    row["counts"] = counts
    row["valid_rows"] = sum(counts)
    return row


def main() -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--repeats", type=int, default=3)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_fp8_batched.py needs an H100: the batched FP8 GEMM has no CPU fallback")
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    cases = {}
    for i, (g, m, n, k, fill) in enumerate(CASES):
        cases[f"{g}x{m}_{n}_{k}_fill{fill}"] = fp8_batched_case(g, m, n, k, fill, args, gen, seed=20261017 + i)
        torch.cuda.empty_cache()
    head = cases["32x128_4096_7168_fill1.0"]["ours"]
    print(json.dumps({
        "metric": "masked batched FP8 GEMM TFLOP/s (2 * valid rows * N * K per call), median of repeats",
        "value": head["tflops"], "unit": "TFLOP/s", "steps": args.steps, "warmup": args.warmup,
        "repeats": args.repeats, "data": "synthetic N(0,1), quantised per 1 x 128 and 128 x 128 block",
        "card": card_info(), "cases": cases,
    }))
    return 0


if __name__ == "__main__":
    sys.exit(main())
