#!/usr/bin/env python
"""Time the block-scaled FP8 grouped GEMM over contiguous row groups (libb200_grouped_fp8.so) on an H100.

    python tools/bench_fp8_grouped.py [--steps K] [--warmup W] [--repeats R]

Cases, the routed experts of a DeepSeek-V3-style FP8 MoE layer (tokens sorted by expert into one [T, K] tensor, one
e4m3 [N, K] weight with 128 x 128 block scales per expert, activations with 1 x 128 block scales): gate/up projections
N = 4096, K = 7168 and down projections N = 7168, K = 2048, for G in {8, 32} local experts and T in {8192, 32768}
routed rows; and one ragged case, N = 2056, K = 2064 (both off the 128 blocks). The group sizes are
bench_grouped.py's: seeded and uneven, two empty experts, the last group ending before T. bf16 output.

Legs, each case timed R times with its legs alternating, reported as the median and the range:
* ``ours``: the dispatched grouped FP8 call, offsets and scales on the device;
* ``bf16_hgemm_grouped``: the bf16 grouped call (libb200_grouped.so) on the same problem with dequantised operands;
* ``loop_fp8_blockwise``: a Python loop of the 2-D block-scaled call (libb200_fp8block.so) over each expert's rows,
  the offsets known on the host and each expert's scale rows copied out beforehand (neither is timed);
* ``loop_torch_scaled_mm``: the same loop with torch._scaled_mm's blockwise scales, where this torch accepts them
  (otherwise the leg is skipped with torch's message).
Each timing: warm-up, then K back-to-back calls between two CUDA events on the current stream, rotating over seeded
operand sets whose footprint exceeds the 50 MB L2 four times (at least two sets). TFLOP/s count valid rows only,
2 * T_valid * N * K per call. Prints one JSON line with the card's name and enforced power limit. Writes nothing.
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

CASES = [(g, t, n, k) for (n, k) in ((4096, 7168), (7168, 2048)) for g in (8, 32) for t in (8192, 32768)]
RAGGED = (8, 8192, 2056, 2064)


def operand_sets(g, t, n, k, starts, ends, gen):
    from cuda_l2_b200 import capi, ops

    set_bytes = t * k + g * n * k + 2 * t * n + 2 * (t * k + g * n * k)
    nsets = max(2, min(8, -(-4 * L2_BYTES // set_bytes)))
    sets = []
    for _ in range(nsets):
        a, sa = ops.quantize_e4m3_blockwise(torch.randn((t, k), device="cuda", generator=gen))
        bt, sb = ops.quantize_e4m3_block128x128(torch.randn((g, n, k), device="cuda", generator=gen))
        nkb = sa.shape[1]
        # the bf16 leg's operands: the dequantised values, rounded once to bf16
        a16 = (a.float() * sa.repeat_interleave(128, dim=1)[:, :k]).bfloat16()
        bt16 = torch.empty((g, n, k), dtype=torch.bfloat16, device="cuda")
        for e in range(g):
            bt16[e] = (bt[e].float() * sb[e].repeat_interleave(128, dim=0)[:n].repeat_interleave(128, dim=1)[:, :k]
                       ).bfloat16()
        per_expert = [capi.m_major(sa[r0:r1]) if r1 > r0 else None for r0, r1 in zip(starts, ends)]
        sets.append(dict(a=a, sa=sa, bt=bt, sb=sb, a16=a16, bt16=bt16, sa_e=per_expert, nkb=nkb,
                         c=torch.empty((t, n), dtype=torch.bfloat16, device="cuda")))
    return sets


def fp8_grouped_case(g, t, n, k, args, gen, seed):
    from cuda_l2_b200 import capi

    sizes = group_sizes(g, t, seed)
    ends = [int(x) for x in np.cumsum(sizes)]
    starts = [0] + ends[:-1]
    offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
    sets = operand_sets(g, t, n, k, starts, ends, gen)
    stream = lambda: torch.cuda.current_stream().cuda_stream   # noqa: E731
    experts = [(e, r0, r1) for e, (r0, r1) in enumerate(zip(starts, ends)) if r1 > r0]

    def loop_blockwise(s):
        for e, r0, r1 in experts:
            capi.fp8_gemm(s["a"][r0:r1], s["bt"][e], s["c"][r0:r1], s["sa_e"][e], s["sb"][e], stream=stream())

    def loop_scaled_mm(s):
        for e, r0, r1 in experts:
            torch._scaled_mm(s["a"][r0:r1], s["bt"][e].t(), scale_a=s["sa_e"][e], scale_b=s["sb"][e].t(),
                             out_dtype=torch.bfloat16)

    legs = {
        "ours": lambda s: capi.fp8_grouped_gemm(s["a"], s["bt"], s["c"], s["sa"], s["sb"], offs, stream=stream()),
        "bf16_hgemm_grouped": lambda s: capi.gemm_grouped(s["a16"], s["bt16"], s["c"], offs, "fp32", stream=stream()),
        "loop_fp8_blockwise": loop_blockwise,
    }
    skipped = {}
    try:
        loop_scaled_mm(sets[0])
        torch.cuda.synchronize()
        legs["loop_torch_scaled_mm"] = loop_scaled_mm
    except (RuntimeError, NotImplementedError, ValueError) as e:
        skipped["loop_torch_scaled_mm"] = str(e).splitlines()[0][:200]
    row = time_legs(legs, sets, 2.0 * ends[-1] * n * k, args.steps, args.warmup, args.repeats)
    row["ours"]["dispatch"] = dict(zip(("config", "group_m"), capi.fp8_grouped_select(g, t, n, k)))
    row["bf16_hgemm_grouped"]["dispatch"] = dict(zip(("config", "group_m"), capi.grouped_select(2, g, t, n, k)))
    row["skipped"] = skipped
    row["group_sizes"] = sizes
    row["t_valid"] = ends[-1]
    return row


def main() -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--repeats", type=int, default=3)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_fp8_grouped.py needs an H100: the grouped FP8 GEMM has no CPU fallback")
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    cases = {}
    for i, (g, t, n, k) in enumerate(CASES + [RAGGED]):
        cases[f"{g}x_{t}_{n}_{k}"] = fp8_grouped_case(g, t, n, k, args, gen, seed=20261016 + i)
        torch.cuda.empty_cache()
    head = cases["8x_8192_4096_7168"]["ours"]
    print(json.dumps({
        "metric": "grouped FP8 GEMM TFLOP/s (2 * valid rows * N * K per call), median of repeats",
        "value": head["tflops"], "unit": "TFLOP/s", "steps": args.steps, "warmup": args.warmup,
        "repeats": args.repeats, "data": "synthetic N(0,1), quantised per 1 x 128 and 128 x 128 block",
        "card": card_info(), "cases": cases,
    }))
    return 0


if __name__ == "__main__":
    sys.exit(main())
