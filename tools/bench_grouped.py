#!/usr/bin/env python
"""Time the grouped fp16 / bf16 GEMM over contiguous row groups (libb200_grouped.so) on an H100.

    python tools/bench_grouped.py [--steps K] [--warmup W] [--repeats R]

Cases, the MoE prefill layout (tokens sorted by expert into one [T, K] tensor, one [N, K] weight per expert), each in
bf16 and fp16 (fp32 accumulation): 8 experts of T = 8192, N = 14336, K = 4096, and 64 experts of T = 16384, N = 2048,
K = 7168. The group sizes are seeded and uneven: T - 5 - 3G tokens split by Dirichlet(2) weights, then two experts
lose all of theirs and every non-empty size that is a multiple of 16 gains 3 rows. So the last group ends before T
(rows past it belong to no group), and T_valid, not T, is the work counted.

Legs, each case timed R times with its legs alternating (ours, theirs, ours, ...), reported as the median and the range:
* ``ours``: the dispatched grouped call, offsets on the device;
* ``torch_grouped_mm`` (bf16 only): ``torch._grouped_mm(a, bt.transpose(-2, -1), offs=offs)``;
* ``loop_of_ops_hgemm``: a Python loop of ops.hgemm over each expert's rows, the offsets known on the host (which the
  grouped call does not need);
* ``batched_masked_padded``: the masked batched call (libb200_batched.so) on the equivalent padded layout
  [G, max group, K], excluding the scatter into it and the gather out of it.
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


def group_sizes(g: int, t: int, seed: int) -> list[int]:
    """Seeded, uneven sizes summing to less than T: two empty groups, none a multiple of 16 unless empty."""
    rng = np.random.default_rng(seed)
    sizes = rng.multinomial(t - 5 - 3 * g, rng.dirichlet(np.full(g, 2.0)))
    sizes[rng.choice(g, size=2, replace=False)] = 0
    sizes = [int(s) + (3 if s % 16 == 0 and s else 0) for s in sizes]
    return sizes


def operand_sets(g, t, n, k, m_max, dtype, gen):
    set_bytes = 2 * (t * k + g * n * k + t * n + g * m_max * (k + n))
    nsets = max(2, min(16, -(-4 * L2_BYTES // set_bytes)))
    sets = []
    for _ in range(nsets):
        a = torch.randn((t, k), device="cuda", generator=gen).to(dtype)
        bt = torch.randn((g, n, k), device="cuda", generator=gen).to(dtype)
        sets.append(dict(a=a, bt=bt, c=torch.empty((t, n), dtype=dtype, device="cuda"),
                         a_pad=torch.randn((g, m_max, k), device="cuda", generator=gen).to(dtype),
                         c_pad=torch.empty((g, m_max, n), dtype=dtype, device="cuda")))
    return sets


def grouped_case(g, t, n, k, dtype, args, gen, seed):
    from cuda_l2_b200 import capi, ops

    sizes = group_sizes(g, t, seed)
    ends = [int(x) for x in np.cumsum(sizes)]
    starts = [0] + ends[:-1]
    offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
    counts = torch.tensor(sizes, dtype=torch.int32, device="cuda")
    m_max = max(sizes)
    sets = operand_sets(g, t, n, k, m_max, dtype, gen)
    stream = lambda: torch.cuda.current_stream().cuda_stream   # noqa: E731

    def loop(s):
        for e, (r0, r1) in enumerate(zip(starts, ends)):
            if r1 > r0:
                ops.hgemm(s["a"][r0:r1], s["bt"][e])

    legs = {"ours": lambda s: capi.gemm_grouped(s["a"], s["bt"], s["c"], offs, "fp32", stream=stream())}
    if dtype == torch.bfloat16:
        legs["torch_grouped_mm"] = lambda s: torch._grouped_mm(s["a"], s["bt"].transpose(-2, -1), offs=offs)
    legs["loop_of_ops_hgemm"] = loop
    legs["batched_masked_padded"] = lambda s: capi.gemm_batched(s["a_pad"], s["bt"], s["c_pad"], "fp32",
                                                                masked_m=counts, stream=stream())
    row = time_legs(legs, sets, 2.0 * ends[-1] * n * k, args.steps, args.warmup, args.repeats)
    variant = capi.batched_variant(dtype)
    row["ours"]["dispatch"] = dict(zip(("config", "group_m"), capi.grouped_select(variant, g, t, n, k)))
    row["batched_masked_padded"]["dispatch"] = dict(zip(("config", "group_m"),
                                                        capi.batched_select(variant, g, m_max, n, k)))
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
        raise SystemExit("tools/bench_grouped.py needs an H100: the grouped GEMM has no CPU fallback")
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    cases = {}
    for i, (g, t, n, k) in enumerate(((8, 8192, 14336, 4096), (64, 16384, 2048, 7168))):
        for dtype in (torch.bfloat16, torch.float16):
            cases[f"{str(dtype)[6:]}_{g}x_{t}_{n}_{k}"] = grouped_case(g, t, n, k, dtype, args, gen, seed=20261016 + i)
            torch.cuda.empty_cache()
    head = cases["bfloat16_8x_8192_14336_4096"]["ours"]
    print(json.dumps({
        "metric": "grouped GEMM TFLOP/s (2 * valid rows * N * K per call), median of repeats", "value": head["tflops"],
        "unit": "TFLOP/s", "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats,
        "data": "synthetic N(0,1)", "card": card_info(), "cases": cases,
    }))
    return 0


if __name__ == "__main__":
    sys.exit(main())
