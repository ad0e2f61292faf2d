#!/usr/bin/env python
"""Time the batched fp16 / bf16 GEMM (libb200_batched.so) on an H100 against torch.bmm and per-matrix launches.

    python tools/bench_batched.py [--steps K] [--warmup W] [--repeats R]

Legs, each case timed R times with its legs alternating (ours, theirs, ours, ...), reported as the median and the range:
* dense, attention-like: B = 64 of 1024x1024x128 and of 1024x128x1024 (M x N x K), fp16 (fp32 accumulation) and bf16:
  the dispatched batched call against torch.bmm;
* masked, MoE-like (bf16): 8 experts of M = 512, N = 14336, K = 4096 and 32 experts of M = 256, N = 4096, K = 7168, with
  seeded per-expert row counts uniform in [0, M/2] (a quarter of M on average): the masked batched call against
  torch.bmm over the padded tensors and against a Python loop of ops.hgemm over each expert's valid rows (counts known
  on the host, which the masked call does not need);
* overhead: B = 1 at 4096^3 and 2048x11008x4096 (fp16): the batched kernel against the 2-D kernel of the same
  configuration and group_m on the plain schedule.
Each timing: warm-up, then K back-to-back calls between two CUDA events on the current stream, rotating over seeded
operand sets whose footprint exceeds the 50 MB L2 four times (at least two sets). TFLOP/s count valid rows only,
2 * sum(rows) * N * K per call. Prints one JSON line with the card's name and enforced power limit. Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

import torch  # noqa: E402

from bench_fp8 import L2_BYTES, card_info  # noqa: E402


def operand_sets(bsz, m, n, k, dtype, gen):
    set_bytes = 2 * bsz * (m * k + n * k + m * n)
    nsets = max(2, min(16, -(-4 * L2_BYTES // set_bytes)))
    sets = []
    for _ in range(nsets):
        a = torch.randn((bsz, m, k), device="cuda", generator=gen).to(dtype)
        bt = torch.randn((bsz, n, k), device="cuda", generator=gen).to(dtype)
        sets.append(dict(a=a, bt=bt, c=torch.empty((bsz, m, n), dtype=dtype, device="cuda")))
    return sets


def time_legs(legs: dict, sets: list, flops: float, steps: int, warmup: int, repeats: int) -> dict:
    for fn in legs.values():
        for i in range(max(warmup, 3)):
            fn(sets[i % len(sets)])
    torch.cuda.synchronize()
    ms = {name: [] for name in legs}
    for _ in range(repeats):
        for name, fn in legs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(steps):
                fn(sets[i % len(sets)])
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / steps)
    out = {}
    for name, xs in ms.items():
        tf = [flops / (x * 1e-3) * 1e-12 for x in xs]
        out[name] = {"tflops": statistics.median(tf), "tflops_min": min(tf), "tflops_max": max(tf),
                     "ms_per_call": statistics.median(xs)}
    return out


def dense_case(bsz, m, n, k, dtype, args, gen):
    from cuda_l2_b200 import capi

    sets = operand_sets(bsz, m, n, k, dtype, gen)
    legs = {"ours": lambda s: capi.gemm_batched(s["a"], s["bt"], s["c"], "fp32",
                                                stream=torch.cuda.current_stream().cuda_stream),
            "torch_bmm": lambda s: torch.bmm(s["a"], s["bt"].transpose(1, 2), out=s["c"])}
    row = time_legs(legs, sets, 2.0 * bsz * m * n * k, args.steps, args.warmup, args.repeats)
    row["ours"]["dispatch"] = dict(zip(("config", "group_m"), capi.batched_select(capi.batched_variant(dtype), bsz, m, n, k)))
    return row


def masked_case(bsz, m, n, k, args, gen, seed):
    from cuda_l2_b200 import capi, ops

    dtype = torch.bfloat16
    g = torch.Generator().manual_seed(seed)
    counts = torch.randint(0, m // 2 + 1, (bsz,), generator=g, dtype=torch.int32)
    host = [int(x) for x in counts]
    mm = counts.cuda()
    sets = operand_sets(bsz, m, n, k, dtype, gen)

    def loop(s):
        for e, r in enumerate(host):
            if r:
                ops.hgemm(s["a"][e, :r], s["bt"][e])

    legs = {"ours_masked": lambda s: capi.gemm_batched(s["a"], s["bt"], s["c"], "fp32", masked_m=mm,
                                                       stream=torch.cuda.current_stream().cuda_stream),
            "torch_bmm_padded": lambda s: torch.bmm(s["a"], s["bt"].transpose(1, 2), out=s["c"]),
            "loop_of_ops_hgemm": loop}
    row = time_legs(legs, sets, 2.0 * sum(host) * n * k, args.steps, args.warmup, args.repeats)
    row["counts"] = host
    row["mean_count_over_m"] = sum(host) / (bsz * m)
    row["ours_masked"]["dispatch"] = dict(zip(("config", "group_m"), capi.batched_select(2, bsz, m, n, k)))
    return row


def overhead_case(m, n, k, args, gen):
    from cuda_l2_b200 import capi

    sets = operand_sets(1, m, n, k, torch.float16, gen)
    cid, gm = capi.batched_select(0, 1, m, n, k)
    legs = {"batched_b1": lambda s: capi.gemm_batched(s["a"], s["bt"], s["c"], "fp32", config_id=cid, group_m=gm,
                                                      stream=torch.cuda.current_stream().cuda_stream),
            "kernel_2d": lambda s: capi.gemm_kmajor(s["a"][0], s["bt"][0], s["c"][0], "fp32", config_id=cid,
                                                    group_m=gm, splits=1,
                                                    stream=torch.cuda.current_stream().cuda_stream)}
    row = time_legs(legs, sets, 2.0 * m * n * k, args.steps, args.warmup, args.repeats)
    row["config"], row["group_m"] = cid, gm
    return row


def main() -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--repeats", type=int, default=5)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_batched.py needs an H100: the batched GEMM has no CPU fallback")
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    dense, masked, overhead = {}, {}, {}
    for dtype in (torch.float16, torch.bfloat16):
        for (bsz, m, n, k) in ((64, 1024, 1024, 128), (64, 1024, 128, 1024)):
            dense[f"{str(dtype)[6:]}_{bsz}x{m}_{n}_{k}"] = dense_case(bsz, m, n, k, dtype, args, gen)
            torch.cuda.empty_cache()
    for i, (bsz, m, n, k) in enumerate(((8, 512, 14336, 4096), (32, 256, 4096, 7168))):
        masked[f"bf16_{bsz}x{m}_{n}_{k}"] = masked_case(bsz, m, n, k, args, gen, seed=20261015 + i)
        torch.cuda.empty_cache()
    for (m, n, k) in ((4096, 4096, 4096), (2048, 11008, 4096)):
        overhead[f"fp16_{m}_{n}_{k}"] = overhead_case(m, n, k, args, gen)
        torch.cuda.empty_cache()
    head = dense["float16_64x1024_1024_128"]["ours"]
    print(json.dumps({
        "metric": "batched GEMM TFLOP/s (2 * valid rows * N * K per call), median of repeats", "value": head["tflops"],
        "unit": "TFLOP/s", "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats,
        "data": "synthetic N(0,1)", "card": card_info(), "dense": dense, "masked": masked, "b1_overhead": overhead,
    }))
    return 0


if __name__ == "__main__":
    sys.exit(main())
