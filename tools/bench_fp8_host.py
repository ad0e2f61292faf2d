#!/usr/bin/env python
"""Time the host side of a decode-size FP8 GEMM: back-to-back ``ops.fp8_gemm`` calls on an H100.

    python tools/bench_fp8_host.py [--calls C] [--warmup W] [--tree DIR]

One product, M = 16 and N = K = 4096, e4m3 operands quantised from N(0,1) data, bf16 output, with rowwise scales
(scale_a [M,1], scale_b [1,N]) and with blockwise scales (scale_a 1 x 128 in the M-major layout the quantiser returns,
scale_b 128 x 128). At this size a call's Python work (argument checks, scale classification and preparation, the
ctypes call) is as long as its kernel, so the time per call is mostly host overhead. Each leg: W warm-up calls, then C
back-to-back calls between two CUDA events on the current stream, reported as microseconds per call. ``--tree`` times
the ``cuda_l2_b200`` package of another checkout (built, with its own ``lib/``) instead of this one's, so that two
versions can be compared in one session by alternating runs of this script. Prints one JSON line with the card's name
and enforced power limit. Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))

import torch  # noqa: E402

from bench_fp8 import card_info  # noqa: E402

M, N, K = 16, 4096, 4096


def time_calls(fn, calls: int, warmup: int) -> float:
    """Microseconds per call of ``fn`` over ``calls`` back-to-back calls, after ``warmup`` untimed ones."""
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1000.0 / calls


def main() -> None:
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    p.add_argument("--calls", type=int, default=10000)
    p.add_argument("--warmup", type=int, default=500)
    p.add_argument("--tree", type=Path, default=Path(__file__).resolve().parent.parent)
    args = p.parse_args()
    sys.path.insert(0, str(args.tree.resolve()))
    from cuda_l2_b200 import ops

    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((M, K), device="cuda", generator=gen).bfloat16()
    w = torch.randn((N, K), device="cuda", generator=gen).bfloat16()
    (a_r, sa_r), (bt_r, sb_r) = ops.quantize_e4m3_rowwise(x), ops.quantize_e4m3_rowwise(w)
    (a_b, sa_b), (bt_b, sb_b) = ops.quantize_e4m3_blockwise(x), ops.quantize_e4m3_block128x128(w)
    sb_r = sb_r.reshape(1, N)
    legs = {
        "rowwise": lambda: ops.fp8_gemm(a_r, bt_r, sa_r, sb_r, torch.bfloat16),
        "blockwise": lambda: ops.fp8_gemm(a_b, bt_b, sa_b, sb_b, torch.bfloat16),
    }
    us = {name: round(time_calls(fn, args.calls, args.warmup), 3) for name, fn in legs.items()}
    print(json.dumps({"tree": str(args.tree), "shape": [M, N, K], "out": "bf16", "calls": args.calls,
                      "us_per_call": us, "card": card_info()}))


if __name__ == "__main__":
    main()
