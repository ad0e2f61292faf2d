#!/usr/bin/env python
"""Row-major B (NN) GEMM on the H100: what reading B [K,N] in place costs or saves.

    python tools/bench_nn.py [--rounds R] [--ms MS] [--out FILE]

Legs, timed with CUDA events on one stream, alternating within every round (median over the rounds):
  nn         C = A B through the row-major B kernels (libb200_nn.so), B [K,N] row-major, read in place;
  tn         the K-major kernels on a B transposed ahead of time (Bt [N,K], not timed): the same configuration and
             schedule with the other B layout;
  copy+tn    B.t().contiguous() and then the K-major kernels: what a caller holding B [K,N] paid before;
  torch      torch.matmul(A, B) (cuBLAS), for scale;
and one B200Linear training step (forward + backward of the hgemm operator, fp16, x [2048, 4096] -> [2048, 11008]):
  linear.parent  the backward on transposed copies (dA = hgemm(dC, Bt^T copy), dBt = hgemm(dC^T copy, A^T copy));
  linear.nn      the backward through the NN kernels (dA = hgemm_nn(dC, Bt), dBt = hgemm_nn(dC^T copy, A)).
Shapes (fp16 operands, fp32 accumulation): 4096^3, 2048 x 11008 x 4096 and attention's P.V per head (P [2048, 2048]
by V [2048, 128], B.H = 64 heads run as 64 2-D calls per step). The card and its power limit are recorded with the
results. Needs an H100; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))

import torch  # noqa: E402

from cuda_l2_b200 import capi, ops  # noqa: E402


def card() -> dict:
    """The GPU's name, power limit and maximum SM clock (nvidia-smi, read only)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:   # noqa: BLE001 - the numbers still stand, the record says why the card is unknown
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def time_ms(fn, iters: int) -> float:
    """Milliseconds per call of ``fn`` over ``iters`` back-to-back calls, CUDA events on the current stream."""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def alternate(legs: dict, rounds: int, ms: float) -> dict:
    """Median ms per call of every leg, the legs alternating within each round; each timing covers about ``ms``."""
    iters = {}
    for name, fn in legs.items():   # warm-up, and the call count of a timing
        fn()
        torch.cuda.synchronize()
        iters[name] = max(3, int(ms / max(time_ms(fn, 3), 1e-3)))
    samples = {name: [] for name in legs}
    for _ in range(rounds):
        for name, fn in legs.items():
            samples[name].append(time_ms(fn, iters[name]))
    return {name: {"ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for name, v in samples.items()}


def gemm_legs(m: int, n: int, k: int, calls: int, seed: int) -> tuple[dict, float]:
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = [torch.randn((m, k), device="cuda", generator=g).half() for _ in range(calls)]
    b = [torch.randn((k, n), device="cuda", generator=g).half() for _ in range(calls)]
    bt = [x.t().contiguous() for x in b]
    c = [torch.empty((m, n), dtype=torch.half, device="cuda") for _ in range(calls)]
    s = torch.cuda.current_stream().cuda_stream

    def nn():
        for i in range(calls):
            capi.gemm_rowmajor(a[i], b[i], c[i], "fp32", stream=s)

    def tn():
        for i in range(calls):
            capi.gemm_kmajor(a[i], bt[i], c[i], "fp32", stream=s)

    def copy_tn():
        for i in range(calls):
            capi.gemm_kmajor(a[i], b[i].t().contiguous(), c[i], "fp32", stream=s)

    def matmul():
        for i in range(calls):
            torch.matmul(a[i], b[i], out=c[i])

    # the two layouts compute the same bits (tests/test_gpu_nn.py); checked here on the timed operands as well
    nn()
    want = torch.empty_like(c[-1])
    capi.gemm_kmajor(a[-1], bt[-1], want, "fp32", stream=s)
    torch.cuda.synchronize()
    assert torch.equal(c[-1].view(torch.int16), want.view(torch.int16)), "NN and TN differ"
    return {"nn": nn, "tn": tn, "copy+tn": copy_tn, "torch": matmul}, 2.0 * m * n * k * calls


class _ParentBackward(torch.autograd.Function):
    """The hgemm operator with the backward it had before the NN kernels: three transposed copies."""

    @staticmethod
    def forward(ctx, a, bt):
        ctx.save_for_backward(a, bt)
        return torch.ops.cuda_l2_b200.hgemm(a, bt, "fp32")

    @staticmethod
    def backward(ctx, g):
        a, bt = ctx.saved_tensors
        g = g.contiguous()
        return (torch.ops.cuda_l2_b200.hgemm(g, bt.t().contiguous(), "fp32"),
                torch.ops.cuda_l2_b200.hgemm(g.t().contiguous(), a.t().contiguous(), "fp32"))


def linear_legs(tokens: int, d_in: int, d_out: int, seed: int) -> tuple[dict, float]:
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((tokens, d_in), device="cuda", generator=g).half().requires_grad_(True)
    lin = ops.B200Linear(d_in, d_out, bias=False, device="cuda", dtype=torch.half)
    dy = torch.randn((tokens, d_out), device="cuda", generator=g).half()

    def new():
        x.grad = lin.weight.grad = None
        lin(x).backward(dy)

    def parent():
        x.grad = lin.weight.grad = None
        _ParentBackward.apply(x, lin.weight).backward(dy)

    # same gradients, bit for bit
    new()
    gx, gw = x.grad.clone(), lin.weight.grad.clone()
    parent()
    assert torch.equal(gx.view(torch.int16), x.grad.view(torch.int16)), "dA differs from the parent formula"
    assert torch.equal(gw.view(torch.int16), lin.weight.grad.view(torch.int16)), "dBt differs from the parent formula"
    return {"linear.parent": parent, "linear.nn": new}, 3 * 2.0 * tokens * d_in * d_out


def main() -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=7)
    p.add_argument("--ms", type=float, default=100.0, help="length of one timing of one leg")
    p.add_argument("--out", type=str, default=None, help="also write the JSON result here")
    args = p.parse_args()
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        raise SystemExit("bench_nn.py needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)
    result = {"card": card(), "rounds": args.rounds, "results": {}}
    cases = {"4096_4096_4096": (4096, 4096, 4096, 1), "2048_11008_4096": (2048, 11008, 4096, 1),
             "pv_bh64_s2048_d128": (2048, 128, 2048, 64)}
    for seed, (name, (m, n, k, calls)) in enumerate(cases.items()):
        legs, flops = gemm_legs(m, n, k, calls, seed)
        times = alternate(legs, args.rounds, args.ms)
        for v in times.values():
            v["tflops"] = flops / (v["ms"] * 1e-3) / 1e12
        result["results"][name] = times
        del legs
        torch.cuda.empty_cache()
    legs, flops = linear_legs(2048, 4096, 11008, 99)
    times = alternate(legs, args.rounds, args.ms)
    for v in times.values():
        v["tflops"] = flops / (v["ms"] * 1e-3) / 1e12
    result["results"]["b200linear_fwd_bwd_2048x4096x11008"] = times
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
