#!/usr/bin/env python
"""FP8 training of linear layers on the H100: the dual-orientation rowwise quantiser of libb200_quant_dual.so against
the torch composition it replaces, and one layer's training step in FP8 against the same step with the torch
quantisers and against bf16.

    python tools/bench_fp8_train.py [--rounds R] [--ms MS] [--out FILE] [--no-profile]

Quantiser legs, bf16 input at 2048 x 4096, 4096 x 11008, 11008 x 4096 and 16384 x 7168: the kernel
(ops.quantize_e4m3_rowwise_dual) and the composition (ops.quantize_e4m3_rowwise_dual_reference, rowwise quantisation
of x and of x^T padded), timed with CUDA events on one stream, alternating within every round (median and range over
the rounds). A second pass under torch.profiler sums the device time of the library's kernels (b200_quant_dual_*) and
its workspace memset per call; the algorithmic bytes over that time give the bandwidth, counting both reads of x (the
column maxima need every row first), e4m3 written once in each orientation and the scales, against the H100 SXM
data-sheet 3.35 TB/s.

Step legs, tokens x in -> out at 2048 x 4096 -> 11008, 4096 x 11008 -> 4096, 4096 x 4096 -> 4096 and
8192 x 3072 -> 768, bf16 with a bias, x requiring a gradient (a layer inside a network): forward, then backward of a
fixed output gradient, the gradients set to None before each eager step. Four legs, each eager and captured in one CUDA
graph (replayed):
  fp8        B200Fp8TrainLinear (dual quantiser, three rowwise fp8_gemm calls);
  fp8_torch  the same step with the torch quantisers (the composition, x.t() padded and quantised): the "before";
  b200_bf16  B200Linear (hgemm with its gradient);
  torch_bf16 nn.Linear (cuBLAS).
  fp8_blockwise  B200Fp8TrainLinear(granularity="blockwise") (dual block quantisers, two block-scaled fp8_gemm calls
             and one with 1 x 128 scales on both operands);
fp8 and fp8_torch are checked bit for bit (y, dX, dW, db) before timing.

Blockwise legs: the dual 1 x 128 quantiser (ops.quantize_e4m3_blockwise_dual, one launch, x read once) at the quantiser
shapes, its kernel time from torch.profiler (b200_quant_block_dual_*) and its bandwidth; and the weight gradient of each
step shape, dW [out, in] = dY^T [out, T] x X^T [in, T], run by the 1 x 128 x 1 x 128 kernel and by the 128 x 128 kernel
on the same e4m3 operands (Bt's scales per 128 x 128 block), alternating, as TFLOP/s. The card and its power limit are
recorded with the results. Needs an H100; there is no CPU path.
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

from bench_nn import alternate, card  # noqa: E402
from cuda_l2_b200 import capi, ops  # noqa: E402

HBM_TBPS = 3.35   # H100 SXM data sheet
QUANT_SHAPES = [(2048, 4096), (4096, 11008), (11008, 4096), (16384, 7168)]
STEP_SHAPES = [(2048, 4096, 11008), (4096, 11008, 4096), (4096, 4096, 4096), (8192, 3072, 768)]   # tokens, in, out


def dual_bytes(rows: int, cols: int) -> int:
    """Algorithmic bytes of one dual quantisation of bf16 [rows, cols]: x read twice, e4m3 written in both
    orientations (q_t with its padding), fp32 scales once."""
    ld_t = -(-rows // 16) * 16
    return 2 * rows * cols * 2 + rows * cols + cols * ld_t + 4 * (rows + cols)


def block_dual_bytes(rows: int, cols: int) -> int:
    """Algorithmic bytes of one dual 1 x 128 quantisation of bf16 [rows, cols]: x read once, e4m3 written in both
    orientations (q_t with its padding), fp32 scales once each."""
    ld_t = -(-rows // 16) * 16
    return rows * cols * 2 + rows * cols + cols * ld_t + 4 * (rows * -(-cols // 128) + cols * -(-rows // 128))


def kernel_us(fn, calls: int, key: str = "b200_quant_dual_", memset: bool = True) -> float:
    """Device time of the kernels whose names contain ``key`` (and, with ``memset``, the workspace memsets) per call of
    ``fn`` (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    total = sum(ev.device_time_total for ev in prof.key_averages()
                if key in ev.key or (memset and ev.key.lower().startswith("memset")))
    return total / calls


class _TorchQuantFp8Linear(torch.autograd.Function):
    """fp8_linear's step with the torch quantisers: the same GEMMs on the same bits."""

    @staticmethod
    def forward(ctx, x2, w):
        xq, xs, xqt, xst = ops.quantize_e4m3_rowwise_dual_reference(x2)
        wq, ws, wqt, wst = ops.quantize_e4m3_rowwise_dual_reference(w)
        ctx.save_for_backward(xqt, xst, wqt, wst)
        return ops.fp8_gemm(xq, wq, xs.reshape(-1, 1), ws.reshape(1, -1), x2.dtype)

    @staticmethod
    def backward(ctx, gy):
        xqt, xst, wqt, wst = ctx.saved_tensors
        gq, gs, gqt, gst = ops.quantize_e4m3_rowwise_dual_reference(gy.contiguous())
        dx = ops.fp8_gemm(gq, wqt, gs.reshape(-1, 1), wst.reshape(1, -1), gy.dtype)
        dw = ops.fp8_gemm(gqt, xqt, gst.reshape(-1, 1), xst.reshape(1, -1), gy.dtype)
        return dx, dw


def step_legs(t: int, k: int, n: int, seed: int) -> dict:
    g = torch.Generator(device="cuda").manual_seed(seed)
    lin = torch.nn.Linear(k, n, device="cuda", dtype=torch.bfloat16)
    fp8 = ops.B200Fp8TrainLinear.from_linear(lin)
    fp8_blockwise = ops.B200Fp8TrainLinear.from_linear(lin, granularity="blockwise")
    b200 = ops.B200Linear.from_linear(lin)
    x = torch.randn((t, k), device="cuda", generator=g).bfloat16().requires_grad_()
    gy = torch.randn((t, n), device="cuda", generator=g).bfloat16()
    forwards = {"fp8": fp8, "fp8_torch": lambda a: _TorchQuantFp8Linear.apply(a, lin.weight) + lin.bias,
                "fp8_blockwise": fp8_blockwise, "b200_bf16": b200, "torch_bf16": lin}

    def eager(fwd):
        def step():
            lin.weight.grad = lin.bias.grad = x.grad = None
            fwd(x).backward(gy)
        return step

    outs = {}
    for name in ("fp8", "fp8_torch"):
        eager(forwards[name])()
        y = forwards[name](x).detach()
        outs[name] = [y, x.grad, lin.weight.grad, lin.bias.grad]
    for a, b in zip(outs["fp8"], outs["fp8_torch"]):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "fp8 and fp8_torch differ"
    del outs
    legs = {}
    for name, fwd in forwards.items():
        legs[f"{name}_eager"] = eager(fwd)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                eager(fwd)()
        torch.cuda.current_stream().wait_stream(side)
        lin.weight.grad = lin.bias.grad = x.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fwd(x).backward(gy)
        legs[f"{name}_graph"] = graph.replay
    return legs


def wgrad_legs(t: int, k: int, n: int, seed: int) -> tuple[dict, float]:
    """dW = dY^T X of a step shape on e4m3 operands from the dual 1 x 128 quantiser: the 1 x 128 x 1 x 128 kernel, and
    the 128 x 128 kernel with X^T's scales taken per 128 x 128 block (their maxima); and the product's FLOPs."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    _, _, gqt, gst = ops.quantize_e4m3_blockwise_dual(torch.randn((t, n), device="cuda", generator=g).bfloat16())
    _, _, xqt, xst = ops.quantize_e4m3_blockwise_dual(torch.randn((t, k), device="cuda", generator=g).bfloat16())
    nkb = xst.shape[1]
    pad = torch.zeros((-(-k // 128) * 128, nkb), device="cuda")
    pad[:k] = xst
    xst_block = pad.view(-1, 128, nkb).amax(1).contiguous()
    one_d = torch.empty((n, k), dtype=torch.bfloat16, device="cuda")
    block = torch.empty_like(one_d)
    legs = {"1x128_1x128": lambda: capi.fp8_gemm(gqt, xqt, one_d, gst, xst, stream=torch.cuda.current_stream().cuda_stream),
            "1x128_128x128": lambda: capi.fp8_gemm(gqt, xqt, block, gst, xst_block,
                                                   stream=torch.cuda.current_stream().cuda_stream)}
    return legs, 2.0 * n * k * gqt.shape[1]


def main() -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=7)
    p.add_argument("--ms", type=float, default=100.0, help="length of one timing of one leg")
    p.add_argument("--out", type=str, default=None, help="also write the JSON result here")
    p.add_argument("--no-profile", action="store_true", help="skip the torch.profiler pass (no kernel times)")
    args = p.parse_args()
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
        raise SystemExit("bench_fp8_train.py needs an H100 (compute capability 9.0)")
    torch.cuda.set_device(0)
    result = {"card": card(), "rounds": args.rounds, "hbm_tbps_datasheet": HBM_TBPS, "dual_quantiser": {},
              "block_dual_quantiser": {}, "wgrad": {}, "step": {}}
    g = torch.Generator(device="cuda").manual_seed(1)
    for rows, cols in QUANT_SHAPES:
        x = torch.randn((rows, cols), device="cuda", generator=g).bfloat16()
        fns = {"kernel": lambda a=x: ops.quantize_e4m3_rowwise_dual(a),
               "torch": lambda a=x: ops.quantize_e4m3_rowwise_dual_reference(a)}
        for got, want in zip(fns["kernel"](), fns["torch"]()):
            dt = torch.uint8 if got.dtype == torch.float8_e4m3fn else torch.int32
            assert torch.equal(got.view(dt), want.view(dt)), (rows, cols)
        nbytes = dual_bytes(rows, cols)
        times = alternate(fns, args.rounds, args.ms)
        for v in times.values():
            v["us"] = v["ms"] * 1e3
        times["bytes"] = nbytes
        times["speedup"] = times["torch"]["ms"] / times["kernel"]["ms"]
        if not args.no_profile:   # a pass of its own: tracing slows the host
            us = kernel_us(fns["kernel"], 50)
            times["kernel_us"] = us
            times["kernel_gbps"] = nbytes / (us * 1e-6) / 1e9
            times["share_of_hbm"] = nbytes / (us * 1e-6) / (HBM_TBPS * 1e12)
        result["dual_quantiser"][f"{rows}x{cols}"] = times
        del x, fns
        torch.cuda.empty_cache()
    for rows, cols in QUANT_SHAPES:
        x = torch.randn((rows, cols), device="cuda", generator=g).bfloat16()
        fns = {"kernel": lambda a=x: ops.quantize_e4m3_blockwise_dual(a),
               "torch": lambda a=x: ops.quantize_e4m3_blockwise_dual_reference(a)}
        for got, want in zip(fns["kernel"](), fns["torch"]()):
            dt = torch.uint8 if got.dtype == torch.float8_e4m3fn else torch.int32
            assert torch.equal(got.view(dt), want.view(dt)), (rows, cols)
        nbytes = block_dual_bytes(rows, cols)
        times = alternate(fns, args.rounds, args.ms)
        for v in times.values():
            v["us"] = v["ms"] * 1e3
        times["bytes"] = nbytes
        if not args.no_profile:
            us = kernel_us(fns["kernel"], 50, "b200_quant_block_dual_", memset=False)
            times["kernel_us"] = us
            times["kernel_gbps"] = nbytes / (us * 1e-6) / 1e9
            times["share_of_hbm"] = nbytes / (us * 1e-6) / (HBM_TBPS * 1e12)
        result["block_dual_quantiser"][f"{rows}x{cols}"] = times
        del x, fns
        torch.cuda.empty_cache()
    for t, k, n in STEP_SHAPES:
        legs, flops = wgrad_legs(t, k, n, seed=t + k + n)
        times = alternate(legs, args.rounds, args.ms)
        for v in times.values():
            v["us"] = v["ms"] * 1e3
            v["tflops"] = flops / (v["ms"] * 1e-3) * 1e-12
        result["wgrad"][f"{n}x{k}x{t}"] = times
        del legs
        torch.cuda.empty_cache()
    for t, k, n in STEP_SHAPES:
        legs = step_legs(t, k, n, seed=t + k + n)
        times = alternate(legs, args.rounds, args.ms)
        for v in times.values():
            v["us"] = v["ms"] * 1e3
        result["step"][f"{t}x{k}->{n}"] = times
        del legs
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
