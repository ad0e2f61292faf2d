#!/usr/bin/env python
"""fp32 weight-gradient accumulation on the H100: the weight gradient added into an fp32 main-grad buffer by the GEMM
epilogue (libb200_wgrad_accum.so) against the existing 16-bit dW followed by ``main_grad.add_(dW)``.

    python tools/bench_wgrad_accum.py [--rounds R] [--ms MS] [--out FILE]

dW legs, at the step shapes of tools/bench_fp8_train.py (tokens x in -> out: 2048 x 4096 -> 11008, 4096 x 11008 ->
4096, 4096 x 4096 -> 4096, 8192 x 3072 -> 768), dW [out, in] reducing over the tokens, on the same operands:
  bf16   fused: ops.wgrad_accumulate_ (the K-grouped kernel, dY and X read in place);
         unfused: B200Linear's dW (hgemm_nn on a dY^T copy, T % 8 == 0 at every shape), then main_grad.add_(dW);
         kgrouped_add: the K-grouped kernel's bf16 dW (the fused kernel's sibling), then main_grad.add_(dW);
         addmm: torch.addmm(main_grad, dy.t(), x, out_dtype=torch.float32) (cuBLAS), where torch accepts it;
  fp8 rowwise / fp8 blockwise   fused: ops.fp8_gemm_accumulate_ on the e4m3 operands dW is computed from;
         unfused: ops.fp8_gemm to bf16, then main_grad.add_(dW).
Step legs: one layer step over 4 micro-batches of the shape (x requiring a gradient, bf16 with a bias), forward and
backward, captured in one CUDA graph and replayed: B200Linear and B200Fp8TrainLinear in both recipes, fused
(fuse_wgrad_accumulation) and unfused (the 16-bit .grad added into main_grad after each micro-batch and set to None).
A captured graph keeps only its own memory pool alive, not the tensors it reads and writes that were allocated before
the capture (the inputs, the layer's weight, bias and main_grad), so each graph is kept with them: a tensor freed
while its graph lives hands its memory back, and the next capture's empty_cache() returns it to the driver.
Every set of legs alternates within each round (median and range over the rounds, CUDA events). The card and its
power limit are recorded with the results. Needs an H100; there is no CPU path.
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

STEP_SHAPES = [(2048, 4096, 11008), (4096, 11008, 4096), (4096, 4096, 4096), (8192, 3072, 768)]   # tokens, in, out
MICRO = 4


def dw_legs(tokens: int, k_in: int, n_out: int) -> dict:
    g = torch.Generator(device="cuda").manual_seed(tokens + n_out)
    dy = torch.randn((tokens, n_out), device="cuda", generator=g).bfloat16()
    x = torch.randn((tokens, k_in), device="cuda", generator=g).bfloat16()
    mg = torch.zeros((n_out, k_in), device="cuda")
    ends = torch.tensor([tokens], dtype=torch.int32, device="cuda")
    dw = torch.empty((1, n_out, k_in), dtype=torch.bfloat16, device="cuda")
    legs = {
        "bf16_fused": lambda: ops.wgrad_accumulate_(mg, dy, x),
        "bf16_unfused": lambda: mg.add_(torch.ops.cuda_l2_b200.hgemm_nn(dy.t().contiguous(), x, "fp32")),
        "bf16_kgrouped_add": lambda: (capi.gemm_grouped_wgrad(dy, x, dw, ends,
                                                              stream=torch.cuda.current_stream().cuda_stream),
                                      mg.add_(dw[0])),
    }
    try:
        torch.addmm(mg, dy.t(), x, out_dtype=torch.float32)
        legs["bf16_addmm"] = lambda: torch.addmm(mg, dy.t(), x, out_dtype=torch.float32, out=mg)
    except (RuntimeError, TypeError) as e:
        print(f"torch.addmm(out_dtype=float32) refused: {e}")
    # the e4m3 operands of dW = q(dY^T) q(X^T)^T, as the training layers quantise them
    gy_q, gy_s, gy_qt, gy_st = ops.quantize_e4m3_rowwise_dual(dy)
    x_q, x_s, x_qt, x_st = ops.quantize_e4m3_rowwise_dual(x)
    rw = (gy_qt, x_qt, gy_st.reshape(-1, 1), x_st.reshape(1, -1))
    _, _, bgy_qt, bgy_st = ops.quantize_e4m3_blockwise_dual(dy)
    _, _, bx_qt, bx_st = ops.quantize_e4m3_blockwise_dual(x)
    bw = (bgy_qt, bx_qt, bgy_st, bx_st)
    for name, ops_ in (("fp8_rowwise", rw), ("fp8_blockwise", bw)):
        legs[f"{name}_fused"] = lambda o=ops_: ops.fp8_gemm_accumulate_(mg, *o)
        legs[f"{name}_unfused"] = lambda o=ops_: mg.add_(ops.fp8_gemm(*o, torch.bfloat16))
    return legs


def step_legs(tokens: int, k_in: int, n_out: int) -> tuple[dict, list]:
    """The captured step of each layer kind, fused and unfused: {leg: replay}, and what must outlive the replays (the
    inputs, and each graph with its layer)."""
    torch.manual_seed(0)
    makers = {
        "bf16": lambda fuse: ops.B200Linear(k_in, n_out, device="cuda", dtype=torch.bfloat16,
                                            fuse_wgrad_accumulation=fuse),
        "fp8_rowwise": lambda fuse: ops.B200Fp8TrainLinear(k_in, n_out, device="cuda", fuse_wgrad_accumulation=fuse),
        "fp8_blockwise": lambda fuse: ops.B200Fp8TrainLinear(k_in, n_out, device="cuda", granularity="blockwise",
                                                             fuse_wgrad_accumulation=fuse),
    }
    xs = [torch.randn((tokens, k_in), device="cuda").bfloat16().requires_grad_() for _ in range(MICRO)]
    gy = torch.randn((tokens, n_out), device="cuda").bfloat16()
    legs, keep = {}, [xs, gy]   # the inputs every graph reads
    for name, make in makers.items():
        for fuse in (True, False):
            layer = make(fuse)
            layer.weight.main_grad = torch.zeros(layer.weight.shape, device="cuda")

            def step(layer=layer, fuse=fuse):
                for x in xs:
                    layer(x).backward(gy)
                    if not fuse:
                        layer.weight.main_grad.add_(layer.weight.grad)
                        layer.weight.grad = None

            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                step()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            for x in xs:
                x.grad = None
            layer.bias.grad = None
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                step()
            keep.append((layer, graph))
            legs[f"{name}_{'fused' if fuse else 'unfused'}"] = graph.replay
    return legs, keep


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--ms", type=float, default=200.0)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wgrad_accum.py needs an H100")
    capi.wgrad_accum_prewarm(torch.cuda.current_stream().cuda_stream)
    result = {"card": card(), "dw": {}, "step": {}}
    for shape in STEP_SHAPES:
        key = "x".join(map(str, shape))
        result["dw"][key] = alternate(dw_legs(*shape), args.rounds, args.ms)
        legs, keep = step_legs(*shape)
        result["step"][key] = alternate(legs, args.rounds, args.ms)
        del legs, keep
        print(key, json.dumps({k: round(v["ms"], 4) for k, v in {**result["dw"][key], **result["step"][key]}.items()}),
              flush=True)
    result["card"] = {**result["card"], "after": card()}
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(text)


if __name__ == "__main__":
    main()
