#!/usr/bin/env python
"""The fused SwiGLU gate / up projection on the H100 (libb200_swiglu.so) against the compositions it replaces.

    python tools/bench_swiglu.py [--rounds R] [--ms MS] [--out FILE]

Shapes (tokens M, hidden H, intermediate I), bf16: H = 4096 with I = 11008 and 14336 at M in {16, 2048, 8192}, and the
small decode shape M = 16, H = 2048, I = 1408, where the TN dispatcher picks split-K for (M, 2I, K) and the gated
kernel, which has only the plain schedule, runs unsplit. Legs, alternating within each round (CUDA events, median and
range over the rounds):
  fused:        ops.swiglu_linear under no_grad (one launch, h never written);
  hgemm_torch:  ops.hgemm into h = [g | u], then F.silu(g) * u;
  cublas_torch: F.linear twice (cuBLAS), then F.silu(g) * u;
  train_fused:  forward + backward of ops.swiglu_linear (x and w_gu requiring gradients);
  train_hgemm:  forward + backward of ops.hgemm + F.silu(g) * u through torch autograd;
  bwd_kernel:   the SwiGLU backward alone, with its bytes (dy, h read, dh written) over its time in GB/s against the
                3.35 TB/s HBM3 data-sheet figure of the H100 SXM.
The card and its power limit are recorded with the results. Needs an H100; there is no CPU path.
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
from cuda_l2_b200 import capi, ops  # noqa: E402

SHAPES = [(16, 4096, 11008), (2048, 4096, 11008), (8192, 4096, 11008), (16, 4096, 14336), (2048, 4096, 14336),
          (8192, 4096, 14336), (16, 2048, 1408)]
HBM_TBPS = 3.35


def legs(m: int, hid: int, i: int) -> tuple[dict, int]:
    g = torch.Generator(device="cuda").manual_seed(m + i)
    x = (torch.randn((m, hid), device="cuda", generator=g) / 4).bfloat16()
    w_gate = (torch.randn((i, hid), device="cuda", generator=g) / hid ** 0.5).bfloat16()
    w_up = (torch.randn((i, hid), device="cuda", generator=g) / hid ** 0.5).bfloat16()
    w_gu = ops.interleave_gate_up(w_gate, w_up)
    w_cat = torch.cat((w_gate, w_up))   # [g | u] for the hgemm composition
    dy = torch.randn((m, i), device="cuda", generator=g).bfloat16()
    xr, wr, wcr = (t.clone().requires_grad_() for t in (x, w_gu, w_cat))
    h = torch.empty((m, 2 * i), dtype=torch.bfloat16, device="cuda")
    dh = torch.empty_like(h)
    stream = torch.cuda.current_stream().cuda_stream

    def fused():
        with torch.no_grad():
            ops.swiglu_linear(x, w_gu)

    def hgemm_torch():
        hh = ops.hgemm(x, w_cat)
        return F.silu(hh[:, :i]) * hh[:, i:]

    def cublas_torch():
        return F.silu(F.linear(x, w_gate)) * F.linear(x, w_up)

    def train_fused():
        xr.grad = wr.grad = None
        ops.swiglu_linear(xr, wr).backward(dy)

    def train_hgemm():
        xr.grad = wcr.grad = None
        hh = ops.hgemm(xr, wcr)
        (F.silu(hh[:, :i]) * hh[:, i:]).backward(dy)

    capi.swiglu(x, w_gu, torch.empty((m, i), dtype=torch.bfloat16, device="cuda"), h, stream=stream)
    bwd_bytes = 2 * (m * i + 2 * m * 2 * i)
    return {"fused": fused, "hgemm_torch": hgemm_torch, "cublas_torch": cublas_torch, "train_fused": train_fused,
            "train_hgemm": train_hgemm,
            "bwd_kernel": lambda: capi.swiglu_backward(dy, h, dh, stream=stream)}, bwd_bytes


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--ms", type=float, default=100.0)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_swiglu.py needs an H100")
    result = {"card": card(), "shapes": {}}
    for m, hid, i in SHAPES:
        key = f"{m}x{hid}x{i}"
        fns, bwd_bytes = legs(m, hid, i)
        r = alternate(fns, args.rounds, args.ms)
        r["bwd_kernel"]["gbps"] = bwd_bytes / (r["bwd_kernel"]["ms"] * 1e-3) / 1e9
        r["bwd_kernel"]["share_of_hbm_peak"] = r["bwd_kernel"]["gbps"] / (HBM_TBPS * 1e3)
        r["choice"] = {"swiglu": capi.swiglu_select(2, m, i, hid), "tn_2i": capi.select("fp32", m, 2 * i, hid)}
        result["shapes"][key] = r
        print(key, json.dumps({k: round(v["ms"], 4) for k, v in r.items() if "ms" in v}),
              f"bwd {r['bwd_kernel']['gbps']:.0f} GB/s", r["choice"], flush=True)
        del fns
        torch.cuda.empty_cache()
    result["card"] = {**result["card"], "after": card()}
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(text)


if __name__ == "__main__":
    main()
