#!/usr/bin/env python
"""Generate tests/golden/fp8_rowwise_cases.npz — the FP8 (e4m3) fixtures with rowwise scales. Needs torch only.

The truth is torch's CPU expression ``(((qa.float() @ qbt.float().t()) * sb[None, :]) * sa[:, None]).to(out_dtype)``,
never this repository's code. Stored: float8_e4m3fn operands as uint8 codes (a [M,K], bt [N,K]), the fp32 scale
vectors sa [M] and sb [N], the truth as uint16 bits (fp16 or bf16 output) and
meta = [m, n, k, kind (0 small integers, 1 randn), out_bf16, seed].

* small-integer cases: operands in [-lim, lim] with lim * lim * k inside the exact range (2047 for fp16 out, 256 for
  bf16 out), per-row and per-column scales that are powers of two or arbitrary fp32 values, ragged M, N and K — exact;
* N(0,1) cases quantised per row (amax / 448 for each row of a and of bt) — tolerance tests (torch's fp32 matmul sums
  in its own order).

    python tests/golden/make_fp8_rowwise_golden.py
"""
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent

ROWWISE_CASES = [
    # (m, n, k, kind, out, scales, seed)   kind "int<lim>" or "randn"; scales "pow2" | "any" (int cases only)
    (64, 256, 64, "int2", "fp16", "pow2", 61),
    (200, 328, 144, "int2", "fp16", "any", 62),            # ragged M, N and K (144 = one k-block of 128 + 16)
    (129, 136, 272, "int1", "fp16", "any", 63),
    (1, 8, 16, "int2", "fp16", "any", 64),
    (64, 256, 64, "int2", "bf16", "pow2", 65),
    (200, 328, 144, "int1", "bf16", "any", 66),
    (37, 24, 208, "int1", "bf16", "pow2", 67),
    (64, 128, 64, "randn", "fp16", None, 71), (200, 328, 144, "randn", "bf16", None, 72),
    (128, 128, 1024, "randn", "fp16", None, 73),
]


def bits(t):
    return t.contiguous().view(torch.int16).numpy().view(np.uint16)


def scale_vector(size: int, kind: str, gen: torch.Generator) -> torch.Tensor:
    if kind == "pow2":
        return torch.pow(2.0, torch.randint(-3, 4, (size,), generator=gen).float())
    return torch.rand(size, generator=gen) * 2.9 + 0.1      # arbitrary fp32 values in [0.1, 3)


def main():
    out = {}
    for i, (m, n, k, kind, out_name, scales, seed) in enumerate(ROWWISE_CASES):
        gen = torch.Generator().manual_seed(seed)
        out_dtype = {"fp16": torch.float16, "bf16": torch.bfloat16}[out_name]
        if kind.startswith("int"):
            lim = int(kind[3:])
            a = (torch.randint(0, 2 * lim + 1, (m, k), generator=gen) - lim).float()
            bt = (torch.randint(0, 2 * lim + 1, (n, k), generator=gen) - lim).float()
            assert lim * lim * k <= (2047 if out_name == "fp16" else 256)
            sa, sb = scale_vector(m, scales, gen), scale_vector(n, scales, gen)
        else:
            a, bt = torch.randn((m, k), generator=gen), torch.randn((n, k), generator=gen)
            sa, sb = a.abs().amax(dim=1) / 448, bt.abs().amax(dim=1) / 448
            a, bt = a / sa[:, None], bt / sb[:, None]
        qa, qbt = a.to(torch.float8_e4m3fn), bt.to(torch.float8_e4m3fn)
        truth = (((qa.float() @ qbt.float().t()) * sb[None, :]) * sa[:, None]).to(out_dtype)
        out[f"a{i}"], out[f"bt{i}"] = qa.view(torch.uint8).numpy(), qbt.view(torch.uint8).numpy()
        out[f"sa{i}"], out[f"sb{i}"] = sa.numpy().astype(np.float32), sb.numpy().astype(np.float32)
        out[f"truth{i}"] = bits(truth)
        out[f"meta{i}"] = np.array([m, n, k, 0 if kind.startswith("int") else 1, int(out_name == "bf16"), seed])
    np.savez_compressed(HERE / "fp8_rowwise_cases.npz", **out)
    print("fp8 rowwise fixtures written to", HERE / "fp8_rowwise_cases.npz")


if __name__ == "__main__":
    main()
