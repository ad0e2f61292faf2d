#!/usr/bin/env python
"""Generate tests/golden/fp8_cases.npz — the FP8 (e4m3) fixtures. Needs torch only.

The FP8 variant is this repository's extension (the reference has no fp8 path), so there is no reference code to run;
the truth is torch's expression ``((a.float() @ bt.float().t()) * (sa * sb)).to(out_dtype)`` on the CPU, never this
repository's oracle. Stored: float8_e4m3fn operands as uint8 codes (a [M,K], bt [N,K]), the two fp32 per-tensor scales,
the truth as uint16 bits (fp16 or bf16 output) and meta = [m, n, k, kind (0 small integers, 1 randn), out_bf16, seed].

* small-integer cases: operands in [-lim, lim] with lim * lim * k inside the exact range (2047 for fp16 out, 256 for
  bf16 out), power-of-two scales and one non-power-of-two pair per output type — exact;
* N(0,1) cases quantised per tensor with amax / 448 scales — tolerance tests (torch's fp32 matmul sums in its own order).

    python tests/golden/make_fp8_golden.py
"""
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent

FP8_CASES = [
    # (m, n, k, kind, out, scale_a, scale_b, seed)   kind "int<lim>" or "randn" (scales then come from amax / 448)
    (64, 256, 64, "int2", "fp16", 0.5, 4.0, 41),
    (200, 328, 144, "int2", "fp16", 0.125, 2.0, 42),       # ragged M, N and K (144 = one k-block of 128 + 16)
    (128, 64, 512, "int1", "fp16", 1.0, 1.0, 43),
    (384, 264, 208, "int2", "fp16", 0.3, 1.7, 44),         # the non-power-of-two pair
    (1, 8, 16, "int2", "fp16", 2.0, 0.25, 45),
    (64, 256, 64, "int2", "bf16", 0.5, 4.0, 46),
    (200, 328, 144, "int1", "bf16", 0.25, 1.0, 47),
    (128, 136, 192, "int1", "bf16", 0.3, 1.7, 48),
    (64, 128, 64, "randn", "fp16", 0, 0, 51), (200, 328, 144, "randn", "bf16", 0, 0, 52),
    (128, 128, 1024, "randn", "fp16", 0, 0, 53),
]


def bits(t):
    return t.contiguous().view(torch.int16).numpy().view(np.uint16)


def main():
    out = {}
    for i, (m, n, k, kind, out_name, sa, sb, seed) in enumerate(FP8_CASES):
        gen = torch.Generator().manual_seed(seed)
        out_dtype = {"fp16": torch.float16, "bf16": torch.bfloat16}[out_name]
        if kind.startswith("int"):
            lim = int(kind[3:])
            a = (torch.randint(0, 2 * lim + 1, (m, k), generator=gen) - lim).float()
            bt = (torch.randint(0, 2 * lim + 1, (n, k), generator=gen) - lim).float()
            assert lim * lim * k <= (2047 if out_name == "fp16" else 256)
            sa_t, sb_t = torch.tensor(sa, dtype=torch.float32), torch.tensor(sb, dtype=torch.float32)
        else:
            a, bt = torch.randn((m, k), generator=gen), torch.randn((n, k), generator=gen)
            sa_t, sb_t = a.abs().amax() / 448, bt.abs().amax() / 448
            a, bt = a / sa_t, bt / sb_t
        qa, qbt = a.to(torch.float8_e4m3fn), bt.to(torch.float8_e4m3fn)
        truth = ((qa.float() @ qbt.float().t()) * (sa_t * sb_t)).to(out_dtype)
        out[f"a{i}"], out[f"bt{i}"] = qa.view(torch.uint8).numpy(), qbt.view(torch.uint8).numpy()
        out[f"scales{i}"] = np.array([sa_t.item(), sb_t.item()], dtype=np.float32)
        out[f"truth{i}"] = bits(truth)
        out[f"meta{i}"] = np.array([m, n, k, 0 if kind.startswith("int") else 1, int(out_name == "bf16"), seed])
    np.savez_compressed(HERE / "fp8_cases.npz", **out)
    print("fp8 fixtures written to", HERE / "fp8_cases.npz")


if __name__ == "__main__":
    main()
