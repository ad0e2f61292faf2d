#!/usr/bin/env python
"""Generate tests/golden/fp8_block_cases.npz — the FP8 (e4m3) fixtures with block scales. Needs torch only.

The truth is torch's CPU expression, never this repository's code: for every 128-wide k-block kb,
``p = qa[:, blk].float() @ qbt[:, blk].float().t()`` and ``s = sa[:, kb:kb+1] * sb_cols[kb]`` (sb_cols: Bt's block scales
repeated over each block's 128 columns), ``acc = p * s`` for the first block and ``acc = acc + p * s`` after it, then
``acc.to(out_dtype)``. Stored: float8_e4m3fn operands as uint8 codes (a [M,K], bt [N,K]), the fp32 scales sa [M, nkb]
and sb [ceil(N/128), nkb], the truth as uint16 bits (fp16 or bf16 output) and
meta = [m, n, k, kind (0 small integers, 1 randn), out_bf16, seed].

* small-integer cases: operands in [-lim, lim] and power-of-two scales, so every product, sum and scaling is exact in
  fp32 and the bits are pinned whatever the order (fused or not); ragged in M (M % 4 != 0), N (N % 128 != 0) and K
  (K % 128 != 0);
* N(0,1) cases quantised per 1 x 128 (a) and 128 x 128 (bt) block, amax / 448 — tolerance tests (torch's fp32 matmul
  sums in its own order and does not fuse the promotion).

    python tests/golden/make_fp8_block_golden.py
"""
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent

BLOCK_CASES = [
    # (m, n, k, kind, out, seed)   kind "int<lim>" or "randn"
    (64, 256, 256, "int2", "fp16", 81),
    (201, 328, 400, "int2", "fp16", 82),          # ragged M, N and K (400 = three k-blocks of 128 + 16)
    (67, 136, 272, "int1", "bf16", 83),
    (1, 8, 16, "int2", "fp16", 84),
    (130, 264, 1040, "int1", "bf16", 85),
    (3, 128, 128, "int2", "bf16", 86),
    (64, 128, 512, "randn", "fp16", 91), (201, 328, 400, "randn", "bf16", 92),
]


def bits(t):
    return t.contiguous().view(torch.int16).numpy().view(np.uint16)


def truth_of(qa, qbt, sa, sb, out_dtype):
    m, k = qa.shape
    n = qbt.shape[0]
    nkb = -(-k // 128)
    sb_cols = sb.repeat_interleave(128, dim=0)[:n]          # [N, nkb]
    acc = None
    for kb in range(nkb):
        blk = slice(kb * 128, min(k, (kb + 1) * 128))
        p = qa[:, blk].float() @ qbt[:, blk].float().t()
        s = sa[:, kb:kb + 1] * sb_cols[:, kb][None, :]
        acc = p * s if acc is None else acc + p * s
    return acc.to(out_dtype)


def main():
    out = {}
    for i, (m, n, k, kind, out_name, seed) in enumerate(BLOCK_CASES):
        gen = torch.Generator().manual_seed(seed)
        out_dtype = {"fp16": torch.float16, "bf16": torch.bfloat16}[out_name]
        nkb, nnb = -(-k // 128), -(-n // 128)
        if kind.startswith("int"):
            lim = int(kind[3:])
            a = (torch.randint(0, 2 * lim + 1, (m, k), generator=gen) - lim).float()
            bt = (torch.randint(0, 2 * lim + 1, (n, k), generator=gen) - lim).float()
            sa = torch.pow(2.0, torch.randint(-2, 3, (m, nkb), generator=gen).float())
            sb = torch.pow(2.0, torch.randint(-2, 3, (nnb, nkb), generator=gen).float())
        else:
            a, bt = torch.randn((m, k), generator=gen), torch.randn((n, k), generator=gen)
            ap = torch.nn.functional.pad(a, (0, nkb * 128 - k)).view(m, nkb, 128)
            sa = ap.abs().amax(dim=2) / 448
            a = (ap / sa[:, :, None]).view(m, -1)[:, :k]
            bp = torch.nn.functional.pad(bt, (0, nkb * 128 - k, 0, nnb * 128 - n)).view(nnb, 128, nkb, 128)
            sb = bp.abs().amax(dim=(1, 3)) / 448
            bt = (bp / sb[:, None, :, None]).reshape(nnb * 128, nkb * 128)[:n, :k]
        qa, qbt = a.to(torch.float8_e4m3fn), bt.to(torch.float8_e4m3fn)
        truth = truth_of(qa, qbt, sa, sb, out_dtype)
        out[f"a{i}"], out[f"bt{i}"] = qa.view(torch.uint8).numpy(), qbt.view(torch.uint8).numpy()
        out[f"sa{i}"], out[f"sb{i}"] = sa.numpy().astype(np.float32), sb.numpy().astype(np.float32)
        out[f"truth{i}"] = bits(truth)
        out[f"meta{i}"] = np.array([m, n, k, 0 if kind.startswith("int") else 1, int(out_name == "bf16"), seed])
    np.savez_compressed(HERE / "fp8_block_cases.npz", **out)
    print("fp8 block fixtures written to", HERE / "fp8_block_cases.npz")


if __name__ == "__main__":
    main()
