#!/usr/bin/env python
"""Time the FP8 (e4m3) GEMM on an H100 against torch._scaled_mm and this library's fp16 path, in one run.

    python tools/bench_fp8.py [--steps K] [--warmup W] [--mnk M_N_K]

Shapes: --mnk (default 4096_4096_4096), 4096^3 and 2048x11008x4096. Per shape, six legs with the same rules:
b200_fp8gemm (e4m3 operands quantised per tensor from N(0,1) data, fp16 out, the dispatcher's choice),
torch._scaled_mm with fast accumulation on and off (same operands and scales), b200_hgemm_f32acc on the fp16 data, and
two bf16-out legs on the same data quantised per row (scales [M,1] and [1,N]): b200_fp8gemm_rowwise and
torch._scaled_mm with rowwise scales and fast accumulation, and two bf16-out legs on the same data quantised per block
(1 x 128 for a, 128 x 128 for bt): b200_fp8gemm_blockwise (libb200_fp8block.so) and torch._scaled_mm with blockwise
scales, the latter reported as {"skipped": reason} where torch refuses it.
Each leg: warm-up, then K back-to-back calls between two CUDA events on the legacy default stream, rotating over seeded
operand sets whose fp16 footprint exceeds the 50 MB L2 four times. TFLOP/s = 2MNK per call. Prints one JSON line with
the card's name and enforced power limit (figures are only comparable at the same limit). Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))

import torch  # noqa: E402

L2_BYTES = 50 * 1024 * 1024


def card_info() -> dict:
    """Name and enforced power limit of the device (read-only NVML queries)."""
    info = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        import pynvml as nv
        nv.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        idx = int(vis.split(",")[torch.cuda.current_device()]) if vis else torch.cuda.current_device()
        info["power_limit_w"] = nv.nvmlDeviceGetEnforcedPowerLimit(nv.nvmlDeviceGetHandleByIndex(idx)) / 1000.0
    except Exception:
        pass
    return info


def time_shape(m: int, n: int, k: int, steps: int, warmup: int, gen: torch.Generator) -> dict:
    from cuda_l2_b200 import capi, ops

    set_bytes = 2 * (m * k + n * k + m * n)
    nsets = max(2, min(16, -(-4 * L2_BYTES // set_bytes)))
    sets = []
    for _ in range(nsets):
        a = torch.randn((m, k), device="cuda", generator=gen).half()
        bt = torch.randn((n, k), device="cuda", generator=gen).half()
        qa, sa = ops.quantize_e4m3(a)
        qb, sb = ops.quantize_e4m3(bt)
        qa_r, sa_r = ops.quantize_e4m3_rowwise(a)
        qb_r, sb_r = ops.quantize_e4m3_rowwise(bt)
        qa_b, sa_b = ops.quantize_e4m3_blockwise(a)
        qb_b, sb_b = ops.quantize_e4m3_block128x128(bt)
        sets.append(dict(a=a, bt=bt, qa=qa, qb=qb, sa=sa, sb=sb, c=torch.empty((m, n), dtype=torch.half, device="cuda"),
                         qa_r=qa_r, qb_r=qb_r, sa_r=sa_r, sb_r=sb_r.reshape(1, n),
                         c_bf16=torch.empty((m, n), dtype=torch.bfloat16, device="cuda"),
                         qa_b=qa_b, qb_b=qb_b, sa_b=sa_b, sb_b=sb_b))

    def ours_fp8(st):
        capi.fp8_gemm(st["qa"], st["qb"], st["c"], st["sa"], st["sb"])

    def ours_fp16(st):
        capi.gemm_kmajor(st["a"], st["bt"], st["c"], "fp32")

    def scaled(fast):
        return lambda st: torch._scaled_mm(st["qa"], st["qb"].t(), scale_a=st["sa"].reshape(()),
                                           scale_b=st["sb"].reshape(()), out_dtype=torch.half, use_fast_accum=fast)

    def ours_rowwise(st):
        capi.fp8_gemm(st["qa_r"], st["qb_r"], st["c_bf16"], st["sa_r"], st["sb_r"])

    def scaled_rowwise(st):
        return torch._scaled_mm(st["qa_r"], st["qb_r"].t(), scale_a=st["sa_r"], scale_b=st["sb_r"],
                                out_dtype=torch.bfloat16, use_fast_accum=True)

    def ours_blockwise(st):
        capi.fp8_gemm(st["qa_b"], st["qb_b"], st["c_bf16"], st["sa_b"], st["sb_b"])

    def scaled_blockwise(st):
        return torch._scaled_mm(st["qa_b"], st["qb_b"].t(), scale_a=st["sa_b"], scale_b=st["sb_b"].t(),
                                out_dtype=torch.bfloat16)

    legs = {"ours_e4m3": ours_fp8, "scaled_mm_fast_accum": scaled(True), "scaled_mm_no_fast_accum": scaled(False),
            "ours_fp16_fp32acc": ours_fp16, "ours_e4m3_rowwise_bf16": ours_rowwise,
            "scaled_mm_rowwise_fast_accum_bf16": scaled_rowwise, "ours_e4m3_blockwise_bf16": ours_blockwise,
            "scaled_mm_blockwise_bf16": scaled_blockwise}
    row = {}
    for name, fn in legs.items():
        if name == "scaled_mm_blockwise_bf16":
            try:
                fn(sets[0])
                torch.cuda.synchronize()
            except (RuntimeError, NotImplementedError, ValueError) as e:
                row[name] = {"skipped": str(e).splitlines()[0]}
                continue
        for i in range(max(warmup, 3)):
            fn(sets[i % nsets])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            fn(sets[i % nsets])
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        row[name] = {"tflops": 2.0 * m * n * k / (ms * 1e-3) * 1e-12, "ms_per_call": ms}
    cfg_id, group_m, splits = capi.fp8_select(m, n, k)
    row["ours_e4m3"]["dispatch"] = {"config": cfg_id, "group_m": group_m, "splits": splits}
    cfg_id, group_m, splits = capi.fp8_blockwise_select(m, n, k)
    row["ours_e4m3_blockwise_bf16"]["dispatch"] = {"config": cfg_id, "group_m": group_m, "splits": splits}
    return row


def main() -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--mnk", type=str, default="4096_4096_4096")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_fp8.py needs an H100: the FP8 path has no CPU fallback")
    torch.cuda.set_device(0)
    shapes = []
    for s in (args.mnk, "4096_4096_4096", "2048_11008_4096"):
        mnk = tuple(int(x) for x in s.split("_"))
        if mnk not in shapes:
            shapes.append(mnk)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    results = {}
    for (m, n, k) in shapes:
        results[f"{m}_{n}_{k}"] = time_shape(m, n, k, args.steps, args.warmup, gen)
        torch.cuda.empty_cache()
    head = results["_".join(map(str, shapes[0]))]["ours_e4m3"]
    print(json.dumps({
        "metric": "FP8 GEMM TFLOP/s (2MNK per call), offline mode, per (M,N,K)", "value": head["tflops"], "unit": "TFLOP/s",
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": head["ms_per_call"],
        "dtype": "e4m3 x e4m3 -> f32 accumulate -> f16, per-tensor scales",
        "data": "synthetic N(0,1), quantised per tensor (amax / 448)", "card": card_info(), "shapes": results,
    }))
    return 0


if __name__ == "__main__":
    sys.exit(main())
