#!/usr/bin/env python
"""Time the grouped SwiGLU GEMM (libb200_grouped_swiglu.so) against the compositions it replaces, on an H100.

    python tools/bench_grouped_swiglu.py [--rounds R] [--ms MS]

Shapes, bf16 with fp32 accumulation, the gate / up projection of MoE experts: Mixtral (G = 8, H = 4096, I = 14336) at
T = 4096 and 16384 tokens, and a fine-grained MoE (G = 64, H = 2048, I = 1408) at T = 16384. The group sizes are
seeded and uneven: T - 5 - 3G tokens split by Dirichlet(2) weights, then two experts lose all of theirs, so the last
group ends before T.

Forward legs:
* ``fused``: the dispatched grouped SwiGLU call, y only;
* ``hgemm_grouped_torch``: libb200_grouped.so's grouped call for h, then ``F.silu(g) * u`` in torch;
* ``torch_grouped_mm_torch``: ``torch._grouped_mm`` for h, then the same.
Training legs (forward + backward under autograd, dX and dW): ``grouped_swiglu_linear`` against ``grouped_linear`` +
``F.silu(g) * u``. The backward kernel alone is reported in GB/s: dy and h read, dh written, valid rows only.

Each leg rotates over seeded operand sets whose footprint exceeds the 50 MB L2 (at least two), the legs alternate
within each of R rounds, each timing covers about MS milliseconds of back-to-back calls between CUDA events, and the
median and range are reported. TFLOP/s count valid rows only, 2 * T_valid * 2I * H per forward call. Prints one JSON
line with the card's name, power limit and maximum SM clock, read in the same run. Writes nothing.
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

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench_nn import card  # noqa: E402

L2_BYTES = 50 * 1024 * 1024
SHAPES = [(8, 4096, 4096, 14336), (8, 16384, 4096, 14336), (64, 16384, 2048, 1408)]   # (G, T, H, I)


def group_sizes(g: int, t: int, seed: int) -> list[int]:
    """Seeded, uneven sizes summing to less than T, two of them empty."""
    rng = np.random.default_rng(seed)
    sizes = rng.multinomial(t - 5 - 3 * g, rng.dirichlet(np.full(g, 2.0)))
    sizes[rng.choice(g, size=2, replace=False)] = 0
    return [int(s) for s in sizes]


def time_ms(fn, sets, iters: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for j in range(iters):
        fn(sets[j % len(sets)])
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def alternate(legs: dict, sets: list, rounds: int, ms: float) -> dict:
    """Median, min and max ms per call of every leg, the legs alternating within each round."""
    iters = {}
    for name, fn in legs.items():   # warm-up, and the call count of a timing
        for j in range(3):
            fn(sets[j % len(sets)])
        torch.cuda.synchronize()
        iters[name] = max(len(sets), int(ms / max(time_ms(fn, sets, len(sets)), 1e-3)))
    samples = {name: [] for name in legs}
    for _ in range(rounds):
        for name, fn in legs.items():
            samples[name].append(time_ms(fn, sets, iters[name]))
    return {name: {"ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for name, v in samples.items()}


def case(g: int, t: int, hid: int, i: int, rounds: int, ms: float, seed: int) -> dict:
    from cuda_l2_b200 import capi, ops

    dtype = torch.bfloat16
    sizes = group_sizes(g, t, seed)
    ends = [int(v) for v in np.cumsum(sizes)]
    t_valid = ends[-1]
    offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(seed)
    set_bytes = 2 * (t * hid + g * 2 * i * hid + 3 * t * 2 * i)
    nsets = max(2, min(8, -(-2 * L2_BYTES // set_bytes)))
    sets = []
    for _ in range(nsets):
        x = (torch.randn((t, hid), device="cuda", generator=gen) * 0.5).to(dtype)
        w = (torch.randn((g, 2 * i, hid), device="cuda", generator=gen) * hid ** -0.5).to(dtype)
        sets.append(dict(x=x, w=w, y=torch.empty((t, i), dtype=dtype, device="cuda"),
                         h=torch.empty((t, 2 * i), dtype=dtype, device="cuda"),
                         dy=torch.randn((t, i), device="cuda", generator=gen).to(dtype),
                         dh=torch.empty((t, 2 * i), dtype=dtype, device="cuda")))
    stream = lambda: torch.cuda.current_stream().cuda_stream   # noqa: E731

    def silu_mul(h):
        gg, uu = h.view(t, i // 64, 2, 64).unbind(2)
        return F.silu(gg.reshape(t, i)) * uu.reshape(t, i)

    def hgemm_grouped_torch(s):
        capi.gemm_grouped(s["x"], s["w"], s["h"], offs, stream=stream())
        return silu_mul(s["h"])

    forward = {
        "fused": lambda s: capi.grouped_swiglu(s["x"], s["w"], offs, s["y"], stream=stream()),
        "hgemm_grouped_torch": hgemm_grouped_torch,
        "torch_grouped_mm_torch": lambda s: silu_mul(torch._grouped_mm(s["x"], s["w"].transpose(-2, -1), offs=offs)),
    }

    def train_fused(s):
        x, w = s["x"].detach().requires_grad_(), s["w"].detach().requires_grad_()
        ops.grouped_swiglu_linear(x, w, offs).backward(s["dy"])

    def train_composed(s):
        x, w = s["x"].detach().requires_grad_(), s["w"].detach().requires_grad_()
        silu_mul(ops.grouped_linear(x, w, offs)).backward(s["dy"])

    training = {"fused": train_fused, "grouped_linear_torch": train_composed}
    backward = {"dh": lambda s: capi.grouped_swiglu_backward(s["dy"], s["h"], s["dh"], offs, stream=stream())}
    flops = 2.0 * t_valid * 2 * i * hid
    row = {"group_sizes": sizes, "t_valid": t_valid, "operand_sets": nsets,
           "dispatch": dict(zip(("config", "group_m"), capi.grouped_swiglu_select(2, g, t, i, hid)))}
    fw = alternate(forward, sets, rounds, ms)
    tr = alternate(training, sets, rounds, ms)
    bw = alternate(backward, sets, rounds, ms)
    for legs in (fw, tr):
        for v in legs.values():
            v["tflops"] = flops / (v["ms"] * 1e-3) * 1e-12 if legs is fw else 3 * flops / (v["ms"] * 1e-3) * 1e-12
    row["forward"] = fw
    row["training"] = tr
    moved = 2.0 * t_valid * (i + 2 * i + 2 * i)   # bytes of dy and h read and dh written
    row["backward_dh"] = {**bw["dh"], "gb_per_s": moved / (bw["dh"]["ms"] * 1e-3) * 1e-9}
    row["forward_speedup_vs_hgemm_grouped_torch"] = fw["hgemm_grouped_torch"]["ms"] / fw["fused"]["ms"]
    row["forward_speedup_vs_torch_grouped_mm_torch"] = fw["torch_grouped_mm_torch"]["ms"] / fw["fused"]["ms"]
    row["training_speedup"] = tr["grouped_linear_torch"]["ms"] / tr["fused"]["ms"]
    return row


def main() -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=7)
    p.add_argument("--ms", type=float, default=100.0)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_grouped_swiglu.py needs an H100: the grouped SwiGLU GEMM has no CPU fallback")
    torch.cuda.set_device(0)
    result = {"metric": "grouped SwiGLU gate / up projection, bf16, median ms per call", "rounds": args.rounds,
              "card": card(), "cases": {}}
    for n, (g, t, hid, i) in enumerate(SHAPES):
        result["cases"][f"G{g}_T{t}_H{hid}_I{i}"] = case(g, t, hid, i, args.rounds, args.ms, seed=20261018 + n)
        torch.cuda.empty_cache()
    print(json.dumps(result))
    return 0


if __name__ == "__main__":
    sys.exit(main())
