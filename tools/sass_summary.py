#!/usr/bin/env python
"""SASS evidence that libb200_hgemm.so is a Hopper-native kernel family: counts of wgmma (HGMMA for 16-bit operands,
QGMMA for e4m3), TMA and cluster mnemonics, of the wgmma waits (one WARPGROUP.DEPBAR per HGMMA would mean ptxas serialised the pipeline), of
GPU-scope memory barriers inside the consumer k-loop (one there runs every k-block of every consumer warp), and of the
legacy tensor-core paths that must be 0.

    python tools/sass_summary.py      # no GPU needed (cuobjdump reads the cubin)
"""
import collections
import re
import subprocess
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
LIB = REPO / "cuda_l2_b200" / "lib" / "libb200_hgemm.so"
WANT = ["HGMMA", "QGMMA", "WARPGROUP.DEPBAR", "WARPGROUP.ARRIVE", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "UCGABAR", "USETMAXREG",
        "ACQBULK", "HMMA", "LDGSTS"]
INSN = re.compile(r"^\s+/\*([0-9a-f]+)\*/\s+((?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)[^;]*)", re.M)


def sass_by_kernel(sass: str) -> dict[str, list[tuple[int, str, str]]]:
    """(address, mnemonic, instruction text) of every instruction of every kernel in `cuobjdump -sass` output."""
    parts = re.split(r"\n\s+Function : (\S+)\n", sass)
    return {name: [(int(m.group(1), 16), m.group(3), m.group(2)) for m in INSN.finditer(body)]
            for name, body in zip(parts[1::2], parts[2::2])}


def k_loop(insns: list[tuple[int, str, str]]) -> list[tuple[int, str, str]]:
    """The consumer k-loop: the shortest range from a backward branch's target to the branch that holds a wgmma
    (HGMMA / QGMMA). It runs once per k-block, from the full-barrier wait to the stage release; empty if there is none."""
    index = {addr: i for i, (addr, _, _) in enumerate(insns)}
    best = []
    for i, (addr, op, text) in enumerate(insns):
        m = re.search(r"\bBRA(?:\.\S+)?\s+0x([0-9a-f]+)", text) if op.startswith("BRA") else None
        if not m or int(m.group(1), 16) >= addr or int(m.group(1), 16) not in index:
            continue
        body = insns[index[int(m.group(1), 16)]:i + 1]
        if any(o.startswith(("HGMMA", "QGMMA")) for _, o, _ in body) and (not best or len(body) < len(best)):
            best = body
    return best


def k_loop_gpu_membars(insns: list[tuple[int, str, str]]) -> int:
    return sum(1 for _, op, _ in k_loop(insns) if op.startswith("MEMBAR") and op.endswith(".GPU"))


def operand_kind(func: str) -> str:
    """Operand / accumulator / output types of a kernel, from the Config<..., BF16, E4M3> arguments in its mangled name."""
    if re.search(r"Lb1EEELi\d", func):
        return "e4m3 in, fp32 acc, " + ("bf16 out" if re.search(r"Lb1ELb1EEELi\d", func) else "fp16 out")
    if re.search(r"Lb1ELb0EEELi\d", func):
        return "bf16"
    return "fp16 in, fp32 acc" if re.search(r"ELi[12]ELb1E", func) else "fp16 in, fp16 acc"


def main():
    sass = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function : (\S+)", sass)
    ops = collections.Counter()
    for m in re.finditer(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)", sass, re.M):
        ops[m.group(1)] += 1
    print(f"# cuobjdump -sass {LIB.relative_to(REPO)}   ({len(funcs)} kernels, {sum(ops.values())} instructions)")
    print("# kernels by K-mode (last template argument): " +
          ", ".join(f"{k}: {v}" for k, v in sorted(collections.Counter(re.search(r"ELi(\d)EEEv", f).group(1) for f in funcs
                                                                       if re.search(r"ELi(\d)EEEv", f)).items())) +
          "   (0 plain, 1 workspace split-K, 2 cluster split-K, 3 stream-K)")
    print("# operand types: " + ", ".join(f"{k}: {v}" for k, v in sorted(collections.Counter(
        operand_kind(f) for f in funcs).items())))
    print()
    for w in WANT:
        match = lambda k: k == w or k.startswith(w + ".") or k.startswith(w + "_")
        exact = sum(v for k, v in ops.items() if match(k))
        variants = sorted(k for k in ops if match(k))
        note = {"HMMA": "   <- legacy mma.sync path: must be 0", "HGMMA": "   <- Hopper wgmma", "QGMMA": "   <- Hopper wgmma, e4m3",
                "WARPGROUP.DEPBAR": "   <- wgmma waits: about two per kernel, not one per HGMMA",
                "LDGSTS": "   <- cp.async (not used: every bulk load is TMA)"}.get(w, "")
        print(f"{w:14s} {exact:6d}   {' '.join(variants[:8])}{note}")
        if w == "WARPGROUP.DEPBAR":
            per_kernel = collections.Counter(k_loop_gpu_membars(insns) for insns in sass_by_kernel(sass).values())
            print(f"{'MEMBAR.*.GPU':14s} {sum(n * c for n, c in per_kernel.items()):6d}   in the consumer k-loop, per kernel: " +
                  ", ".join(f"{n} in {c} kernels" for n, c in sorted(per_kernel.items())) + "   <- must be 0")
    return 0


if __name__ == "__main__":
    sys.exit(main())
