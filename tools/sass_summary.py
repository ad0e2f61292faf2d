#!/usr/bin/env python
"""SASS evidence that libb200_hgemm.so is a Hopper-native kernel family: counts of wgmma (HGMMA), TMA and cluster
mnemonics, of the wgmma waits (one WARPGROUP.DEPBAR per HGMMA would mean ptxas serialised the pipeline), and of the
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
WANT = ["HGMMA", "WARPGROUP.DEPBAR", "WARPGROUP.ARRIVE", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "UCGABAR", "USETMAXREG",
        "ACQBULK", "HMMA", "LDGSTS"]


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
        ("bf16" if re.search(r"Lb1EEELi\d", f) else "fp16 in, fp32 acc" if re.search(r"ELi[12]ELb1E", f) else "fp16 in, fp16 acc")
        for f in funcs).items())))
    print()
    for w in WANT:
        match = lambda k: k == w or k.startswith(w + ".") or k.startswith(w + "_")
        exact = sum(v for k, v in ops.items() if match(k))
        variants = sorted(k for k in ops if match(k))
        note = {"HMMA": "   <- legacy mma.sync path: must be 0", "HGMMA": "   <- Hopper wgmma",
                "WARPGROUP.DEPBAR": "   <- wgmma waits: about two per kernel, not one per HGMMA",
                "LDGSTS": "   <- cp.async (not used: every bulk load is TMA)"}.get(w, "")
        print(f"{w:14s} {exact:6d}   {' '.join(variants[:8])}{note}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
