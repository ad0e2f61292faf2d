#!/usr/bin/env python
"""README-style summary of eval_results/: the mean speed-up table and the bar chart the reference publishes
(README.md:18-23, assets/speedup_summary_all.png) for the b200 CSVs.

    python tools/make_results_summary.py            # writes eval_results/SUMMARY.md and assets/speedup_summary_b200.svg

For every eval_results/cuda_l2_b200_<ACC>_speedup_<mode>*.csv: the mean over shapes of the speed-up in each of the
reference's four headline columns (torch.matmul, cuBLAS-max, cuBLASLt-heuristic-max, cuBLASLt-auto-tuning-max), the
number of shapes and the fraction at or above 1.0 against cuBLASLt-auto-tuning-max. The chart is plain SVG (no
plotting library in this image).
"""
import csv
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
COLS = ["torch.matmul", "cuBLAS-max", "cuBLASLt-heuristic-max", "cuBLASLt-auto-tuning-max"]
COLORS = ["#8da0cb", "#66c2a5", "#fc8d62", "#e78ac3"]


def load(path: Path):
    rows = list(csv.DictReader(open(path)))
    out = {"file": path.name, "shapes": len(rows)}
    for c in COLS:
        v = [float(r[c]) for r in rows if r.get(c) not in (None, "")]
        out[c] = (sum(v) / len(v), len(v)) if v else (None, 0)
    v = [float(r[COLS[3]]) for r in rows if r.get(COLS[3]) not in (None, "")]
    out["won"] = sum(x >= 1.0 for x in v)
    out["n_auto"] = len(v)
    return out


def label(name: str) -> str:
    stem = name[len("cuda_l2_b200_"):-len(".csv")]
    acc, rest = stem.split("_speedup_", 1)
    return f"H100 {acc} {rest.replace('_', ' ')}"


def svg(groups, path: Path):
    bar_w, gap, group_gap, h, top, left = 26, 4, 46, 260, 40, 60
    vmax = max([1.2] + [g[c][0] for g in groups for c in COLS if g[c][0]]) * 1.1
    width = left + len(groups) * (len(COLS) * (bar_w + gap) + group_gap) + 20
    y = lambda v: top + h - h * v / vmax
    parts = [f'<svg xmlns="http://www.w3.org/2000/svg" width="{width}" height="{top + h + 90}" font-family="sans-serif" font-size="11">',
             f'<rect width="100%" height="100%" fill="white"/>',
             f'<text x="{left}" y="20" font-size="14" font-weight="bold">Mean speed-up of the H100 kernels over each baseline (all shapes of the file)</text>']
    t = 0.0
    while t <= vmax:
        parts.append(f'<line x1="{left}" x2="{width - 10}" y1="{y(t):.1f}" y2="{y(t):.1f}" stroke="{"#444" if abs(t - 1.0) < 1e-9 else "#ddd"}"/>')
        parts.append(f'<text x="{left - 6}" y="{y(t) + 4:.1f}" text-anchor="end">{t:.1f}x</text>')
        t += 0.2
    x = left + 10
    for g in groups:
        x0 = x
        for c, col in zip(COLS, COLORS):
            mean = g[c][0]
            if mean:
                parts.append(f'<rect x="{x}" y="{y(mean):.1f}" width="{bar_w}" height="{top + h - y(mean):.1f}" fill="{col}"/>')
                parts.append(f'<text x="{x + bar_w / 2}" y="{y(mean) - 3:.1f}" text-anchor="middle" font-size="10">{mean:.2f}</text>')
            x += bar_w + gap
        parts.append(f'<text x="{(x0 + x) / 2}" y="{top + h + 16}" text-anchor="middle">{label(g["file"])}</text>')
        parts.append(f'<text x="{(x0 + x) / 2}" y="{top + h + 30}" text-anchor="middle" fill="#555">{g["shapes"]} shapes</text>')
        x += group_gap
    lx = left
    for c, col in zip(COLS, COLORS):
        parts.append(f'<rect x="{lx}" y="{top + h + 50}" width="12" height="12" fill="{col}"/><text x="{lx + 16}" y="{top + h + 60}">{c}</text>')
        lx += 170
    parts.append("</svg>")
    path.write_text("\n".join(parts))


def main():
    files = sorted((REPO / "eval_results").glob("cuda_l2_b200_*_speedup_*.csv"))
    files = [f for f in files if not f.name.endswith("_absolute.csv")]
    groups = [load(f) for f in files]
    lines = ["# H100 results in the reference's format", "",
             "Mean speed-up over each baseline (the reference's README figure), per results file; `won` = shapes at or above",
             "1.0 against cuBLASLt-auto-tuning-max (the harder of its two layouts). Files tagged `harness_sample` / `server` come",
             "from the real `eval_one_file.sh` flow or the harness's Python loop on a stratified sample (see DESIGN.md §6).", "",
             "| results file | shapes | " + " | ".join(COLS) + " | won vs auto-tuning-max |", "|---|---|" + "---|" * (len(COLS) + 1)]
    for g in groups:
        cells = [f"{g[c][0]:.3f}" + (f" ({g[c][1]})" if g[c][1] != g["shapes"] else "") if g[c][0] else "-" for c in COLS]
        lines.append(f"| `{g['file']}` | {g['shapes']} | " + " | ".join(cells) + f" | {g['won']} / {g['n_auto']} = {100.0 * g['won'] / max(g['n_auto'], 1):.1f} % |")
    lines += ["", "![speed-up summary](speedup_summary.svg)", ""]
    (REPO / "eval_results" / "SUMMARY.md").write_text("\n".join(lines))
    svg(groups, REPO / "eval_results" / "speedup_summary.svg")   # next to the tables it summarises (git-ignored)
    print("\n".join(lines))
    return 0


if __name__ == "__main__":
    sys.exit(main())
