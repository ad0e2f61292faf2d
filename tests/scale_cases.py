"""Production-scale GEMM cases, where a 32-bit element or byte index would wrap — TEST INFRASTRUCTURE (imports and
runs without a GPU; test_gpu_scale.py runs the cases, test_scale_cpu.py checks this file).

* CASES: for each case, the tensors the GPU test allocates, the one whose size crosses 2^31 (or 2^32) elements or
  bytes, the row, batch, group or expert where that crossing falls, and the device memory the case needs.
* routing_histogram: seeded, Zipf-like group sizes for G = 256 experts with the edges the grouped kernels have to get
  right (empty groups, 1-row groups, one very long group, group starts at every residue mod 128, and a short group
  holding a crossing row with an empty group on each side).
* fill_ints_: exact-domain operands generated on the device, in place (16-bit) or band by band (e4m3), never through a
  full-size int64 or fp32 intermediate. The bounds are exact_domain.py's.
* matmul64 / first_mismatch: the float64 reference in row bands (and reduction chunks) of at most BAND_BYTES, rounded
  once per band to the output type and compared bit for bit with the kernel's band; the whole output is compared.
* guarded: an output inside a buffer with GUARD_BYTES of NaN sentinel on each side, so an element never written and a
  write past either end are both caught.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

import exact_domain as ed

NUM_EXPERTS = 256
BIG_GROUP = 65536
GUARD_BYTES = 1 << 20
BAND_BYTES = 1 << 29          # one float64 working band of the reference (512 MiB)
REF_SLACK = 1 << 26           # cuBLAS workspace and small tensors of the reference
SENTINEL = {torch.float16: 0x7D5A, torch.bfloat16: 0x7FA5,    # NaN payloads no kernel produces
            torch.float8_e4m3fn: 0xFF}                     # -NaN: the quantisers write NaN as 0x7F
_BITS = {1: torch.uint8, 2: torch.int16}
DTYPES = {"16": None, "fp16": torch.float16, "bf16": torch.bfloat16, "e4m3": torch.float8_e4m3fn,
          "fp32": torch.float32, "int32": torch.int32}
ITEMSIZE = {"16": 2, "fp16": 2, "bf16": 2, "e4m3": 1, "fp32": 4, "int32": 4}

# 2-D problems of cases 1 to 5 (M, N, K)
TN = (24600, 131080, 256)
TALL = (196616, 264, 16384)
NN_LONG = (136, 12296, 262216)
T_GROUPED, N_GROUPED, K_GROUPED = 262216, 12296, 64
WGRAD = dict(g=NUM_EXPERTS, m=2048, n=9216, t=24576)
FP8_EXPERTS = dict(g=NUM_EXPERTS, n=2560, k=7168, t=8192, slots=64)
# The weight gradient of blockwise FP8 training (1 x 128 scales on both operands) over FP8_DW_TOKENS tokens: K is the
# token count padded to 16 (capi.dual_ld_t), and A [M, K] passes 2^31 bytes along K.
FP8_DW_TOKENS = 4500007
FP8_DW = (640, 1152, -(-FP8_DW_TOKENS // 16) * 16)
# One bf16 activation past 2^31 elements for every quantiser that takes it: rows % 16 != 0 (q_t's padded columns),
# cols % 128 != 0 and cols / 2 % 128 != 0 (the last 1 x 128 group of x and of the SwiGLU output is partial).
QUANT = (349203, 8200)

# Long-reduction groups of the K-grouped case: one of 140 001 rows, one holding row 174 648 (dY's crossing) in its
# middle, a 1-row, an empty one and a short last group.
WGRAD_LONG_SIZES = (3, 0, 140001, 29996, 10017, 0, 1, 82198)


@dataclass(frozen=True)
class Tensor:
    name: str
    shape: tuple
    dtype: str        # a key of DTYPES; "16" is the run's fp16 / bf16 type

    @property
    def numel(self) -> int:
        return math.prod(self.shape)

    @property
    def nbytes(self) -> int:
        return self.numel * ITEMSIZE[self.dtype]


@dataclass(frozen=True)
class Case:
    name: str
    path: str
    tensors: tuple            # Tensor, in allocation order
    outputs: tuple            # names of the outputs, each inside a guarded buffer
    crosses: str              # the tensor whose size crosses the boundaries
    unit: str                 # "elements" or "bytes"
    crossings: tuple          # ((boundary, index along the tensor's first dimension where it falls), ...)

    def tensor(self, name: str) -> Tensor:
        return next(t for t in self.tensors if t.name == name)

    def crossing_index(self, boundary: int) -> int:
        """The index along the crossing tensor's first dimension that holds element (or byte) ``boundary``."""
        t = self.tensor(self.crosses)
        step = math.prod(t.shape[1:]) * (ITEMSIZE[t.dtype] if self.unit == "bytes" else 1)
        return boundary // step

    def size(self) -> int:
        t = self.tensor(self.crosses)
        return t.nbytes if self.unit == "bytes" else t.numel

    def tensor_bytes(self) -> int:
        """What allocate() takes: every tensor, the outputs with their two guard bands."""
        return sum(t.nbytes for t in self.tensors) + 2 * GUARD_BYTES * len(self.outputs)

    def memory_bytes(self) -> int:
        """Device memory the case needs at its peak: its tensors, and the reference's working set (a float64 row band,
        the float64 chunks of both operands, the band's float32 and 16-bit roundings and the comparison)."""
        return self.tensor_bytes() + 4 * BAND_BYTES + REF_SLACK


def _t(name, shape, dtype="16"):
    return Tensor(name, tuple(shape), dtype)


def _cases() -> dict:
    m, n, k = TN
    nkb = -(-k // 128)
    tall_m, tall_n, tall_k = TALL
    lm, ln, lk = NN_LONG
    t, gn, gk = T_GROUPED, N_GROUPED, K_GROUPED
    w, e = WGRAD, FP8_EXPERTS
    enkb, enb = e["k"] // 128, -(-e["n"] // 128)
    dm, dn, dk = FP8_DW
    dnkb = -(-dk // 128)
    qr, qc = QUANT
    qld_t = -(-qr // 16) * 16
    i31, i32 = 2 ** 31, 2 ** 32
    out = [
        Case("tn", "2-D TN: dispatcher (fp16 with fp32 and fp16 accumulation, bf16), pinned CTA pair, cluster and "
             "stream-K", (_t("a", (m, k)), _t("bt", (n, k)), _t("c", (m, n))), ("c",), "c", "elements",
             ((i31, 16383),)),
        Case("nn", "2-D NN (row-major B), fp16 and bf16", (_t("a", (m, k)), _t("b", (k, n)), _t("c", (m, n))), ("c",),
             "c", "elements", ((i31, 16383),)),
        Case("block", "block-scaled e4m3 2-D, bf16 out",
             (_t("a", (m, k), "e4m3"), _t("bt", (n, k), "e4m3"), _t("sa", (nkb, -(-m // 4) * 4), "fp32"),
              _t("sb", (-(-n // 128), nkb), "fp32"), _t("c", (m, n), "bf16")), ("c",), "c", "elements",
             ((i31, 16383),)),
        Case("tall", "2-D TN, fp16, A past 2^31 elements",
             (_t("a", (tall_m, tall_k)), _t("bt", (tall_n, tall_k)), _t("c", (tall_m, tall_n))), ("c",), "a",
             "elements", ((i31, 131072),)),
        Case("nn_long", "NN long reduction, fp16 and bf16: dispatcher, pinned cluster split-K and stream-K",
             (_t("a", (lm, lk)), _t("b", (lk, ln)), _t("c", (lm, ln))), ("c",), "b", "elements", ((i31, 174648),)),
        Case("batched", "batched, dense (fp16) and masked (bf16)",
             (_t("a", (64, 4104, 64)), _t("bt", (64, 12296, 64)), _t("masked_m", (64,), "int32"),
              _t("c", (64, 4104, 12296))), ("c",), "c", "elements", ((i31, 42),)),
        Case("grouped", "grouped forward, fp16, 256-expert routing histogram",
             (_t("a", (t, gk)), _t("bt", (NUM_EXPERTS, gn, gk)), _t("offs", (NUM_EXPERTS,), "int32"),
              _t("c", (t, gn))), ("c",), "c", "elements", ((i31, 174648),)),
        Case("grouped_nn", "grouped row-major B (dX), bf16, the same histogram",
             (_t("a", (t, gk)), _t("b", (NUM_EXPERTS, gk, gn)), _t("offs", (NUM_EXPERTS,), "int32"),
              _t("c", (t, gn))), ("c",), "c", "elements", ((i31, 174648),)),
        Case("wgrad", "K-grouped weight gradient, fp16, then T == 0 on the same output",
             (_t("dy", (w["t"], w["m"])), _t("x", (w["t"], w["n"])), _t("offs", (w["g"],), "int32"),
              _t("c", (w["g"], w["m"], w["n"]))), ("c",), "c", "elements", ((i31, 113), (i32, 227))),
        Case("wgrad_long", "K-grouped weight gradient, fp16, long reductions",
             (_t("dy", (t, gn)), _t("x", (t, gk)), _t("offs", (len(WGRAD_LONG_SIZES),), "int32"),
              _t("c", (len(WGRAD_LONG_SIZES), gn, gk))), ("c",), "dy", "elements", ((i31, 174648),)),
        Case("fp8_experts", "block-scaled e4m3 grouped and masked batched, bf16 out, one weight stack",
             (_t("bt", (e["g"], e["n"], e["k"]), "e4m3"), _t("sb", (e["g"], enb, enkb), "fp32"),
              _t("a", (e["t"], e["k"]), "e4m3"), _t("sa", (enkb, e["t"]), "fp32"),
              _t("offs", (e["g"],), "int32"), _t("c", (e["t"], e["n"]), "bf16"),
              _t("ab", (e["g"], e["slots"], e["k"]), "e4m3"), _t("sab", (e["g"], enkb, e["slots"]), "fp32"),
              _t("masked_m", (e["g"],), "int32"), _t("cb", (e["g"], e["slots"], e["n"]), "bf16")),
             ("c", "cb"), "bt", "bytes", ((i31, 117), (i32, 234))),
        Case("fp8_dw", "1 x 128 x 1 x 128 e4m3 weight gradient, bf16 out, A past 2^31 bytes along K",
             (_t("a", (dm, dk), "e4m3"), _t("bt", (dn, dk), "e4m3"), _t("sa", (dnkb, -(-dm // 4) * 4), "fp32"),
              _t("sb", (dnkb, -(-dn // 4) * 4), "fp32"), _t("c", (dm, dn), "bf16")), ("c",), "a", "bytes",
             ((i31, 477),)),
        Case("fp8_dw_out", "1 x 128 x 1 x 128 e4m3 2-D, bf16 out",
             (_t("a", (m, k), "e4m3"), _t("bt", (n, k), "e4m3"), _t("sa", (nkb, -(-m // 4) * 4), "fp32"),
              _t("sb", (nkb, -(-n // 4) * 4), "fp32"), _t("c", (m, n), "bf16")), ("c",), "c", "elements",
             ((i31, 16383),)),
        Case("quant", "every e4m3 quantiser of a bf16 activation, outputs sharing two guarded buffers and two scale "
             "buffers (each sized for the largest layout it holds)",
             (_t("x", (qr, qc), "bf16"), _t("q", (qr, qc), "e4m3"), _t("q_t", (qc, qld_t), "e4m3"),
              _t("scale", (-(-qc // 128), -(-qr // 4) * 4), "fp32"), _t("scale_t", (-(-qr // 128), -(-qc // 4) * 4), "fp32"),
              _t("workspace", (qr + qc + 1024,), "fp32")), ("q", "q_t"), "x", "elements", ((i31, 261888),)),
    ]
    return {c.name: c for c in out}


CASES = _cases()


def allocate(case: Case, dtype16=torch.float16, device="cuda") -> dict:
    """The case's tensors (uninitialised), the outputs inside guarded buffers filled with the sentinel: name ->
    tensor, and "<output>:buf" -> its buffer. ``device="meta"`` allocates nothing."""
    out = {}
    for t in case.tensors:
        dt = dtype16 if t.dtype == "16" else DTYPES[t.dtype]
        if t.name in case.outputs:
            out[f"{t.name}:buf"], out[t.name] = guarded(t.shape, dt, device)
        else:
            out[t.name] = torch.empty(t.shape, dtype=dt, device=device)
    return out


# ------------------------------------------------------------------------------------------------ guard bands
def guarded(shape, dtype, device="cuda"):
    """(buffer, view): the view of ``shape`` lies in the buffer with GUARD_BYTES on each side, all of it holding the
    NaN sentinel of ``dtype``."""
    size = torch.empty((), dtype=dtype).element_size()
    g = GUARD_BYTES // size
    buf = torch.empty((2 * g + math.prod(shape),), dtype=dtype, device=device)
    if device != "meta":
        buf.view(_BITS[size]).fill_(SENTINEL[dtype])
    return buf, buf[g:g + math.prod(shape)].view(shape)


def guards_intact(buf) -> bool:
    g = GUARD_BYTES // buf.element_size()
    s = SENTINEL[buf.dtype]
    bits = buf.view(_BITS[buf.element_size()])
    return bool((bits[:g] == s).all()) and bool((bits[-g:] == s).all())


# ------------------------------------------------------------------------------------------------ operands
# Integer ranges [lo, hi] (and the share of nonzeros) of each case's operands, and the bound each obeys:
# max over elements of sum_k |i * j| <= reduction * max|i| * max|j|.
DOMAINS = {
    "fp16": dict(a=(-15, 15), b=(-15, 15)),                 # K = 256 and 64: <= 57 600 (fp16 out, few infs)
    "fp16acc16": dict(a=(-1, 1), b=(-7, 7)),                # K = 256: <= 1 792 < 2048
    "bf16": dict(a=(-127, 127), b=(-127, 127)),             # K = 256: < 2^22
    "tall": dict(a=(-7, 7), b=(-7, 7)),                     # K = 16 384: < 2^20
    "nn_long": dict(a=(1, 1, 0.125), b=(1, 1, 0.5)),        # 0/1, K = 262 216: row sums of A asserted < 65 504
    "wgrad": dict(a=(-7, 7), b=(-7, 7)),                    # groups of <= 24 576 rows: < 2^21
    "wgrad_long": dict(a=(-1, 1), b=(-7, 7)),               # groups of <= 140 001 rows: < 2^20
    "e4m3": dict(a=(-1, 1, 0.2), b=(-1, 1)),                # nonzeros per row of A asserted <= 2047
}


def sum_bound(domain: dict, reduction: int) -> int:
    """The largest sum_k |i * j| the domain allows over a reduction of that length."""
    return reduction * max(map(abs, domain["a"][:2])) * max(map(abs, domain["b"][:2]))


def exact_bound(kind: str) -> int:
    """exact_domain.py's bound for a kind of product (sums must stay below it, e4m3: at or below)."""
    return {"fp16acc16": ed.FP16_ACC_SUM_BOUND, "e4m3": ed.E4M3_SUM_BOUND + 1}.get(kind, ed.EXACT_SUM_BOUND)


def generator(seed: int, device="cuda") -> torch.Generator:
    return torch.Generator(device=device).manual_seed(seed)


def fill_ints_(x: torch.Tensor, spec: tuple, gen: torch.Generator, band: int = 1 << 27) -> torch.Tensor:
    """``x`` <- integers drawn uniformly from [lo, hi] (``spec`` = (lo, hi) or (lo, hi, p): each kept with probability
    p, else 0). fp16 / bf16 are filled in place (random_ / bernoulli_ on the tensor); e4m3 band by band through an fp16
    band of ``band`` elements. Nothing full-size besides ``x``."""
    lo, hi = spec[:2]
    p = spec[2] if len(spec) > 2 else None
    flat = x.view(-1)
    direct = x.dtype in (torch.float16, torch.bfloat16)
    step = flat.numel() if direct and p is None else band
    for s in range(0, flat.numel(), step):
        part = flat[s:s + step]
        tmp = part if direct else torch.empty(part.shape, dtype=torch.float16, device=x.device)
        tmp.random_(lo, hi + 1, generator=gen)
        if p is not None:
            tmp.mul_(torch.empty_like(tmp).bernoulli_(p, generator=gen))
        if tmp is not part:
            part.copy_(tmp)
    return x


def pow2_scales_(x: torch.Tensor, gen: torch.Generator) -> torch.Tensor:
    """Block scales 2^-1, 2^0 or 2^1 (exact in every product and fp32 sum of the e4m3 domain), in place."""
    return x.random_(-1, 2, generator=gen).exp2_()


# ------------------------------------------------------------------------------------------------ routing
def routing_histogram(t: int, seed: int, g: int = NUM_EXPERTS, cross_rows=(), empty=(), nonempty=(),
                      big: int | None = BIG_GROUP, residues: bool = True) -> np.ndarray:
    """Group sizes (int64 [g], sum t) of a seeded, Zipf-like routing of t tokens to g experts: groups 0 and g-1 and
    g/16 others empty (and ``empty``), six of 1 row, the others Zipf-sized, one of them at least ``big`` rows. Each row
    of ``cross_rows`` lies in a group of fewer than 128 rows (so the tile holding the row straddles its end) with an
    empty group on each side. ``nonempty`` groups get rows. ``residues``: group starts at every residue mod 128 (and
    so mod 4), set by moving boundaries between Zipf groups."""
    rng = np.random.default_rng(seed)
    role = np.array(["z"] * g, dtype=object)
    role[[0, g - 1]] = "e"
    fixed = {}
    for r in cross_rows:
        c = int(np.clip(round(g * r / t), 3, g - 4))
        role[[c - 1, c + 1]], role[c] = "e", "x"
        fixed[c] = (r - int(rng.integers(1, 60)), r + int(rng.integers(1, 60)))
    role[list(empty)] = "e"
    assert all(role[i] not in ("e",) for i in nonempty), "a group is asked to be both empty and nonempty"
    spare = rng.permutation([i for i in range(1, g - 1) if role[i] == "z" and i not in nonempty])
    role[spare[:g // 16]] = "e"
    role[spare[g // 16:g // 16 + 6]] = "1"
    sizes = np.zeros(g, dtype=np.int64)
    # segments between the fixed (crossing) groups, each with the rows it must hold
    cuts = sorted(fixed)
    segs, prev_end, prev_g = [], 0, -1
    for c in cuts + [g]:
        start = fixed[c][0] if c < g else t
        segs.append((list(range(prev_g + 1, c)), start - prev_end))
        if c < g:
            sizes[c] = fixed[c][1] - fixed[c][0]
            prev_end, prev_g = fixed[c][1], c
    big_seg = max(range(len(segs)), key=lambda i: segs[i][1]) if big else -1
    for i, (members, rows) in enumerate(segs):
        ones = [j for j in members if role[j] == "1"]
        zipf = [j for j in members if role[j] == "z"]
        sizes[ones] = 1
        rest = rows - len(ones) - 2 * len(zipf)
        if i == big_seg:
            b = zipf[int(rng.integers(len(zipf)))]
            role[b] = "b"
            sizes[b] += big
            rest -= big
        assert rest >= 0 and zipf, f"{rows} rows cannot hold the groups of segment {i}"
        w = 1.0 / (1.0 + rng.permutation(len(zipf))) ** 1.1
        share = np.floor(rest * w / w.sum()).astype(np.int64)
        share[np.argmax(w)] += rest - share.sum()
        sizes[zipf] += 2 + share
    assert sizes.sum() == t
    if residues:
        _cover_residues(sizes, role)
    return sizes


def _cover_residues(sizes: np.ndarray, role: np.ndarray) -> None:
    """Move boundaries between consecutive Zipf groups (empty groups between them move along) until the starts of the
    nonempty groups take every residue mod 128; every group keeps at least one row."""
    nz = [i for i in range(len(sizes)) if role[i] == "z"]
    pairs = []   # (i, j): Zipf groups with only empty groups between them
    for i, j in zip(nz, nz[1:]):
        if all(role[x] == "e" for x in range(i + 1, j)):
            pairs.append((i, j))
    for r in range(128):
        starts = np.concatenate(([0], np.cumsum(sizes)[:-1]))
        have = [int(starts[i]) % 128 for i in range(len(sizes)) if sizes[i] > 0]
        if r in have:
            continue
        for i, j in pairs:
            s_j = int(starts[j])
            if have.count(s_j % 128) < 2:
                continue
            lo, hi = int(starts[i]) + 1, s_j + int(sizes[j]) - 1
            x = lo + (r - lo) % 128
            if x <= hi:
                sizes[i], sizes[j] = x - starts[i], s_j + sizes[j] - x
                break
        else:
            raise AssertionError(f"no boundary can take residue {r}")


def group_ends(sizes) -> list:
    return [int(v) for v in np.cumsum(sizes)]


def histogram_report(sizes, cross_rows=()) -> dict:
    """What a histogram offers: its empty, 1-row and largest groups, the residues of its nonempty groups' starts, and
    for each crossing row the group holding it with its neighbours' sizes."""
    sizes = np.asarray(sizes)
    starts = np.concatenate(([0], np.cumsum(sizes)[:-1]))
    ends = np.cumsum(sizes)
    out = {"empty": [int(i) for i in np.flatnonzero(sizes == 0)], "one_row": int((sizes == 1).sum()),
           "largest": int(sizes.max()), "res4": {int(s) % 4 for s, z in zip(starts, sizes) if z > 0},
           "res128": {int(s) % 128 for s, z in zip(starts, sizes) if z > 0}, "crossings": []}
    for r in cross_rows:
        c = int(np.searchsorted(ends, r, side="right"))
        out["crossings"].append(dict(group=c, start=int(starts[c]), size=int(sizes[c]),
                                     before=int(sizes[c - 1]), after=int(sizes[c + 1])))
    return out


HISTOGRAMS = {
    "grouped": dict(t=T_GROUPED, seed=7, cross_rows=(174648,)),
    "wgrad": dict(t=WGRAD["t"], seed=9, nonempty=(113, 227), empty=(114, 228), big=None, residues=False),
    "fp8_experts": dict(t=FP8_EXPERTS["t"], seed=11, nonempty=(117, 234), big=None, residues=False),
}


def histogram(name: str) -> np.ndarray:
    return routing_histogram(**HISTOGRAMS[name])


def masked_counts(b: int, m: int, seed: int) -> list:
    """Row counts of a masked batched case, every kind in each run of six batches: 0, 1, M, more than M, negative,
    and a ragged count in (1, M)."""
    rng = np.random.default_rng(seed)
    kinds = (0, 1, m, m + 37, -5, None)
    return [int(rng.integers(2, m)) if kinds[i % 6] is None else kinds[i % 6] for i in range(b)]


# ------------------------------------------------------------------------------------------------ the reference
def band_rows(n: int) -> int:
    """Rows of a float64 band of n columns that fit BAND_BYTES."""
    return max(1, BAND_BYTES // (8 * n))


def matmul64(a: torch.Tensor, b: torch.Tensor, band_bytes: int = BAND_BYTES) -> torch.Tensor:
    """a [R, K] @ b [K, N] in float64 (any float dtypes, views allowed), the reduction in chunks so that no float64
    chunk of a or b passes ``band_bytes``; partial products summed in float64 (exact on the domain)."""
    r, k = a.shape
    n = b.shape[1]
    out = torch.zeros((r, n), dtype=torch.float64, device=a.device)
    kc = max(1, band_bytes // (8 * max(r, n)))
    for k0 in range(0, k, kc):
        out.addmm_(a[:, k0:k0 + kc].to(torch.float64), b[k0:k0 + kc].to(torch.float64))
    return out


def round_bits(x64: torch.Tensor, dtype) -> torch.Tensor:
    """float64 values of the domain -> int16 bits of ``dtype`` (fp16 / bf16): to float32 exactly (+0.0 makes every
    zero positive, as the kernels' sums are), then one rounding to nearest even."""
    return (x64.to(torch.float32) + 0.0).to(dtype).view(torch.int16)


def first_mismatch(out: torch.Tensor, ref_rows, rows: int | None = None, base: int = 0, boundary: int = 2 ** 31,
                   what: str = "") -> str | None:
    """Compare rows [0, rows) of the 2-D ``out`` bit for bit with ``ref_rows(r0, r1)`` (float64 [r1 - r0, N]) rounded
    once, band by band. None if all equal, else where the first mismatch is: its flat element index (``base``: that of
    out[0, 0] in the tensor the index is counted in), its distance from ``boundary`` and its band."""
    rows = out.shape[0] if rows is None else rows
    n = out.shape[1]
    step = band_rows(n)
    for i, r0 in enumerate(range(0, rows, step)):
        r1 = min(rows, r0 + step)
        want = round_bits(ref_rows(r0, r1), out.dtype)
        got = out[r0:r1].view(torch.int16)
        bad = got != want
        if bool(bad.any()):
            j = int(bad.view(-1).nonzero()[0])
            idx = base + r0 * n + j
            return (f"{what}: first mismatch at element {idx} ({idx - boundary:+d} from 2^{boundary.bit_length() - 1}), "
                    f"row {r0 + j // n} col {j % n}, band {i} (rows [{r0}, {r1})): got {int(got.view(-1)[j]) & 0xFFFF:#06x}, "
                    f"want {int(want.view(-1)[j]) & 0xFFFF:#06x}")
    return None


def grouped_rows(a: torch.Tensor, b_kn, ends):
    """ref_rows of a grouped product: rows [s, e) of group g are a[s:e] @ b_kn(g) ([K, N], float64-convertible)."""
    starts = [0] + list(ends[:-1])

    def ref(r0, r1):
        out = torch.empty((r1 - r0, b_kn(0).shape[1]), dtype=torch.float64, device=a.device)
        for g, (s, e) in enumerate(zip(starts, ends)):
            lo, hi = max(s, r0), min(e, r1)
            if lo < hi:
                out[lo - r0:hi - r0] = matmul64(a[lo:hi], b_kn(g))
        return out
    return ref


def block_expand(s: torch.Tensor, rows: int, cols: int, rb: int = 1) -> torch.Tensor:
    """Block scales [ceil(rows / rb), ceil(cols / 128)] spread to one per element [rows, cols] (float64)."""
    x = s.to(torch.float64)
    if rb > 1:
        x = x.repeat_interleave(rb, dim=0)
    return x.repeat_interleave(128, dim=1)[:rows, :cols]


# ------------------------------------------------------------------------------------------------ quantisers
QUANTISERS = ("tensor", "rowwise", "blockwise", "silu_mul", "rowwise_dual", "blockwise_dual", "block128x128_dual")


def quant_band_rows(cols: int) -> int:
    """Rows of x per reference band: a multiple of 128 (whole 128-row groups of the transposed and 128 x 128 results)
    whose float32 copy takes at most a quarter of BAND_BYTES (the reference holds a few of them)."""
    return max(128, BAND_BYTES // (16 * cols) // 128 * 128)


def quant_bands(kind: str, x: torch.Tensor, band_rows: int):
    """The reference of quantiser ``kind`` (a key of QUANTISERS) on x [rows, cols], band by band: yields (result,
    index, want) with ``want`` the bits the unbanded ``ops.*_reference`` gives at ``index`` (a tuple of slices) of its
    ``result`` ("q", "scale", "q_t" or "scale_t", laid out as that reference lays it out). Each band holds ``band_rows``
    rows of x (a multiple of 128). The global quantities are reduced over all bands first: the per-tensor amax, and the
    column maxima behind the rowwise dual's scale_t. q_t's band is its columns [lo, hi); its padding columns [rows,
    ld_t) come with the last band (blockwise dual) or on their own (rowwise dual)."""
    from cuda_l2_b200 import capi, ops
    assert band_rows % 128 == 0 and kind in QUANTISERS
    rows, cols = x.shape
    e4, big, tiny = torch.float8_e4m3fn, ops.E4M3_MAX, torch.finfo(torch.float32).tiny
    bands = [(lo, min(rows, lo + band_rows)) for lo in range(0, rows, band_rows)]
    ld_t = capi.dual_ld_t(rows)
    every = slice(None)
    if kind == "tensor":
        # abs() again: a NaN that reduction returns keeps the sign the unbanded reference's does (+), as in its abs()
        amax = torch.stack([x[lo:hi].abs().amax() for lo, hi in bands]).amax().abs()
        scale = (amax.float() / big).clamp_min(tiny).reshape(1)
        yield "scale", (every,), scale
        for lo, hi in bands:
            yield "q", (slice(lo, hi),), (x[lo:hi].float() / scale).clamp(-big, big).to(e4)
        return
    if kind == "rowwise_dual":
        col_max = torch.stack([x[lo:hi].abs().amax(dim=0) for lo, hi in bands]).amax(dim=0).abs()
        scale_t = (col_max.float() / big).clamp_min(tiny)
        yield "scale_t", (every,), scale_t
        pad = torch.zeros((cols, ld_t - rows), dtype=torch.float32, device=x.device)
        yield "q_t", (every, slice(rows, ld_t)), (pad / scale_t[:, None]).clamp(-big, big).to(e4)
    for lo, hi in bands:
        xb, r = x[lo:hi], slice(lo, hi)
        if kind == "rowwise":
            q, s = ops.quantize_e4m3_rowwise_reference(xb)
            yield "q", (r,), q
            yield "scale", (r,), s
        elif kind in ("blockwise", "blockwise_dual", "silu_mul"):
            ref = ops.silu_mul_quantize_e4m3_blockwise_reference if kind == "silu_mul" else \
                ops.quantize_e4m3_blockwise_reference
            q, s = ref(xb)
            yield "q", (r,), q
            yield "scale", (r,), s
            if kind == "blockwise_dual":
                xt = xb.t()
                if hi == rows:
                    xt = torch.nn.functional.pad(xt, (0, ld_t - rows))
                qt, st = ops.quantize_e4m3_blockwise_reference(xt.contiguous())
                yield "q_t", (every, slice(lo, lo + qt.shape[1])), qt
                yield "scale_t", (every, slice(lo // 128, lo // 128 + st.shape[1])), st
        elif kind == "rowwise_dual":
            q, s = ops.quantize_e4m3_rowwise_reference(xb)
            yield "q", (r,), q
            yield "scale", (r,), s.reshape(-1)
            yield "q_t", (every, r), (xb.t().float() / scale_t[:, None]).clamp(-big, big).to(e4)
        else:
            q, s = ops.quantize_e4m3_block128x128(xb)
            sr = slice(lo // 128, lo // 128 + s.shape[0])
            yield "q", (r,), q
            yield "scale", (sr,), s
            yield "q_t", (every, r), q.t()
            yield "scale_t", (every, sr), s.t()
