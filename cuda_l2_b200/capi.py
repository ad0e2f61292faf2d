"""ctypes binding of the C-ABI libraries (include/b200_hgemm.h, include/b200_baselines.h).

This is the Python face of the drop-in boundary: the same entry points the torch extension
(``pybind/hgemm_b200_fp32.cc`` / ``hgemm_b200_fp16.cc``) wraps, reachable without a JIT build.  Tensors
are torch CUDA tensors used purely as device-memory handles (``data_ptr()``); all arithmetic happens in
``libb200_hgemm.so``.  There is no CPU or PyTorch fallback: if the library is missing or the device is
not an H100, these functions raise.
"""
from __future__ import annotations

import ctypes
from pathlib import Path

LIB_DIR = Path(__file__).resolve().parent / "lib"
_hgemm = None
_baselines = None

ACC_BITS = {"fp32": 32, "fp16": 16, 32: 32, 16: 16}


class B200HgemmError(RuntimeError):
    pass


def _load(name: str) -> ctypes.CDLL:
    path = LIB_DIR / name
    if not path.exists():
        raise B200HgemmError(
            f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `python cuda_l2_b200/build.py`). There is no fallback path.")
    return ctypes.CDLL(str(path))


def hgemm_lib() -> ctypes.CDLL:
    global _hgemm
    if _hgemm is None:
        lib = _load("libb200_hgemm.so")
        vp, i = ctypes.c_void_p, ctypes.c_int
        for fn in ("b200_hgemm_f32acc", "b200_hgemm_f16acc"):
            getattr(lib, fn).argtypes = [vp, vp, vp, vp, i, i, i, vp]
            getattr(lib, fn).restype = i
        lib.b200_bgemm_f32acc.argtypes = [vp, vp, vp, vp, i, i, i, vp]
        lib.b200_bgemm_f32acc.restype = i
        lib.b200_bgemm_run_config.argtypes = [i, vp, vp, vp, i, i, i, i, i, i, vp]
        lib.b200_hgemm_num_configs.restype = i
        lib.b200_hgemm_config_info.argtypes = [i, ctypes.POINTER(i), ctypes.POINTER(i), ctypes.POINTER(i)]
        lib.b200_hgemm_config_cluster.argtypes = [i, ctypes.POINTER(i), ctypes.POINTER(i)]
        lib.b200_hgemm_config_m_rep.argtypes = [i]
        lib.b200_hgemm_config_stages_requested.argtypes = [i]
        lib.b200_hgemm_select_config.argtypes = [i, i, i, i]
        lib.b200_hgemm_select.argtypes = [i, i, i, i, ctypes.POINTER(i), ctypes.POINTER(i), ctypes.POINTER(i)]
        lib.b200_hgemm_run_config.argtypes = [i, i, vp, vp, vp, i, i, i, i, i, i, vp]
        lib.b200_hgemm_host.argtypes = [i, vp, vp, vp, i, i, i]
        ip = ctypes.POINTER(i)
        lib.b200_hgemm_schedule_units.argtypes = [i, i, i, i, i, i, i, ip, i, ip, ip, ip]
        lib.b200_hgemm_schedule_units.restype = i
        lib.b200_hgemm_prewarm.argtypes = [vp]
        lib.b200_hgemm_release.argtypes = []
        lib.b200_hgemm_launch_count.restype = ctypes.c_ulonglong
        lib.b200_hgemm_strerror.argtypes = [i]
        lib.b200_hgemm_strerror.restype = ctypes.c_char_p
        _hgemm = lib
    return _hgemm


def baselines_lib() -> ctypes.CDLL:
    global _baselines
    if _baselines is None:
        lib = _load("libb200_baselines.so")
        vp, i = ctypes.c_void_p, ctypes.c_int
        lib.b200_bl_init.argtypes = [i]
        lib.b200_bl_destroy.argtypes = [i]
        lib.b200_bl_destroy.restype = None
        for fn in ("b200_bl_cublas", "b200_bl_lt_heuristic", "b200_bl_lt_autotune"):
            getattr(lib, fn).argtypes = [i, i, vp, vp, vp, i, i, i]
        lib.b200_bl_lt_autotune_find.argtypes = [i, i, i, i, i, i, i]
        lib.b200_bl_lt_autotune_info.argtypes = [i, i, ctypes.POINTER(i), ctypes.POINTER(ctypes.c_float)]
        _baselines = lib
    return _baselines


def exported_symbols() -> dict[str, list[str]]:
    """Symbols each header declares — used by the CPU tests to check the libraries export all of them."""
    return {
        "libb200_hgemm.so": [
            "b200_hgemm_f32acc", "b200_hgemm_f16acc", "b200_hgemm_num_configs", "b200_hgemm_config_info",
            "b200_hgemm_config_cluster", "b200_hgemm_config_m_rep", "b200_hgemm_config_stages_requested",
            "b200_hgemm_select_config", "b200_hgemm_select", "b200_hgemm_run_config", "b200_hgemm_host", "b200_hgemm_launch_count",
            "b200_hgemm_strerror", "b200_hgemm_schedule_units", "b200_hgemm_prewarm", "b200_hgemm_release",
            "b200_bgemm_f32acc", "b200_bgemm_run_config",
        ],
        "libb200_baselines.so": [
            "b200_bl_init", "b200_bl_destroy", "b200_bl_cublas", "b200_bl_lt_heuristic", "b200_bl_lt_autotune_find",
            "b200_bl_lt_autotune", "b200_bl_lt_autotune_info",
        ],
    }


def strerror(status: int) -> str:
    return hgemm_lib().b200_hgemm_strerror(status).decode()


def _check(status: int, what: str) -> None:
    if status != 0:
        raise B200HgemmError(f"{what} failed: status {status} ({strerror(status)})")


def _shape_check(a, b_col_major, c):
    import torch

    for name, t in (("a", a), ("b_col_major", b_col_major), ("c", c)):
        if t.dtype != torch.half:
            raise B200HgemmError(f"{name} must be torch.half, got {t.dtype}")
        if not t.is_cuda:
            raise B200HgemmError(f"{name} must be a CUDA tensor")
        if not t.is_contiguous():
            raise B200HgemmError(f"{name} must be contiguous")
    m, k = a.shape
    # b_col_major is shape-labelled [K,N] but its memory is [N,K] (tools/utils.py:110-115 in the reference)
    kb, n = b_col_major.shape
    if kb != k or tuple(c.shape) != (m, n):
        raise B200HgemmError(f"shape mismatch: a {tuple(a.shape)}, b_col_major {tuple(b_col_major.shape)}, c {tuple(c.shape)}")
    return m, n, k


def hgemm(a, b_col_major, c, acc: str | int = "fp32", stream: int | None = None) -> None:
    """c[M,N] = a[M,K] @ B[K,N] where ``b_col_major`` holds B K-major. Asynchronous on ``stream``
    (``None`` = the legacy default stream, like the reference's launches)."""
    m, n, k = _shape_check(a, b_col_major, c)
    bits = ACC_BITS[acc]
    fn = hgemm_lib().b200_hgemm_f32acc if bits == 32 else hgemm_lib().b200_hgemm_f16acc
    _check(fn(a.data_ptr(), None, b_col_major.data_ptr(), c.data_ptr(), m, n, k, stream), "b200_hgemm")


def gemm_kmajor(a, b_kmajor, c, acc: str | int = "fp32", stream: int | None = None, config_id: int | None = None,
                group_m: int = 0, splits: int = 1) -> None:
    """c[M,N] = a[M,K] @ b_kmajor[N,K]^T with the operands' dtype deciding the kernel family: fp16 (fp32 or fp16
    accumulation) or bf16 (fp32 accumulation). ``b_kmajor`` is shaped as stored, [N,K] — an ``nn.Linear`` weight.
    ``config_id`` pins one kernel configuration (tests); default is the dispatcher."""
    import torch

    if a.dtype not in (torch.half, torch.bfloat16) or b_kmajor.dtype != a.dtype or c.dtype != a.dtype:
        raise B200HgemmError(f"operands must all be fp16 or all bf16, got {a.dtype}, {b_kmajor.dtype}, {c.dtype}")
    for name, t in (("a", a), ("b_kmajor", b_kmajor), ("c", c)):
        if not t.is_cuda or not t.is_contiguous():
            raise B200HgemmError(f"{name} must be a contiguous CUDA tensor")
    (m, k), (n, k2) = a.shape, b_kmajor.shape
    if k2 != k or tuple(c.shape) != (m, n):
        raise B200HgemmError(f"shape mismatch: a {tuple(a.shape)}, b_kmajor {tuple(b_kmajor.shape)}, c {tuple(c.shape)}")
    lib = hgemm_lib()
    bits = ACC_BITS[acc]
    if a.dtype == torch.bfloat16:
        if bits != 32:
            raise B200HgemmError("bf16 operands accumulate in fp32 only")
        if config_id is None:
            st = lib.b200_bgemm_f32acc(a.data_ptr(), None, b_kmajor.data_ptr(), c.data_ptr(), m, n, k, stream)
        else:
            st = lib.b200_bgemm_run_config(config_id, a.data_ptr(), b_kmajor.data_ptr(), c.data_ptr(), m, n, k, group_m, 0, splits, stream)
    elif config_id is None:
        fn = lib.b200_hgemm_f32acc if bits == 32 else lib.b200_hgemm_f16acc
        st = fn(a.data_ptr(), None, b_kmajor.data_ptr(), c.data_ptr(), m, n, k, stream)
    else:
        st = lib.b200_hgemm_run_config(bits, config_id, a.data_ptr(), b_kmajor.data_ptr(), c.data_ptr(), m, n, k, group_m, 0, splits, stream)
    _check(st, "b200 gemm")


def hgemm_config(a, b_col_major, c, config_id: int, acc: str | int = "fp32", group_m: int = 0, max_ctas: int = 0,
                 splits: int = 1, stream: int | None = None) -> None:
    m, n, k = _shape_check(a, b_col_major, c)
    _check(hgemm_lib().b200_hgemm_run_config(ACC_BITS[acc], config_id, a.data_ptr(), b_col_major.data_ptr(),
                                            c.data_ptr(), m, n, k, group_m, max_ctas, splits, stream), "b200_hgemm_run_config")


def hgemm_host(a_host, b_col_major_host, c_host, acc: str | int = "fp32") -> None:
    """End-to-end call on HOST tensors (H2D + GEMM + D2H, synchronous) — what bench.py's e2e leg times."""
    m, k = a_host.shape
    kb, n = b_col_major_host.shape
    assert kb == k and tuple(c_host.shape) == (m, n)
    for t in (a_host, b_col_major_host, c_host):
        assert (not t.is_cuda) and t.is_contiguous()
    _check(hgemm_lib().b200_hgemm_host(ACC_BITS[acc], a_host.data_ptr(), b_col_major_host.data_ptr(),
                                       c_host.data_ptr(), m, n, k), "b200_hgemm_host")


def configs() -> list[dict]:
    lib = hgemm_lib()
    out = []
    for cid in range(lib.b200_hgemm_num_configs()):
        bn, st, cg = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        lib.b200_hgemm_config_info(cid, ctypes.byref(bn), ctypes.byref(st), ctypes.byref(cg))
        cm, cn = ctypes.c_int(), ctypes.c_int()
        lib.b200_hgemm_config_cluster(cid, ctypes.byref(cm), ctypes.byref(cn))
        out.append({"id": cid, "bn": bn.value, "stages": st.value, "cta_group": cg.value,
                    "stages_requested": lib.b200_hgemm_config_stages_requested(cid),
                    "cluster_m": cm.value, "cluster_n": cn.value, "m_rep": lib.b200_hgemm_config_m_rep(cid)})
    return out


def select_config(acc: str | int, m: int, n: int, k: int) -> int:
    return hgemm_lib().b200_hgemm_select_config(ACC_BITS[acc], m, n, k)


def select(acc: str | int, m: int, n: int, k: int) -> tuple[int, int, int]:
    """(config id, rasterisation group, split-K factor) the dispatcher uses for this problem."""
    cid, gm, sp = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _check(hgemm_lib().b200_hgemm_select(ACC_BITS[acc], m, n, k, ctypes.byref(cid), ctypes.byref(gm), ctypes.byref(sp)),
           "b200_hgemm_select")
    return cid.value, gm.value, sp.value


STREAMK_TAIL, STREAMK_TAIL_PLUS_WAVE = 100, 101      # `splits` codes of b200_hgemm_run_config


def schedule(config_id: int, m: int, n: int, k: int, splits: int = 1, num_sms: int = 132) -> dict:
    """Host-side view of the kernel's schedule (no GPU needed; the kernel walks the same code).

    Returns ``{"workers": W, "sk_tiles": S, "units": [[(tile, kb0, kb1, contributors), ...] per worker]}``."""
    lib = hgemm_lib()
    nw, sk = ctypes.c_int(), ctypes.c_int()
    cap = 64
    buf, contrib = (ctypes.c_int * (3 * cap))(), (ctypes.c_int * cap)()
    st = lib.b200_hgemm_schedule_units(config_id, m, n, k, splits, num_sms, 0, buf, cap, ctypes.byref(nw),
                                       ctypes.byref(sk), contrib)
    _check(min(st, 0), "b200_hgemm_schedule_units")
    units = []
    for w in range(nw.value):
        cnt = lib.b200_hgemm_schedule_units(config_id, m, n, k, splits, num_sms, w, buf, cap, None, None, contrib)
        _check(min(cnt, 0), "b200_hgemm_schedule_units")
        if cnt > cap:
            cap = cnt
            buf, contrib = (ctypes.c_int * (3 * cap))(), (ctypes.c_int * cap)()
            cnt = lib.b200_hgemm_schedule_units(config_id, m, n, k, splits, num_sms, w, buf, cap, None, None, contrib)
        units.append([(buf[3 * j], buf[3 * j + 1], buf[3 * j + 2], contrib[j]) for j in range(cnt)])
    return {"workers": nw.value, "sk_tiles": sk.value, "units": units}


def prewarm(stream: int | None = None) -> None:
    """Allocate the split-K / stream-K scratch of (current device, stream) now — needed before a CUDA-graph capture."""
    _check(hgemm_lib().b200_hgemm_prewarm(stream), "b200_hgemm_prewarm")


def release() -> None:
    """Free every device allocation the library holds (scratch, host-entry staging). Nothing may be in flight."""
    _check(hgemm_lib().b200_hgemm_release(), "b200_hgemm_release")


def gpu_local_cpus(device_index: int = 0) -> set[int] | None:
    """The CPUs NVML reports as local to the GPU (same NUMA node / PCIe root), intersected with the CPUs this process
    may use; None when NVML or the answer is unavailable."""
    import os

    try:
        import pynvml as nv
        nv.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        phys = device_index
        if vis:
            try:
                phys = int(vis.split(",")[device_index])
            except (ValueError, IndexError):
                pass
        h = nv.nvmlDeviceGetHandleByIndex(phys)
        words = nv.nvmlDeviceGetCpuAffinity(h, ((os.cpu_count() or 64) + 63) // 64)
        cpus = {64 * w + b for w, word in enumerate(words) for b in range(64) if (int(word) >> b) & 1}
        cpus &= os.sched_getaffinity(0)
        return cpus or None
    except Exception:
        return None


class host_near_gpu:
    """Context manager: run the calling thread on the CPUs local to ``device_index`` while HOST buffers for
    b200_hgemm_host are allocated (and, ideally, while the calls are made). Pinned memory lands on the NUMA node of the
    allocating thread; a buffer on the far socket costs the PCIe copies a cross-socket hop — in round 1 the same
    end-to-end call measured 55.7 TFLOP/s per GPU from a far node against 71.4 from the near one. Equivalent to
    launching under ``numactl --cpunodebind``; a no-op when NVML cannot tell."""

    def __init__(self, device_index: int = 0):
        self.device_index, self.saved, self.cpus = device_index, None, None

    def __enter__(self):
        import os
        self.cpus = gpu_local_cpus(self.device_index)
        if self.cpus:
            self.saved = os.sched_getaffinity(0)
            try:
                os.sched_setaffinity(0, self.cpus)
            except OSError:
                self.saved, self.cpus = None, None
        return self

    def __exit__(self, *exc):
        import os
        if self.saved is not None:
            os.sched_setaffinity(0, self.saved)
        return False


def launch_count() -> int:
    return int(hgemm_lib().b200_hgemm_launch_count())


# ------------------------------------------------------------------------------------------ comparators
class Baselines:
    """cuBLAS / cuBLASLt comparators (library calls; never part of the product path)."""

    NN, TN = 0, 1

    def __init__(self, acc: str | int = "fp32"):
        self.bits = ACC_BITS[acc]
        self.lib = baselines_lib()
        if self.lib.b200_bl_init(self.bits) != 0:
            raise B200HgemmError("cuBLAS/cuBLASLt handle creation failed")

    def close(self):
        self.lib.b200_bl_destroy(self.bits)

    def _call(self, fn, layout, a, b, c):
        m, k = a.shape
        n = c.shape[1]
        st = fn(self.bits, layout, a.data_ptr(), b.data_ptr(), c.data_ptr(), m, n, k)
        if st != 0:
            raise B200HgemmError(f"baseline call failed with status {st}")

    def cublas(self, layout, a, b, c):
        self._call(self.lib.b200_bl_cublas, layout, a, b, c)

    def lt_heuristic(self, layout, a, b, c):
        self._call(self.lib.b200_bl_lt_heuristic, layout, a, b, c)

    def lt_autotune_find(self, layout, m, n, k, warm_rounds=0, bench_rounds=0):
        st = self.lib.b200_bl_lt_autotune_find(self.bits, layout, m, n, k, warm_rounds, bench_rounds)
        if st != 0:
            raise B200HgemmError(f"cuBLASLt auto-tuning failed with status {st}")
        cand, ms = ctypes.c_int(), ctypes.c_float()
        self.lib.b200_bl_lt_autotune_info(self.bits, layout, ctypes.byref(cand), ctypes.byref(ms))
        return cand.value, ms.value

    def lt_autotune(self, layout, a, b, c):
        self._call(self.lib.b200_bl_lt_autotune, layout, a, b, c)
