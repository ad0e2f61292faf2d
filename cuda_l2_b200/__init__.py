"""cuda_l2_b200 — an H100-native (sm_90a) HGEMM kernel family behind the CUDA-L2 evaluation harness.

Scope: ONE hot path, ``C[M,N] (fp16) = A[M,K] (fp16) x B[K,N] (fp16)`` with fp32 or fp16 accumulation,
as hand-written wgmma/TMA CUDA in ``csrc/``, exposed through a C ABI (``include/b200_hgemm.h``),
a torch-extension binding with the reference's names (``pybind/hgemm_b200_fp{32,16}.cc``) and this
package's ctypes binding (:mod:`cuda_l2_b200.capi`).
"""
__version__ = "0.1.0"
