"""Deployable face of the kernel: a ``torch.library`` custom op and an ``nn.Linear`` drop-in.

The reference's README lists "easy deployment for open-source LLMs" as to-do and tells users of off-grid shapes to pad
to the nearest larger configuration (README.md:75,83-86). Here nothing is padded — the kernels take any
``M, N, K > 0`` with ``N % 8 == 0`` and ``K % 8 == 0`` and the dispatcher maps an off-grid shape to the tuned entry of
the nearest grid shape — so deployment is a plain operator:

* ``torch.ops.cuda_l2_b200.hgemm(a, b_kmajor, acc)``: ``a`` [M,K] times B given K-major as ``b_kmajor`` [N,K]
  (exactly the layout of an ``nn.Linear`` weight: ``[out_features, in_features]``), returns [M,N]. fp16 or bf16
  operands (bf16 always accumulates in fp32); ``acc`` = "fp32" | "fp16".
* ``torch.ops.cuda_l2_b200.hgemm_nn(a, b, acc)``: ``a`` [M,K] times ``b`` [K,N] row-major (``torch.matmul(a, b)``'s
  layout, such as attention's P·V), returns [M,N]. ``b`` is read in place by the row-major B kernels: no transposed
  copy. Its gradient needs no transposed copy of ``b`` either.
* ``torch.ops.cuda_l2_b200.hgemm_batched(a, b_kmajor, acc, masked_m=None)``: ``a`` [B,M,K] times ``b_kmajor``
  [B,N,K] per batch, returns [B,M,N] — ``torch.bmm(a, b_kmajor.transpose(1, 2))`` in one launch (per-head attention
  products, per-expert projections). ``masked_m``, an int32 CUDA tensor [B] read by the kernel (no host
  synchronisation), limits batch b to its first ``masked_m[b]`` rows: the layout of an MoE layer's experts, whose token
  counts live on the GPU. Inference only in that form; the dense form has a gradient.
* ``torch.ops.cuda_l2_b200.hgemm_grouped(a, b_kmajor, offs, acc)``: ``a`` [T,K] whose rows are sorted into contiguous
  groups, ``b_kmajor`` [G,N,K] one weight per group, ``offs`` the int32 cumulative group ends on the GPU; returns
  [T,N] — ``torch._grouped_mm(a, b_kmajor.transpose(-2, -1), offs=offs)`` in one launch, the MoE prefill layout.
  Inference only.
* ``torch.ops.cuda_l2_b200.hgemm_grouped_nn(a, b, offs, acc)``: ``a`` [T,K] in the same groups times ``b`` [G,K,N]
  row-major per group -> [T,N] (``torch._grouped_mm(a, b, offs=offs)``): an expert weight stack [G, N_model,
  K_model] is read in place as the B of the input gradient. Rows at or past ``offs[-1]`` are unspecified.
* ``torch.ops.cuda_l2_b200.hgemm_grouped_wgrad(a, b, offs, acc)``: ``a`` [T,M] and ``b`` [T,N] in the same groups ->
  [G,M,N], ``a[start_g:end_g]^T @ b[start_g:end_g]`` per group (``torch._grouped_mm(a.t(), b, offs=offs)``), the
  weight gradient; an empty group's matrix is zero.
* :func:`grouped_linear` (``torch.ops.cuda_l2_b200.grouped_linear(x, w, offs, acc)``) and :class:`B200GroupedLinear`:
  ``hgemm_grouped``'s product with a gradient. The forward is ``hgemm_grouped``'s kernel; ``dX`` runs
  ``hgemm_grouped_nn`` on the weight stack in place and ``dW`` ``hgemm_grouped_wgrad``, so a training step of the
  experts copies no operand. fp16 or bf16 with fp32 accumulation.
* ``torch.ops.cuda_l2_b200.hgemm_bias_act(a, b_kmajor, bias=None, activation='none')``: ``act(a @ b_kmajor^T + bias)``
  in one launch, fp16 or bf16 with fp32 accumulation; ``activation`` is "none", "relu" or "gelu_tanh" (torch's
  ``_addmm_activation`` set). The bias is added to the fp32 sum and the activation applied before the one rounding to
  the output type (libb200_epilogue.so, csrc/b200_epilogue.h). Its gradient reads relu's mask from the output and
  recomputes gelu_tanh's pre-activation with one more launch. :func:`linear` is ``F.linear`` plus the activation on it,
  for any leading dimensions. ``fp8_gemm_bias_act(a, b_kmajor, scale_a, scale_b, bias, activation, out_dtype)`` is the
  same epilogue after ``fp8_gemm``'s per-tensor or rowwise scales (inference only).
* :class:`B200Linear`: ``y = x @ W^T (+ b)`` for any leading dimensions; :func:`replace_linear_modules` swaps the
  eligible ``nn.Linear`` layers of a model in place.
* ``torch.ops.cuda_l2_b200.fp8_gemm(a, b_kmajor, scale_a, scale_b, out_dtype)``: ``float8_e4m3fn`` operands in the same
  layout, per-tensor fp32 scales as one-element CUDA tensors, ``(a @ b_kmajor^T) * scale_a * scale_b`` rounded once to
  ``out_dtype`` (fp16 or bf16) — ``torch._scaled_mm`` with per-tensor scales and fast accumulation. Rowwise scales
  follow ``torch._scaled_mm``'s shapes, ``scale_a`` [M,1] and ``scale_b`` [1,N]: ``((a @ b_kmajor^T) * scale_b) * scale_a``.
  Blockwise scales (DeepSeek-V3-style checkpoints): ``scale_a`` [M, ceil(K/128)] (one per token and 128 input
  channels), ``scale_b`` [ceil(N/128), ceil(K/128)] (one per 128 x 128 weight block); every 128-wide k-block's sum is
  scaled and accumulated in fp32 (include/b200_fp8_block.h).
* :class:`B200Fp8Linear`: inference-only FP8 version of an ``nn.Linear`` (weight quantised once, activation per call;
  per tensor, rowwise or blockwise), or of a checkpoint's e4m3 weight and block scales (:meth:`B200Fp8Linear.from_fp8`).
* ``torch.ops.cuda_l2_b200.fp8_grouped_gemm(a, b_kmajor, scale_a, scale_b, offs, out_dtype)``: the grouped product of
  ``hgemm_grouped`` with e4m3 operands and block scales, ``scale_a`` [T, ceil(K/128)] (one per token and 128 input
  channels), ``scale_b`` [G, ceil(N/128), ceil(K/128)] (each expert's ``weight_scale_inv``): the routed experts of an
  FP8 mixture-of-experts checkpoint in one launch (include/b200_grouped_fp8.h). Inference only.
* ``torch.ops.cuda_l2_b200.fp8_batched_gemm(a, b_kmajor, scale_a, scale_b, out_dtype, masked_m=None)``: the batched
  product of ``hgemm_batched`` with e4m3 operands and block scales, ``scale_a`` [B, M, ceil(K/128)], ``scale_b``
  [B, ceil(N/128), ceil(K/128)], and the optional per-batch row counts on the GPU: the same experts in the padded
  decode layout (include/b200_batched_fp8.h). Inference only.
* :class:`B200Fp8GroupedLinear`: those experts as a module, from a checkpoint's stacked e4m3 weights and block scales
  (:meth:`B200Fp8GroupedLinear.from_fp8`) or from a 16-bit stack (:meth:`B200Fp8GroupedLinear.from_weights`);
  ``forward`` takes the prefill layout, ``forward_masked`` the decode layout.
* ``torch.ops.cuda_l2_b200.quantize_e4m3(x)``, ``quantize_e4m3_rowwise(x)``, ``quantize_e4m3_blockwise(x,
  masked_m=None)`` and ``silu_mul_quantize_e4m3_blockwise(h, masked_m=None)``: the FP8 GEMMs' A operand and scales in
  one pass over a 16-bit or fp32 activation (libb200_quant.so, csrc/b200_quant.h), each returning ``(q, scale)`` with
  the bits of the torch composition :func:`quantize_e4m3` and its siblings keep as ``*_reference``. The last one
  quantises ``F.silu(g) * u`` of a gate/up product ``h = [g | u]``. :func:`quantize_e4m3` and its siblings route CUDA
  tensors to them. Inference only.
* :class:`B200Fp8GroupedMLP`: the routed experts of an FP8 MoE checkpoint as a gated MLP, four launches per forward
  (quantise, gate/up GEMM, SwiGLU + quantise, down GEMM), in the prefill or the decode layout.
* ``torch.ops.cuda_l2_b200.quantize_e4m3_rowwise_dual(x)``: ``(q, scale, q_t, scale_t)``, the rowwise quantisation of
  ``x`` [rows, cols] and of ``x^T`` zero-padded to a multiple of 16 columns, from one tensor (libb200_quant_dual.so,
  csrc/b200_quant_dual.h): the two K-major e4m3 operands FP8 training needs of each tensor. Inference only itself.
* :func:`fp8_linear` and :class:`B200Fp8TrainLinear`: ``x @ W^T`` trained in FP8, a rowwise-scaled e4m3 forward and
  backward (three ``fp8_gemm`` calls per step) over a trainable 16-bit weight.
* :func:`swiglu_linear` and :class:`B200SwiGLULinear`: ``F.silu(x @ W_gate^T) * (x @ W_up^T)``, the gate / up
  projection of a SwiGLU MLP, as one GEMM whose epilogue applies the activation (libb200_swiglu.so,
  csrc/b200_swiglu.h), over a fused weight whose gate and up rows interleave in blocks of 64
  (:func:`interleave_gate_up`, :func:`split_gate_up`). The backward is one element-wise pass for dh, then the
  product's dX and dW. Plain functions, not operators.
* ``fuse_wgrad_accumulation=True`` on :class:`B200Linear`, :class:`B200Fp8TrainLinear` and :class:`B200GroupedLinear`
  (and ``fp8_linear(..., main_grad=...)``): the backward adds dW into the weight's fp32 ``main_grad`` in the GEMM
  epilogue (libb200_wgrad_accum.so, csrc/b200_wgrad_accum.h) and returns no weight gradient. The plain functions
  :func:`wgrad_accumulate_`, :func:`grouped_wgrad_accumulate_` and :func:`fp8_gemm_accumulate_` are the pieces; they are
  not operators.

There is no CPU or PyTorch fallback on the forward path: a non-CUDA tensor, a missing library or a non-H100 device
raises. Backward (training is not what the reference targets) is provided through the same kernels, so a fine-tuning
loop works: ``hgemm``'s input gradient reads the weight in place through the row-major B kernels, and its weight
gradient pays one transposed copy (of the output gradient). The weight gradient reduces over the tokens M, which the
forward takes in any number: when M % 8 != 0 that copy would have rows of M % 8 != 0 elements, which no kernel reads,
so the weight gradients of ``hgemm``, ``hgemm_nn``, ``hgemm_batched`` and ``hgemm_bias_act`` run
``hgemm_grouped_wgrad`` instead, on both operands in place, with one group (one per batch) whose end it writes on the
device. The grouped product trains through :func:`grouped_linear`
(``hgemm_grouped`` itself stays inference only). The FP8 operators have no gradient: a backward through them raises.
FP8 training goes through :func:`fp8_linear`, whose own backward runs those operators.
"""
from __future__ import annotations

import torch
from torch import nn

from . import capi

_LIB = "cuda_l2_b200"


def _define_op(name: str, schema: str, shape, launch, why: str = "", outputs=None, backward=None,
               setup_context=None) -> None:
    """Defines the operator cuda_l2_b200::<name> with ``schema``. ``shape(*args)`` checks the arguments by the kernel's
    rules (meta tensors pass) and returns the result's shape and dtype: the fake implementation is an empty tensor of
    those, and the CUDA one allocates the result ``c`` on the operands' device and calls ``launch(c, *args,
    stream=...)`` there, on torch's current stream, so that it orders with the surrounding torch ops. Whatever more
    ``shape`` returns (the FP8 operators: the scale granularity it found) is passed to ``launch`` after the arguments,
    so that the launch does not work it out again.
    An operator with several results passes ``outputs`` instead of ``shape``: ``outputs(*args)`` checks the arguments
    the same way and returns the tuple of empty results, allocated on the device of ``args[0]`` in their final layout;
    the CUDA and the fake implementation both call it, so the fake results have the real ones' shapes and strides, and
    ``launch`` receives the tuple. The CPU implementation raises (there is no fallback). ``backward`` and
    ``setup_context`` are the operator's gradient, as torch.library.register_autograd takes them; without them it is
    inference only, and a backward through it raises (``why`` says why)."""
    qualname = f"{_LIB}::{name}"
    torch.library.define(qualname, schema)

    def cuda(*args):
        found = ()
        if outputs is not None:
            c = outputs(*args)
            device = args[0].device
        else:
            out_shape, dtype, *found = shape(*args)
            c = torch.empty(out_shape, dtype=dtype, device=args[0].device)
            device = c.device
        with torch.cuda.device(device):
            launch(c, *args, *found, stream=torch.cuda.current_stream(device).cuda_stream)
        return c

    def cpu(*args):
        raise capi.B200HgemmError(f"{qualname} has no CPU implementation (and no fallback): move the tensors to an H100")

    def fake(*args):
        if outputs is not None:
            return outputs(*args)
        out_shape, dtype, *_ = shape(*args)
        return args[0].new_empty(out_shape, dtype=dtype)

    def no_backward(ctx, *grads):
        raise capi.B200HgemmError(f"{qualname} is inference only: it has no gradient{why}")

    torch.library.impl(qualname, "CUDA")(cuda)
    torch.library.impl(qualname, "CPU")(cpu)
    torch.library.register_fake(qualname)(fake)
    # Without a gradient formula autograd would only warn and hand back no gradient for the inputs: no_backward raises.
    torch.library.register_autograd(qualname, backward or no_backward, setup_context=setup_context)


def _empty_product(c: torch.Tensor, k: int) -> bool:
    """Whether the product into ``c`` needs no kernel, as torch.matmul's: ``c`` has no element (M, N or B == 0), or
    the reduction is empty (K == 0), which makes ``c`` zero here. The C ABI rejects both with kBadShape."""
    if c.numel() == 0:
        return True
    if k == 0:
        c.zero_()
        return True
    return False


def _hgemm_shape(a, b_kmajor, acc="fp32"):
    m, n, _, _ = capi.check_operands(a, b_kmajor, a.dtype, acc)
    return (m, n), a.dtype


def _hgemm_launch(c, a, b_kmajor, acc="fp32", *, stream):
    if not _empty_product(c, a.shape[1]):
        capi.gemm_kmajor(a.contiguous(), b_kmajor.contiguous(), c, acc, stream=stream)


def _token_ends(m: int, groups: int, device) -> torch.Tensor:
    """The int32 group ends m, 2m, ..., groups * m of ``groups`` blocks of m tokens, written on the device by one kernel:
    no host copy, so a backward that passes them to the K-grouped kernel can be captured in a CUDA graph."""
    return torch.arange(m, m * groups + 1, m, dtype=torch.int32, device=device)


def _product_grads(a, b_kmajor, grad_c, need_a: bool, need_b: bool):
    """(dA, dBt) of C = A Bt^T for the output gradient ``grad_c`` (None where not needed)."""
    grad_a = grad_b = None
    g = grad_c.contiguous()
    # C = A Bt^T  =>  dA = dC Bt  (reduction over N: Bt [N,K] is B row-major),  dBt = dC^T A  (reduction over M: A [M,K]
    # is B row-major). The row-major B kernels read both in place; only dC^T is copied. They compute what the K-major
    # kernels compute on transposed copies, bit for bit.
    if need_a:
        grad_a = torch.ops.cuda_l2_b200.hgemm_nn(g, b_kmajor, "fp32")
    if need_b:
        m = a.shape[0]
        if m % 8 == 0:
            grad_b = torch.ops.cuda_l2_b200.hgemm_nn(g.t().contiguous(), a, "fp32")
        else:   # dC^T would have M % 8 != 0 columns (no 16-byte rows): the K-grouped kernel reduces any M, in place
            grad_b = torch.ops.cuda_l2_b200.hgemm_grouped_wgrad(g, a, _token_ends(m, 1, g.device), "fp32")[0]
    return grad_a, grad_b


def _hgemm_backward(ctx, grad_c):
    a, b_kmajor = ctx.saved_tensors
    return (*_product_grads(a, b_kmajor, grad_c, ctx.needs_input_grad[0], ctx.needs_input_grad[1]), None)


def _hgemm_setup_context(ctx, inputs, output):
    a, b_kmajor, _ = inputs
    ctx.save_for_backward(a, b_kmajor)


_define_op("hgemm", "(Tensor a, Tensor b_kmajor, str acc='fp32') -> Tensor", _hgemm_shape, _hgemm_launch,
           backward=_hgemm_backward, setup_context=_hgemm_setup_context)


def hgemm(a: torch.Tensor, b_kmajor: torch.Tensor, acc: str = "fp32") -> torch.Tensor:
    """``a`` [M,K] @ ``b_kmajor`` [N,K]^T -> [M,N] through the H100 kernel (see the module docstring)."""
    return torch.ops.cuda_l2_b200.hgemm(a, b_kmajor, acc)


# ------------------------------------------------------------------------------------------ row-major B (libb200_nn.so)
def _hgemm_nn_shape(a, b, acc="fp32"):
    m, n, _ = capi.check_rowmajor_operands(a, b, a.dtype, acc)
    return (m, n), a.dtype


def _hgemm_nn_launch(c, a, b, acc="fp32", *, stream):
    if not _empty_product(c, a.shape[1]):
        capi.gemm_rowmajor(a.contiguous(), b.contiguous(), c, acc, stream=stream)


def _hgemm_nn_backward(ctx, grad_c):
    a, b = ctx.saved_tensors
    grad_a = grad_b = None
    g = grad_c.contiguous()
    # C = A B  =>  dA = dC B^T (B [K,N] is K-major in the reduced N: the K-major kernels read it in place),
    # dB = A^T dC (dC [M,N] is row-major in the reduced M; A^T is copied)
    if ctx.needs_input_grad[0]:
        grad_a = torch.ops.cuda_l2_b200.hgemm(g, b, "fp32")
    if ctx.needs_input_grad[1]:
        m = a.shape[0]
        if m % 8 == 0:
            grad_b = torch.ops.cuda_l2_b200.hgemm_nn(a.t().contiguous(), g, "fp32")
        else:   # A^T would have M % 8 != 0 columns: the K-grouped kernel reads A and dC in place
            grad_b = torch.ops.cuda_l2_b200.hgemm_grouped_wgrad(a, g, _token_ends(m, 1, g.device), "fp32")[0]
    return grad_a, grad_b, None


def _hgemm_nn_setup_context(ctx, inputs, output):
    a, b, _ = inputs
    ctx.save_for_backward(a, b)


_define_op("hgemm_nn", "(Tensor a, Tensor b, str acc='fp32') -> Tensor", _hgemm_nn_shape, _hgemm_nn_launch,
           backward=_hgemm_nn_backward, setup_context=_hgemm_nn_setup_context)


def hgemm_nn(a: torch.Tensor, b: torch.Tensor, acc: str = "fp32") -> torch.Tensor:
    """``a`` [M,K] @ ``b`` [K,N] -> [M,N] (``torch.matmul(a, b)``) with ``b`` row-major, read in place by the H100
    row-major B kernels (see the module docstring)."""
    return torch.ops.cuda_l2_b200.hgemm_nn(a, b, acc)


# ------------------------------------------------------------------------------------------ batched (libb200_batched.so)
def _hgemm_batched_shape(a, b_kmajor, acc="fp32", masked_m=None):
    bsz, m, n, _ = capi.check_batched_operands(a, b_kmajor, acc, masked_m)
    return (bsz, m, n), a.dtype


def _hgemm_batched_launch(c, a, b_kmajor, acc="fp32", masked_m=None, *, stream):
    if _empty_product(c, a.shape[2]):
        return
    if masked_m is not None:
        masked_m = masked_m.contiguous()
    capi.gemm_batched(a.contiguous(), b_kmajor.contiguous(), c, acc, masked_m=masked_m, stream=stream)


def _hgemm_batched_backward(ctx, grad_c):
    if ctx.masked:
        raise capi.B200HgemmError("cuda_l2_b200::hgemm_batched with masked_m is inference only: it has no gradient")
    a, b_kmajor = ctx.saved_tensors
    grad_a = grad_b = None
    g = grad_c.contiguous()
    # per batch, as _hgemm_backward: dA = dC Bt (B operand Bt^T, K-major in N), dBt = dC^T A (reduction over M)
    if ctx.needs_input_grad[0]:
        grad_a = torch.ops.cuda_l2_b200.hgemm_batched(g, b_kmajor.transpose(1, 2).contiguous(), "fp32")
    if ctx.needs_input_grad[1]:
        bsz, m, k = a.shape
        if m % 8 == 0:
            grad_b = torch.ops.cuda_l2_b200.hgemm_batched(g.transpose(1, 2).contiguous(),
                                                          a.transpose(1, 2).contiguous(), "fp32")
        elif bsz:   # ragged M: the K-grouped kernel, batch b being the group of rows [b M, (b + 1) M), one launch
            grad_b = torch.ops.cuda_l2_b200.hgemm_grouped_wgrad(g.reshape(bsz * m, -1), a.reshape(bsz * m, k),
                                                                _token_ends(m, bsz, g.device), "fp32")
        else:       # no batch: the gradient has no element
            grad_b = torch.zeros_like(b_kmajor)
    return grad_a, grad_b, None, None


def _hgemm_batched_setup_context(ctx, inputs, output):
    a, b_kmajor, _, masked_m = inputs
    ctx.masked = masked_m is not None
    ctx.save_for_backward(a, b_kmajor)


_define_op("hgemm_batched", "(Tensor a, Tensor b_kmajor, str acc='fp32', Tensor? masked_m=None) -> Tensor",
           _hgemm_batched_shape, _hgemm_batched_launch, backward=_hgemm_batched_backward,
           setup_context=_hgemm_batched_setup_context)


def hgemm_batched(a: torch.Tensor, b_kmajor: torch.Tensor, acc: str = "fp32",
                  masked_m: torch.Tensor | None = None) -> torch.Tensor:
    """``a`` [B,M,K] @ ``b_kmajor`` [B,N,K]^T per batch -> [B,M,N] (``torch.bmm(a, b_kmajor.transpose(1, 2))``) through
    the H100 kernel (see the module docstring). ``masked_m``: optional int32 CUDA tensor [B]; only rows
    [0, clamp(masked_m[b], 0, M)) of batch b are computed, the rest of the result is unspecified."""
    return torch.ops.cuda_l2_b200.hgemm_batched(a, b_kmajor, acc, masked_m)


# ------------------------------------------------------------------------------------------ grouped (libb200_grouped.so)
def _hgemm_grouped_shape(a, b_kmajor, offs, acc="fp32"):
    _, t, n, _ = capi.check_grouped_operands(a, b_kmajor, offs, acc)
    return (t, n), a.dtype


def _hgemm_grouped_launch(c, a, b_kmajor, offs, acc="fp32", *, stream):
    if b_kmajor.shape[0] == 0 or _empty_product(c, a.shape[1]):   # no group, no element or no reduction
        return
    a, b_kmajor, offs = a.contiguous(), b_kmajor.contiguous(), offs.contiguous()
    capi.gemm_grouped(a, b_kmajor, c, offs, acc, stream=stream)


_define_op("hgemm_grouped", "(Tensor a, Tensor b_kmajor, Tensor offs, str acc='fp32') -> Tensor", _hgemm_grouped_shape,
           _hgemm_grouped_launch, " (train through grouped_linear, the same product with a gradient)")


def hgemm_grouped(a: torch.Tensor, b_kmajor: torch.Tensor, offs: torch.Tensor, acc: str = "fp32") -> torch.Tensor:
    """``a`` [T,K] by ``b_kmajor`` [G,N,K] over contiguous row groups -> [T,N]: rows [offs[g-1], offs[g]) of the
    result are those rows of ``a`` times ``b_kmajor[g]^T`` (``torch._grouped_mm(a, b_kmajor.transpose(-2, -1),
    offs=offs)``), in one launch. ``offs``: int32 CUDA tensor [G] of cumulative group ends, read by the kernel (no host
    synchronisation) and clamped to [previous end, T]. Rows at or past ``offs[-1]`` are unspecified. Inference only."""
    return torch.ops.cuda_l2_b200.hgemm_grouped(a, b_kmajor, offs, acc)


# ------------------------------------------------------------------------------------------ grouped backward
#                                                                                            (libb200_grouped_bwd.so)
def _hgemm_grouped_nn_shape(a, b, offs, acc="fp32"):
    _, t, n, _ = capi.check_grouped_nn_operands(a, b, offs, acc)
    return (t, n), a.dtype


def _hgemm_grouped_nn_launch(c, a, b, offs, acc="fp32", *, stream):
    if b.shape[0] == 0 or _empty_product(c, a.shape[1]):   # no group, no element or no reduction
        return
    capi.gemm_grouped_nn(a.contiguous(), b.contiguous(), c, offs.contiguous(), acc, stream=stream)


_define_op("hgemm_grouped_nn", "(Tensor a, Tensor b, Tensor offs, str acc='fp32') -> Tensor", _hgemm_grouped_nn_shape,
           _hgemm_grouped_nn_launch, " (it is a backward kernel: train through grouped_linear)")


def hgemm_grouped_nn(a: torch.Tensor, b: torch.Tensor, offs: torch.Tensor, acc: str = "fp32") -> torch.Tensor:
    """``a`` [T,K] by ``b`` [G,K,N] row-major over contiguous row groups -> [T,N]: rows [offs[g-1], offs[g]) of the
    result are those rows of ``a`` times ``b[g]`` (``torch._grouped_mm(a, b, offs=offs)``), in one launch. ``offs`` as
    for :func:`hgemm_grouped`. Rows at or past ``offs[-1]`` are unspecified. fp16 or bf16, fp32 accumulation."""
    return torch.ops.cuda_l2_b200.hgemm_grouped_nn(a, b, offs, acc)


def _hgemm_grouped_wgrad_shape(a, b, offs, acc="fp32"):
    g, _, m, n = capi.check_grouped_wgrad_operands(a, b, offs, acc)
    return (g, m, n), a.dtype


def _hgemm_grouped_wgrad_launch(c, a, b, offs, acc="fp32", *, stream):
    if c.numel() == 0:
        return
    capi.gemm_grouped_wgrad(a.contiguous(), b.contiguous(), c, offs.contiguous(), acc, stream=stream)


_define_op("hgemm_grouped_wgrad", "(Tensor a, Tensor b, Tensor offs, str acc='fp32') -> Tensor",
           _hgemm_grouped_wgrad_shape, _hgemm_grouped_wgrad_launch,
           " (it is a backward kernel: train through grouped_linear)")


def hgemm_grouped_wgrad(a: torch.Tensor, b: torch.Tensor, offs: torch.Tensor, acc: str = "fp32") -> torch.Tensor:
    """``a`` [T,M] and ``b`` [T,N] over contiguous row groups -> [G,M,N]: matrix g is ``a[start_g:end_g]^T @
    b[start_g:end_g]`` (``torch._grouped_mm(a.t(), b, offs=offs)``), in one launch, with the groups of
    :func:`hgemm_grouped`; an empty group's matrix is zero. fp16 or bf16, fp32 accumulation."""
    return torch.ops.cuda_l2_b200.hgemm_grouped_wgrad(a, b, offs, acc)


def _grouped_linear_shape(x, w, offs, acc="fp32"):
    capi._bwd_variant(x.dtype, acc)   # a product the backward can run
    return _hgemm_grouped_shape(x, w, offs, acc)


def _grouped_input_grad(g, x, w, offs, acc):
    """dX of the grouped product for the contiguous output gradient ``g``: dX[s:e] = dY[s:e] W[g] (W [G, N, K] is a
    row-major B over the reduced N, read in place), into zeros, so that rows at or past the last end stay zero."""
    grad_x = torch.zeros_like(x)
    if x.numel() > 0 and g.shape[1] > 0:   # an empty reduction (N == 0) leaves dX zero
        with torch.cuda.device(x.device):
            capi.gemm_grouped_nn(g, w.contiguous(), grad_x, offs.contiguous(), acc,
                                 stream=torch.cuda.current_stream(x.device).cuda_stream)
    return grad_x


def _grouped_linear_backward(ctx, grad_y):
    x, w, offs = ctx.saved_tensors
    grad_x = grad_w = None
    g = grad_y.contiguous()
    # Y[s:e] = X[s:e] W[g]^T  =>  dX[s:e] = dY[s:e] W[g], dW[g] = dY[s:e]^T X[s:e] (the K-grouped product). Rows of dY at
    # or past the last end are never read.
    if ctx.needs_input_grad[0]:
        grad_x = _grouped_input_grad(g, x, w, offs, ctx.acc)
    if ctx.needs_input_grad[1]:
        grad_w = torch.ops.cuda_l2_b200.hgemm_grouped_wgrad(g, x, offs, ctx.acc)
    return grad_x, grad_w, None, None


def _grouped_linear_setup_context(ctx, inputs, output):
    x, w, offs, acc = inputs
    ctx.acc = acc
    ctx.save_for_backward(x, w, offs)


_define_op("grouped_linear", "(Tensor x, Tensor w, Tensor offs, str acc='fp32') -> Tensor", _grouped_linear_shape,
           _hgemm_grouped_launch, backward=_grouped_linear_backward, setup_context=_grouped_linear_setup_context)


def grouped_linear(x: torch.Tensor, w: torch.Tensor, offs: torch.Tensor, acc: str = "fp32") -> torch.Tensor:
    """The experts of a mixture-of-experts layer with a gradient: ``x`` [T,K] sorted into contiguous groups by the
    int32 cumulative ends ``offs`` [G] (on the GPU), ``w`` [G,N,K] one weight per group -> [T,N], rows [offs[g-1],
    offs[g]) being ``x[rows] @ w[g]^T``. The forward is :func:`hgemm_grouped`'s kernel, bit for bit; the backward
    gives ``dX`` (rows at or past ``offs[-1]`` zero) from :func:`hgemm_grouped_nn` on ``w`` in place and ``dW`` from
    :func:`hgemm_grouped_wgrad`, and never reads rows of the output gradient at or past ``offs[-1]``. Rows of the
    result at or past ``offs[-1]`` are unspecified. fp16 or bf16 with fp32 accumulation."""
    return torch.ops.cuda_l2_b200.grouped_linear(x, w, offs, acc)


# ------------------------------------------------------- fp32 weight-gradient accumulation (libb200_wgrad_accum.so)
def _on_stream(t: torch.Tensor):
    """(device context, torch's current stream handle) for a launch on ``t``'s device."""
    return torch.cuda.device(t.device), torch.cuda.current_stream(t.device).cuda_stream


def grouped_wgrad_accumulate_(main_grad: torch.Tensor, grad_y: torch.Tensor, x: torch.Tensor,
                              offs: torch.Tensor) -> torch.Tensor:
    """``main_grad[g] += grad_y[start_g:end_g]^T @ x[start_g:end_g]`` for every group g, in place, and returns
    ``main_grad``: the weight gradient of :func:`grouped_linear` added into an fp32 buffer [G, N, K] by the epilogue of
    its K-grouped kernel (csrc/b200_wgrad_accum.h). ``grad_y`` [T, N] and ``x`` [T, K] fp16 or bf16, ``offs`` the int32
    group ends [G] on the GPU. Each element gets exactly the fp32 sum that :func:`hgemm_grouped_wgrad` rounds, added
    with one rounding; an empty group's matrix and, with T == 0, all of ``main_grad`` stay as they are, bits included.
    Not an operator and not differentiable: it is the fused layers' backward."""
    g, t, n, k = capi.check_grouped_wgrad_operands(grad_y, x, offs)
    capi.check_main_grad(main_grad, (g, n, k), grad_y.device)
    if main_grad.device.type != "meta":
        ctx, stream = _on_stream(main_grad)
        with ctx:
            capi.wgrad_accum_grouped(grad_y.contiguous(), x.contiguous(), main_grad, offs.contiguous(), stream=stream)
    return main_grad


def wgrad_accumulate_(main_grad: torch.Tensor, grad_y: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """``main_grad += grad_y^T @ x`` in place for a 16-bit linear layer, and returns ``main_grad``: ``grad_y`` [T, N]
    and ``x`` [T, K] fp16 or bf16, ``main_grad`` [N, K] fp32 (the weight's shape). Any token count T; T == 0 changes
    nothing and launches nothing. :func:`grouped_wgrad_accumulate_` with one group, both operands read in place."""
    if grad_y.dim() != 2 or x.dim() != 2:
        raise capi.B200HgemmError(f"wgrad_accumulate_: grad_y [T, N] and x [T, K] expected, got {tuple(grad_y.shape)} "
                                  f"and {tuple(x.shape)}")
    t, n = grad_y.shape
    capi.check_main_grad(main_grad, (n, x.shape[1]), grad_y.device)
    offs = _token_ends(t, 1, grad_y.device) if t > 0 else grad_y.new_empty((1,), dtype=torch.int32)
    grouped_wgrad_accumulate_(main_grad.view(1, *main_grad.shape), grad_y, x, offs)
    return main_grad


def fp8_gemm_accumulate_(c32: torch.Tensor, a: torch.Tensor, b_kmajor: torch.Tensor, scale_a: torch.Tensor,
                         scale_b: torch.Tensor) -> torch.Tensor:
    """``c32 +=`` the e4m3 product :func:`fp8_gemm` computes for ``a`` [M, K] and ``b_kmajor`` [N, K], in place, and
    returns ``c32`` ([M, N] fp32): exactly the fp32 value fp8_gemm rounds to its output is added, with one rounding. The
    scales are rowwise (``scale_a`` [M, 1], ``scale_b`` [1, N]: the weight gradient of rowwise :func:`fp8_linear`) or
    1 x 128 on both operands (``scale_a`` [M, ceil(K/128)], ``scale_b`` [N, ceil(K/128)], in any layout: the blockwise
    one); per-tensor and 128 x 128 scales raise. Not an operator and not differentiable."""
    m, n, k, granularity = capi.check_operands(a, b_kmajor, torch.bfloat16, scales=(scale_a, scale_b))
    if granularity not in capi.WGRAD_ACCUM_FORMS:
        raise capi.B200HgemmError(f"fp8_gemm_accumulate_ takes rowwise or 1 x 128 x 1 x 128 scales, got {granularity}")
    capi.check_main_grad(c32, (m, n), a.device, "c32")
    if c32.device.type != "meta" and m > 0 and k > 0:
        ctx, stream = _on_stream(c32)
        with ctx:
            capi.wgrad_accum_fp8(a.contiguous(), b_kmajor.contiguous(), c32,
                                 *_kernel_scales(granularity, scale_a, scale_b), stream=stream)
    return c32


def _fused_main_grad(weight: torch.Tensor) -> torch.Tensor:
    """``weight.main_grad`` of a layer with ``fuse_wgrad_accumulation``: an fp32 tensor of the weight's shape,
    contiguous, on its device. B200HgemmError naming the rule otherwise."""
    main_grad = getattr(weight, "main_grad", None)
    capi.check_main_grad(main_grad, tuple(weight.shape), weight.device, "weight.main_grad (fuse_wgrad_accumulation)")
    return main_grad


class _LinearWgradAccumFunction(torch.autograd.Function):
    """``hgemm(x2, weight)`` whose backward adds dW into ``weight.main_grad`` (:func:`wgrad_accumulate_`), read when
    the backward runs as Megatron-LM reads it, and returns no gradient for the weight; a frozen weight gets nothing
    added. The forward and dX are the ``hgemm`` operator's, bit for bit."""

    @staticmethod
    def forward(ctx, x2, weight, acc):
        ctx.acc, ctx.weight = acc, weight
        ctx.save_for_backward(x2, weight)
        return torch.ops.cuda_l2_b200.hgemm(x2, weight, acc)

    @staticmethod
    def backward(ctx, grad_y):
        x2, weight = ctx.saved_tensors
        grad_x, _ = _product_grads(x2, weight, grad_y, ctx.needs_input_grad[0], False)
        if ctx.needs_input_grad[1]:
            wgrad_accumulate_(_fused_main_grad(ctx.weight), grad_y.contiguous(), x2)
        return grad_x, None, None


class _GroupedLinearWgradAccumFunction(torch.autograd.Function):
    """:func:`grouped_linear` whose backward adds dW into ``w.main_grad`` (:func:`grouped_wgrad_accumulate_`), read
    when the backward runs, and returns no gradient for the weight stack; a frozen stack gets nothing added. The forward
    and dX are ``grouped_linear``'s, bit for bit."""

    @staticmethod
    def forward(ctx, x, w, offs, acc):
        ctx.acc, ctx.weight = acc, w
        ctx.save_for_backward(x, w, offs)
        return torch.ops.cuda_l2_b200.hgemm_grouped(x, w, offs, acc)

    @staticmethod
    def backward(ctx, grad_y):
        x, w, offs = ctx.saved_tensors
        g = grad_y.contiguous()
        grad_x = _grouped_input_grad(g, x, w, offs, ctx.acc) if ctx.needs_input_grad[0] else None
        if ctx.needs_input_grad[1]:
            grouped_wgrad_accumulate_(_fused_main_grad(ctx.weight), g, x, offs)
        return grad_x, None, None, None


class B200GroupedLinear(nn.Module):
    """Trainable experts of a mixture-of-experts layer: G ``nn.Linear`` weights [N, K] without bias, stacked as the
    Parameter ``weight`` [G, N, K] (fp16 or bf16). ``forward(x, offs)`` takes the tokens sorted by expert, ``x`` [T, K],
    and the int32 cumulative group ends ``offs`` [G] on the GPU, and runs :func:`grouped_linear`: no host
    synchronisation in either direction. Rows at or past ``offs[-1]`` of the result are unspecified. Needs
    K % 8 == 0 and N % 8 == 0.

    ``fuse_wgrad_accumulation=True``: the weight must carry ``weight.main_grad``, an fp32 tensor of its shape (checked
    in forward); the backward adds dW into it (:func:`grouped_wgrad_accumulate_`) and leaves ``weight.grad`` None. y
    and dX are the unfused layer's, bit for bit."""

    def __init__(self, num_groups: int, in_features: int, out_features: int, device=None,
                 dtype: torch.dtype = torch.bfloat16, acc: str = "fp32", fuse_wgrad_accumulation: bool = False):
        super().__init__()
        self._check(num_groups, in_features, out_features, dtype, acc)
        self.num_groups, self.in_features, self.out_features, self.acc = num_groups, in_features, out_features, acc
        self.fuse_wgrad_accumulation = fuse_wgrad_accumulation
        self.weight = nn.Parameter(torch.empty((num_groups, out_features, in_features), device=device, dtype=dtype))
        bound = 1.0 / (in_features ** 0.5)
        with torch.no_grad():
            self.weight.uniform_(-bound, bound)

    @staticmethod
    def _check(g: int, k: int, n: int, dtype: torch.dtype, acc: str) -> None:
        if g < 1 or not linear_supported(k, n, dtype):
            raise capi.B200HgemmError(f"B200GroupedLinear needs G >= 1, fp16 / bf16 and feature counts divisible by 8, "
                                      f"got G={g}, {k}->{n} {dtype}")
        capi._bwd_variant(dtype, acc)

    @classmethod
    def from_weights(cls, w: torch.Tensor, acc: str = "fp32",
                     fuse_wgrad_accumulation: bool = False) -> "B200GroupedLinear":
        """The experts of a weight stack ``w`` [G, N, K] (a Parameter or a tensor), sharing its storage: no copy."""
        if w.dim() != 3:
            raise capi.B200HgemmError(f"from_weights needs a weight stack [G, N, K], got {list(w.shape)}")
        g, n, k = w.shape
        cls._check(g, k, n, w.dtype, acc)
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        new.num_groups, new.in_features, new.out_features, new.acc = g, k, n, acc
        new.fuse_wgrad_accumulation = fuse_wgrad_accumulation
        new.weight = w if isinstance(w, nn.Parameter) else nn.Parameter(w)
        return new

    def forward(self, x: torch.Tensor, offs: torch.Tensor) -> torch.Tensor:
        if self.fuse_wgrad_accumulation:
            _fused_main_grad(self.weight)
            if torch.is_grad_enabled() and (x.requires_grad or self.weight.requires_grad):
                return _GroupedLinearWgradAccumFunction.apply(x, self.weight, offs, self.acc)
        return grouped_linear(x, self.weight, offs, self.acc)

    def extra_repr(self) -> str:
        return (f"num_groups={self.num_groups}, in_features={self.in_features}, out_features={self.out_features}, "
                f"acc={self.acc}" + (", fuse_wgrad_accumulation=True" if self.fuse_wgrad_accumulation else ""))


def linear_supported(in_features: int, out_features: int, dtype: torch.dtype) -> bool:
    t = capi.gemm_type(dtype, dtype)
    return t is not None and t.fits(out_features, in_features)


class B200Linear(nn.Module):
    """``nn.Linear`` whose matmul runs on the H100 HGEMM kernel. The weight keeps ``nn.Linear``'s layout
    ``[out_features, in_features]`` — which IS the kernel's K-major B operand — so swapping a layer copies nothing.

    ``fuse_wgrad_accumulation=True`` (Megatron-LM's gradient-accumulation fusion): the weight must carry
    ``weight.main_grad``, an fp32 tensor of its shape, contiguous, on its device (checked in forward); the backward adds
    dW = dY^T X into it with the K-grouped kernel's epilogue (:func:`wgrad_accumulate_`, any token count) and leaves
    ``weight.grad`` None. y, dX and the bias gradient are the unfused layer's, bit for bit."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, device=None,
                 dtype: torch.dtype = torch.float16, acc: str = "fp32", fuse_wgrad_accumulation: bool = False):
        super().__init__()
        if not linear_supported(in_features, out_features, dtype):
            raise capi.B200HgemmError(f"B200Linear needs fp16/bf16 and feature counts divisible by 8, got "
                                      f"{in_features}->{out_features} {dtype}")
        self.in_features, self.out_features, self.acc = in_features, out_features, acc
        self.fuse_wgrad_accumulation = fuse_wgrad_accumulation
        self.weight = nn.Parameter(torch.empty((out_features, in_features), device=device, dtype=dtype))
        self.bias = nn.Parameter(torch.empty(out_features, device=device, dtype=dtype)) if bias else None
        self.reset_parameters()

    def reset_parameters(self) -> None:
        bound = 1.0 / (self.in_features ** 0.5)
        with torch.no_grad():
            self.weight.uniform_(-bound, bound)
            if self.bias is not None:
                self.bias.uniform_(-bound, bound)

    @classmethod
    def from_linear(cls, lin: nn.Linear, acc: str = "fp32", fuse_wgrad_accumulation: bool = False) -> "B200Linear":
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        if not linear_supported(lin.in_features, lin.out_features, lin.weight.dtype):
            raise capi.B200HgemmError(f"cannot convert {lin}: needs fp16/bf16 weights and feature counts divisible by 8")
        new.in_features, new.out_features, new.acc = lin.in_features, lin.out_features, acc
        new.fuse_wgrad_accumulation = fuse_wgrad_accumulation
        new.weight, new.bias = lin.weight, lin.bias          # shared storage, no copy
        return new

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        lead = x.shape[:-1]
        x2 = x.reshape(-1, self.in_features)
        fused = False
        if self.fuse_wgrad_accumulation:
            _fused_main_grad(self.weight)
            fused = torch.is_grad_enabled() and (x.requires_grad or self.weight.requires_grad)
        if fused:
            y = _LinearWgradAccumFunction.apply(x2, self.weight, self.acc)
        else:
            y = torch.ops.cuda_l2_b200.hgemm(x2, self.weight, self.acc)
        if self.bias is not None:
            y = y + self.bias
        return y.view(*lead, self.out_features)

    def extra_repr(self) -> str:
        fused = ", fuse_wgrad_accumulation=True" if self.fuse_wgrad_accumulation else ""
        return (f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, "
                f"acc={self.acc}{fused}")


# ------------------------------------------------------------------------------------------ SwiGLU (libb200_swiglu.so)
def interleave_gate_up(w_gate: torch.Tensor, w_up: torch.Tensor) -> torch.Tensor:
    """The fused gate / up weight ``w_gu`` [2I, H] of a SwiGLU MLP from its gate and up weights [I, H] (a copy): rows
    [128 b, 128 b + 64) are gate rows [64 b, 64 b + 64), rows [128 b + 64, 128 b + 128) the matching up rows. I must be
    a multiple of 64. An expert stack ([G, I, H] each) gives [G, 2I, H], every expert's matrix interleaved so."""
    if w_gate.dim() == 3:
        if w_gate.shape != w_up.shape or w_gate.shape[1] % capi.SWIGLU_BLOCK:
            raise capi.B200HgemmError(f"gate and up expert stacks must both be [G, I, H] with I % {capi.SWIGLU_BLOCK} "
                                      f"== 0, got {tuple(w_gate.shape)} and {tuple(w_up.shape)}")
    elif w_gate.dim() != 2 or w_gate.shape != w_up.shape or w_gate.shape[0] % capi.SWIGLU_BLOCK:
        raise capi.B200HgemmError(f"gate and up weights must both be [I, H] with I % {capi.SWIGLU_BLOCK} == 0, got "
                                  f"{tuple(w_gate.shape)} and {tuple(w_up.shape)}")
    lead, (i, h) = w_gate.shape[:-2], w_gate.shape[-2:]
    blk = capi.SWIGLU_BLOCK
    return torch.stack((w_gate.reshape(*lead, i // blk, blk, h), w_up.reshape(*lead, i // blk, blk, h)),
                       dim=-3).reshape(*lead, 2 * i, h)


def split_gate_up(w_gu: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """``(w_gate, w_up)``, each [I, H], of a fused gate / up weight ``w_gu`` [2I, H] (copies): the inverse of
    :func:`interleave_gate_up`. An expert stack [G, 2I, H] gives two stacks [G, I, H]."""
    blk = capi.SWIGLU_BLOCK
    if w_gu.dim() == 3:
        if w_gu.shape[1] % (2 * blk):
            raise capi.B200HgemmError(f"w_gu expert stack must be [G, 2I, H] with I % {blk} == 0, got {tuple(w_gu.shape)}")
    elif w_gu.dim() != 2 or w_gu.shape[0] % (2 * blk):
        raise capi.B200HgemmError(f"w_gu must be [2I, H] with I % {blk} == 0, got {tuple(w_gu.shape)}")
    lead, (n, h) = w_gu.shape[:-2], w_gu.shape[-2:]
    v = w_gu.reshape(*lead, n // (2 * blk), 2, blk, h)
    return tuple(v.select(-3, j).clone(memory_format=torch.contiguous_format).view(*lead, n // 2, h) for j in (0, 1))


def _swiglu_forward(x2: torch.Tensor, w_gu: torch.Tensor, want_h: bool):
    """(y [M, I], h [M, 2I] or None) of the fused gate / up product of ``x2`` [M, H]: one launch of libb200_swiglu.so.
    M == 0 launches nothing, and K == 0 makes y (and h) zero, as :func:`_empty_product` does for the products."""
    m, i, k = capi.check_swiglu_operands(x2, w_gu)
    if not x2.is_cuda or not w_gu.is_cuda:
        raise capi.B200HgemmError("swiglu_linear has no CPU implementation (and no fallback): move the tensors to an H100")
    y = torch.empty((m, i), dtype=x2.dtype, device=x2.device)
    h = torch.empty((m, 2 * i), dtype=x2.dtype, device=x2.device) if want_h else None
    if m == 0:
        return y, h
    if k == 0:   # h = 0, so y = silu(0) * 0 = +0
        y.zero_()
        if h is not None:
            h.zero_()
        return y, h
    with torch.cuda.device(x2.device):
        capi.swiglu(x2.contiguous(), w_gu.contiguous(), y, h, stream=torch.cuda.current_stream(x2.device).cuda_stream)
    return y, h


class _SwiGLULinearFunction(torch.autograd.Function):
    """y = silu(g) * u of h = x2 w_gu^T, saving x2, w_gu and h (not silu(g)). The backward is one pass of
    libb200_swiglu.so's SwiGLU gradient (dh from dy and h), then dX and dW of the product through
    :func:`_product_grads` (any token count)."""

    @staticmethod
    def forward(ctx, x2, w_gu):
        x2, w_gu = x2.contiguous(), w_gu.contiguous()
        y, h = _swiglu_forward(x2, w_gu, True)
        ctx.save_for_backward(x2, w_gu, h)
        return y

    @staticmethod
    def backward(ctx, grad_y):
        x2, w_gu, h = ctx.saved_tensors
        dh = torch.empty_like(h)
        if dh.numel():
            with torch.cuda.device(h.device):
                capi.swiglu_backward(grad_y.contiguous(), h, dh, stream=torch.cuda.current_stream(h.device).cuda_stream)
        return _product_grads(x2, w_gu, dh, ctx.needs_input_grad[0], ctx.needs_input_grad[1])


def swiglu_linear(x: torch.Tensor, w_gu: torch.Tensor) -> torch.Tensor:
    """``F.silu(x @ W_gate^T) * (x @ W_up^T)`` for ``x`` [..., H] and the fused weight ``w_gu`` [2I, H]
    (:func:`interleave_gate_up`), as one GEMM whose epilogue applies the SwiGLU: fp16 or bf16 with fp32 accumulation,
    y [..., I] bit for bit torch's ``F.silu(g) * u`` on the 16-bit gate / up product. Differentiable in ``x`` and
    ``w_gu``; without a gradient to compute, h is never written. No host synchronisation in either direction, so a
    training step can be captured in a CUDA graph. I % 64 == 0 and H % 8 == 0."""
    lead = x.shape[:-1]
    x2 = x.reshape(lead.numel(), x.shape[-1])   # explicit rows: -1 is ambiguous when H == 0
    if torch.is_grad_enabled() and (x.requires_grad or w_gu.requires_grad):
        y = _SwiGLULinearFunction.apply(x2, w_gu)
    else:
        y, _ = _swiglu_forward(x2, w_gu, False)
    return y.view(*lead, y.shape[-1])


class B200SwiGLULinear(nn.Module):
    """The gate and up projections of a SwiGLU MLP (Llama, Mistral, Qwen) with the activation, as one layer:
    ``forward(x) = F.silu(gate_proj(x)) * up_proj(x)`` through :func:`swiglu_linear`. The Parameter ``weight`` is the
    fused ``w_gu`` [2I, H], gate and up rows interleaved in blocks of 64 (:func:`interleave_gate_up`,
    :func:`split_gate_up`). No bias. fp16 or bf16; I % 64 == 0 and H % 8 == 0."""

    def __init__(self, in_features: int, intermediate_features: int, device=None, dtype: torch.dtype = torch.bfloat16):
        super().__init__()
        self._check(in_features, intermediate_features, dtype)
        self.in_features, self.intermediate_features = in_features, intermediate_features
        self.weight = nn.Parameter(torch.empty((2 * intermediate_features, in_features), device=device, dtype=dtype))
        bound = 1.0 / (in_features ** 0.5)
        with torch.no_grad():
            self.weight.uniform_(-bound, bound)

    @staticmethod
    def _check(h: int, i: int, dtype: torch.dtype) -> None:
        if dtype not in (torch.float16, torch.bfloat16) or h <= 0 or h % 8 or i <= 0 or i % capi.SWIGLU_BLOCK:
            raise capi.B200HgemmError(f"B200SwiGLULinear needs fp16 / bf16, in_features % 8 == 0 and "
                                      f"intermediate_features % {capi.SWIGLU_BLOCK} == 0, got {h} -> {i} {dtype}")

    @classmethod
    def from_linears(cls, gate_proj: nn.Linear, up_proj: nn.Linear) -> "B200SwiGLULinear":
        """The layer of two bias-free ``nn.Linear`` projections H -> I of one dtype and device, their weights
        interleaved into a new Parameter (a copy)."""
        if gate_proj.bias is not None or up_proj.bias is not None:
            raise capi.B200HgemmError("from_linears needs bias-free gate and up projections (a SwiGLU MLP has none)")
        wg, wu = gate_proj.weight, up_proj.weight
        if wg.shape != wu.shape or wg.dtype != wu.dtype or wg.device != wu.device:
            raise capi.B200HgemmError(f"gate and up projections must match in shape, dtype and device, got "
                                      f"{tuple(wg.shape)} {wg.dtype} {wg.device} and {tuple(wu.shape)} {wu.dtype} "
                                      f"{wu.device}")
        i, h = wg.shape
        cls._check(h, i, wg.dtype)
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        new.in_features, new.intermediate_features = h, i
        with torch.no_grad():
            new.weight = nn.Parameter(interleave_gate_up(wg, wu), requires_grad=wg.requires_grad or wu.requires_grad)
        return new

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return swiglu_linear(x, self.weight)

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, intermediate_features={self.intermediate_features}"


# ------------------------------------------------------------------ grouped SwiGLU (libb200_grouped_swiglu.so)
def _grouped_swiglu_forward(x: torch.Tensor, w_gu: torch.Tensor, offs: torch.Tensor, want_h: bool):
    """(y [T, I], h [T, 2I] or None) of the fused grouped gate / up product of ``x`` [T, H] by the expert stack ``w_gu``
    [G, 2I, H]: one launch of libb200_grouped_swiglu.so. T == 0 launches nothing, and H == 0 makes y (and h) zero, as
    :func:`_swiglu_forward` does."""
    _, t, i, k = capi.check_grouped_swiglu_operands(x, w_gu, offs)
    if not x.is_cuda or not w_gu.is_cuda or not offs.is_cuda:
        raise capi.B200HgemmError("grouped_swiglu_linear has no CPU implementation (and no fallback): move the tensors "
                                  "to an H100")
    y = torch.empty((t, i), dtype=x.dtype, device=x.device)
    h = torch.empty((t, 2 * i), dtype=x.dtype, device=x.device) if want_h else None
    if t == 0:
        return y, h
    if k == 0:   # h = 0, so y = silu(0) * 0 = +0
        y.zero_()
        if h is not None:
            h.zero_()
        return y, h
    with torch.cuda.device(x.device):
        capi.grouped_swiglu(x.contiguous(), w_gu.contiguous(), offs.contiguous(), y, h,
                            stream=torch.cuda.current_stream(x.device).cuda_stream)
    return y, h


class _GroupedSwiGLULinearFunction(torch.autograd.Function):
    """y = silu(g) * u of the grouped product h = x w_gu[g]^T per group, saving x, w_gu, offs and h. The backward is one
    pass of libb200_grouped_swiglu.so's SwiGLU gradient over the groups' rows (dh from dy and h), then dX from
    :func:`_grouped_input_grad` (zero past the last end) and dW [G, 2I, H] from :func:`hgemm_grouped_wgrad`. Rows of dy
    at or past the last end are never read. No host synchronisation."""

    @staticmethod
    def forward(ctx, x, w_gu, offs):
        x, w_gu, offs = x.contiguous(), w_gu.contiguous(), offs.contiguous()
        y, h = _grouped_swiglu_forward(x, w_gu, offs, True)
        ctx.save_for_backward(x, w_gu, offs, h)
        return y

    @staticmethod
    def backward(ctx, grad_y):
        x, w_gu, offs, h = ctx.saved_tensors
        dh = torch.empty_like(h)
        if dh.numel():
            with torch.cuda.device(h.device):
                capi.grouped_swiglu_backward(grad_y.contiguous(), h, dh, offs,
                                             stream=torch.cuda.current_stream(h.device).cuda_stream)
        grad_x = _grouped_input_grad(dh, x, w_gu, offs, "fp32") if ctx.needs_input_grad[0] else None
        grad_w = None
        if ctx.needs_input_grad[1]:
            grad_w = torch.ops.cuda_l2_b200.hgemm_grouped_wgrad(dh, x, offs, "fp32")
        return grad_x, grad_w, None


def grouped_swiglu_linear(x: torch.Tensor, w_gu: torch.Tensor, offs: torch.Tensor) -> torch.Tensor:
    """The gate and up projections of SwiGLU experts with the activation: ``x`` [T, H] sorted into contiguous groups by
    the int32 cumulative ends ``offs`` [G] (on the GPU), ``w_gu`` [G, 2I, H] one fused gate / up weight per expert
    (:func:`interleave_gate_up` of expert stacks) -> y [T, I], rows [offs[g-1], offs[g]) being ``F.silu(x[rows] @
    W_gate[g]^T) * (x[rows] @ W_up[g]^T)``, as one grouped GEMM whose epilogue applies the SwiGLU: fp16 or bf16 with
    fp32 accumulation, bit for bit torch's ``F.silu(g) * u`` on the 16-bit grouped product. Rows at or past
    ``offs[-1]`` are unspecified. Differentiable in ``x`` and ``w_gu``; without a gradient to compute, h is never
    written. The backward never reads rows of the output gradient at or past ``offs[-1]`` and gives dX zero there. No
    host synchronisation in either direction, so a training step can be captured in a CUDA graph with the offsets
    changing between replays. I % 64 == 0 and H % 8 == 0."""
    if torch.is_grad_enabled() and (x.requires_grad or w_gu.requires_grad):
        return _GroupedSwiGLULinearFunction.apply(x, w_gu, offs)
    y, _ = _grouped_swiglu_forward(x, w_gu, offs, False)
    return y


class B200GroupedSwiGLULinear(nn.Module):
    """The gate and up projections of the SwiGLU experts of a mixture-of-experts layer (Mixtral, Qwen-MoE, DeepSeek)
    with the activation, as one layer: ``forward(x, offs)`` takes the tokens sorted by expert, ``x`` [T, H], and the
    int32 cumulative group ends ``offs`` [G] on the GPU, and runs :func:`grouped_swiglu_linear`. The Parameter
    ``weight`` is the expert stack ``w_gu`` [G, 2I, H], each expert's gate and up rows interleaved in blocks of 64
    (:func:`interleave_gate_up`, :func:`split_gate_up`). Rows at or past ``offs[-1]`` of the result are unspecified.
    No bias. fp16 or bf16; I % 64 == 0 and H % 8 == 0."""

    def __init__(self, num_groups: int, in_features: int, intermediate_features: int, device=None,
                 dtype: torch.dtype = torch.bfloat16):
        super().__init__()
        self._check(num_groups, in_features, intermediate_features, dtype)
        self.num_groups, self.in_features, self.intermediate_features = num_groups, in_features, intermediate_features
        self.weight = nn.Parameter(torch.empty((num_groups, 2 * intermediate_features, in_features), device=device,
                                               dtype=dtype))
        bound = 1.0 / (in_features ** 0.5)
        with torch.no_grad():
            self.weight.uniform_(-bound, bound)

    @staticmethod
    def _check(g: int, h: int, i: int, dtype: torch.dtype) -> None:
        if g < 1 or dtype not in (torch.float16, torch.bfloat16) or h <= 0 or h % 8 or i <= 0 or \
                i % capi.SWIGLU_BLOCK:
            raise capi.B200HgemmError(f"B200GroupedSwiGLULinear needs G >= 1, fp16 / bf16, in_features % 8 == 0 and "
                                      f"intermediate_features % {capi.SWIGLU_BLOCK} == 0, got G={g}, {h} -> {i} {dtype}")

    @classmethod
    def from_weights(cls, w_gate: torch.Tensor, w_up: torch.Tensor) -> "B200GroupedSwiGLULinear":
        """The layer of the expert stacks ``w_gate`` and ``w_up`` [G, I, H] of one dtype and device, interleaved into a
        new, trainable Parameter (a copy), as :meth:`B200GroupedLinear.from_weights` makes one. A vLLM-style ``w13``
        [G, 2I, H] (gate rows first) is ``from_weights(w13[:, :I], w13[:, I:])``."""
        if w_gate.dim() != 3 or w_gate.shape != w_up.shape or w_gate.dtype != w_up.dtype or \
                w_gate.device != w_up.device:
            raise capi.B200HgemmError(f"gate and up stacks must both be [G, I, H] of one dtype and device, got "
                                      f"{tuple(w_gate.shape)} {w_gate.dtype} {w_gate.device} and {tuple(w_up.shape)} "
                                      f"{w_up.dtype} {w_up.device}")
        g, i, h = w_gate.shape
        cls._check(g, h, i, w_gate.dtype)
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        new.num_groups, new.in_features, new.intermediate_features = g, h, i
        with torch.no_grad():
            new.weight = nn.Parameter(interleave_gate_up(w_gate, w_up))
        return new

    def forward(self, x: torch.Tensor, offs: torch.Tensor) -> torch.Tensor:
        return grouped_swiglu_linear(x, self.weight, offs)

    def extra_repr(self) -> str:
        return (f"num_groups={self.num_groups}, in_features={self.in_features}, "
                f"intermediate_features={self.intermediate_features}")


def replace_linear_modules(model: nn.Module, acc: str = "fp32", skip: tuple[str, ...] = ()) -> list[str]:
    """Swap every eligible ``nn.Linear`` of ``model`` (fp16/bf16 weights, features divisible by 8) for a
    :class:`B200Linear` sharing its parameters. Returns the qualified names that were replaced."""
    done = []
    for name, mod in list(model.named_modules()):
        for child_name, child in list(mod.named_children()):
            full = f"{name}.{child_name}" if name else child_name
            if type(child) is nn.Linear and full not in skip and \
                    linear_supported(child.in_features, child.out_features, child.weight.dtype):
                setattr(mod, child_name, B200Linear.from_linear(child, acc))
                done.append(full)
    return done


# ------------------------------------------------------------------------ bias + activation epilogue (libb200_epilogue.so)
def _activate(z: torch.Tensor, activation: str) -> torch.Tensor:
    if activation == "relu":
        return torch.relu(z)
    if activation == "gelu_tanh":
        return torch.nn.functional.gelu(z, approximate="tanh")
    return z


def _bias_act_empty(c: torch.Tensor, k: int, bias, activation: str) -> bool:
    """Whether the fused product into ``c`` needs no kernel: ``c`` has no element (M or N == 0), or the reduction is
    empty (K == 0), which makes ``c`` act(bias) broadcast over the rows (act(0) without a bias), rounded once, as
    ``addmm`` with an empty reduction gives. The C ABI rejects both with kBadShape."""
    if c.numel() == 0:
        return True
    if k == 0:
        z = torch.zeros(c.shape[1], dtype=torch.float32, device=c.device)
        if bias is not None:
            z = z + bias.float()
        c.copy_(_activate(z, activation).expand_as(c))
        return True
    return False


def _hgemm_bias_act_shape(a, b_kmajor, bias, activation="none"):
    m, n, k, _ = capi.check_operands(a, b_kmajor, a.dtype, "fp32")
    capi.epilogue_variant(a.dtype, a.dtype)
    capi.check_bias(bias, n, a.dtype)
    capi.activation_code(activation)
    return (m, n), a.dtype


def _hgemm_bias_act_launch(c, a, b_kmajor, bias=None, activation="none", *, stream):
    if not _bias_act_empty(c, a.shape[1], bias, activation):
        capi.gemm_bias_act(a.contiguous(), b_kmajor.contiguous(), c, bias, activation, stream=stream)


def _hgemm_bias_act_backward(ctx, grad_y):
    a, b_kmajor, bias, y = ctx.saved_tensors
    # dZ, the gradient at the pre-activation z = A Bt^T + bias: relu's mask from the saved output (y > 0 exactly where
    # z > 0 survived the rounding); gelu_tanh's derivative at z recomputed by the same kernel without the activation,
    # so that the forward saves no pre-activation tensor.
    if ctx.activation == "relu":
        grad_z = grad_y * (y > 0)
    elif ctx.activation == "gelu_tanh":
        z = torch.ops.cuda_l2_b200.hgemm_bias_act(a, b_kmajor, bias, "none")
        grad_z = torch.ops.aten.gelu_backward(grad_y, z, approximate="tanh")
    else:
        grad_z = grad_y
    grad_a, grad_b = _product_grads(a, b_kmajor, grad_z, ctx.needs_input_grad[0], ctx.needs_input_grad[1])
    grad_bias = None
    if bias is not None and ctx.needs_input_grad[2]:
        grad_bias = grad_z.sum(0, dtype=torch.float32).to(bias.dtype)
    return grad_a, grad_b, grad_bias, None


def _hgemm_bias_act_setup_context(ctx, inputs, output):
    a, b_kmajor, bias, activation = inputs
    ctx.activation = activation
    ctx.save_for_backward(a, b_kmajor, bias, output if activation == "relu" else None)


_define_op("hgemm_bias_act", "(Tensor a, Tensor b_kmajor, Tensor? bias, str activation='none') -> Tensor",
           _hgemm_bias_act_shape, _hgemm_bias_act_launch, backward=_hgemm_bias_act_backward,
           setup_context=_hgemm_bias_act_setup_context)


def hgemm_bias_act(a: torch.Tensor, b_kmajor: torch.Tensor, bias: torch.Tensor | None = None,
                   activation: str = "none") -> torch.Tensor:
    """act(``a`` [M,K] @ ``b_kmajor`` [N,K]^T + ``bias``) -> [M,N] in one launch, fp32 until one rounding (see the
    module docstring)."""
    return torch.ops.cuda_l2_b200.hgemm_bias_act(a, b_kmajor, bias, activation)


def linear(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None = None,
           activation: str = "none") -> torch.Tensor:
    """``act(F.linear(x, weight, bias))`` for ``x`` [..., in_features] and ``weight`` [out_features, in_features]
    (``F.linear``'s shapes), one fused launch of :func:`hgemm_bias_act`, with a gradient."""
    if x.dim() == 0 or weight.dim() != 2:
        raise capi.B200HgemmError(f"linear: x [..., in_features] and weight [out_features, in_features] expected, got "
                                  f"{tuple(x.shape)} and {tuple(weight.shape)}")
    y = torch.ops.cuda_l2_b200.hgemm_bias_act(x.reshape(-1, x.shape[-1]), weight, bias, activation)
    return y.view(*x.shape[:-1], weight.shape[0])


# ------------------------------------------------------------------------------------------ FP8 (e4m3), inference only
E4M3_MAX = 448.0   # largest finite float8_e4m3fn value

def _kernel_scales(granularity: str, scale_a: torch.Tensor, scale_b: torch.Tensor):
    """Scales of ``granularity`` (what :func:`capi.scale_granularity` found) as the kernels read them, copied only
    where they are not laid out so: per-tensor scales one contiguous element each; a blockwise ``scale_a``, and a
    1 x 128 ``scale_b``, M-major (:func:`capi.m_major`); rowwise vectors and the block scales of Bt contiguous and
    16-byte aligned."""
    if granularity == "tensor":
        return scale_a.reshape(1).contiguous(), scale_b.reshape(1).contiguous()
    if granularity == "rowwise":
        return capi._aligned(scale_a), capi._aligned(scale_b)
    return capi.m_major(scale_a), (capi.m_major(scale_b) if granularity == "blockwise_1d1d" else
                                   capi._aligned(scale_b))


def _fp8_gemm_shape(a, b_kmajor, scale_a, scale_b, out_dtype):
    m, n, _, granularity = capi.check_operands(a, b_kmajor, out_dtype, scales=(scale_a, scale_b))
    return (m, n), out_dtype, granularity


def _fp8_gemm_launch(c, a, b_kmajor, scale_a, scale_b, out_dtype, granularity, *, stream):
    if c.shape[0] > 0:
        capi.fp8_gemm(a.contiguous(), b_kmajor.contiguous(), c, *_kernel_scales(granularity, scale_a, scale_b),
                      stream=stream)


_define_op("fp8_gemm", "(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, ScalarType out_dtype) -> Tensor",
           _fp8_gemm_shape, _fp8_gemm_launch,
           " (train with the fp16 / bf16 operator and quantise afterwards)")


def fp8_gemm(a: torch.Tensor, b_kmajor: torch.Tensor, scale_a: torch.Tensor, scale_b: torch.Tensor,
             out_dtype: torch.dtype = torch.float16) -> torch.Tensor:
    """(``a`` [M,K] @ ``b_kmajor`` [N,K]^T), scaled, -> [M,N] ``out_dtype``, e4m3 operands (see the module docstring).
    Per-tensor scales: one element each. Rowwise scales: ``scale_a`` [M,1], ``scale_b`` [1,N]. Blockwise scales:
    ``scale_a`` [M, ceil(K/128)] in any layout, ``scale_b`` [ceil(N/128), ceil(K/128)]. 1 x 128 scales on both
    operands (the weight gradient of blockwise FP8 training): ``scale_a`` [M, ceil(K/128)] and ``scale_b``
    [N, ceil(K/128)], each in any layout (the M-major one of :func:`quantize_e4m3_blockwise` is read in place)."""
    return torch.ops.cuda_l2_b200.fp8_gemm(a, b_kmajor, scale_a, scale_b, out_dtype)


def _fp8_bias_act_shape(a, b_kmajor, scale_a, scale_b, bias, activation, out_dtype):
    m, n, _, granularity = capi.check_operands(a, b_kmajor, out_dtype, scales=(scale_a, scale_b))
    if granularity in ("blockwise", "blockwise_1d1d"):
        raise capi.B200HgemmError("fp8_gemm_bias_act: blockwise scales have no bias + activation kernel (per-tensor or "
                                  "rowwise scales only; run fp8_gemm and add the bias)")
    capi.check_bias(bias, n, out_dtype)
    capi.activation_code(activation)
    return (m, n), out_dtype, granularity


def _fp8_bias_act_launch(c, a, b_kmajor, scale_a, scale_b, bias, activation, out_dtype, granularity, *, stream):
    if not _bias_act_empty(c, a.shape[1], bias, activation):
        capi.gemm_bias_act(a.contiguous(), b_kmajor.contiguous(), c, bias, activation,
                           *_kernel_scales(granularity, scale_a, scale_b), stream=stream)


_define_op("fp8_gemm_bias_act",
           "(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, Tensor? bias, str activation, "
           "ScalarType out_dtype) -> Tensor",
           _fp8_bias_act_shape, _fp8_bias_act_launch,
           " (train with the fp16 / bf16 operator hgemm_bias_act and quantise afterwards)")


def fp8_gemm_bias_act(a: torch.Tensor, b_kmajor: torch.Tensor, scale_a: torch.Tensor, scale_b: torch.Tensor,
                      bias: torch.Tensor | None = None, activation: str = "none",
                      out_dtype: torch.dtype = torch.float16) -> torch.Tensor:
    """act((``a`` @ ``b_kmajor``^T) scaled + ``bias``) -> [M,N] ``out_dtype``, e4m3 operands with per-tensor or rowwise
    scales (as :func:`fp8_gemm`), in one launch."""
    return torch.ops.cuda_l2_b200.fp8_gemm_bias_act(a, b_kmajor, scale_a, scale_b, bias, activation, out_dtype)


# ------------------------------------------------------------------------------------------ e4m3 quantisers of
#                                                                                            activations (libb200_quant.so)
# Each quantiser has a torch composition, the ``*_reference`` function, and an operator that runs the one-pass kernel
# of libb200_quant.so with the reference's bits on CUDA (csrc/b200_quant.h). The public function routes a non-empty
# CUDA tensor of a dtype a kernel takes to the operator and anything else (CPU tensors in particular) to the reference.
def quantize_e4m3_reference(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """:func:`quantize_e4m3` as a composition of torch ops."""
    scale = (x.abs().amax().float() / E4M3_MAX).clamp_min(torch.finfo(torch.float32).tiny).reshape(1)
    q = (x.float() / scale).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q, scale


def quantize_e4m3_rowwise_reference(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """:func:`quantize_e4m3_rowwise` as a composition of torch ops."""
    scale = (x.abs().amax(dim=1, keepdim=True).float() / E4M3_MAX).clamp_min(torch.finfo(torch.float32).tiny)
    q = (x.float() / scale).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q, scale


def quantize_e4m3_blockwise_reference(x: torch.Tensor, masked_m: torch.Tensor | None = None
                                      ) -> tuple[torch.Tensor, torch.Tensor]:
    """:func:`quantize_e4m3_blockwise` as a composition of torch ops. ``masked_m`` changes nothing here: every row is
    computed."""
    if x.dim() not in (2, 3):
        raise capi.B200HgemmError(f"quantize_e4m3_blockwise takes [M, K] or [B, M, K], got {list(x.shape)}")
    *lead, m, k = x.shape
    nkb = capi.num_k_blocks(k)
    xb = nn.functional.pad(x.float(), (0, nkb * capi.BLOCK - k)).view(*lead, m, nkb, capi.BLOCK)
    scale = (xb.abs().amax(dim=-1) / E4M3_MAX).clamp_min(torch.finfo(torch.float32).tiny)
    q = (xb / scale[..., None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(*lead, m, nkb * capi.BLOCK)
    return q[..., :k].contiguous(), capi.empty_m_major(lead, m, nkb, x.device).copy_(scale)


def silu_mul_quantize_e4m3_blockwise_reference(h: torch.Tensor, masked_m: torch.Tensor | None = None
                                               ) -> tuple[torch.Tensor, torch.Tensor]:
    """:func:`silu_mul_quantize_e4m3_blockwise` as a composition of torch ops: ``F.silu(g) * u``, then
    :func:`quantize_e4m3_blockwise_reference`. ``masked_m`` changes nothing here."""
    i = _swiglu_width(h)
    return quantize_e4m3_blockwise_reference(nn.functional.silu(h[..., :i]) * h[..., i:])


def _swiglu_width(h: torch.Tensor) -> int:
    """I of a SwiGLU input h [(B,) M, 2I]; B200HgemmError for any other shape."""
    if h.dim() not in (2, 3) or h.shape[-1] % 2:
        raise capi.B200HgemmError(f"h must be [M, 2I] or [B, M, 2I], got {list(h.shape)}")
    return h.shape[-1] // 2


def _quant_routed(x: torch.Tensor, silu_mul: bool = False) -> bool:
    """Whether a quantiser of libb200_quant.so runs on ``x``: a non-empty CUDA tensor of a dtype it takes."""
    return x.is_cuda and x.numel() > 0 and capi.quant_dtype(x.dtype, silu_mul) is not None


def _quant_input(x: torch.Tensor, silu_mul: bool = False) -> None:
    if capi.quant_dtype(x.dtype, silu_mul) is None:
        raise capi.B200HgemmError(f"no e4m3 quantiser for {x.dtype} input (fp16, bf16{'' if silu_mul else ', fp32'})")
    if x.numel() == 0:
        raise capi.B200HgemmError(f"the e4m3 quantisers take non-empty inputs, got {list(x.shape)}")


def _check_masked_m(masked_m, bsz: int) -> None:
    if masked_m is not None and (masked_m.dtype != torch.int32 or tuple(masked_m.shape) != (bsz,)):
        raise capi.B200HgemmError(f"masked_m must be an int32 tensor of shape [{bsz}], got {masked_m.dtype} "
                                  f"{tuple(masked_m.shape)}")


def _quantize_e4m3_outputs(x):
    _quant_input(x)
    return x.new_empty(x.shape, dtype=torch.float8_e4m3fn), x.new_empty((1,), dtype=torch.float32)


def _quantize_e4m3_launch(out, x, *, stream):
    workspace = torch.empty(capi.QUANT_TENSOR_WORKSPACE, dtype=torch.float32, device=x.device)
    capi.quantize_e4m3(x.contiguous(), *out, workspace, stream=stream)


def _quantize_e4m3_rowwise_outputs(x):
    _quant_input(x)
    if x.dim() != 2:
        raise capi.B200HgemmError(f"quantize_e4m3_rowwise takes [rows, cols], got {list(x.shape)}")
    return x.new_empty(x.shape, dtype=torch.float8_e4m3fn), x.new_empty((x.shape[0], 1), dtype=torch.float32)


def _quantize_e4m3_rowwise_launch(out, x, *, stream):
    capi.quantize_e4m3_rowwise(x.contiguous(), *out, stream=stream)


def _blockwise_outputs(x, k: int, masked_m):
    *lead, m, _ = x.shape
    _check_masked_m(masked_m, lead[0] if lead else 1)
    return (x.new_empty((*lead, m, k), dtype=torch.float8_e4m3fn),
            capi.empty_m_major(lead, m, capi.num_k_blocks(k), x.device))


def _quantize_e4m3_blockwise_outputs(x, masked_m=None):
    _quant_input(x)
    if x.dim() not in (2, 3):
        raise capi.B200HgemmError(f"quantize_e4m3_blockwise takes [M, K] or [B, M, K], got {list(x.shape)}")
    return _blockwise_outputs(x, x.shape[-1], masked_m)


def _quantize_e4m3_blockwise_launch(out, x, masked_m=None, *, stream):
    capi.quantize_e4m3_blockwise(x.contiguous(), *out, None if masked_m is None else masked_m.contiguous(),
                                 stream=stream)


def _silu_mul_outputs(h, masked_m=None):
    _quant_input(h, silu_mul=True)
    return _blockwise_outputs(h, _swiglu_width(h), masked_m)


def _silu_mul_launch(out, h, masked_m=None, *, stream):
    capi.silu_mul_quantize_e4m3_blockwise(h.contiguous(), *out, None if masked_m is None else masked_m.contiguous(),
                                          stream=stream)


_QUANT_WHY = " (quantisation is not differentiable: train the 16-bit model and quantise afterwards)"
_define_op("quantize_e4m3", "(Tensor x) -> (Tensor, Tensor)", None, _quantize_e4m3_launch, _QUANT_WHY,
           outputs=_quantize_e4m3_outputs)
_define_op("quantize_e4m3_rowwise", "(Tensor x) -> (Tensor, Tensor)", None, _quantize_e4m3_rowwise_launch,
           _QUANT_WHY, outputs=_quantize_e4m3_rowwise_outputs)
_define_op("quantize_e4m3_blockwise", "(Tensor x, Tensor? masked_m=None) -> (Tensor, Tensor)", None,
           _quantize_e4m3_blockwise_launch, _QUANT_WHY, outputs=_quantize_e4m3_blockwise_outputs)
_define_op("silu_mul_quantize_e4m3_blockwise", "(Tensor h, Tensor? masked_m=None) -> (Tensor, Tensor)", None,
           _silu_mul_launch, _QUANT_WHY, outputs=_silu_mul_outputs)


def quantize_e4m3(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Per-tensor quantisation on x's device: scale = amax(|x|) / 448 (a one-element fp32 tensor), q = e4m3(x / scale).
    No host synchronisation. A CUDA fp16 / bf16 / fp32 tensor runs ``cuda_l2_b200::quantize_e4m3`` (two launches),
    anything else :func:`quantize_e4m3_reference`, with the same bits."""
    if _quant_routed(x):
        return torch.ops.cuda_l2_b200.quantize_e4m3(x)
    return quantize_e4m3_reference(x)


def quantize_e4m3_rowwise(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Per-row quantisation of a 2-D ``x`` [rows, cols] on its device: scale[r] = amax(|x[r]|) / 448 (an fp32
    [rows, 1] tensor), q = e4m3(x / scale). One outlier row no longer squeezes every other row into e4m3's few low
    codes. No host synchronisation. A 2-D CUDA fp16 / bf16 / fp32 tensor runs ``cuda_l2_b200::quantize_e4m3_rowwise``
    (one launch), anything else :func:`quantize_e4m3_rowwise_reference`, with the same bits."""
    if x.dim() == 2 and _quant_routed(x):
        return torch.ops.cuda_l2_b200.quantize_e4m3_rowwise(x)
    return quantize_e4m3_rowwise_reference(x)


def quantize_e4m3_blockwise(x: torch.Tensor, masked_m: torch.Tensor | None = None
                            ) -> tuple[torch.Tensor, torch.Tensor]:
    """Per 1 x 128 block quantisation of activations ``x`` [M, K] on its device: scale[m, kb] = amax(|x[m, 128 kb :
    128 kb + 128]|) / 448, q = e4m3(x / scale). The scale comes back as the M-major [M, ceil(K/128)] view the kernel
    reads in place (strides (1, ld_a), ld_a = M rounded up to 4). A batch ``x`` [B, M, K] is quantised per matrix, the
    same way: its scale is [B, M, ceil(K/128)], a view of a [B, ceil(K/128), ld_a] buffer that the batched kernel reads
    in place (strides (ceil(K/128) * ld_a, 1, ld_a)). No host synchronisation. A CUDA fp16 / bf16 / fp32 tensor runs
    ``cuda_l2_b200::quantize_e4m3_blockwise`` (one launch), anything else :func:`quantize_e4m3_blockwise_reference`,
    with the same bits. ``masked_m``: optional int32 tensor [B] on x's device, the per-matrix row counts of the
    masked batched GEMM; the kernel then reads and writes only rows [0, clamp(masked_m[b], 0, M)) of matrix b (the
    rest of q and scale is unspecified), the reference computes every row."""
    if x.dim() in (2, 3) and _quant_routed(x):
        return torch.ops.cuda_l2_b200.quantize_e4m3_blockwise(x, masked_m)
    return quantize_e4m3_blockwise_reference(x, masked_m)


def silu_mul_quantize_e4m3_blockwise(h: torch.Tensor, masked_m: torch.Tensor | None = None
                                     ) -> tuple[torch.Tensor, torch.Tensor]:
    """The SwiGLU of a gated MLP, quantised for the next FP8 GEMM: ``h`` [(B,) M, 2I] holds the gate g = h[..., :I]
    and the up projection u = h[..., I:] (the fused w13 layout of vLLM / SGLang checkpoints); returns
    :func:`quantize_e4m3_blockwise` of ``F.silu(g) * u`` [(B,) M, I], bit for bit. A CUDA fp16 / bf16 tensor runs
    ``cuda_l2_b200::silu_mul_quantize_e4m3_blockwise`` (one launch, no intermediate in memory), anything else
    :func:`silu_mul_quantize_e4m3_blockwise_reference`. ``masked_m`` as for :func:`quantize_e4m3_blockwise`."""
    if _quant_routed(h, silu_mul=True) and h.dim() in (2, 3) and h.shape[-1] % 2 == 0:
        return torch.ops.cuda_l2_b200.silu_mul_quantize_e4m3_blockwise(h, masked_m)
    return silu_mul_quantize_e4m3_blockwise_reference(h, masked_m)


def quantize_e4m3_block128x128(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Per 128 x 128 block quantisation of a weight ``w`` [N, K] on its device (the layout of DeepSeek-V3-style
    checkpoints' ``weight_scale_inv``): scale [ceil(N/128), ceil(K/128)] = amax(|block|) / 448, q = e4m3(w / scale).
    A stack of experts' weights [G, N, K] is quantised per expert, with scales [G, ceil(N/128), ceil(K/128)]. Torch ops
    only, no host synchronisation."""
    *lead, n, k = w.shape
    nnb, nkb, b = -(-n // capi.BLOCK), capi.num_k_blocks(k), capi.BLOCK
    wb = nn.functional.pad(w.float(), (0, nkb * b - k, 0, nnb * b - n)).view(*lead, nnb, b, nkb, b)
    scale = (wb.abs().amax(dim=(-3, -1)) / E4M3_MAX).clamp_min(torch.finfo(torch.float32).tiny)
    q = (wb / scale[..., :, None, :, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(*lead, nnb * b,
                                                                                                      nkb * b)
    return q[..., :n, :k].contiguous(), scale.contiguous()


FP8_GRANULARITIES = ("tensor", "rowwise", "blockwise")


class B200Fp8Linear(nn.Module):
    """Inference-only FP8 ``nn.Linear``: the weight is quantised once to e4m3 (buffers ``weight_fp8`` / ``weight_scale``);
    every call quantises the activation on the device and runs ``cuda_l2_b200::fp8_gemm``, then adds the bias (shared
    with the source layer). ``granularity="tensor"``: one scale for the weight (``weight_scale`` [1]) and one per call
    for the activation. ``"rowwise"``: one scale per output channel (``weight_scale`` [1, out_features], the layout of
    common FP8 checkpoints) and one per activation row (token). ``"blockwise"``: one scale per 128 x 128 weight block
    (``weight_scale`` [ceil(out/128), ceil(in/128)], DeepSeek-V3-style checkpoints, loadable as they are with
    :meth:`from_fp8`) and one per token and 128 input channels. No ``.item()`` and no host synchronisation, so the
    forward can be captured in a CUDA graph. Needs in_features % 16 == 0, out_features % 8 == 0."""

    @staticmethod
    def _check_fits(in_features: int, out_features: int, out_dtype: torch.dtype, what) -> None:
        t = capi.gemm_type(torch.float8_e4m3fn, out_dtype)
        if t is None or not t.fits(out_features, in_features):
            raise capi.B200HgemmError(f"cannot convert {what} to FP8: needs in_features % 16 == 0, out_features % 8 == 0 "
                                      f"and an fp16 / bf16 output type (got {out_dtype})")

    @classmethod
    def from_linear(cls, lin: nn.Linear, out_dtype: torch.dtype | None = None,
                    granularity: str = "tensor") -> "B200Fp8Linear":
        out_dtype = out_dtype or lin.weight.dtype
        cls._check_fits(lin.in_features, lin.out_features, out_dtype, lin)
        if granularity not in FP8_GRANULARITIES:
            raise capi.B200HgemmError(f"granularity must be one of {FP8_GRANULARITIES}, got {granularity!r}")
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        new.in_features, new.out_features, new.out_dtype = lin.in_features, lin.out_features, out_dtype
        new.granularity = granularity
        with torch.no_grad():
            if granularity == "rowwise":
                w_q, w_scale = quantize_e4m3_rowwise(lin.weight)
                w_scale = w_scale.reshape(1, lin.out_features)   # [1, N]: the column scales of the product
            elif granularity == "blockwise":
                w_q, w_scale = quantize_e4m3_block128x128(lin.weight)
            else:
                w_q, w_scale = quantize_e4m3(lin.weight)
        new.register_buffer("weight_fp8", w_q)
        new.register_buffer("weight_scale", w_scale)
        new.bias = lin.bias                                  # shared with the source layer
        return new

    @classmethod
    def from_fp8(cls, weight_fp8: torch.Tensor, weight_scale: torch.Tensor, bias: torch.Tensor | None = None,
                 out_dtype: torch.dtype = torch.bfloat16) -> "B200Fp8Linear":
        """A blockwise layer from a checkpoint's e4m3 weight [out, in] and its fp32 128 x 128 block scales
        [ceil(out/128), ceil(in/128)] (``weight_scale_inv``), taken as they are: no re-quantisation."""
        out_features, in_features = weight_fp8.shape
        cls._check_fits(in_features, out_features, out_dtype, f"a [{out_features}, {in_features}] weight")
        want = (-(-out_features // capi.BLOCK), capi.num_k_blocks(in_features))
        if weight_fp8.dtype != torch.float8_e4m3fn or weight_scale.dtype != torch.float32 or tuple(weight_scale.shape) != want:
            raise capi.B200HgemmError(f"from_fp8 needs a float8_e4m3fn weight and fp32 block scales of shape {list(want)}, "
                                      f"got {weight_fp8.dtype} and {weight_scale.dtype} {list(weight_scale.shape)}")
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        new.in_features, new.out_features, new.out_dtype = in_features, out_features, out_dtype
        new.granularity = "blockwise"
        new.register_buffer("weight_fp8", weight_fp8.contiguous())
        new.register_buffer("weight_scale", weight_scale.contiguous())
        new.bias = bias
        return new

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        lead = x.shape[:-1]
        x2 = x.reshape(-1, self.in_features)
        if x2.shape[0] == 0:
            y = x2.new_empty((0, self.out_features), dtype=self.out_dtype)
        else:
            quantize = {"rowwise": quantize_e4m3_rowwise, "blockwise": quantize_e4m3_blockwise}.get(self.granularity,
                                                                                                 quantize_e4m3)
            x_q, x_scale = quantize(x2)
            y = torch.ops.cuda_l2_b200.fp8_gemm(x_q, self.weight_fp8, x_scale, self.weight_scale, self.out_dtype)
        if self.bias is not None:
            y = y + self.bias
        return y.view(*lead, self.out_features)

    def extra_repr(self) -> str:
        return (f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, "
                f"out_dtype={self.out_dtype}, granularity={self.granularity}")


# ------------------------------------------------------------------------------------------ FP8 training of linear layers
#                                                                                            (libb200_quant_dual.so)
# e4m3 wgmma reads K-major operands only, so the input gradient dX = dY W and the weight gradient dW = dY^T X need W,
# dY and X transposed, each quantised along its other axis. The dual quantiser writes both orientations of a tensor
# from one read of it; every GEMM of the step is then fp8_gemm with rowwise scales.
def quantize_e4m3_rowwise_dual_reference(x: torch.Tensor
                                         ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """:func:`quantize_e4m3_rowwise_dual` as a composition of torch ops: the rowwise quantisation of ``x`` and of
    ``x^T`` zero-padded to a multiple of 16 columns, with the scales as vectors."""
    if x.dim() != 2:
        raise capi.B200HgemmError(f"quantize_e4m3_rowwise_dual takes [rows, cols], got {list(x.shape)}")
    rows, cols = x.shape
    q, scale = quantize_e4m3_rowwise_reference(x)
    q_t, scale_t = quantize_e4m3_rowwise_reference(
        nn.functional.pad(x.t(), (0, capi.dual_ld_t(rows) - rows)).contiguous())
    return q, scale.reshape(rows), q_t, scale_t.reshape(cols)


def _quantize_e4m3_rowwise_dual_outputs(x):
    _quant_input(x)
    if x.dim() != 2:
        raise capi.B200HgemmError(f"quantize_e4m3_rowwise_dual takes [rows, cols], got {list(x.shape)}")
    rows, cols = x.shape
    return (x.new_empty((rows, cols), dtype=torch.float8_e4m3fn), x.new_empty((rows,), dtype=torch.float32),
            x.new_empty((cols, capi.dual_ld_t(rows)), dtype=torch.float8_e4m3fn),
            x.new_empty((cols,), dtype=torch.float32))


def _quantize_e4m3_rowwise_dual_launch(out, x, *, stream):
    workspace = torch.empty(capi.quant_dual_workspace(*x.shape), dtype=torch.float32, device=x.device)
    capi.quantize_e4m3_rowwise_dual(x.contiguous(), *out, workspace, stream=stream)


_define_op("quantize_e4m3_rowwise_dual", "(Tensor x) -> (Tensor, Tensor, Tensor, Tensor)", None,
           _quantize_e4m3_rowwise_dual_launch, _QUANT_WHY, outputs=_quantize_e4m3_rowwise_dual_outputs)


def quantize_e4m3_rowwise_dual(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """Both rowwise quantisations of a 2-D ``x`` [rows, cols] on its device: ``(q, scale, q_t, scale_t)``, where
    ``q`` [rows, cols] and ``scale`` [rows] are :func:`quantize_e4m3_rowwise`'s (the scale as a vector), and ``q_t``
    [cols, ld_t] and ``scale_t`` [cols] are the same for ``x^T`` zero-padded to ``ld_t`` = rows rounded up to 16
    columns: a K-major FP8 GEMM operand whose reduction runs along x's rows. A padding byte is e4m3(0 / scale_t), 0x00
    unless the column's scale is NaN. No host synchronisation. A non-empty 2-D CUDA fp16 / bf16 / fp32 tensor runs
    ``cuda_l2_b200::quantize_e4m3_rowwise_dual`` (a memset and two launches, x read twice), anything else
    :func:`quantize_e4m3_rowwise_dual_reference`, with the same bits."""
    if x.dim() == 2 and _quant_routed(x):
        return torch.ops.cuda_l2_b200.quantize_e4m3_rowwise_dual(x)
    return quantize_e4m3_rowwise_dual_reference(x)


# ------------------------------------------------------------------------------------------ blockwise FP8 training
#                                                                                            (libb200_quant_block_dual.so)
# The DeepSeek-V3 recipe: x and dY get one scale per token and 128 channels, W one per 128 x 128 block. A 128 x 128 tile
# holds complete groups in both orientations, so one launch writes both e4m3 copies of a tensor. These quantisers are
# plain functions, not operators: the blockwise training path is not traceable by FakeTensor or torch.compile.
def quantize_e4m3_blockwise_dual_reference(x: torch.Tensor
                                           ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """:func:`quantize_e4m3_blockwise_dual` as a composition of torch ops: :func:`quantize_e4m3_blockwise_reference`
    of ``x`` and of ``x^T`` zero-padded to a multiple of 16 columns."""
    if x.dim() != 2:
        raise capi.B200HgemmError(f"quantize_e4m3_blockwise_dual takes [rows, cols], got {list(x.shape)}")
    rows = x.shape[0]
    q, scale = quantize_e4m3_blockwise_reference(x)
    q_t, scale_t = quantize_e4m3_blockwise_reference(
        nn.functional.pad(x.t(), (0, capi.dual_ld_t(rows) - rows)).contiguous())
    return q, scale, q_t, scale_t


def _block_dual_routed(x: torch.Tensor) -> bool:
    """Whether libb200_quant_block_dual.so runs on ``x``: a non-empty 2-D fp16 / bf16 CUDA tensor."""
    return x.dim() == 2 and _quant_routed(x, silu_mul=True)


def quantize_e4m3_blockwise_dual(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """Both 1 x 128 quantisations of a 2-D ``x`` [rows, cols] on its device: ``(q, scale, q_t, scale_t)``, where ``q``
    [rows, cols] and ``scale`` [rows, ceil(cols/128)] are :func:`quantize_e4m3_blockwise`'s, and ``q_t`` [cols, ld_t]
    and ``scale_t`` [cols, ceil(rows/128)] are the same for ``x^T`` zero-padded to ``ld_t`` = rows rounded up to 16
    columns: a K-major FP8 GEMM operand whose reduction runs along x's rows, scaled per 128 of them. Both scales come
    back in the M-major layout the block-scaled GEMMs read in place. A padding byte is e4m3(0 / s), 0x00 unless the
    group's scale is NaN. A non-empty CUDA fp16 / bf16 tensor runs one launch of libb200_quant_block_dual.so on the
    current stream (x read once), anything else :func:`quantize_e4m3_blockwise_dual_reference`, with the same bits. Not
    an operator: FakeTensor and torch.compile cannot trace it."""
    if not _block_dual_routed(x):
        return quantize_e4m3_blockwise_dual_reference(x)
    rows, cols = x.shape
    q = x.new_empty((rows, cols), dtype=torch.float8_e4m3fn)
    q_t = x.new_empty((cols, capi.dual_ld_t(rows)), dtype=torch.float8_e4m3fn)
    scale = capi.empty_m_major((), rows, capi.num_k_blocks(cols), x.device)
    scale_t = capi.empty_m_major((), cols, capi.num_k_blocks(rows), x.device)
    with torch.cuda.device(x.device):
        capi.quantize_e4m3_blockwise_dual(x.contiguous(), q, scale, q_t, scale_t,
                                          stream=torch.cuda.current_stream(x.device).cuda_stream)
    return q, scale, q_t, scale_t


def quantize_e4m3_block128x128_dual_reference(w: torch.Tensor
                                              ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """:func:`quantize_e4m3_block128x128_dual` as a composition of torch ops: :func:`quantize_e4m3_block128x128` and
    its transpose."""
    if w.dim() != 2:
        raise capi.B200HgemmError(f"quantize_e4m3_block128x128_dual takes [rows, cols], got {list(w.shape)}")
    q, scale = quantize_e4m3_block128x128(w)
    return q, scale, q.t().contiguous(), scale.t().contiguous()


def quantize_e4m3_block128x128_dual(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """Both 128 x 128 block quantisations of a weight ``w`` [N, K] on its device: ``(q, scale, q_t, scale_t)`` with
    ``q`` [N, K] and ``scale`` [ceil(N/128), ceil(K/128)] those of :func:`quantize_e4m3_block128x128`, ``q_t`` = q^T
    [K, N] and ``scale_t`` = scale^T (with 128 x 128 blocks, the quantisation of w^T is the transpose of that of w, bit
    for bit). A non-empty CUDA fp16 / bf16 tensor runs one launch of libb200_quant_block_dual.so on the current stream,
    anything else :func:`quantize_e4m3_block128x128_dual_reference`, with the same bits. Not an operator."""
    if not _block_dual_routed(w):
        return quantize_e4m3_block128x128_dual_reference(w)
    n, k = w.shape
    nnb, nkb = -(-n // capi.BLOCK), capi.num_k_blocks(k)
    q = w.new_empty((n, k), dtype=torch.float8_e4m3fn)
    q_t = w.new_empty((k, n), dtype=torch.float8_e4m3fn)
    scale = w.new_empty((nnb, nkb), dtype=torch.float32)
    scale_t = w.new_empty((nkb, nnb), dtype=torch.float32)
    with torch.cuda.device(w.device):
        capi.quantize_e4m3_block128x128_dual(w.contiguous(), q, scale, q_t, scale_t,
                                             stream=torch.cuda.current_stream(w.device).cuda_stream)
    return q, scale, q_t, scale_t


FP8_TRAIN_GRANULARITIES = ("rowwise", "blockwise")


def _check_fp8_train_granularity(granularity: str) -> None:
    if granularity not in FP8_TRAIN_GRANULARITIES:
        raise capi.B200HgemmError(f"granularity must be one of {FP8_TRAIN_GRANULARITIES}, got {granularity!r}")


def _check_fp8_linear(in_features: int, out_features: int, dtype: torch.dtype, what) -> None:
    """The rules of :func:`fp8_linear`'s three GEMMs: fp16 / bf16, and in_features and out_features multiples of 16
    (each is the reduction of one of them, and e4m3 rows must be 16 bytes)."""
    if dtype not in (torch.float16, torch.bfloat16) or in_features % 16 or out_features % 16:
        raise capi.B200HgemmError(f"FP8 training of {what} needs fp16 / bf16 and in_features % 16 == 0, "
                                  f"out_features % 16 == 0, got {in_features}->{out_features} {dtype}")


def _rowwise_gemm(a, a_scale, b_kmajor, b_scale, out_dtype):
    """fp8_gemm with rowwise scales given as vectors: a_scale [M], b_scale [N]."""
    return torch.ops.cuda_l2_b200.fp8_gemm(a, b_kmajor, a_scale.reshape(-1, 1), b_scale.reshape(1, -1), out_dtype)


class _Fp8LinearFunction(torch.autograd.Function):
    """y = x W^T with a gradient, every product an e4m3 rowwise-scaled fp8_gemm. The forward saves the transposed e4m3
    copies its backward reads, not x and W, and only those of the gradients that will be asked for."""

    @staticmethod
    def forward(ctx, x2, weight, main_grad=None):
        need_x, need_w = ctx.needs_input_grad[:2]
        ctx.shapes = (x2.shape, weight.shape)
        ctx.dtypes = (x2.dtype, weight.dtype)
        ctx.main_grad = main_grad
        if x2.shape[0] == 0:
            ctx.save_for_backward()
            return x2.new_empty((0, weight.shape[0]))
        # dW = q(dY^T) q(X^T)^T needs X transposed; dX = q(dY) q(W^T)^T needs W transposed
        if need_w:
            x_q, x_s, x_qt, x_st = quantize_e4m3_rowwise_dual(x2)
        else:
            x_q, x_s = quantize_e4m3_rowwise(x2)
            x_qt = x_st = None
        if need_x:
            w_q, w_s, w_qt, w_st = quantize_e4m3_rowwise_dual(weight)
        else:
            w_q, w_s = quantize_e4m3_rowwise(weight)
            w_qt = w_st = None
        ctx.save_for_backward(x_qt, x_st, w_qt, w_st)
        return _rowwise_gemm(x_q, x_s, w_q, w_s, x2.dtype)

    @staticmethod
    def backward(ctx, grad_y):
        (x_shape, w_shape), (x_dtype, w_dtype) = ctx.shapes, ctx.dtypes
        need_x, need_w = ctx.needs_input_grad[:2]
        grad_x = grad_w = None
        if x_shape[0] == 0:
            if need_x:
                grad_x = grad_y.new_empty(x_shape, dtype=x_dtype)
            if need_w and ctx.main_grad is None:
                grad_w = grad_y.new_zeros(w_shape, dtype=w_dtype)
            return grad_x, grad_w, None
        x_qt, x_st, w_qt, w_st = ctx.saved_tensors
        g = grad_y.contiguous()
        if need_w:
            g_q, g_s, g_qt, g_st = quantize_e4m3_rowwise_dual(g)
            if ctx.main_grad is None:
                grad_w = _rowwise_gemm(g_qt, g_st, x_qt, x_st, w_dtype)   # [N, ld_t(M)] x [K, ld_t(M)] -> [N, K]
            else:   # the same product's fp32 value, added into main_grad
                fp8_gemm_accumulate_(ctx.main_grad, g_qt, x_qt, g_st.reshape(-1, 1), x_st.reshape(1, -1))
        else:
            g_q, g_s = quantize_e4m3_rowwise(g)
        if need_x:
            grad_x = _rowwise_gemm(g_q, g_s, w_qt, w_st, x_dtype)         # [M, N] x [K, N] -> [M, K]
        return grad_x, grad_w, None


class _Fp8BlockwiseLinearFunction(torch.autograd.Function):
    """y = x W^T with a gradient in the blockwise recipe: x and dY quantised per token and 128 channels, W per 128 x 128
    block, every k-block of every product promoted into an fp32 accumulator. The forward saves the transposed e4m3
    copies its backward reads, not x and W, and only those of the gradients that will be asked for."""

    @staticmethod
    def forward(ctx, x2, weight, main_grad=None):
        need_x, need_w = ctx.needs_input_grad[:2]
        ctx.shapes = (x2.shape, weight.shape)
        ctx.dtypes = (x2.dtype, weight.dtype)
        ctx.main_grad = main_grad
        if x2.shape[0] == 0:
            ctx.save_for_backward()
            return x2.new_empty((0, weight.shape[0]))
        # dW = q(dY^T) q(X^T)^T needs X transposed; dX = q(dY) q(W^T)^T needs W transposed
        if need_w:
            x_q, x_s, x_qt, x_st = quantize_e4m3_blockwise_dual(x2)
        else:
            x_q, x_s = quantize_e4m3_blockwise(x2)
            x_qt = x_st = None
        if need_x:
            w_q, w_s, w_qt, w_st = quantize_e4m3_block128x128_dual(weight)
        else:
            w_q, w_s = quantize_e4m3_block128x128(weight)
            w_qt = w_st = None
        ctx.save_for_backward(x_qt, x_st, w_qt, w_st)
        return torch.ops.cuda_l2_b200.fp8_gemm(x_q, w_q, x_s, w_s, x2.dtype)

    @staticmethod
    def backward(ctx, grad_y):
        (x_shape, w_shape), (x_dtype, w_dtype) = ctx.shapes, ctx.dtypes
        need_x, need_w = ctx.needs_input_grad[:2]
        grad_x = grad_w = None
        if x_shape[0] == 0:
            if need_x:
                grad_x = grad_y.new_empty(x_shape, dtype=x_dtype)
            if need_w and ctx.main_grad is None:
                grad_w = grad_y.new_zeros(w_shape, dtype=w_dtype)
            return grad_x, grad_w, None
        x_qt, x_st, w_qt, w_st = ctx.saved_tensors
        g = grad_y.contiguous()
        gemm = torch.ops.cuda_l2_b200.fp8_gemm
        if need_w:
            g_q, g_s, g_qt, g_st = quantize_e4m3_blockwise_dual(g)
            if ctx.main_grad is None:
                grad_w = gemm(g_qt, x_qt, g_st, x_st, w_dtype)   # [N, ld_t(M)] x [K, ld_t(M)], 1 x 128 scales -> [N, K]
            else:   # the same product's fp32 value, added into main_grad
                fp8_gemm_accumulate_(ctx.main_grad, g_qt, x_qt, g_st, x_st)
        else:
            g_q, g_s = quantize_e4m3_blockwise(g)
        if need_x:
            grad_x = gemm(g_q, w_qt, g_s, w_st, x_dtype)     # [M, N] x [K, N], 128 x 128 scales of W^T -> [M, K]
        return grad_x, grad_w, None


def fp8_linear(x: torch.Tensor, weight: torch.Tensor, granularity: str = "rowwise",
               main_grad: torch.Tensor | None = None) -> torch.Tensor:
    """``x @ weight^T`` for ``x`` [..., K] and ``weight`` [N, K] of one dtype (fp16 or bf16), K % 16 == 0 and
    N % 16 == 0, in FP8 with a gradient.

    ``granularity="rowwise"``: x and W are quantised to e4m3 with one fp32 scale per row (per token, per output
    channel) and multiplied by ``fp8_gemm`` into x's dtype. The backward quantises dY the same way and runs two more
    ``fp8_gemm`` calls, dX = dY W (scales per token and per input channel) and dW = dY^T X (both operands scaled along
    the tokens), from the transposed e4m3 copies of W and x that the forward kept. Every product accumulates in the FP8
    tensor cores' fast mode. Without a gradient to compute, the forward is ``B200Fp8Linear``'s rowwise one, bit for
    bit. No host synchronisation: a forward and backward can be captured in one CUDA graph.

    ``granularity="blockwise"`` (the DeepSeek-V3 recipe): x and dY get one scale per token and 128 channels, W one per
    128 x 128 block, and every 128-wide k-block of the three products is promoted into an fp32 accumulator. y and dX
    are block-scaled ``fp8_gemm`` calls; dW = q(dY^T) q(X^T)^T reduces over the tokens with 1 x 128 scales on both
    operands, so one outlier token squeezes only its own 128-token group. Both orientations of x, dY and W come from
    one launch each (:func:`quantize_e4m3_blockwise_dual`, :func:`quantize_e4m3_block128x128_dual`). Without a
    gradient to compute, the forward is ``B200Fp8Linear``'s blockwise one, bit for bit. Also no host synchronisation;
    its quantisers are not operators, so this path is not traceable by FakeTensor or torch.compile.

    ``main_grad``: an fp32 tensor of the weight's shape, contiguous, on its device. The backward then adds dW into it
    (:func:`fp8_gemm_accumulate_`: exactly the fp32 value the unfused dW rounds, one rounding per element) and returns
    no gradient for the weight. y and dX are the unfused call's, bit for bit. The backward writes the tensor given here.
    A frozen weight (``requires_grad=False``) gets nothing added."""
    if x.dim() == 0 or weight.dim() != 2 or x.shape[-1] != weight.shape[1] or x.dtype != weight.dtype:
        raise capi.B200HgemmError(f"fp8_linear: x [..., K] and weight [N, K] of one dtype expected, got "
                                  f"{x.dtype} {tuple(x.shape)} and {weight.dtype} {tuple(weight.shape)}")
    _check_fp8_train_granularity(granularity)
    n, k = weight.shape
    _check_fp8_linear(k, n, weight.dtype, f"a [{n}, {k}] weight")
    if main_grad is not None:
        capi.check_main_grad(main_grad, (n, k), weight.device)
    x2 = x.reshape(-1, k)
    blockwise = granularity == "blockwise"
    if torch.is_grad_enabled() and (x.requires_grad or weight.requires_grad):
        y = (_Fp8BlockwiseLinearFunction if blockwise else _Fp8LinearFunction).apply(x2, weight, main_grad)
    elif x2.shape[0] == 0:
        y = x2.new_empty((0, n))
    elif blockwise:
        (x_q, x_s), (w_q, w_s) = quantize_e4m3_blockwise(x2), quantize_e4m3_block128x128(weight)
        y = torch.ops.cuda_l2_b200.fp8_gemm(x_q, w_q, x_s, w_s, x.dtype)
    else:
        (x_q, x_s), (w_q, w_s) = quantize_e4m3_rowwise(x2), quantize_e4m3_rowwise(weight)
        y = torch.ops.cuda_l2_b200.fp8_gemm(x_q, w_q, x_s, w_s.reshape(1, n), x.dtype)
    return y.view(*x.shape[:-1], n)


class B200Fp8TrainLinear(nn.Module):
    """``nn.Linear`` trained in FP8: a trainable 16-bit ``weight`` [out_features, in_features] (and optional ``bias``),
    the product run by :func:`fp8_linear` with ``granularity`` ("rowwise", the default, or "blockwise": e4m3 forward and
    backward with those scales), the bias added by torch after it as :class:`B200Linear` does. In eval or no-grad mode
    the output is :class:`B200Fp8Linear`'s of the same granularity, bit for bit. Needs fp16 / bf16 and
    in_features % 16 == 0, out_features % 16 == 0.

    ``fuse_wgrad_accumulation=True``: the weight must carry ``weight.main_grad``, an fp32 tensor of its shape (checked
    in forward); the backward adds dW into it (``fp8_linear``'s ``main_grad``) and leaves ``weight.grad`` None. The buffer
    written is the ``weight.main_grad`` of the forward: replacing it between forward and backward leaves the new one
    untouched, and a step captured in a CUDA graph keeps writing the buffer it was captured with (zero it in place)."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, device=None,
                 dtype: torch.dtype = torch.bfloat16, granularity: str = "rowwise",
                 fuse_wgrad_accumulation: bool = False):
        super().__init__()
        _check_fp8_linear(in_features, out_features, dtype, "B200Fp8TrainLinear")
        _check_fp8_train_granularity(granularity)
        self.in_features, self.out_features, self.granularity = in_features, out_features, granularity
        self.fuse_wgrad_accumulation = fuse_wgrad_accumulation
        self.weight = nn.Parameter(torch.empty((out_features, in_features), device=device, dtype=dtype))
        self.bias = nn.Parameter(torch.empty(out_features, device=device, dtype=dtype)) if bias else None
        self.reset_parameters()

    reset_parameters = B200Linear.reset_parameters

    @classmethod
    def from_linear(cls, lin: nn.Linear, granularity: str = "rowwise",
                    fuse_wgrad_accumulation: bool = False) -> "B200Fp8TrainLinear":
        """A layer sharing ``lin``'s Parameters (no copy), as :meth:`B200Linear.from_linear`."""
        _check_fp8_linear(lin.in_features, lin.out_features, lin.weight.dtype, lin)
        _check_fp8_train_granularity(granularity)
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        new.in_features, new.out_features, new.granularity = lin.in_features, lin.out_features, granularity
        new.fuse_wgrad_accumulation = fuse_wgrad_accumulation
        new.weight, new.bias = lin.weight, lin.bias          # shared storage, no copy
        return new

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        main_grad = _fused_main_grad(self.weight) if self.fuse_wgrad_accumulation else None
        y = fp8_linear(x, self.weight, self.granularity, main_grad)
        if self.bias is not None:
            y = y + self.bias
        return y

    def extra_repr(self) -> str:
        return (f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, "
                f"granularity={self.granularity}" + (", fuse_wgrad_accumulation=True" if self.fuse_wgrad_accumulation
                                                     else ""))


# ------------------------------------------------------------------------------------------ grouped FP8 (libb200_grouped_fp8.so)
def _fp8_grouped_shape(a, b_kmajor, scale_a, scale_b, offs, out_dtype):
    _, t, n, _ = capi.check_grouped_operands(a, b_kmajor, offs, "fp32", out_dtype, (scale_a, scale_b))
    return (t, n), out_dtype


def _fp8_grouped_launch(c, a, b_kmajor, scale_a, scale_b, offs, out_dtype, *, stream):
    if b_kmajor.shape[0] == 0 or c.shape[0] == 0:   # no group or no row
        return
    a, b_kmajor, offs = a.contiguous(), b_kmajor.contiguous(), offs.contiguous()
    scale_a, scale_b = _kernel_scales("blockwise", scale_a, scale_b)   # the only form the shape check accepts
    capi.fp8_grouped_gemm(a, b_kmajor, c, scale_a, scale_b, offs, stream=stream)


_define_op("fp8_grouped_gemm", "(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, Tensor offs, "
           "ScalarType out_dtype) -> Tensor", _fp8_grouped_shape, _fp8_grouped_launch)


def fp8_grouped_gemm(a: torch.Tensor, b_kmajor: torch.Tensor, scale_a: torch.Tensor, scale_b: torch.Tensor,
                     offs: torch.Tensor, out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``a`` [T,K] by ``b_kmajor`` [G,N,K], e4m3 operands with block scales, over contiguous row groups -> [T,N]
    ``out_dtype``: rows [offs[g-1], offs[g]) of the result are the block-scaled product of those rows of ``a`` and
    ``b_kmajor[g]^T``, in one launch. ``scale_a`` [T, ceil(K/128)] in any layout (the M-major one of
    :func:`quantize_e4m3_blockwise` is read in place), ``scale_b`` [G, ceil(N/128), ceil(K/128)]. ``offs`` as for
    :func:`hgemm_grouped`; rows at or past ``offs[-1]`` are unspecified. Inference only."""
    return torch.ops.cuda_l2_b200.fp8_grouped_gemm(a, b_kmajor, scale_a, scale_b, offs, out_dtype)


# ------------------------------------------------------------------------------------------ batched FP8 (libb200_batched_fp8.so)
def _fp8_batched_shape(a, b_kmajor, scale_a, scale_b, out_dtype, masked_m=None):
    bsz, m, n, _ = capi.check_batched_operands(a, b_kmajor, "fp32", masked_m, out_dtype, (scale_a, scale_b))
    return (bsz, m, n), out_dtype


def _fp8_batched_launch(c, a, b_kmajor, scale_a, scale_b, out_dtype, masked_m=None, *, stream):
    if c.shape[0] == 0 or c.shape[1] == 0:   # no matrix or no row
        return
    a, b_kmajor = a.contiguous(), b_kmajor.contiguous()
    scale_a, scale_b = _kernel_scales("blockwise", scale_a, scale_b)   # the only form the shape check accepts
    if masked_m is not None:
        masked_m = masked_m.contiguous()
    capi.fp8_batched_gemm(a, b_kmajor, c, scale_a, scale_b, masked_m=masked_m, stream=stream)


_define_op("fp8_batched_gemm", "(Tensor a, Tensor b_kmajor, Tensor scale_a, Tensor scale_b, ScalarType out_dtype, "
           "Tensor? masked_m=None) -> Tensor", _fp8_batched_shape, _fp8_batched_launch)


def fp8_batched_gemm(a: torch.Tensor, b_kmajor: torch.Tensor, scale_a: torch.Tensor, scale_b: torch.Tensor,
                     out_dtype: torch.dtype = torch.bfloat16, masked_m: torch.Tensor | None = None) -> torch.Tensor:
    """``a`` [B,M,K] by ``b_kmajor`` [B,N,K] per batch, e4m3 operands with block scales -> [B,M,N] ``out_dtype``, in
    one launch. ``scale_a`` [B, M, ceil(K/128)] in any layout (the one :func:`quantize_e4m3_blockwise` returns for a
    [B,M,K] input is read in place), ``scale_b`` [B, ceil(N/128), ceil(K/128)]. ``masked_m``: optional int32 CUDA
    tensor [B], read by the kernel; only rows [0, clamp(masked_m[b], 0, M)) of batch b are computed, the rest of the
    result is unspecified (the MoE decode layout). Inference only."""
    return torch.ops.cuda_l2_b200.fp8_batched_gemm(a, b_kmajor, scale_a, scale_b, out_dtype, masked_m)


class B200Fp8GroupedLinear(nn.Module):
    """Inference-only FP8 experts of a mixture-of-experts layer: G ``nn.Linear`` weights [N, K] without bias, stacked
    as e4m3 ``weight_fp8`` [G, N, K] with 128 x 128 block scales ``weight_scale`` [G, ceil(N/128), ceil(K/128)]. The
    forward takes the tokens sorted by expert, ``x`` [T, K], and the int32 cumulative group ends ``offs`` [G] on the
    GPU, quantises ``x`` per token and 128 input channels on the device and runs ``cuda_l2_b200::fp8_grouped_gemm``:
    no ``.item()`` and no host synchronisation, so it can be captured in a CUDA graph. Rows at or past ``offs[-1]``
    of the result are unspecified. Needs K % 16 == 0, N % 8 == 0."""

    @classmethod
    def from_fp8(cls, weight_fp8: torch.Tensor, weight_scale_inv: torch.Tensor,
                 out_dtype: torch.dtype = torch.bfloat16) -> "B200Fp8GroupedLinear":
        """The experts of a checkpoint, taken as they are: the e4m3 weights [G, N, K] and their fp32 128 x 128 block
        scales [G, ceil(N/128), ceil(K/128)] (each expert's ``weight_scale_inv``, stacked). No re-quantisation."""
        try:
            g, n, k = weight_fp8.shape
        except ValueError:
            raise capi.B200HgemmError(f"from_fp8 needs a stacked weight [G, N, K], got {list(weight_fp8.shape)}") from None
        B200Fp8Linear._check_fits(k, n, out_dtype, f"a [{g}, {n}, {k}] weight stack")
        want = (g, -(-n // capi.BLOCK), capi.num_k_blocks(k))
        if weight_fp8.dtype != torch.float8_e4m3fn or weight_scale_inv.dtype != torch.float32 or \
                tuple(weight_scale_inv.shape) != want:
            raise capi.B200HgemmError(f"from_fp8 needs a float8_e4m3fn weight stack and fp32 block scales of shape "
                                      f"{list(want)}, got {weight_fp8.dtype} and {weight_scale_inv.dtype} "
                                      f"{list(weight_scale_inv.shape)}")
        new = cls()
        new.num_groups, new.in_features, new.out_features, new.out_dtype = g, k, n, out_dtype
        new.register_buffer("weight_fp8", weight_fp8.contiguous())
        new.register_buffer("weight_scale", weight_scale_inv.contiguous())
        return new

    @classmethod
    def from_weights(cls, w: torch.Tensor) -> "B200Fp8GroupedLinear":
        """The experts from a 16-bit weight stack ``w`` [G, N, K], quantised per 128 x 128 block; the output dtype is
        ``w``'s."""
        if w.dtype not in (torch.float16, torch.bfloat16) or w.dim() != 3:
            raise capi.B200HgemmError(f"from_weights needs an fp16 / bf16 weight stack [G, N, K], got {w.dtype} "
                                      f"{list(w.shape)}")
        with torch.no_grad():
            w_q, w_scale = quantize_e4m3_block128x128(w)
        return cls.from_fp8(w_q, w_scale, w.dtype)

    def forward(self, x: torch.Tensor, offs: torch.Tensor) -> torch.Tensor:
        x_q, x_scale = quantize_e4m3_blockwise(x)
        return torch.ops.cuda_l2_b200.fp8_grouped_gemm(x_q, self.weight_fp8, x_scale, self.weight_scale, offs,
                                                       self.out_dtype)

    def forward_masked(self, x: torch.Tensor, masked_m: torch.Tensor) -> torch.Tensor:
        """The same experts in the padded decode layout: ``x`` [G, M, K], one fixed slot of M tokens per expert, and the
        int32 token counts ``masked_m`` [G] on the GPU -> [G, M, N]. Rows [0, clamp(masked_m[g], 0, M)) of expert g are
        computed; the rest of its slot in the result is unspecified. Quantises ``x`` per token and 128 input channels
        on the device and runs ``cuda_l2_b200::fp8_batched_gemm``: no host synchronisation, so it can be captured in a
        CUDA graph. The quantiser, too, reads and writes only the counted rows: the others are rows the GEMM treats
        as unspecified."""
        x_q, x_scale = quantize_e4m3_blockwise(x, masked_m)
        return torch.ops.cuda_l2_b200.fp8_batched_gemm(x_q, self.weight_fp8, x_scale, self.weight_scale,
                                                       self.out_dtype, masked_m)

    def extra_repr(self) -> str:
        return (f"num_groups={self.num_groups}, in_features={self.in_features}, out_features={self.out_features}, "
                f"out_dtype={self.out_dtype}")


class B200Fp8GroupedMLP(nn.Module):
    """Inference-only routed experts of an FP8 mixture-of-experts checkpoint as a gated MLP: for the tokens of expert
    g, ``y = (silu(x W1[g]^T) * (x W3[g]^T)) W2[g]^T``, with the gate and up projections fused in one stack
    ``w13_fp8`` [G, 2I, H] (W1 in rows [0, I), W3 in rows [I, 2I): the w13 layout of vLLM / SGLang checkpoints) and
    ``w2_fp8`` [G, H, I], both e4m3 with 128 x 128 block scales. A forward is four launches and no host
    synchronisation: :func:`quantize_e4m3_blockwise` of x, the gate/up FP8 GEMM (out_dtype h [.., 2I]),
    :func:`silu_mul_quantize_e4m3_blockwise` of h, and the down FP8 GEMM. Needs H % 16 == 0 and I % 16 == 0."""

    @classmethod
    def from_fp8(cls, w13_fp8: torch.Tensor, w13_scale: torch.Tensor, w2_fp8: torch.Tensor, w2_scale: torch.Tensor,
                 out_dtype: torch.dtype = torch.bfloat16) -> "B200Fp8GroupedMLP":
        """The experts of a checkpoint, taken as they are: the e4m3 stacks ``w13_fp8`` [G, 2I, H] and ``w2_fp8``
        [G, H, I] with their fp32 128 x 128 block scales [G, ceil(2I/128), ceil(H/128)] and [G, ceil(H/128),
        ceil(I/128)]. ``out_dtype`` (fp16 or bf16) is that of the gate/up product and of the result."""
        try:
            g, two_i, hid = w13_fp8.shape
            g2, hid2, i = w2_fp8.shape
        except ValueError:
            raise capi.B200HgemmError(f"from_fp8 needs stacks w13 [G, 2I, H] and w2 [G, H, I], got "
                                      f"{list(w13_fp8.shape)} and {list(w2_fp8.shape)}") from None
        if g < 1 or g2 != g or hid2 != hid or two_i != 2 * i or hid % 16 or i % 16:
            raise capi.B200HgemmError(f"B200Fp8GroupedMLP needs w13 [G, 2I, H] and w2 [G, H, I] with G >= 1, "
                                      f"H % 16 == 0 and I % 16 == 0, got {list(w13_fp8.shape)} and "
                                      f"{list(w2_fp8.shape)}")
        if out_dtype not in (torch.float16, torch.bfloat16):
            raise capi.B200HgemmError(f"out_dtype must be fp16 or bf16, got {out_dtype}")
        for name, w, s in (("w13", w13_fp8, w13_scale), ("w2", w2_fp8, w2_scale)):
            want = (g, -(-w.shape[1] // capi.BLOCK), capi.num_k_blocks(w.shape[2]))
            if w.dtype != torch.float8_e4m3fn or s.dtype != torch.float32 or tuple(s.shape) != want:
                raise capi.B200HgemmError(f"{name} must be a float8_e4m3fn stack with fp32 block scales of shape "
                                          f"{list(want)}, got {w.dtype} and {s.dtype} {list(s.shape)}")
        new = cls()
        new.num_experts, new.hidden_size, new.intermediate_size, new.out_dtype = g, hid, i, out_dtype
        new.register_buffer("w13_fp8", w13_fp8.contiguous())
        new.register_buffer("w13_scale", w13_scale.contiguous())
        new.register_buffer("w2_fp8", w2_fp8.contiguous())
        new.register_buffer("w2_scale", w2_scale.contiguous())
        return new

    @classmethod
    def from_weights(cls, w13: torch.Tensor, w2: torch.Tensor) -> "B200Fp8GroupedMLP":
        """The experts from 16-bit stacks ``w13`` [G, 2I, H] and ``w2`` [G, H, I] of one dtype, quantised per
        128 x 128 block; the output dtype is theirs."""
        if w13.dtype not in (torch.float16, torch.bfloat16) or w2.dtype != w13.dtype or w13.dim() != 3 or \
                w2.dim() != 3:
            raise capi.B200HgemmError(f"from_weights needs fp16 / bf16 stacks w13 [G, 2I, H] and w2 [G, H, I] of one "
                                      f"dtype, got {w13.dtype} {list(w13.shape)} and {w2.dtype} {list(w2.shape)}")
        with torch.no_grad():
            w13_q, w13_s = quantize_e4m3_block128x128(w13)
            w2_q, w2_s = quantize_e4m3_block128x128(w2)
        return cls.from_fp8(w13_q, w13_s, w2_q, w2_s, w13.dtype)

    def forward(self, x: torch.Tensor, offs: torch.Tensor) -> torch.Tensor:
        """``x`` [T, H], the tokens sorted by expert, and the int32 cumulative group ends ``offs`` [G] on the GPU ->
        [T, H]. Rows at or past ``offs[-1]`` of the result are unspecified."""
        x_q, x_scale = quantize_e4m3_blockwise(x)
        h = torch.ops.cuda_l2_b200.fp8_grouped_gemm(x_q, self.w13_fp8, x_scale, self.w13_scale, offs, self.out_dtype)
        p_q, p_scale = silu_mul_quantize_e4m3_blockwise(h)
        return torch.ops.cuda_l2_b200.fp8_grouped_gemm(p_q, self.w2_fp8, p_scale, self.w2_scale, offs,
                                                       self.out_dtype)

    def forward_masked(self, x: torch.Tensor, masked_m: torch.Tensor) -> torch.Tensor:
        """The same experts in the padded decode layout: ``x`` [G, M, H], one slot of M tokens per expert, and the
        int32 token counts ``masked_m`` [G] on the GPU -> [G, M, H]. Rows [0, clamp(masked_m[g], 0, M)) of expert g
        are computed; the rest of its slot in the result is unspecified. Both quantisers take ``masked_m`` too, so
        no launch reads or writes a row past the counts."""
        x_q, x_scale = quantize_e4m3_blockwise(x, masked_m)
        h = torch.ops.cuda_l2_b200.fp8_batched_gemm(x_q, self.w13_fp8, x_scale, self.w13_scale, self.out_dtype,
                                                    masked_m)
        p_q, p_scale = silu_mul_quantize_e4m3_blockwise(h, masked_m)
        return torch.ops.cuda_l2_b200.fp8_batched_gemm(p_q, self.w2_fp8, p_scale, self.w2_scale, self.out_dtype,
                                                       masked_m)

    def extra_repr(self) -> str:
        return (f"num_experts={self.num_experts}, hidden_size={self.hidden_size}, "
                f"intermediate_size={self.intermediate_size}, out_dtype={self.out_dtype}")


__all__ = ["hgemm", "hgemm_nn", "hgemm_batched", "hgemm_grouped", "hgemm_grouped_nn", "hgemm_grouped_wgrad",
           "grouped_linear", "B200GroupedLinear", "B200Linear", "replace_linear_modules", "linear_supported", "fp8_gemm", "quantize_e4m3",
           "quantize_e4m3_rowwise", "quantize_e4m3_blockwise", "quantize_e4m3_block128x128", "B200Fp8Linear",
           "fp8_grouped_gemm", "fp8_batched_gemm", "B200Fp8GroupedLinear", "silu_mul_quantize_e4m3_blockwise",
           "B200Fp8GroupedMLP", "quantize_e4m3_rowwise_dual", "fp8_linear", "B200Fp8TrainLinear",
           "quantize_e4m3_blockwise_dual", "quantize_e4m3_block128x128_dual"]
