"""Fused softmax + CTC loss for the AN4 DeepSpeech model (``csrc/ctc.cu``).

``ctc_loss(logits, targets, input_lengths, target_lengths)`` computes

    F.ctc_loss(F.log_softmax(logits, -1).float(), targets.long(), input_lengths.long(), target_lengths.long(),
               blank=0, reduction="sum", zero_infinity=True)

for time-major ``[T, N, C]`` logits and concatenated 1-D targets, on CUDA with two kernels forward and one backward.  The
softmax is taken inside the kernels, so there is no ``[T, N, C]`` log-softmax tensor, no widening copy and no
log-softmax backward.  The lengths are read on the device: device lengths are used as they are, host lengths are copied
over from pinned memory without a synchronisation.  Host input lengths are checked against ``T`` on the host and raise
as the stock op does.  The launch geometry and the workspace depend on the shapes only, and the per-utterance losses
are added in a fixed order without atomics, so the op is bitwise reproducible, runs under
``torch.use_deterministic_algorithms(True)`` and can be captured in a CUDA graph.

Types: logits are fp32, bf16 or fp16 (under autocast the 16-bit ``fc`` output is taken as it is, widened exactly in the
kernels); targets int32 or int64.  The loss is a 0-d fp32 tensor.  The logits' gradient has the logits' type:
``(softmax(x) - posterior) · g`` computed in fp32 and rounded once (to nearest even; an fp16 gradient past 65504 becomes
inf, so a loss-scaled overflow reaches the scaler's check).  ``g`` is read on the device.

Edge cases, per utterance: ``Ln = 0`` is the all-blank alignment; an infeasible utterance (or ``Tn = 0`` with
``Ln > 0``) contributes exactly 0 to the loss and the gradient; a label outside ``[0, C)`` or a device input length
outside ``[0, T]`` makes that utterance's loss and gradient NaN, where torch device-asserts.  A negative target length,
or one that takes the running sum of target lengths past ``targets.numel()``, leaves the target offsets undefined from
that utterance on: it and every later utterance are NaN, the earlier ones unaffected.  Frames ``t >= Tn`` are never
read: their gradient is exactly 0 even if they hold inf or NaN.  A ``-inf`` logit leaves the loss finite (as torch's)
and makes the gradient of its frame NaN in every class (as torch's).

Falls back to exactly the stock expression above wherever the fast path does not apply: CPU logits, no native
extension, logits not 3-D or not fp32 / bf16 / fp16, ``C`` outside ``[1, 128]``, more than 2047 targets in the batch,
padded 2-D targets, or lengths that are not ``N`` integers.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ext
from .ext import DTYPE_CODE


def _stock(logits, targets, input_lengths, target_lengths):
    return F.ctc_loss(F.log_softmax(logits, -1).float(), targets.long(), input_lengths.long(), target_lengths.long(),
                      blank=0, reduction="sum", zero_infinity=True)


def _is_lengths(t, N: int) -> bool:
    return (isinstance(t, torch.Tensor) and t.numel() == N and t.dim() <= 1 and not t.is_floating_point()
            and not t.is_complex() and t.dtype != torch.bool)


def _fast_path_ok(logits, targets, input_lengths, target_lengths) -> bool:
    if not (isinstance(logits, torch.Tensor) and logits.is_cuda and logits.dim() == 3 and ext.available()):
        return False
    T, N, C = logits.shape
    return (logits.dtype in DTYPE_CODE and isinstance(targets, torch.Tensor) and targets.dim() == 1
            and targets.dtype in (torch.int32, torch.int64) and _is_lengths(input_lengths, N)
            and _is_lengths(target_lengths, N) and ext.require().ctc_supported(T, N, C, targets.numel()))


def _on_device(t: torch.Tensor, dtype, device) -> torch.Tensor:
    """``t`` as a contiguous ``dtype`` tensor on ``device``; a host tensor goes through pinned memory, asynchronously."""
    if t.is_cuda:
        return t.to(device, dtype).contiguous()
    return t.to(dtype).contiguous().pin_memory().to(device, non_blocking=True)


class _CTCLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, targets, tn, ln):
        C_ = ext.require()
        T, N, C = logits.shape
        nt = targets.numel()
        ws = torch.empty(C_.ctc_workspace_floats(T, N, nt), dtype=torch.float32, device=logits.device)
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        C_.ctc_forward(logits.data_ptr(), targets.data_ptr() if nt else 0, int(targets.dtype == torch.int64),
                       tn.data_ptr(), ln.data_ptr(), ws.data_ptr(), loss.data_ptr(), T, N, C, nt,
                       DTYPE_CODE[logits.dtype], torch.cuda.current_stream().cuda_stream)
        ctx.save_for_backward(logits, targets, tn, ln, ws)
        return loss

    @staticmethod
    def backward(ctx, g):
        C_ = ext.require()
        logits, targets, tn, ln, ws = ctx.saved_tensors
        T, N, C = logits.shape
        nt = targets.numel()
        g = g.float().contiguous()                      # the loss is fp32, so is its gradient
        ab = torch.empty(C_.ctc_ab_floats(T, N, nt), dtype=torch.float32, device=logits.device)
        dx = torch.empty_like(logits)
        C_.ctc_backward(logits.data_ptr(), targets.data_ptr() if nt else 0, int(targets.dtype == torch.int64),
                        tn.data_ptr(), ln.data_ptr(), ws.data_ptr(), ab.data_ptr(), g.data_ptr(), dx.data_ptr(), T, N, C,
                        nt, DTYPE_CODE[logits.dtype], torch.cuda.current_stream().cuda_stream)
        return dx, None, None, None


def ctc_loss(logits: torch.Tensor, targets: torch.Tensor, input_lengths: torch.Tensor,
             target_lengths: torch.Tensor) -> torch.Tensor:
    """Summed CTC loss (blank 0, zero_infinity) of ``softmax(logits)``, logits ``[T, N, C]``; see the module docstring."""
    if not _fast_path_ok(logits, targets, input_lengths, target_lengths):
        return _stock(logits, targets, input_lengths, target_lengths)
    T = logits.size(0)
    dev = logits.device
    if not input_lengths.is_cuda and input_lengths.numel() and int(input_lengths.max()) > T:
        raise RuntimeError("Expected input_lengths to have value at most %d, but got value %d"
                           % (T, int(input_lengths.max())))
    tn = _on_device(input_lengths.reshape(-1), torch.int32, dev)
    ln = _on_device(target_lengths.reshape(-1), torch.int32, dev)
    return _CTCLoss.apply(logits.contiguous(), _on_device(targets, targets.dtype, dev), tn, ln)
