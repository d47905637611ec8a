"""Fused softmax cross-entropy for BERT's masked-LM loss (``csrc/xent.cu``).

``softmax_cross_entropy(logits, target, ignore_index)`` computes ``F.cross_entropy(logits, target,
ignore_index=ignore_index)`` for 2-D logits with the mean reduction, on CUDA with two kernels forward and one backward.
Only the rows whose target is not ``ignore_index`` carry loss: the forward pass reads only those rows and keeps one fp32
log-sum-exp per row, and the backward pass reads them again and writes the gradient once, with 128-bit zero stores on
the ignored rows.  Between the passes the op holds the logits (which the autograd graph keeps anyway), the targets and
the ``[R + 1]`` fp32 log-sum-exps and label count.  The loss is reduced on the device in a fixed order: no host
synchronisation, bitwise reproducible, and CUDA-graph safe.

Types: logits are fp32, bf16 or fp16; the loss is a 0-d fp32 tensor, as ``F.cross_entropy`` returns it under autocast,
and the logits' gradient has the logits' type: ``(softmax(x) - onehot(t)) · g / n`` computed in fp32 and rounded once
(to nearest even; an fp16 gradient past 65504 becomes inf, so a loss-scaled overflow reaches the scaler's check).  The
incoming gradient ``g`` and the label count ``n`` are read on the device, so a loss scale takes effect without a sync.

Edge cases: no labelled row gives a NaN loss and an all-zero gradient, as torch.  An inf or NaN in a labelled row
propagates to that row's loss and gradient; isolated ``-inf`` logits contribute 0.  A target outside ``[0, V)`` that is
not ``ignore_index`` gives a NaN loss and a NaN gradient row, where torch's kernel device-asserts.  Unlike the stock
op, an ignored row is never read, so its gradient is exactly 0 even if it holds inf or NaN.

Falls back to exactly ``F.cross_entropy(logits, target, ignore_index=ignore_index)`` wherever the fast path does not
apply: CPU tensors, no native extension, logits not 2-D, not fp32 / bf16 / fp16 or without rows or columns, a target
that is not int64 of shape ``[R]`` on the logits' device.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ext
from .ext import DTYPE_CODE, dense16


def _fast_path_ok(logits: torch.Tensor, target: torch.Tensor) -> bool:
    if not (logits.is_cuda and logits.dim() == 2 and ext.available()):
        return False
    R, V = logits.shape
    return (logits.dtype in DTYPE_CODE and 0 < R < 2 ** 31 and V > 0 and target.dtype == torch.int64
            and tuple(target.shape) == (R,) and target.device == logits.device)


class _SoftmaxCrossEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, ignore_index):
        C = ext.require()
        R, V = logits.shape
        lse = torch.empty(R + 1, dtype=torch.float32, device=logits.device)      # per-row log-sum-exp, then n
        rowloss = torch.empty(R, dtype=torch.float32, device=logits.device)
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        C.xent_forward(logits.data_ptr(), target.data_ptr(), lse.data_ptr(), rowloss.data_ptr(), loss.data_ptr(), R, V,
                       ignore_index, DTYPE_CODE[logits.dtype], torch.cuda.current_stream().cuda_stream)
        ctx.save_for_backward(logits, target, lse)
        ctx.ignore_index = ignore_index
        return loss

    @staticmethod
    def backward(ctx, g):
        C = ext.require()
        logits, target, lse = ctx.saved_tensors
        R, V = logits.shape
        g = g.float().contiguous()                      # the loss is fp32, so is its gradient
        dx = torch.empty_like(logits)
        C.xent_backward(logits.data_ptr(), target.data_ptr(), lse.data_ptr(), g.data_ptr(), dx.data_ptr(), R, V,
                        ctx.ignore_index, DTYPE_CODE[logits.dtype], torch.cuda.current_stream().cuda_stream)
        return dx, None, None


def softmax_cross_entropy(logits: torch.Tensor, target: torch.Tensor, ignore_index: int = -100) -> torch.Tensor:
    """``F.cross_entropy(logits, target, ignore_index=ignore_index)`` (mean over the labelled rows); see the module
    docstring."""
    if _fast_path_ok(logits, target):
        return _SoftmaxCrossEntropy.apply(dense16(logits), target.contiguous(), int(ignore_index))
    return F.cross_entropy(logits, target, ignore_index=ignore_index)
