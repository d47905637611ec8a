"""Fused batch-norm of the AN4 DeepSpeech model over the frames of the longest utterance (``csrc/frame_bn.cu``).

``lens`` are the utterances' output frame lengths (``DeepSpeech.get_seq_lens``), an int32 tensor on the input's device,
read there only.  With ``T_b`` the input's frame width, ``Tm = min(max(lens), T_b)``.

- ``conv_block_bn(x, bn, lens)``, x ``[N, C, F, T_b]`` the output of a conv (with its bias), replaces
  ``mask(hardtanh(mask(bn(mask(x))), 0, 20))`` of ``_TimeMaskedConv``, the mask zeroing the frames ``t >= lens[n]``.
  The statistics are over ``(n, f, t < Tm)``, a masked frame counted as 0.
- ``seq_bn(x, bn, lens)``, x ``[T_b, N, H]``, replaces ``bn(x.reshape(T_b N, H)).view(T_b, N, H)`` (``_SeqBN``).  The
  statistics are over the rows of the first ``Tm`` frames; the output and the input gradient are exactly +0 after them.

``lens`` must hold exactly N integer lengths (``ValueError`` otherwise, checked on the host from the shape).

For the AN4 collate (sorted, padded to the longest utterance) ``Tm = T_b``, and the op equals the stock modules to
rounding.  Where the longest utterance is shorter than the tensor, ``Tm < T_b``, it equals the stock modules run on the
tensor cropped to ``Tm`` frames, so that a batch padded to a frame multiple gives the unpadded batch's statistics, loss
and gradients to rounding.  The
summation order depends on ``Tm`` (never on ``T_b``), so a padded launch equals the cropped one bit for bit; there are
no atomics, and the results are reproducible run to run.  No value is read on the host: the op can be captured in a
CUDA graph.

The running statistics move as torch's (``momentum``, unbiased variance, ``num_batches_tracked`` + 1) with the counted
frames as the count ``n``.  For ``n = 1``, where the stock module raises, the biased variance (0) takes the place of the
unbiased one, so ``running_var`` stays finite.

Types: x fp32, bf16 or fp16 (under autocast the 16-bit conv / LSTM / look-ahead output as it is); the affine parameters,
statistics and their gradients fp32, as torch's batch-norm under autocast.  y and dx have x's type, computed in fp32
and rounded once.  One kernel forward and one backward per call.

Falls back to exactly the stock expression wherever the kernels do not apply: CPU input, no native extension, eval mode,
``track_running_stats=False``, no affine parameters or non-fp32 ones, ``momentum=None``, a type other than fp32 / bf16
/ fp16, a non-contiguous input, or too large a channel.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ext
from .ext import DTYPE_CODE


def _stock_conv_block(x, bn, lens):
    mask = torch.arange(x.size(3), device=x.device).view(1, 1, 1, -1) >= lens.to(x.device).view(-1, 1, 1, 1)
    x = bn(x.masked_fill(mask, 0)).masked_fill(mask, 0)
    return F.hardtanh(x, 0, 20, inplace=True).masked_fill(mask, 0)


def _stock_seq(x, bn):
    t, n = x.size(0), x.size(1)
    return bn(x.reshape(t * n, -1)).view(t, n, -1)


def _fast_path_ok(x: torch.Tensor, bn: nn.modules.batchnorm._BatchNorm, conv: int) -> bool:
    if not (x.is_cuda and bn.training and bn.track_running_stats and bn.running_mean is not None and bn.affine
            and bn.momentum is not None and x.dtype in DTYPE_CODE and x.is_contiguous() and x.dim() == (4 if conv else 3)
            and ext.available()):
        return False
    if not all(t.dtype == torch.float32 and t.is_cuda for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var)):
        return False
    if conv:
        N, C, Fq, Tb = x.shape
    else:
        Tb, N, C = x.shape
        Fq = 1
    return C == bn.num_features and ext.require().frame_bn_supported(conv, N, C, Fq, Tb)


class _FrameBN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, lens, bn, conv):
        C_ = ext.require()
        if conv:
            N, C, Fq, Tb = x.shape
        else:
            Tb, N, C = x.shape
            Fq = 1
        y = torch.empty_like(x)
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        nbt = bn.num_batches_tracked
        C_.frame_bn_forward(conv, x.data_ptr(), lens.data_ptr(), weight.data_ptr(), bias.data_ptr(), y.data_ptr(),
                            mean.data_ptr(), rstd.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
                            nbt.data_ptr() if nbt is not None and nbt.is_cuda else 0, N, C, Fq, Tb, float(bn.eps),
                            float(bn.momentum), DTYPE_CODE[x.dtype], torch.cuda.current_stream().cuda_stream)
        ctx.save_for_backward(x, weight, bias, lens, mean, rstd)
        ctx.dims = (conv, N, C, Fq, Tb)
        return y

    @staticmethod
    def backward(ctx, dy):
        C_ = ext.require()
        x, weight, bias, lens, mean, rstd = ctx.saved_tensors
        conv, N, C, Fq, Tb = ctx.dims
        dy = dy.to(x.dtype).contiguous()
        dx = torch.empty_like(x)
        dgamma = torch.empty_like(mean)
        dbeta = torch.empty_like(mean)
        C_.frame_bn_backward(conv, x.data_ptr(), dy.data_ptr(), lens.data_ptr(), weight.data_ptr(), bias.data_ptr(),
                             mean.data_ptr(), rstd.data_ptr(), dx.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), N, C,
                             Fq, Tb, DTYPE_CODE[x.dtype], torch.cuda.current_stream().cuda_stream)
        return dx, dgamma, dbeta, None, None, None


def _device_lens(lens: torch.Tensor, device) -> torch.Tensor:
    return lens.to(device=device, dtype=torch.int32).contiguous()


def _check_lens(lens, N: int) -> None:
    """The kernels read ``lens[0..N)`` on the device: anything but N integer lengths is refused on the host (shape and
    type only, no synchronisation)."""
    if not (isinstance(lens, torch.Tensor) and lens.dim() == 1 and lens.numel() == N and not lens.is_floating_point()
            and not lens.is_complex() and lens.dtype != torch.bool):
        raise ValueError("lens must be a 1-D integer tensor of the batch's %d lengths, got %s" % (
            N, tuple(lens.shape) if isinstance(lens, torch.Tensor) else type(lens).__name__))


def conv_block_bn(x: torch.Tensor, bn: nn.BatchNorm2d, lens: torch.Tensor) -> torch.Tensor:
    """``mask(hardtanh(mask(bn(mask(x))), 0, 20))`` over x ``[N, C, F, T_b]``, statistics over the first ``Tm`` frames;
    see the module docstring."""
    _check_lens(lens, x.size(0))
    if not _fast_path_ok(x, bn, 1):
        return _stock_conv_block(x, bn, lens)
    return _FrameBN.apply(x, bn.weight, bn.bias, _device_lens(lens, x.device), bn, 1)


def seq_bn(x: torch.Tensor, bn: nn.BatchNorm1d, lens: torch.Tensor) -> torch.Tensor:
    """``bn`` on the ``T_b N`` rows of x ``[T_b, N, H]``, statistics over the rows of the first ``Tm`` frames; see the
    module docstring."""
    _check_lens(lens, x.size(1))
    if not _fast_path_ok(x, bn, 0):
        return _stock_seq(x, bn)
    return _FrameBN.apply(x, bn.weight, bn.bias, _device_lens(lens, x.device), bn, 0)
