"""Fused look-ahead convolution + Hardtanh(0, 20) of the AN4 DeepSpeech model (``csrc/lookahead.cu``).

``lookahead_hardtanh(x, weight, lens)`` replaces ``nn.Sequential(Lookahead(H, context), nn.Hardtanh(0, 20))`` on x
``[T_b, N, H]`` with the ``[H, context + 1]`` weight.  ``lens`` are the output frame lengths, an int32 tensor on the
input's device, read there only (the lengths ``fused_frame_bn`` takes).  With ``Tm = min(max(lens), T_b)`` and
``L_n = min(lens[n], Tm)``::

    z[t, n, h] = sum_{k = 0..context} W[h, k] x[t + k, n, h]     (x read as 0 where t + k >= L_n)
    y[t, n, h] = t < L_n ? clamp(z, 0, 20) : +0

Backward: ``dz = dy`` where the frame is valid and ``0 < y < 20`` (torch's strict Hardtanh backward, y alone decides
it), else 0; ``dx[t] = sum_k W[h, k] dz[t - k]`` on valid frames and exactly +0 on the frames ``t >= lens[n]``;
``dW[h, k] = sum over t < Tm and n of x[t + k] dz[t]``.

Relation to the stock module: the LSTM layers write exact zeros past each utterance's length, so on the model y and dW
equal the stock module's to rounding.  The stock dx is not zero on padded frames (the taps of the valid frames before
them reach there); the fused dx is +0.  The LSTM backward ignores those frames either way, so the parameter gradients
agree to rounding.  A non-finite dz reaches dW through the zeros read past a length (0 * inf = NaN) as it does
through the stock convolution's zero padding, so loss scaling still sees an fp16 overflow.

dW is summed in a fixed order that depends on ``(Tm, N, H, context)`` and the lengths, never on ``T_b``: a launch at a
padded width equals the launch on the tensor cropped to ``Tm`` frames bit for bit, and runs repeat bit for bit.  No
value is read on the host, so the op can be captured in a CUDA graph.  It has no state and runs the same in train and
eval mode.

Types: x fp32, bf16 or fp16, as it comes (under autocast, the 16-bit LSTM output); y and dx have x's type, computed in
fp32 and rounded once.  The weight and its gradient stay fp32: autocast does not round the weight.  One kernel forward
and one backward per call.

Falls back to exactly the stock expression (which reads no lengths) wherever the kernels do not apply: CPU input, no
native extension, a type other than fp32 / bf16 / fp16, a weight that is not fp32, a non-contiguous input, or more
taps than ``max_taps()``.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ext
from .ext import DTYPE_CODE
from .fused_frame_bn import _check_lens, _device_lens


def _stock(x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """``nn.Sequential(Lookahead, nn.Hardtanh(0, 20, inplace=True))`` of ``models/deepspeech.py``."""
    context = weight.size(1) - 1
    y = F.pad(x.permute(1, 2, 0), (0, context))
    y = F.conv1d(y, weight.unsqueeze(1), groups=weight.size(0))
    return F.hardtanh(y.permute(2, 0, 1).contiguous(), 0, 20, inplace=True)


def max_taps() -> int:
    """The most taps (``context + 1``) the kernels take."""
    return ext.require().lookahead_max_taps()


def _fast_path_ok(x: torch.Tensor, weight: torch.Tensor) -> bool:
    if not (x.is_cuda and x.dim() == 3 and x.dtype in DTYPE_CODE and x.is_contiguous() and weight.is_cuda
            and weight.dtype == torch.float32 and weight.dim() == 2 and weight.size(0) == x.size(2)
            and ext.available()):
        return False
    Tb, N, H = x.shape
    return ext.require().lookahead_supported(N, H, Tb, weight.size(1))


class _Lookahead(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, lens):
        C_ = ext.require()
        Tb, N, H = x.shape
        K = weight.size(1)
        w = weight.contiguous()
        y = torch.empty_like(x)
        C_.lookahead_forward(x.data_ptr(), w.data_ptr(), lens.data_ptr(), y.data_ptr(), N, H, Tb, K,
                             DTYPE_CODE[x.dtype], torch.cuda.current_stream().cuda_stream)
        ctx.save_for_backward(x, w, lens, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        C_ = ext.require()
        x, w, lens, y = ctx.saved_tensors
        Tb, N, H = x.shape
        K = w.size(1)
        dy = dy.to(x.dtype).contiguous()
        dx = torch.empty_like(x)
        dw = torch.empty_like(w)
        C_.lookahead_backward(x.data_ptr(), y.data_ptr(), dy.data_ptr(), w.data_ptr(), lens.data_ptr(), dx.data_ptr(),
                              dw.data_ptr(), N, H, Tb, K, DTYPE_CODE[x.dtype], torch.cuda.current_stream().cuda_stream)
        return dx, dw, None


def lookahead_hardtanh(x: torch.Tensor, weight: torch.Tensor, lens: torch.Tensor) -> torch.Tensor:
    """``hardtanh(lookahead(x), 0, 20)`` over x ``[T_b, N, H]`` with the frames past each length read as 0 and written
    +0; see the module docstring."""
    _check_lens(lens, x.size(1))
    if not _fast_path_ok(x, weight):
        return _stock(x, weight)
    return _Lookahead.apply(x, weight, _device_lens(lens, x.device))
