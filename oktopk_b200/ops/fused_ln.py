"""Fused dropout + residual add + LayerNorm for BERT's encoder layers (``csrc/layernorm.cu``).

``residual_dropout_layer_norm(x, a, ln, p)`` computes ``ln(x + dropout(a, p))``, the end of a BertLayer's attention and
MLP blocks, on CUDA with one kernel forward and two backward instead of the stock dropout, add and layer_norm kernels
and their backward.  The dropout mask is never stored: the backward pass regenerates it from the seed and recomputes
``x + dropout(a)`` from the saved ``x`` and ``a``.

Dropout: each call draws one int64 seed on the device from torch's default CUDA generator
(``torch.empty(1, dtype=torch.int64, device=x.device).random_()``) and the kernels derive element ``i``'s keep bit from it
with Philox4x32-10 (counter ``i // 4``, word ``i % 4``, kept iff below ``floor((1-p) 2^32)``).  So ``torch.manual_seed``
makes runs reproducible, ``torch.utils.checkpoint`` (which restores the CUDA RNG state) recomputes the same mask, and a
CUDA graph of a whole step draws a fresh mask at each replay.  The masks are not torch's own dropout masks.  ``p = 0``
(what a caller passes in eval mode) runs no generator.

Types: ``x`` and the LayerNorm's parameters are fp32; ``a`` is fp32, bf16 or fp16.  Under CUDA autocast the residual
stream and ``layer_norm`` stay fp32 while the linear layer in front hands over a 16-bit ``a``: that mixed case runs
fused, with ``y`` fp32 as the stock ops return it and ``a``'s gradient in ``a``'s type.  The 16-bit results are bit for
bit the fp32 kernel's on ``a.float()``, with only ``a``'s gradient rounded.

Falls back to exactly ``ln(x + F.dropout(a, p, p > 0))`` wherever the fast path does not apply: CPU tensors, a last
dimension outside 128, 256, ..., 1024 or unlike ``ln.normalized_shape``, ``x`` not fp32 or ``a`` not fp32 / bf16 / fp16,
``x`` and ``a`` of different shapes, a LayerNorm without affine parameters or with parameters that are not fp32,
``p`` outside [0, 1), or no native extension.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from . import ext
from .ext import DTYPE_CODE, dense16


def keep_threshold(p: float) -> int:
    """``floor((1-p) 2^32)``: an element is kept iff its Philox word is below it; ``2^32`` (p = 0) keeps everything."""
    return 1 << 32 if p == 0 else int(math.floor((1.0 - p) * 2.0 ** 32))


def _fast_path_ok(x: torch.Tensor, a: torch.Tensor, ln: torch.nn.LayerNorm, p: float) -> bool:
    if not (x.is_cuda and x.dim() >= 1 and x.numel() > 0 and ext.available()):
        return False
    H = x.size(-1)
    w, b = ln.weight, ln.bias
    return (0.0 <= p < 1.0 and x.dtype == torch.float32 and a.dtype in DTYPE_CODE and a.device == x.device
            and a.shape == x.shape and tuple(ln.normalized_shape) == (H,) and H % 128 == 0 and 128 <= H <= 1024
            and w is not None and b is not None and w.dtype == torch.float32 and b.dtype == torch.float32
            and w.device == x.device and b.device == x.device)


class _ResidualDropoutLN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, a, gamma, beta, p, eps):
        C = ext.require()
        H = x.size(-1)
        R = x.numel() // H
        seed = torch.empty(1, dtype=torch.int64, device=x.device).random_() if p > 0 else None
        y = torch.empty_like(x)
        stats = torch.empty((2, R), dtype=torch.float32, device=x.device)          # [mean; rstd] per row
        thr, scale = keep_threshold(p), 1.0 / (1.0 - p)
        C.ln_forward(x.data_ptr(), a.data_ptr(), y.data_ptr(), gamma.data_ptr(), beta.data_ptr(), stats[0].data_ptr(),
                     stats[1].data_ptr(), 0 if seed is None else seed.data_ptr(), R, H, thr, scale, eps,
                     DTYPE_CODE[a.dtype], torch.cuda.current_stream().cuda_stream)
        ctx.save_for_backward(x, a, gamma, stats, seed)
        ctx.thr, ctx.scale = thr, scale
        return y

    @staticmethod
    def backward(ctx, dy):
        C = ext.require()
        x, a, gamma, stats, seed = ctx.saved_tensors
        H = x.size(-1)
        R = x.numel() // H
        dy = dense16(dy.float())                        # y is fp32, so is its gradient
        dx = torch.empty_like(x)
        da = torch.empty_like(a)
        partial = torch.empty(C.ln_bwd_grid(R) * 2 * H, dtype=torch.float32, device=x.device)
        dgb = torch.empty(2 * H, dtype=torch.float32, device=x.device)              # [dgamma | dbeta]
        C.ln_backward(x.data_ptr(), a.data_ptr(), dy.data_ptr(), gamma.data_ptr(), stats[0].data_ptr(),
                      stats[1].data_ptr(), 0 if seed is None else seed.data_ptr(), dx.data_ptr(), da.data_ptr(),
                      partial.data_ptr(), dgb.data_ptr(), dgb.data_ptr() + 4 * H, R, H, ctx.thr, ctx.scale,
                      DTYPE_CODE[a.dtype], torch.cuda.current_stream().cuda_stream)
        return dx, da, dgb[:H], dgb[H:], None, None


def residual_dropout_layer_norm(x: torch.Tensor, a: torch.Tensor, ln: torch.nn.LayerNorm, p: float) -> torch.Tensor:
    """``ln(x + dropout(a, p))`` (``p = 0``: no dropout, as in eval mode); see the module docstring."""
    p = float(p)
    if _fast_path_ok(x, a, ln, p):
        return _ResidualDropoutLN.apply(dense16(x), dense16(a), ln.weight, ln.bias, p, float(ln.eps))
    return ln(x + F.dropout(a, p, p > 0))
