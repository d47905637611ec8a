"""Fused (conv-bias +) BatchNorm2d [+ residual] + ReLU [+ 2x2 max-pool] for channels_last fp32, bf16 or fp16 activations
(``csrc/bnrelu.cu``).

``bias_bn_relu(x, bn, conv_bias, relu=True, pool=None)`` replaces ``pool(relu(bn(x + conv_bias)))`` in training mode on
CUDA with one kernel forward and one backward instead of the seven stock ones (bias add, batch-norm, clamp, counter
increment; threshold backward, batch-norm backward, bias-gradient reduction) plus the two of the pool.  With a 2x2 /
stride-2 ``pool`` the forward kernel writes only the pooled output and a one-byte arg-max; the pre-pool activation is
never stored.  The convolution is then called WITHOUT its bias: a bias in front of a batch-norm cancels exactly
(``BN(x + b) = BN(x)``, the batch mean absorbs it), so it only enters the running-mean update, and its gradient is
identically zero (returned as ``None``; autograd's own reduction over ``dy`` returns rounding noise for it).
Parameters, buffers and ``state_dict`` keys are the stock modules' ones.  Small layers (``bn_sliced(M, C, W)``: VGG-16's
layers 5 - 13 at 16 images) run the channel-sliced kernels, which have no grid hand-off and compute the same bits.

Residual: ``bias_bn_relu(..., residual=r)`` / ``conv_bn_relu(..., residual=r)`` compute ``relu(bn(x) + r)``, the end of a
ResNet block, in the same two kernels (``relu=True`` and no pool only; anything else is a ``ValueError``).  The
statistics are ``x``'s alone; the backward kernel also writes ``dr = dy * [bn(x) + r > 0]``, which is exact.  ``r`` must
be on ``x``'s device with its shape and dtype (a non-channels_last ``r`` is made contiguous once); otherwise, and
wherever the fast path does not apply, the stock ``F.relu(bn(x) + r)`` runs.

bf16: under ``torch.autocast("cuda", torch.bfloat16)`` (or with bf16 activations and autocast off) the convolution
returns bf16 and the kernels' bf16 instantiation runs.  As torch's batch-norm does under autocast, it takes bf16
activations with fp32 parameters and statistics: ``y`` and ``dx`` are bf16; ``dgamma``, ``dbeta`` and the running
statistics fp32.  Its results are bit for bit those of the fp32 kernels run on ``x.float()`` (and ``dy.float()``), with
``y`` and ``dx`` rounded to bf16.

fp16 is opt-in: every entry point takes ``fp16=False``, and only with ``fp16=True`` do fp16 activations (autocast off
or ``torch.autocast("cuda", torch.float16)``) take the kernels' fp16 instantiation; the fp32 input of a convolution
under fp16 autocast then qualifies too, since the convolution hands the batch-norm fp16.  The kernel is the bf16 one's
spec in fp16: bit for bit the fp32 kernels on the widened input with ``y`` and ``dx`` rounded to fp16.  fp16's narrow
range is kept as torch's ``.half()`` keeps it: a value that rounds past 65504 is stored as inf (under loss scaling that
inf is what the optimizer's overflow check sees), subnormals are not flushed, and an inf or NaN input propagates as in
the fp32 kernel.  Without ``fp16=True`` fp16 activations and fp16 autocast keep the stock ops.

Falls back to the stock ops whenever the fast path does not apply (CPU, eval mode, activations neither fp32 nor bf16
nor opted-in fp16, fp16 autocast without ``fp16=True``, parameters not fp32, not channels_last, channels not a multiple
of 4, cumulative-average momentum).  A pool that cannot be folded in (not 2x2 / stride 2, odd height or width, or
batch-norm tiles that are not whole pairs of image rows) runs after the fused kernel on its own, on stock ``MaxPool2d``
for 16-bit activations (the standalone pool kernels are fp32 only).
"""
from __future__ import annotations

import itertools
from typing import Optional

import torch
import torch.nn.functional as F

from . import ext
from .ext import DTYPE_CODE

# > 0 caps the grid of the fused batch-norm kernels, so that each CTA loops over several tiles (tests use it to cover
# that path on a GPU whose co-resident grid exceeds the tile count).  A cap also keeps a shape the channel-sliced kernels
# would take on the cooperative ones (1 << 30 caps nothing: the cooperative kernels exactly as without a cap).
MAX_CTAS = 0

_SLOTS = itertools.count()


def _sync_slot(bn: torch.nn.BatchNorm2d) -> int:
    """The grid hand-off counters of ``bn``'s kernels (csrc/bnrelu.cu ``g_bn_sync``): one slot per module, so that the
    kernels of two layers never share counters."""
    s = bn.__dict__.get("_okt_bn_slot")
    if s is None:
        s = bn.__dict__["_okt_bn_slot"] = next(_SLOTS)
    return s


def _dtype_ok(x: torch.Tensor, fp16: bool = False) -> bool:
    """fp32 or bf16 activations, with autocast off or in bf16.  With ``fp16``, also fp16 activations with autocast off,
    and fp16 or fp32 ones under fp16 autocast (a convolution there turns fp32 input into fp16, and stock batch-norm runs
    an fp32 activation in fp32).  Without ``fp16``, fp16 activations and fp16 autocast keep the stock ops."""
    if not torch.is_autocast_enabled():
        return x.dtype in (torch.float32, torch.bfloat16) or (fp16 and x.dtype == torch.float16)
    if torch.get_autocast_dtype("cuda") == torch.float16:
        return fp16 and x.dtype in (torch.float32, torch.float16)
    return x.dtype in (torch.float32, torch.bfloat16) and torch.get_autocast_dtype("cuda") == torch.bfloat16


def _bn_params_fp32(bn: torch.nn.BatchNorm2d) -> bool:
    return all(t is None or t.dtype == torch.float32 for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))


def _fast_path_ok(x: torch.Tensor, bn: torch.nn.BatchNorm2d, fp16: bool = False) -> bool:
    return (x.is_cuda and _dtype_ok(x, fp16) and x.dim() == 4 and bn.training and bn.affine
            and bn.momentum is not None and x.size(1) % 4 == 0 and _bn_params_fp32(bn)
            and x.is_contiguous(memory_format=torch.channels_last) and ext.available())


def _is_2x2(pool: torch.nn.MaxPool2d) -> bool:
    ks = pool.kernel_size if isinstance(pool.kernel_size, tuple) else (pool.kernel_size,) * 2
    st = pool.stride if isinstance(pool.stride, tuple) else (pool.stride,) * 2
    pad = pool.padding if isinstance(pool.padding, tuple) else (pool.padding,) * 2
    dil = pool.dilation if isinstance(pool.dilation, tuple) else (pool.dilation,) * 2
    return ks == (2, 2) and st == (2, 2) and pad == (0, 0) and dil == (1, 1) and not pool.return_indices


def _pool_fusable(x: torch.Tensor, pool: torch.nn.MaxPool2d) -> bool:
    N, C, H, W = x.shape
    return (_is_2x2(pool) and H % 2 == 0 and W % 2 == 0
            and ext.require().bn_tile_rows(N * H * W, C) % (2 * W) == 0)


def _residual_ok(x: torch.Tensor, residual: torch.Tensor) -> bool:
    return residual.device == x.device and residual.shape == x.shape and residual.dtype == x.dtype


def _partial(C, x: torch.Tensor, M: int, Ch: int, W: int) -> Optional[torch.Tensor]:
    """The cooperative kernels' per-tile partials; the channel-sliced kernels need none."""
    if MAX_CTAS <= 0 and C.bn_sliced(M, Ch, W):
        return None
    rows = C.bn_tile_rows(M, Ch)
    return torch.empty((M + rows - 1) // rows * 2 * Ch, dtype=torch.float32, device=x.device)


class _BiasBNReLUPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, cbias, rmean, rvar, nbt, momentum, eps, relu, pool, slot, res=None):
        C = ext.require()
        N, Ch, H, W = x.shape
        M = N * H * W
        dtype = DTYPE_CODE[x.dtype]
        if pool:
            y = torch.empty((N, Ch, H // 2, W // 2), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
            arg = torch.empty(y.numel(), dtype=torch.uint8, device=x.device)
        else:
            y = torch.empty_like(x)                   # preserves channels_last
            arg = None
        partial = _partial(C, x, M, Ch, W if pool else 0)
        stats = torch.empty(2 * Ch, dtype=torch.float32, device=x.device)       # [mean | invstd]
        s = torch.cuda.current_stream().cuda_stream
        C.bn_forward(x.data_ptr(), y.data_ptr(), 0 if arg is None else arg.data_ptr(),
                     0 if partial is None else partial.data_ptr(), gamma.data_ptr(),
                     beta.data_ptr(), 0 if cbias is None else cbias.data_ptr(), stats.data_ptr(), stats.data_ptr() + 4 * Ch,
                     0 if rmean is None else rmean.data_ptr(), 0 if rvar is None else rvar.data_ptr(),
                     0 if nbt is None else nbt.data_ptr(), float(momentum), float(eps), int(relu), M, Ch,
                     W if pool else 0, slot, MAX_CTAS, s, dtype, 0 if res is None else res.data_ptr())
        ctx.save_for_backward(x, gamma, beta, stats, arg, res)
        ctx.relu, ctx.pool, ctx.slot, ctx.dtype = bool(relu), bool(pool), slot, dtype
        return y

    @staticmethod
    def backward(ctx, dy):
        C = ext.require()
        x, gamma, beta, stats, arg, res = ctx.saved_tensors
        N, Ch, H, W = x.shape
        M = N * H * W
        assert dy.dtype == x.dtype, (dy.dtype, x.dtype)          # y was allocated in x.dtype
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        dx = torch.empty_like(x)
        partial = _partial(C, x, M, Ch, W if ctx.pool else 0)
        dgb = torch.empty(2 * Ch, dtype=torch.float32, device=x.device)         # [dgamma | dbeta]
        dres = None if res is None else torch.empty_like(x)                       # dy masked by the ReLU
        s = torch.cuda.current_stream().cuda_stream
        C.bn_backward(x.data_ptr(), dy.data_ptr(), 0 if arg is None else arg.data_ptr(), dx.data_ptr(),
                      0 if partial is None else partial.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                      stats.data_ptr(), stats.data_ptr() + 4 * Ch, dgb.data_ptr(), dgb.data_ptr() + 4 * Ch, int(ctx.relu), M, Ch, W if ctx.pool else 0, ctx.slot, MAX_CTAS, s,
                      ctx.dtype, 0 if res is None else res.data_ptr(), 0 if dres is None else dres.data_ptr())
        # conv bias: the loss does not depend on it (see module docstring) -> no gradient
        return dx, dgb[:Ch], dgb[Ch:], None, None, None, None, None, None, None, None, None, dres


def _check_residual(residual: Optional[torch.Tensor], relu: bool, pool: Optional[torch.nn.MaxPool2d]) -> None:
    if residual is not None and (not relu or pool is not None):
        raise ValueError("a residual is added before the ReLU: it needs relu=True and pool=None")


def bias_bn_relu(x: torch.Tensor, bn: torch.nn.BatchNorm2d, conv_bias: Optional[torch.Tensor] = None,
                 relu: bool = True, pool: Optional[torch.nn.MaxPool2d] = None, fp16: bool = False,
                 residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``pool(relu(bn(x + conv_bias)))`` (``relu=False``: without the ReLU; ``pool=None``: without the pool;
    ``fp16``: fp16 activations and fp16 autocast take the fused kernels too).  With a ``residual`` (the end of a
    ResNet block; ``relu=True`` and ``pool=None`` only): ``relu(bn(x + conv_bias) + residual)``."""
    _check_residual(residual, relu, pool)
    if (_fast_path_ok(x, bn, fp16) and (conv_bias is None or conv_bias.dtype == torch.float32)
            and (residual is None or _residual_ok(x, residual))):
        if residual is not None and not residual.is_contiguous(memory_format=torch.channels_last):
            residual = residual.contiguous(memory_format=torch.channels_last)
        track = bn.track_running_stats and bn.running_mean is not None
        fuse = pool is not None and _pool_fusable(x, pool)
        y = _BiasBNReLUPool.apply(x, bn.weight, bn.bias, conv_bias, bn.running_mean if track else None,
                                  bn.running_var if track else None, bn.num_batches_tracked if track else None,
                                  bn.momentum, bn.eps, relu, fuse, _sync_slot(bn), residual)
        return y if pool is None or fuse else max_pool_2x2(y, pool)
    if conv_bias is not None:
        x = x + conv_bias.view(1, -1, 1, 1)
    y = bn(x)
    if residual is not None:
        return F.relu(y + residual)
    y = F.relu(y) if relu else y
    return y if pool is None else max_pool_2x2(y, pool)


def conv_bn_relu(x: torch.Tensor, conv: torch.nn.Conv2d, bn: torch.nn.BatchNorm2d, relu: bool = True,
                 pool: Optional[torch.nn.MaxPool2d] = None, fp16: bool = False,
                 residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``pool(relu(bn(conv(x))))`` with the convolution's bias folded into the fused batch-norm when the fast path
    applies (``fp16``: see ``bias_bn_relu``); with a ``residual``, ``relu(bn(conv(x)) + residual)``."""
    _check_residual(residual, relu, pool)
    if _fast_path_ok_pre(x, conv, bn, fp16):
        z = F.conv2d(x, conv.weight, None, conv.stride, conv.padding, conv.dilation, conv.groups)
        if _fast_path_ok(z, bn, fp16):
            return bias_bn_relu(z, bn, conv.bias, relu, pool, fp16, residual)
        if conv.bias is not None:
            z = z + conv.bias.view(1, -1, 1, 1)
        y = bn(z)
    else:
        y = bn(conv(x))
    if residual is not None:
        return F.relu(y + residual)
    y = F.relu(y) if relu else y
    return y if pool is None else max_pool_2x2(y, pool)


def _fast_path_ok_pre(x: torch.Tensor, conv: torch.nn.Conv2d, bn: torch.nn.BatchNorm2d, fp16: bool = False) -> bool:
    return (x.is_cuda and _dtype_ok(x, fp16) and bn.training and bn.affine and bn.momentum is not None
            and conv.out_channels % 4 == 0 and conv.padding_mode == "zeros" and ext.available()
            and (conv.bias is None or conv.bias.dtype == torch.float32) and _bn_params_fp32(bn)
            and x.is_contiguous(memory_format=torch.channels_last) and not isinstance(conv.padding, str))


class _MaxPool2x2(torch.autograd.Function):
    """2x2 / stride-2 max pooling on channels_last fp32 (``csrc/bnrelu.cu``): the backward pass writes every input position
    (no memset, no atomics: stride-2 windows do not overlap)."""

    @staticmethod
    def forward(ctx, x):
        C = ext.require()
        N, Ch, H, W = x.shape
        y = torch.empty((N, Ch, H // 2, W // 2), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        arg = torch.empty(y.numel(), dtype=torch.uint8, device=x.device)
        C.maxpool2_fwd(x.data_ptr(), y.data_ptr(), arg.data_ptr(), N, H, W, Ch, torch.cuda.current_stream().cuda_stream)
        ctx.save_for_backward(arg)
        ctx.shape = (N, Ch, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        C = ext.require()
        (arg,) = ctx.saved_tensors
        N, Ch, H, W = ctx.shape
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        dx = torch.empty((N, Ch, H, W), dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
        C.maxpool2_bwd(dy.data_ptr(), arg.data_ptr(), dx.data_ptr(), N, H, W, Ch, torch.cuda.current_stream().cuda_stream)
        return dx


def max_pool_2x2(x: torch.Tensor, pool: torch.nn.MaxPool2d) -> torch.Tensor:
    """A pool that does not directly follow a fused batch-norm run (or could not be folded into it)."""
    if (_is_2x2(pool) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.size(1) % 4 == 0
            and x.size(2) % 2 == 0 and x.size(3) % 2 == 0 and x.is_contiguous(memory_format=torch.channels_last)
            and ext.available() and torch.is_grad_enabled() and not torch.is_autocast_enabled()):
        return _MaxPool2x2.apply(x)
    return pool(x)


def run_fused_sequential(seq: torch.nn.Sequential, x: torch.Tensor, fp16: bool = False) -> torch.Tensor:
    """Run an ``nn.Sequential`` fusing every ``Conv2d -> BatchNorm2d [-> ReLU] [-> MaxPool2d]`` run it contains
    (``fp16``: see ``bias_bn_relu``)."""
    mods = list(seq.children())
    i = 0
    while i < len(mods):
        m = mods[i]
        if isinstance(m, torch.nn.Conv2d) and i + 1 < len(mods) and isinstance(mods[i + 1], torch.nn.BatchNorm2d):
            relu = i + 2 < len(mods) and isinstance(mods[i + 2], torch.nn.ReLU)
            j = i + (3 if relu else 2)
            pool = mods[j] if j < len(mods) and isinstance(mods[j], torch.nn.MaxPool2d) else None
            x = conv_bn_relu(x, m, mods[i + 1], relu, pool, fp16)
            i = j + (1 if pool is not None else 0)
        elif isinstance(m, torch.nn.MaxPool2d):
            x = max_pool_2x2(x, m)
            i += 1
        elif isinstance(m, torch.nn.AvgPool2d) and m.kernel_size in (1, (1, 1)) and m.stride in (1, (1, 1)):
            i += 1                                     # 1x1 average pool: the identity (VGG/models/vgg.py:37), no kernel
        else:
            x = m(x)
            i += 1
    return x
