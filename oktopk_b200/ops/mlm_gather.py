"""Fixed-capacity gather of BERT's labelled masked-LM rows (``csrc/mlm_gather.cu``).

``gather_labelled(x, labels, capacity, ignore_index, overflow)`` takes the rows ``x [R, H]`` and their masked-LM
labels ``[R]`` and returns ``(xg [M, H], tgt [M])`` with ``M = capacity``: the rows whose label is not
``ignore_index`` and their labels, so that the head's transform and decoder GEMMs and the loss run on M rows instead
of R while every shape stays fixed by the batch shape (CUDA graphs, recompute and loss scaling work unchanged).

The contract:

* row order is kept: slot s holds the s-th labelled row;
* padding rows (the slots past the number of labelled rows) are zero and carry ``ignore_index``, so the loss skips them;
* labelled rows past the capacity are left out of ``xg`` and of the loss, and ``max(count - M, 0)`` is added to
  ``overflow`` (a device int64 that accumulates over calls; nothing is read on the host);
* the gradient of ``x`` is the gradient of ``xg`` on the gathered rows and exactly 0 on every other row (unlabelled or
  past the capacity).  ``labels`` gets no gradient.

On CUDA with the native extension, for fp32, bf16 or fp16 ``x``, the forward pass is two launches (select, gather) and
the backward pass one (scatter, which writes every row of the gradient once); no host synchronisation.  Everywhere else
(CPU tensors, no extension, another dtype, a ``labels`` that is not int64 ``[R]`` on ``x``'s device) the same
semantics run in torch: the same slots, the same padding and the same overflow rule.

``capacity_rows(R, fraction)`` is the capacity the models use: ``fraction · R`` rounded up to a multiple of 8
(256 at 8 × 128 tokens and 0.25); a fraction of 1.0 can never overflow.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

from . import ext
from .ext import DTYPE_CODE


def capacity_rows(R: int, fraction: float) -> int:
    """The gathered rows for ``R`` token rows: ``fraction · R`` rounded up to a multiple of 8, ``0 < fraction <= 1``."""
    if not 0.0 < fraction <= 1.0:
        raise ValueError("mlm_capacity must be in (0, 1], got %r" % (fraction,))
    return 8 * max(1, math.ceil(fraction * R / 8))


def _native_ok(labels: torch.Tensor, capacity: int, x: Optional[torch.Tensor] = None) -> bool:
    if not (labels.is_cuda and labels.dtype == torch.int64 and labels.dim() == 1 and ext.available()):
        return False
    R = labels.numel()
    if not (0 < R < 2 ** 31 and 0 < capacity < 2 ** 31):
        return False
    if x is None:
        return True
    return (x.dim() == 2 and x.size(0) == R and 0 < x.size(1) < 2 ** 31 and x.dtype in DTYPE_CODE
            and x.device == labels.device)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def select_labelled(labels: torch.Tensor, capacity: int, ignore_index: int = -1,
                    overflow: Optional[torch.Tensor] = None
                    ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """``(rows [M] int32, tgt [M] int64, slot [R] int32, count 0-d int64)`` for ``labels [R]`` and ``M = capacity``: the
    source row of each slot (-1: padding), its label (``ignore_index``: padding), each row's slot (-1: unlabelled or
    past the capacity) and the number of labelled rows.  ``overflow`` (one int64, or None) accumulates
    ``max(count - M, 0)``."""
    M = int(capacity)
    if M <= 0:
        raise ValueError("capacity must be positive, got %d" % M)
    dev = labels.device
    if _native_ok(labels, M):
        C = ext.require()
        R = labels.numel()
        labels = labels.contiguous()
        rows = torch.empty(M, dtype=torch.int32, device=dev)
        tgt = torch.empty(M, dtype=torch.int64, device=dev)
        slot = torch.empty(R, dtype=torch.int32, device=dev)
        count = torch.empty((), dtype=torch.int64, device=dev)
        ov = 0
        if overflow is not None:
            if not (overflow.is_cuda and overflow.dtype == torch.int64 and overflow.numel() == 1
                    and overflow.is_contiguous() and overflow.device == dev):
                raise ValueError("overflow must be one contiguous int64 on the labels' device")
            ov = overflow.data_ptr()
        C.mlm_select(labels.data_ptr(), rows.data_ptr(), tgt.data_ptr(), slot.data_ptr(), count.data_ptr(), ov, R, M,
                     int(ignore_index), _stream())
        return rows, tgt, slot, count
    labels = labels.reshape(-1)
    R = labels.numel()
    on = labels != ignore_index
    pos = torch.cumsum(on, 0) - 1
    kept = on & (pos < M)
    slot = torch.where(kept, pos, -1)
    count = on.sum()
    # every row that is not kept lands in the extra slot M, which is cut off
    rows = torch.full((M + 1,), -1, dtype=torch.int64, device=dev)
    rows.scatter_(0, torch.where(kept, pos, M), torch.arange(R, device=dev))
    rows = rows[:M]
    tgt = torch.cat([labels, labels.new_full((1,), ignore_index)])[torch.where(rows >= 0, rows, R)]
    if overflow is not None:
        overflow.add_((count - M).clamp(min=0).to(overflow.dtype))
    return rows.to(torch.int32), tgt, slot.to(torch.int32), count


def _copy_rows(src: torch.Tensor, idx: torch.Tensor, native: bool, gather: bool) -> torch.Tensor:
    """``out[d] = src[idx[d]]`` where ``idx[d] >= 0``, else 0, for every d."""
    n, H = idx.numel(), src.size(1)
    if native:
        C = ext.require()
        src = src.contiguous()
        out = torch.empty(n, H, dtype=src.dtype, device=src.device)
        fn = C.mlm_gather if gather else C.mlm_scatter
        fn(src.data_ptr(), idx.data_ptr(), out.data_ptr(), n, H, DTYPE_CODE[src.dtype], _stream())
        return out
    padded = torch.cat([src, src.new_zeros(1, H)])
    return padded[torch.where(idx >= 0, idx.long(), src.size(0))]


class _GatherLabelled(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, labels, capacity, ignore_index, overflow):
        native = _native_ok(labels, capacity, x)
        rows, tgt, slot, _ = select_labelled(labels, capacity, ignore_index, overflow)
        xg = _copy_rows(x, rows, native, gather=True)
        ctx.save_for_backward(slot)
        ctx.native = native
        ctx.mark_non_differentiable(tgt)
        return xg, tgt

    @staticmethod
    def backward(ctx, dxg, _dtgt):
        (slot,) = ctx.saved_tensors
        return _copy_rows(dxg, slot, ctx.native, gather=False), None, None, None, None


def gather_labelled(x: torch.Tensor, labels: torch.Tensor, capacity: int, ignore_index: int = -1,
                    overflow: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(xg [M, H], tgt [M])``: the rows of ``x [R, H]`` whose label is not ``ignore_index``, in row order, zero-padded
    to ``M = capacity`` rows; see the module docstring."""
    if x.dim() != 2 or labels.numel() != x.size(0):
        raise ValueError("gather_labelled needs x [R, H] and labels [R], got %s and %s"
                         % (tuple(x.shape), tuple(labels.shape)))
    return _GatherLabelled.apply(x, labels.reshape(-1), int(capacity), int(ignore_index), overflow)
