"""Flat gradient buckets ("tensor fusion", C4) -- gradients are *views* into persistent flat buffers.

The reference copies every gradient into a merged buffer in ``_push_to_buffer`` and slices the
result back in ``_pull_from_buffer`` (``VGG/allreducer.py:272-366``); BERT ``torch.cat``s 534 MB per
step (``optimization.py:149-170``).  Here ``p.grad`` aliases the bucket (autograd accumulates
straight into it), parameters and optimizer state optionally alias equally laid-out flat buffers so
that the optimizer step is one fused kernel per bucket, and the bucket itself is a symmetric
peer-mapped allocation that the dense kernel reduces in place.

Bucketing follows the reference: parameters in reverse registration (= backward) order, a new
bucket once the running size reaches the threshold (``THRESHOLD = 640 Mi`` elements there, i.e. one
bucket; ``OkTopkConfig.bucket_elems`` here).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

ALIGN = 64   # elements: keeps every parameter 256-byte aligned inside the flat buffers (cuDNN/cuBLAS friendly)


@dataclass
class Bucket:
    index: int
    name: str
    params: List[torch.nn.Parameter]
    names: List[str]
    offsets: List[int]
    numel: int
    group_slices: List[Tuple[int, int, int]] = field(default_factory=list)   # (group index, start, end)
    grad: Optional[torch.Tensor] = None
    flat_param: Optional[torch.Tensor] = None
    grad_views: Optional[List[torch.Tensor]] = None
    pending: int = 0
    launched: bool = False
    dirty: bool = True
    event: Optional["torch.cuda.Event"] = None
    held: Optional[List[torch.Tensor]] = None      # gradient tensors a running reduction reads (until synchronize())

    def views(self, flat: torch.Tensor) -> List[torch.Tensor]:
        """Per-parameter aliases of a flat buffer with the PARAMETER'S OWN memory layout: a channels_last conv weight
        gets a channels_last view, so flat parameters, gradients and optimizer state stay element-wise aligned whatever
        the layout (the flat kernels are element-wise, the sparse allreduce is permutation-agnostic)."""
        out = []
        for p, o in zip(self.params, self.offsets):
            sl = flat[o:o + p.numel()]
            if p.is_contiguous() or not _dense_non_overlapping(p):
                out.append(sl.view_as(p))
            else:
                out.append(sl.as_strided(p.size(), p.stride()))
        return out


def _dense_non_overlapping(t: torch.Tensor) -> bool:
    """True if the tensor's elements occupy exactly numel() consecutive storage slots (any permutation of dims)."""
    if t.numel() <= 1:
        return True
    dims = sorted(((st, sz) for st, sz in zip(t.stride(), t.size()) if sz > 1))
    expect = 1
    for st, sz in dims:
        if st != expect:
            return False
        expect *= sz
    return True


def _align(x: int) -> int:
    return (x + ALIGN - 1) // ALIGN * ALIGN


def build_buckets(param_groups: Sequence[dict], names: Dict[torch.nn.Parameter, str], bucket_elems: int) -> List[Bucket]:
    """Reverse-order bucketing.  Inside a bucket parameters are ordered by param group so that each
    group (own lr / weight decay) is one contiguous slice for the fused optimizer kernel."""
    ordered: List[Tuple[int, torch.nn.Parameter]] = []
    for gi, g in enumerate(param_groups):
        for p in g["params"]:
            if p.requires_grad:
                ordered.append((gi, p))
    # registration order == order of appearance; backward produces gradients roughly in reverse
    ordered = ordered[::-1]
    raw: List[List[Tuple[int, torch.nn.Parameter]]] = []
    cur, size = [], 0
    for gi, p in ordered:
        cur.append((gi, p))
        size += _align(p.numel())
        if size >= bucket_elems:
            raw.append(cur)
            cur, size = [], 0
    if cur:
        raw.append(cur)
    buckets = []
    for bi, members in enumerate(raw):
        members = sorted(members, key=lambda m: m[0])      # stable: keeps reverse order inside a group
        params, pnames, offsets, slices = [], [], [], []
        off, cur_g, g_start = 0, None, 0
        for gi, p in members:
            if cur_g is None:
                cur_g, g_start = gi, off
            elif gi != cur_g:
                slices.append((cur_g, g_start, off))
                cur_g, g_start = gi, off
            params.append(p)
            pnames.append(names.get(p, "allreduce.noname.%d" % len(params)))
            offsets.append(off)
            off += _align(p.numel())
        slices.append((cur_g, g_start, off))
        buckets.append(Bucket(index=bi, name="bucket%d:%s" % (bi, pnames[0]), params=params, names=pnames,
                              offsets=offsets, numel=off, group_slices=slices))
    return buckets


def attach(bucket: Bucket, grad_flat: torch.Tensor, flatten_params: bool) -> None:
    """Alias ``p.grad`` (and optionally ``p.data``) to the flat buffers."""
    assert grad_flat.numel() >= bucket.numel
    bucket.grad = grad_flat
    with torch.no_grad():
        if flatten_params:
            fp = torch.zeros(bucket.numel, dtype=torch.float32, device=grad_flat.device)
            for p, v in zip(bucket.params, bucket.views(fp)):
                v.copy_(p.data)
                p.data = v
            bucket.flat_param = fp
        bucket.grad_views = bucket.views(grad_flat)
        for p, v in zip(bucket.params, bucket.grad_views):
            p.grad = v
