"""Per-bucket algorithm state shared by the oracle, the torch.distributed path and the CUDA engine.

The reference keeps this in dicts keyed by the joined parameter names
(``VGG/allreducer.py:312-320``: ``_allreduce_counter``, ``_local_threshold``,
``_global_threshold``, ``_boundaries``, ``_region_offsets``) plus the compressor's class-level
``residuals`` dict (``VGG/compression.py:170``).  Here it is one object per bucket, and it is
checkpointable (the reference never saves any of it, SURVEY 5.4).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch


def uniform_boundaries(n: int, P: int) -> List[int]:
    """``n // P`` per region, remainder on the last (``VGG/allreducer.py:1159-1164``)."""
    s = n // P
    b = [s] * P
    b[P - 1] += n - s * P
    return b


def offsets_of(boundaries: List[int]) -> List[int]:
    off, acc = [], 0
    for b in boundaries:
        off.append(acc)
        acc += b
    return off


@dataclass
class SparseState:
    """State of one bucket on one rank."""

    numel: int
    world: int
    counter: int = 0                       # completed reductions of this bucket (dense warm-up included)
    local_thr: float = 0.0
    global_thr: float = 0.0
    boundaries: List[int] = field(default_factory=list)      # region sizes, sum == numel
    region_offsets: List[int] = field(default_factory=list)  # region starts
    residual: Optional[torch.Tensor] = None
    # bookkeeping for observability (SURVEY 5.1/5.5)
    last_local_count: int = 0
    last_thr_used: float = 0.0             # Ok-Topk: threshold the last call selected with (after the guard), before adaptation
    last_global_count: int = 0
    last_volume_elems: int = 0             # scalars sent + received by this rank in the last call
    last_mode: str = ""

    def __post_init__(self):
        if not self.boundaries:
            self.boundaries = uniform_boundaries(self.numel, self.world)
            self.region_offsets = offsets_of(self.boundaries)

    def ensure_residual(self, like: torch.Tensor) -> torch.Tensor:
        if self.residual is None or self.residual.numel() != like.numel() or self.residual.device != like.device:
            self.residual = torch.zeros_like(like)
        return self.residual

    def state_dict(self) -> Dict:
        return {
            "numel": self.numel, "world": self.world, "counter": self.counter,
            "local_thr": float(self.local_thr), "global_thr": float(self.global_thr),
            "boundaries": list(self.boundaries), "region_offsets": list(self.region_offsets),
            "residual": None if self.residual is None else self.residual.detach().cpu().clone(),
        }

    def load_state_dict(self, sd: Dict, device=None) -> None:
        assert sd["numel"] == self.numel, "bucket size changed"
        self.counter = int(sd["counter"])
        self.local_thr = float(sd["local_thr"])
        self.global_thr = float(sd["global_thr"])
        if sd["world"] == self.world:
            self.boundaries = list(sd["boundaries"])
            self.region_offsets = list(sd["region_offsets"])
        else:  # elastic restart with a different world size: fall back to uniform regions
            self.boundaries = uniform_boundaries(self.numel, self.world)
            self.region_offsets = offsets_of(self.boundaries)
        r = sd.get("residual")
        if r is not None:
            self.residual = r.to(device) if device is not None else r.clone()
