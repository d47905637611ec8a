"""Per-bucket algorithm state shared by the oracle, the torch.distributed path and the CUDA engine.

The reference keeps this in dicts keyed by the joined parameter names
(``VGG/allreducer.py:312-320``: ``_allreduce_counter``, ``_local_threshold``,
``_global_threshold``, ``_boundaries``, ``_region_offsets``) plus the compressor's class-level
``residuals`` dict (``VGG/compression.py:170``).  Here it is one object per bucket, and it is
checkpointable (the reference never saves any of it, SURVEY 5.4).

``plan_call`` decides from the bucket counter what one reduction runs; the CUDA engine, the dist backend, the oracle
and the whole-step CUDA graphs all follow it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

# the kernel family that runs each scheme; the automatic dense switch applies exactly to the "fused" family
FAMILY = {
    "oktopk": "fused", "topkSA": "fused", "topkDSA": "fused", "gaussiankSA": "fused",
    "topkA": "gather", "topkA2": "gather", "topkAopt": "gather", "gaussiank": "gather", "gaussiankconcat": "gather",
    "gtopk": "tree",
}


@dataclass(frozen=True)
class CallPlan:
    """What one bucket reduction runs.  ``kind``: ``"dense"`` (warm-up, ``compressor none``, ``sparse=False``),
    ``"dense_switch"`` or the scheme's ``FAMILY``.  The flags are set only where the launch differs: Ok-Topk's exact
    local threshold, exact global top-k and region re-partition (only at P > 1), and TopkAopt's exact-threshold
    iteration in ``exact_local``.  Equal plans launch the same kernels, so a plan keys a captured CUDA graph."""

    kind: str
    exact_local: bool = False
    exact_global: bool = False
    repartition: bool = False


def plan_call(cfg, compressor: Optional[str], counter: int, density: Optional[float], world_size: int) -> CallPlan:
    """The plan of the reduction a bucket runs at ``counter`` (its completed reductions, warm-up included).  ``density``
    None means ``cfg.density``.  An unknown compressor raises ``KeyError``."""
    if not cfg.sparse or compressor in ("none", None) or counter < cfg.warmup_iters:
        return CallPlan("dense")
    family = FAMILY[compressor]
    d = cfg.density if density is None else density
    if family == "fused" and world_size > 1 and cfg.dense_switch_density > 0 and d >= cfg.dense_switch_density:
        # predicted slower than the dense kernel at this density: the error-compensated gradient is reduced densely
        return CallPlan("dense_switch")
    it = counter - cfg.warmup_iters
    if compressor == "oktopk":
        return CallPlan(family, exact_local=it % cfg.local_recompute_interval == 0,
                        exact_global=it % cfg.global_recompute_interval == 0,
                        repartition=world_size > 1 and it % cfg.repartition_interval == 0)
    if compressor == "topkAopt":
        return CallPlan(family, exact_local=it % cfg.topkaopt_recompute_interval == 0)
    return CallPlan(family)


def schedule_period(cfg, compressor: Optional[str]) -> int:
    """Sparse iterations after which ``plan_call`` repeats itself."""
    if compressor == "oktopk":
        return math.lcm(cfg.local_recompute_interval, cfg.global_recompute_interval, cfg.repartition_interval)
    if compressor == "topkAopt":
        return cfg.topkaopt_recompute_interval
    return 1


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
