"""Whole-step CUDA graphs: forward + backward + fused sparse allreduce + fused optimizer update
captured once per *iteration type* and replayed.

Small-batch workloads (VGG-16 at 16 images/GPU, the reference's configuration) are launch bound: a
step is several hundred kernels of a few microseconds each.  Everything on our path is capturable
because nothing depends on host-visible values: thresholds, region edges, slot cursors, flag epochs
and the learning rate live in device memory, and the persistent cooperative kernel is a normal graph
node.  The only host-side variation is *which* flavour of the kernel a step needs (exact threshold
re-computation / region re-partition iterations, SURVEY 3.3): each engine's ``plan_call``.  One graph
is captured per flavour the first time it occurs and the host picks the graph from the iteration counter.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from ..ops import ext
from ..parallel.state import plan_call, schedule_period
from .data import PaddedAN4Batch
from .trainer import Trainer

# Padded AN4 input shapes (one per T_b at a fixed batch size) that get graphs; batches of further shapes run eagerly.
# Each shape holds a graph per flavour; at m = 32 the synthetic AN4 utterances (96-396 frames) pad to 11 lengths.
MAX_AN4_SHAPES = 16


def ptb_graph_error(net, autocast: Optional[torch.dtype]) -> Optional[str]:
    """Why the PTB language model ``net`` (a ``PTBLSTM``) does not get graphed steps under ``autocast`` (None: fp32), or
    None when it does: the fused stacked-layer LSTM in bf16, fp16 and fp32, and the stock cuDNN layer in fp32, are the
    configurations whose graphed steps are checked against eager ones bit for bit."""
    if net.fuse_lstm and (autocast is not None or net.fuse_lstm_fp32):
        return None
    if autocast is not None:
        return ("the stock nn.LSTM under %s autocast has no graphed step: set fuse_lstm (--fused-lstm-lm) for the "
                "fused 16-bit layers" % str(autocast).replace("torch.", ""))
    return None


class _FixedShape:
    """The input rule of fixed-shape batches (VGG, the ResNets, BERT; a trainer without ``dataset``): one static copy of
    the batch, and a batch of another shape disables the graph step.  Every rule answers: ``why_disabled`` ("" when
    graphs apply); ``inputs(batch)``, for a ``stage``d batch: (the static inputs holding it, the key prefix or None), or
    a string, a ``fallbacks`` counter (this step runs eagerly) or else why the graph step disables itself; and what ends
    a capture: ``store()`` inside the graph, ``rebind()`` after it."""
    fallbacks = ("shapes", "targets")

    def __init__(self, tr):
        self.tr = tr
        self.why_disabled = ""
        self._static_of: Dict[Optional[Tuple], tuple] = {}      # by key prefix

    def stage(self, batch):
        return batch

    def inputs(self, batch):
        return self._fill(None, batch) or "batch shape changed"

    def _fill(self, prefix, batch):
        """(static inputs of ``prefix`` holding ``batch``, ``prefix``); None, the copy stopped, at a shape not theirs."""
        static = self._static_of.get(prefix)
        if static is None:
            vals = [t.clone() if torch.is_tensor(t) else t for t in batch]
            static = self._static_of[prefix] = type(batch)(*vals) if isinstance(batch, PaddedAN4Batch) else tuple(vals)
        for s, t in zip(static, batch):
            if torch.is_tensor(t):
                if s.shape != t.shape:
                    return None
                s.copy_(t, non_blocking=True)
        return static, prefix

    def rebind(self) -> None:
        """After every capture, a failed one too: point the trainer back at the state the graphs read."""

    def store(self) -> None:
        """Inside a capture, after the update: the graph's last nodes."""


class _PaddedAN4(_FixedShape):
    """AN4 batches staged by the trainer's ``an4_pad_multiple`` (``data.PaddedAN4Batch``: frames padded to a multiple of
    m, lengths on the device, targets in a fixed-capacity buffer): static inputs per padded shape, keys (shape, flavour).
    Past ``MAX_AN4_SHAPES`` shapes, or over the target capacity, a step runs eagerly on the same padded form.  Needs
    every LSTM layer fused and the fused CTC loss, the two parts that read the lengths on the device."""

    def __init__(self, tr):
        super().__init__(tr)
        self.why_disabled = tr.net.device_lengths_error(True, tr.autocast is not None) or ""
        if not self.why_disabled and not getattr(tr.net, "fuse_ctc", False):
            self.why_disabled = "fuse_ctc is off: the stock CTC loss copies the lengths to the host"

    def stage(self, batch):
        return self.tr.stage_batch(batch)

    def inputs(self, batch):
        if batch.over_capacity:
            return "targets"
        shape = tuple(batch.inputs.shape)
        if shape not in self._static_of and len(self._static_of) >= MAX_AN4_SHAPES:
            return "shapes"
        return self._fill(shape, batch) or "batch shape changed"


class _CarriedState(_FixedShape):
    """The PTB language model's (h, c), carried across batches: the graphs read it from one static pair ``state``
    [L, N, H] (h in the autocast type on the 16-bit fused path, c fp32) and, as their last node, copy the step's
    (h_n, c_n) into it; ``Trainer.hidden`` *is* that pair between replays.  A short batch, or a state whose dtypes are
    not the pair's, runs that step eagerly and the graphs stay.  Needs ``ptb_graph_error`` to be None."""
    fallbacks = ("shapes", "state")

    def __init__(self, tr):
        super().__init__(tr)
        self.why_disabled = ptb_graph_error(tr.net, tr.autocast) or ""
        self.state: Optional[Tuple[torch.Tensor, torch.Tensor]] = None      # allocated at the first graphed step

    def inputs(self, batch):
        placed = self._fill(None, batch)
        if placed is None:
            return "shapes"
        return placed if self._load(batch[0].size(0)) else "state"

    def _load(self, n: int) -> bool:
        """Before a replay, make ``hidden`` (a reset, ``Trainer.test()``'s, an eager step's) the static pair for ``n``
        sequences by the eager step's rule (``Trainer._forward_loss_impl``): None or another batch size starts from
        zeros, anything else is carried in exactly.  False (nothing changed) when its dtypes are not the pair's."""
        tr = self.tr
        st = self.state
        if st is None:
            shape = (tr.net.num_layers, n, tr.net.embedding_dim)
            h_dt = tr.autocast if tr.net.fuse_lstm and tr.autocast is not None else torch.float32
            st = self.state = (torch.empty(shape, dtype=h_dt, device=tr.device),
                               torch.empty(shape, dtype=torch.float32, device=tr.device))
        hid = tr.hidden
        if hid is not None and hid[0] is st[0] and hid[1] is st[1]:
            return True
        if hid is None or hid[0].size(1) != st[0].size(1):
            for s in st:
                s.zero_()
        elif all(h.dtype == s.dtype and h.shape == s.shape for h, s in zip(hid, st)):
            # detached: a copy from a tensor with autograd history would attach that history to the pair and keep the
            # eager step's graph (its AccumulateGrad nodes, bound to the stream they were made on) alive into a capture
            for h, s in zip(hid, st):
                s.copy_(h.detach())
        else:
            return False
        tr.hidden = st
        return True

    def rebind(self) -> None:
        self.tr.hidden = self.state              # after a failed capture nothing ran: the pair holds this step's state

    def store(self) -> None:
        """Copy the step's (h_n, c_n) into the static pair.  Last, because the backward pass reads (h0, c0) from it."""
        for s, h in zip(self.state, self.tr.hidden):
            if h.dtype != s.dtype or h.shape != s.shape:
                raise RuntimeError("the carried state comes back as %s %s, the static buffer is %s %s"
                                   % (h.dtype, tuple(h.shape), s.dtype, tuple(s.shape)))
            s.copy_(h.detach())


class GraphedTrainStep:
    def __init__(self, trainer, warmup_eager: int = 3):
        self.tr = trainer
        self.opt = trainer.optimizer
        rules = {"an4": _PaddedAN4, "ptb": _CarriedState}      # what depends on the batch: one input rule per kind
        self.rule = rules.get(getattr(trainer, "dataset", None), _FixedShape)(trainer)
        self.why_disabled = self.rule.why_disabled
        self.enabled = not self.why_disabled
        self.fallbacks = dict.fromkeys(self.rule.fallbacks, 0)      # the steps that ran eagerly, by the rule's reason
        self.graphs: Dict[Tuple, torch.cuda.CUDAGraph] = {}
        self.launches: Dict[Tuple, int] = {}
        self.static_loss: Optional[torch.Tensor] = None
        self.eager_left = warmup_eager
        self.pool = None
        self._loss_of: Dict[Tuple, torch.Tensor] = {}
        self._inputs_of: Dict[Tuple, tuple] = {}      # the static inputs each graph reads
        self._precaptured = set()                      # the key prefixes whose sparse flavours are all captured

    @property
    def _state(self) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:      # the PTB rule's static (h, c) pair
        return getattr(self.rule, "state", None)

    # ------------------------------------------------------------------ iteration flavour
    def _engines(self):
        return [self.opt._allreducer._engines.get(b.name) for b in self.opt._buckets]

    def _key(self, counters=None) -> Tuple:
        """The flavour of the step the engines are about to run (or would run at the given iteration counters): the
        density (k and the guard limits are baked into the launch) followed by every engine's ``CallPlan``."""
        engines = self._engines()
        if any(e is None for e in engines):
            return ("nograph",)
        if counters is None:
            counters = [e.host.counter for e in engines]
        cfg, density = self.opt._cfg, self.opt.get_current_density()
        name = self.opt._allreducer.compressor.name
        return (density,) + tuple(plan_call(cfg, name, c, density, e.P) for e, c in zip(engines, counters))

    def _sparse_flavours(self):
        """Every (key, representative sparse-iteration index) the schedule can produce -- a handful: for Ok-Topk the
        common threshold-reuse step, the exact-threshold step (1 in tau) and, at P > 1, the exact + re-partition step."""
        cfg = self.opt._cfg
        seen = {}
        n_eng = len(self._engines())
        for it in range(min(schedule_period(cfg, self.opt._allreducer.compressor.name), 1 << 16)):
            seen.setdefault(self._key([cfg.warmup_iters + it] * n_eng), it)
        return seen

    def precapture_sparse(self, static, prefix) -> None:
        """Capture the graph of EVERY sparse-phase flavour of the static inputs ``static`` (key prefix ``prefix``) now
        (capturing records launches, it executes nothing), so that the rare exact-threshold / re-partition iterations are
        replayed like the common one instead of running eagerly inside somebody's timed region.  Engine iteration
        counters are faked for the capture and restored.  Called by ``step`` when every engine has a plan."""
        cfg = self.opt._cfg
        if not cfg.sparse:
            return
        engines = self._engines()
        real = [e.host.counter for e in engines]
        for flavour, it in self._sparse_flavours().items():
            key = flavour if prefix is None else (prefix, flavour)
            if key in self.graphs or flavour == ("nograph",):
                continue
            for e in engines:
                e.host.counter = cfg.warmup_iters + it
            self._inputs_of[key] = static
            if self._capture(key) is None:
                break
        for e, c in zip(engines, real):
            e.host.counter = c
        if not self._precaptured:
            # every long-lived object of the training process exists now (model, optimizer state, engines, graphs): move
            # them to the permanent generation so that the cyclic collector's full passes stop walking them -- a
            # generation-2 collection otherwise stalls a 1.2 ms step loop for tens of milliseconds.  Once only: a later
            # padded AN4 length adds a few graphs and static inputs, not worth a pause of that size each, and freezing
            # again would also pin whatever garbage exists at that moment
            import gc
            gc.collect()
            gc.freeze()
        self._precaptured.add(prefix)

    # ------------------------------------------------------------------ one step
    def _eager(self, batch) -> torch.Tensor:
        self.opt.zero_grad()
        loss = Trainer._forward_backward(self.tr, batch)
        self.tr.update_model()
        return loss.detach()

    def step(self, batch) -> torch.Tensor:
        """Run one optimizer step on ``batch`` (device tensors; the input rule stages it); returns the (device) loss."""
        batch = self.rule.stage(batch)
        if not self.enabled or self.eager_left > 0:
            self.eager_left -= 1
            return self._eager(batch)
        flavour = self._key()
        if flavour == ("nograph",):
            return self._eager(batch)
        placed = self.rule.inputs(batch)
        if isinstance(placed, str):
            if placed in self.fallbacks:         # this step eagerly, the graphs stay
                self.fallbacks[placed] += 1
            else:
                self.enabled, self.why_disabled = False, placed
            return self._eager(batch)
        static, prefix = placed
        key = flavour if prefix is None else (prefix, flavour)      # the graph key, as in precapture_sparse
        self.opt.refresh_lr()
        if prefix not in self._precaptured and all(plan.kind != "dense" for plan in flavour[1:]):
            self.precapture_sparse(static, prefix)   # first sparse step (of this shape): capture every flavour at once
        g = self.graphs.get(key)
        if g is None:
            self._inputs_of[key] = static
            g = self._capture(key)
            if g is None:
                return self._eager(batch)
        for eng in self._engines():
            eng.host.counter += 1
        if hasattr(self.opt, "counter"):
            self.opt.counter += 1
        g.replay()
        self.opt._allreducer.poll_faults()       # pinned host mirror of the device fault words: a plain load per bucket
        ext.LAUNCH_COUNT["total"] += self.launches.get(key, 0)
        self.static_loss = self._loss_of[key]
        return self.static_loss

    def _capture(self, key) -> Optional[torch.cuda.CUDAGraph]:
        """Capture the step on the static inputs of ``key``; None when that fails, which disables the graph step."""
        counters = [eng.host.counter for eng in self._engines()]
        opt_counter = getattr(self.opt, "counter", None)
        l0 = ext.LAUNCH_COUNT["total"]
        g = torch.cuda.CUDAGraph()
        try:
            torch.cuda.synchronize()
            with torch.cuda.graph(g, pool=self.pool):
                self.opt.zero_grad()
                loss = Trainer._forward_backward(self.tr, self._inputs_of[key])
                self.tr.update_model()
                out = loss.detach()
                self.rule.store()
        except Exception as e:  # noqa: BLE001 - fall back to eager for good
            self.enabled, self.why_disabled, g = False, "capture failed: %r" % (e,), None
            try:
                torch.cuda.synchronize()
            except Exception:  # noqa: BLE001
                pass
            self.opt._after_step()
        self.rule.rebind()
        # capture executed the Python side effects (counters) but no kernels: undo them, the replay is the real step
        for eng, c in zip(self._engines(), counters):
            eng.host.counter = c
        if opt_counter is not None:
            self.opt.counter = opt_counter
        if g is None:
            return None
        # each graph writes a loss buffer of its own; static_loss is the one of the latest capture or replay
        self.static_loss = self._loss_of[key] = out
        if self.pool is None:
            self.pool = g.pool()
        self.launches[key] = ext.LAUNCH_COUNT["total"] - l0
        ext.LAUNCH_COUNT["total"] = l0
        self.graphs[key] = g
        return g
