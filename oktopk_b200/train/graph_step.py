"""Whole-step CUDA graphs: forward + backward + fused sparse allreduce + fused optimizer update
captured once per *iteration type* and replayed.

Small-batch workloads (VGG-16 at 16 images/GPU, the reference's configuration) are launch bound: a
step is several hundred kernels of a few microseconds each.  Everything on our path is capturable
because nothing depends on host-visible values: thresholds, region edges, slot cursors, flag epochs
and the learning rate live in device memory, and the persistent cooperative kernel is a normal graph
node.  The only host-side variation is *which* flavour of the kernel a step needs (exact threshold
re-computation / region re-partition iterations, SURVEY 3.3): each engine's ``plan_call``.  One graph
is captured per flavour the first time it occurs and the host picks the graph from the iteration counter.

AN4 batches vary in length.  With the trainer's ``an4_pad_multiple`` they arrive staged (``data.PaddedAN4Batch``):
frames padded to a multiple of m, lengths on the device, targets in a fixed-capacity buffer, so that a batch's shapes
depend on its padded length T_b only.  Graphs and static inputs are then keyed by (padded input shape, flavour), and
every flavour of a new T_b is captured the first time it appears.  At most ``MAX_AN4_SHAPES`` padded shapes get graphs;
a batch of another shape after that, or one whose targets exceed the capacity, runs that step eagerly on the same
padded form (counted in ``fallbacks``).  The step needs every LSTM layer fused and the fused CTC loss, the two parts that
read the lengths on the device; otherwise the graph step disables itself and the padded batches run eagerly.

The PTB language model carries (h, c) from one batch to the next.  Its graphs read the state from one static pair
[L, N, H] (h in the autocast type on the 16-bit fused path, c fp32; both fp32 in fp32) and, as their last node, after
backward and the update, copy the step's (h_n, c_n) into it; the trainer's ``hidden`` *is* that pair between replays.
Before a replay the eager step's rule is applied to whatever ``hidden`` is then (a reset, ``Trainer.test()``, an eager
step): None or another batch size zeroes the pair, anything else is copied in.  A batch of another shape (the short last
batch of an epoch), or a state whose dtypes differ from the pair's, runs that step eagerly (counted in ``fallbacks``)
and the graphs stay.  Graphed PTB needs the fused LSTM layers or the stock layer in fp32 (``ptb_graph_error``).
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from ..ops import ext
from ..parallel.state import plan_call, schedule_period
from .data import PaddedAN4Batch

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


def _clone(batch):
    vals = [t.clone() if torch.is_tensor(t) else t for t in batch]
    return type(batch)(*vals) if isinstance(batch, PaddedAN4Batch) else tuple(vals)


class GraphedTrainStep:
    def __init__(self, trainer, warmup_eager: int = 3):
        self.tr = trainer
        self.opt = trainer.optimizer
        self.graphs: Dict[Tuple, torch.cuda.CUDAGraph] = {}
        self.launches: Dict[Tuple, int] = {}
        self.static_in: Optional[Tuple[torch.Tensor, ...]] = None
        self.static_loss: Optional[torch.Tensor] = None
        self.eager_left = warmup_eager
        self.enabled = True
        self.pool = None
        self.why_disabled = ""
        self._cap_counters, self._cap_opt_counter = [], None
        self._loss_of: Dict[Tuple, torch.Tensor] = {}
        # AN4 (padded batches): static inputs per padded shape, the shapes whose sparse flavours are all captured, and
        # the steps that ran eagerly because their shape was past MAX_AN4_SHAPES or their targets past the capacity
        self.an4 = getattr(trainer, "dataset", None) == "an4"
        self._static_of: Dict[Tuple, tuple] = {}
        self._precaptured_shapes = set()
        self._shape: Optional[Tuple] = None
        self.fallbacks = {"shapes": 0, "targets": 0}
        # PTB: the static (h, c) every graph reads and writes back (allocated at the first graphed step); the steps that
        # ran eagerly because their batch had another shape or their carried state another dtype
        self.ptb = getattr(trainer, "dataset", None) == "ptb"
        self._state: Optional[Tuple[torch.Tensor, torch.Tensor]] = None
        if self.ptb:
            self.fallbacks = {"shapes": 0, "state": 0}
            why = ptb_graph_error(trainer.net, trainer.autocast)
            if why is not None:
                self.enabled, self.why_disabled = False, why
        if self.an4:
            net = trainer.net
            why = net.device_lengths_error(True, trainer.autocast is not None)
            if why is None and not getattr(net, "fuse_ctc", False):
                why = "fuse_ctc is off: the stock CTC loss copies the lengths to the host"
            if why is not None:
                self.enabled, self.why_disabled = False, why

    # ------------------------------------------------------------------ iteration flavour
    def _engines(self):
        return [self.opt._allreducer._engines.get(b.name) for b in self.opt._buckets]

    def _full_key(self, flavour: Tuple) -> Tuple:
        """The graph key: the flavour, and for AN4 the padded input shape before it."""
        return (self._shape, flavour) if self.an4 else flavour

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

    def precapture_sparse(self) -> int:
        """Capture the graph of EVERY sparse-phase flavour now (capturing records launches, it executes nothing), so that
        the rare exact-threshold / re-partition iterations are replayed like the common one instead of running eagerly
        inside somebody's timed region.  Engine iteration counters are faked for the capture and restored."""
        if not self.enabled or self.static_in is None:
            return 0
        cfg = self.opt._cfg
        if not cfg.sparse:
            return 0
        engines = self._engines()
        if any(e is None for e in engines):
            return 0
        real = [e.host.counter for e in engines]
        real_opt = getattr(self.opt, "counter", None)
        made = 0
        for flavour, it in self._sparse_flavours().items():
            key = self._full_key(flavour)
            if key in self.graphs or flavour == ("nograph",):
                continue
            for e in engines:
                e.host.counter = cfg.warmup_iters + it
            ok = self._capture(key) is not None
            for e, c in zip(engines, real):
                e.host.counter = c
            if real_opt is not None:
                self.opt.counter = real_opt
            if not ok:
                break
            made += 1
        first = not self._precaptured_shapes
        self._precaptured_shapes.add(self._shape)
        if first:
            # every long-lived object of the training process exists now (model, optimizer state, engines, graphs): move
            # them to the permanent generation so that the cyclic collector's full passes stop walking them -- a
            # generation-2 collection otherwise stalls a 1.2 ms step loop for tens of milliseconds.  Once only: a later
            # padded AN4 length adds a few graphs and static inputs, not worth a pause of that size each, and freezing
            # again would also pin whatever garbage exists at that moment
            import gc
            gc.collect()
            gc.freeze()
        return made

    # ------------------------------------------------------------------ one step
    def _eager(self, batch) -> torch.Tensor:
        tr = self.tr
        self.opt.zero_grad()
        loss, _ = tr._forward_loss(batch)
        self._backward(loss)
        tr.update_model()
        return loss.detach()

    def _backward(self, loss: torch.Tensor) -> None:
        # with loss scaling the scale is read from device memory: the captured graph stays valid when it moves
        (self.opt.scale_loss(loss) if getattr(self.opt, "_ls", None) is not None else loss).backward()

    def step(self, batch) -> torch.Tensor:
        """Run one optimizer step on ``batch`` (device tensors; an AN4 batch is staged by the trainer first); returns the
        (device) loss."""
        if self.an4:
            batch = self.tr.stage_batch(batch)
        if not self.enabled or self.eager_left > 0:
            self.eager_left -= 1
            return self._eager(batch)
        flavour = self._key()
        if flavour == ("nograph",):
            return self._eager(batch)
        shape = None
        if self.an4:
            if batch.over_capacity:
                self.fallbacks["targets"] += 1
                return self._eager(batch)
            shape = tuple(batch.inputs.shape)
            if shape not in self._static_of and len(self._static_of) >= MAX_AN4_SHAPES:
                self.fallbacks["shapes"] += 1
                return self._eager(batch)
        static = self._static_of.get(shape)
        if static is None:
            static = self._static_of[shape] = _clone(batch)
        for s, t in zip(static, batch):
            if torch.is_tensor(t):
                if s.shape != t.shape:
                    if self.ptb:                 # a short batch: this step eagerly, the graphs stay
                        self.fallbacks["shapes"] += 1
                        return self._eager(batch)
                    self.enabled, self.why_disabled = False, "batch shape changed"
                    return self._eager(batch)
                s.copy_(t, non_blocking=True)
        if self.ptb and not self._load_state(batch[0].size(0)):
            self.fallbacks["state"] += 1
            return self._eager(batch)
        self.static_in, self._shape = static, shape
        key = self._full_key(flavour)
        self.opt.refresh_lr()
        if shape not in self._precaptured_shapes and all(plan.kind != "dense" for plan in flavour[1:]):
            self.precapture_sparse()             # first sparse step (of this shape): capture every flavour at once
        g = self.graphs.get(key)
        if g is None:
            g = self._capture(key)
            if g is None:
                return self._eager(batch)
            for eng, c in zip(self._engines(), self._cap_counters):
                eng.host.counter = c             # the capture ran the Python side effects; the replay below is the real step
            if hasattr(self.opt, "counter") and self._cap_opt_counter is not None:
                self.opt.counter = self._cap_opt_counter
        for eng in self._engines():
            eng.host.counter += 1
        if hasattr(self.opt, "counter"):
            self.opt.counter += 1
        g.replay()
        self.opt._allreducer.poll_faults()       # pinned host mirror of the device fault words: a plain load per bucket
        ext.LAUNCH_COUNT["total"] += self.launches.get(key, 0)
        self.static_loss = self._loss_of[key]
        return self.static_loss

    # ------------------------------------------------------------------ PTB: the carried state
    def _load_state(self, n: int) -> bool:
        """Make the trainer's ``hidden`` the static pair for a batch of ``n`` sequences, by the eager step's rule
        (``Trainer._forward_loss_impl``): None or another batch size starts from zeros, anything else is carried in
        exactly.  False (nothing changed) when the state cannot be copied exactly: its dtypes are not the pair's."""
        tr = self.tr
        st = self._state
        if st is None:
            shape = (tr.net.num_layers, n, tr.net.embedding_dim)
            h_dt = tr.autocast if tr.net.fuse_lstm and tr.autocast is not None else torch.float32
            st = self._state = (torch.empty(shape, dtype=h_dt, device=tr.device),
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

    def _store_state(self) -> None:
        """Inside a capture, after the update: copy the step's (h_n, c_n) into the static pair.  Last, because the
        backward pass reads (h0, c0) from it."""
        for s, h in zip(self._state, self.tr.hidden):
            if h.dtype != s.dtype or h.shape != s.shape:
                raise RuntimeError("the carried state comes back as %s %s, the static buffer is %s %s"
                                   % (h.dtype, tuple(h.shape), s.dtype, tuple(s.shape)))
            s.copy_(h.detach())

    def _capture(self, key) -> Optional[torch.cuda.CUDAGraph]:
        tr = self.tr
        if self.ptb:
            tr.hidden = self._state
        counters = [eng.host.counter for eng in self._engines()]
        opt_counter = getattr(self.opt, "counter", None)
        self._cap_counters, self._cap_opt_counter = counters, opt_counter
        l0 = ext.LAUNCH_COUNT["total"]
        g = torch.cuda.CUDAGraph()
        try:
            torch.cuda.synchronize()
            with torch.cuda.graph(g, pool=self.pool):
                self.opt.zero_grad()
                loss, _ = tr._forward_loss(self.static_in)
                self._backward(loss)
                tr.update_model()
                out = loss.detach()
                if self.ptb:
                    self._store_state()
            if self.ptb:
                tr.hidden = self._state
            if self.static_loss is None:
                self.static_loss = out
            else:
                # every graph must write the same loss buffer: re-point through a copy node is not possible after
                # capture, so keep one buffer per graph and expose the latest
                self.static_loss = out
            self._loss_of[key] = out
            if self.pool is None:
                self.pool = g.pool()
        except Exception as e:  # noqa: BLE001 - fall back to eager for good
            self.enabled, self.why_disabled = False, "capture failed: %r" % (e,)
            if self.ptb:
                tr.hidden = self._state          # nothing ran: the pair still holds the state this step starts from
            # capture executed the Python side effects (counters) but no kernels: undo them
            for eng, c in zip(self._engines(), counters):
                eng.host.counter = c
            if opt_counter is not None:
                self.opt.counter = opt_counter
            try:
                torch.cuda.synchronize()
            except Exception:  # noqa: BLE001
                pass
            self.opt._after_step()
            return None
        self.launches[key] = ext.LAUNCH_COUNT["total"] - l0
        ext.LAUNCH_COUNT["total"] = l0
        self.graphs[key] = g
        return g

    def loss_tensor(self, key=None) -> torch.Tensor:
        return self.static_loss
