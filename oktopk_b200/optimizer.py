"""User-facing optimizer wrappers (L3): ``DistributedOptimizer`` and ``BertAdam``.

API parity with the reference (SURVEY A.3):
``DistributedOptimizer(optimizer, named_parameters=None, compression=NoneCompressor, is_sparse=False,
err_handler=None, layerwise_times=None, sigma_scale=2.5, density=0.1, norm_clip=None, writer=None)``
(``VGG/distributed_optimizer.py:203-207``) with ``step() / synchronize() / zero_grad() / stop() /
add_train_epoch() / get_current_density()`` and the ``local`` gradient-accumulation gate (:78,186);
``BertAdam(params, lr, warmup, t_total, ..., density, compressor, rank)``
(``BERT/bert/transformers/optimization.py:68-227``).

What is different by design (GPU-first):
  * no consumer thread, no queues, no per-hook ``torch.cuda.synchronize()`` (:58-59,90,93): a
    bucket's reduction is enqueued on a side CUDA stream from the post-accumulate hook of its
    last gradient, in a fixed bucket order on every rank, and ``synchronize()`` is a stream wait;
  * gradients / parameters / momentum are views into flat buffers, the update is one fused kernel
    per (bucket, param group) that also zeroes the gradient bucket (``zero_grad()`` is then free);
  * any torch optimizer can be wrapped (the reference re-implements SGD only, A.4-7): SGD, BertAdam and
    ``torch.optim.Adam`` / ``AdamW`` built with ``fused=True`` take the fused kernels (Adam: fp32 CUDA parameters,
    no amsgrad / maximize / differentiable, Python-number lr and betas) and ``Lamb`` (LAMB, three kernels per bucket and
    param group) take the fused kernels; everything else falls through to its own ``step()``;
  * ``state_dict()`` carries residuals, thresholds, region boundaries and counters (SURVEY 5.4).
"""
from __future__ import annotations

import math
import os
import warnings
from typing import Dict, Iterable, List, Optional

import torch

from .compression import NoneCompressor, compressors, resolve_compressor
from .config import LossScale, OkTopkConfig
from .ops import ext
from .parallel.allreducer import AllReducer
from .parallel.buckets import Bucket, attach, build_buckets
from .parallel.early_pack import PackPlanner
from .parallel.world import World, world as _world


# CTA cap of the early SGD update (sgd_ahead_kernel).  It streams 24 B per element beside backward and must finish before
# backward does, or the update after the call waits for it; every CTA beyond that takes HBM bandwidth from backward.
# VGG-16, 16 images, H100 SXM at 700 W, ms/step against the update off: 8 CTAs +13.6 %, 12 -0.3 %, 16 -3.0 %, 20 -4.4 %,
# 24 -4.2 %, 32 -0.5 % (ROADMAP 2b).  24 keeps a margin from the cliff below.
SGD_AHEAD_CTAS = 24


# ====================================================================================== loss scaling
class _ScaleState:
    """The optimizer's loss-scale state, laid out as the kernels' ``LossScaleDev`` (csrc/oktopk.cuh) in one small
    tensor on the parameters' device: scale, inv_scale (fp32), growth tracker, step verdict (int32), skipped steps and
    the wrapped Adam's applied-step count (int64).  On the CUDA engine the check and the update run on the device
    (csrc/scale.cu); elsewhere the same rules run in torch ops with a host read of the verdict."""

    def __init__(self, ls: LossScale, device: torch.device):
        self.cfg = ls
        self.buf = torch.zeros(32, dtype=torch.uint8, device=device)
        self.f32 = self.buf[0:8].view(torch.float32)          # scale, inv_scale
        self.i32 = self.buf[8:16].view(torch.int32)           # growth_tracker, found_inf
        self.i64 = self.buf[16:32].view(torch.int64)          # skipped, adam_step
        self.native = device.type == "cuda" and ext.available()
        self.reset()

    @property
    def ptr(self) -> int:
        return self.buf.data_ptr()

    @property
    def found_ptr(self) -> int:
        return self.buf.data_ptr() + 12

    def reset(self, scale: Optional[float] = None, growth_tracker: int = 0, skipped: int = 0, adam_step: int = 0) -> None:
        from .parallel.oracle import inv_scale_of
        scale = self.cfg.init_scale if scale is None else scale
        vals = torch.zeros(32, dtype=torch.uint8)
        vals[0:8].view(torch.float32).copy_(torch.tensor([scale, inv_scale_of(scale)], dtype=torch.float32))
        vals[8:16].view(torch.int32).copy_(torch.tensor([growth_tracker, 0], dtype=torch.int32))
        vals[16:32].view(torch.int64).copy_(torch.tensor([skipped, adam_step], dtype=torch.int64))
        self.buf.copy_(vals)

    def scale(self) -> torch.Tensor:
        return self.f32[0]

    def state(self) -> Dict:
        """Synchronous read."""
        h = self.buf.cpu()
        f, i, q = h[0:8].view(torch.float32), h[8:16].view(torch.int32), h[16:32].view(torch.int64)
        return {"scale": float(f[0]), "growth_tracker": int(i[0]), "skipped_steps": int(q[0]), "adam_step": int(q[1]),
                "found_inf": int(i[1])}

    def found_host(self) -> bool:
        return bool(self.i32[1].item())

    def check_host(self, flat: torch.Tensor, world: World) -> bool:
        """The torch-ops form of unscale_check (``backend='dist'``): unscale ``flat`` in place, agree across ranks on
        whether any of them saw a non-finite value (a host read), and fold the verdict into the step's."""
        with torch.no_grad():
            bad = (~torch.isfinite(flat)).any().to(torch.int32).reshape(1)
            flat.mul_(self.f32[1])
            world.all_reduce_sum(bad)
            skip = bool(bad.item())
            if skip:
                self.i32[1].fill_(1)
        return skip

    def update(self) -> None:
        """End of step: growth / backoff, counters, verdict cleared (on the current stream)."""
        c = self.cfg
        if self.native:
            ext.require().scale_update(self.ptr, float(c.growth_factor), float(c.backoff_factor), int(c.growth_interval),
                                       torch.cuda.current_stream().cuda_stream)
            return
        from .parallel.oracle import update_scale
        st = self.state()
        found = bool(st["found_inf"])
        scale, tracker = update_scale(st["scale"], st["growth_tracker"], found, c)
        self.reset(scale, tracker, st["skipped_steps"] + int(found), st["adam_step"] + int(not found))


# ====================================================================================== comm mixin
class _BucketedComm:
    """Bucket bookkeeping, autograd hooks, stream choreography.  Mixed into optimizer classes."""

    def _okt_setup(self, named_parameters, allreducer: AllReducer, flatten_params: bool = True,
                   loss_scale: Optional[LossScale] = None, max_grad_norm: Optional[float] = None,
                   clip_per_param: bool = False) -> None:
        if named_parameters is not None:
            named_parameters = list(named_parameters)
            if any(not isinstance(p, tuple) for p in named_parameters):
                raise ValueError("named_parameters should be a sequence of (name, parameter) tuples, "
                                 "usually produced by model.named_parameters().")
            names = {v: k for k, v in named_parameters}
        else:
            names = {}
        i = 0
        for g in self.param_groups:
            for p in g["params"]:
                if p not in names:
                    names[p] = "allreduce.noname.%d" % i
                i += 1
        self._parameter_names = names
        self._allreducer = allreducer
        self._cfg: OkTopkConfig = allreducer.cfg
        self.local = False
        self._synced = False
        self._ls: Optional[_ScaleState] = None
        self.momentum_correction = False
        self._buckets: List[Bucket] = build_buckets(self.param_groups, names, self._cfg.bucket_elems)
        self._bucket_of: Dict[torch.nn.Parameter, Bucket] = {}
        self._flat_state: Dict[int, Dict[str, torch.Tensor]] = {}
        self._next_launch = 0
        self._hook_handles = []
        self._comm_stream = None
        self._use_streams = False
        # Gradient landing: autograd produces every gradient in a fresh tensor; ONE multi-tensor kernel per bucket copies
        # them into the flat symmetric bucket when the bucket's last gradient is ready (instead of autograd accumulating
        # into pre-existing bucket views = one elementwise add kernel per parameter per step).
        self._land = False
        for b in self._buckets:
            dev = b.params[0].device
            grad = allreducer.register_bucket(b.name, b.numel, dev)
            attach(b, grad, flatten_params)
            if dev.type == "cuda" and self._cfg.land_grads and ext.available():
                self._land = True
            b.pending = len(b.params)
            b.dirty = False                       # freshly zeroed
            if dev.type == "cuda":
                self._use_streams = self._cfg.overlap
                b.event = torch.cuda.Event()
            for p in b.params:
                self._bucket_of[p] = b
                self._hook_handles.append(p.register_post_accumulate_grad_hook(self._make_hook(p)))
        # Ok-Topk with a fused update: the reduction reads the gradients straight from autograd's tensors, with no landing
        # copy (see _source_table).  Its pack pass then leaves the bucket alone, so the bucket must be all-zero when such a
        # call starts: the fused update clears the few entries the reduction wrote (zero_grad=1 after EVERY step, dense
        # warm-up steps included), and CudaBucketEngine.reset_sparse_state / load_state_dict clear it after a fault or a
        # checkpoint load.
        if self._update is _AdamUpdate:           # the fused Adam kernel works on flat fp32 CUDA buckets only
            if not (ext.available() and all(b.flat_param is not None and b.grad.is_cuda for b in self._buckets)):
                self._update = None
        self._direct = (self._land and self._update is not None and allreducer.compressor.name == "oktopk"
                        and all(b.flat_param is not None for b in self._buckets))
        # Early pack (parallel/early_pack.py): on a threshold-reuse Ok-Topk step the hooks pack the ready gradients on the
        # communication stream, once early_pack_frac of the bucket has them, while backward goes on
        self._packs = {}
        self._pos_in_bucket = {p: i for b in self._buckets for i, p in enumerate(b.params)}
        if self._direct and self._use_streams:
            for b in self._buckets:
                if len(b.params) <= ext.require().SRC_SEG_MAX:
                    self._packs[b.index] = PackPlanner(b.offsets, b.numel,
                                                       math.ceil(self._cfg.early_pack_frac * b.numel),
                                                       ext.require().PACK_RANGE_MAX)
            for b in self._buckets:
                b.packing = None                  # this step: None undecided, else whether its hooks pack early
        if self._use_streams:
            # high priority: a bucket's (SM-partitioned) communication kernel should get its SMs as soon as backward
            # kernels retire CTAs, not after the whole backward queue
            self._comm_stream = torch.cuda.Stream(priority=-1)
        # Early SGD update (csrc/optim.cu sgd_ahead_kernel): beside each early-pack segment, the zero-gradient update of
        # its ranges runs on a side stream, forked from the segment's event; the tail after the call recomputes, from the
        # stash of old values, only the elements the call wrote.  The stash is the bucket's length, allocated here.
        self._ahead_stash: Dict[int, tuple] = {}
        self._ahead_stream = None
        self._ahead_ctas = SGD_AHEAD_CTAS
        if (self._packs and self._update is _SGDUpdate and self._cfg.sgd_ahead
                and os.environ.get("OKTOPK_SGD_AHEAD", "1") != "0"):
            self._ahead_stream = torch.cuda.Stream()
            for b in self._buckets:
                if b.index in self._packs:
                    mom = any(self.param_groups[gi].get("momentum", 0.0) != 0 for gi, _, _ in b.group_slices)
                    self._ahead_stash[b.index] = (torch.empty_like(b.grad), torch.empty_like(b.grad) if mom else None)
        for b in self._buckets:
            b.ahead = None                        # this step: None undecided, else whether its segments update early
        allreducer.add_resync_hook(self._resync_replicas)
        if loss_scale is not None:
            allreducer.enable_loss_scaling()
            self._ls = _ScaleState(loss_scale, self._buckets[0].params[0].device if self._buckets else torch.device("cpu"))
        # device-resident per-group scalars (the learning rate; for wrapped Adam the step's decay, step size and bias
        # correction): the fused update kernels read them from memory so that a captured CUDA graph of the whole step
        # stays valid when the schedule moves
        # With loss scaling the wrapped Adam's or Lamb's step count is on the device (a skipped step does not advance it):
        # the host stages {lr, weight_decay, beta1, beta2} per group in double (_hyper_dev) and a kernel derives the
        # scalars.
        self._lr_dev = self._hyper_dev = None
        self._lr_pin, self._lr_ev, self._lr_ring, self._lr_last = [], [], 0, None
        dev0 = self._buckets[0].params[0].device if self._buckets else torch.device("cpu")
        if dev0.type == "cuda" and ext.available() and self._update is not None:
            groups = max(len(self.param_groups), 1)
            self._lr_dev = torch.zeros(groups * self._update.n_scalars, dtype=torch.float32, device=dev0)
            stage = self._lr_dev
            if self._ls is not None and (self._update is _AdamUpdate or self._update is _LambUpdate):
                stage = self._hyper_dev = torch.zeros(groups * 4, dtype=torch.float64, device=dev0)
            self._lr_pin = [torch.zeros_like(stage, device="cpu").pin_memory() for _ in range(8)]
            self._lr_ev = [None] * len(self._lr_pin)
        # gradient clipping: on the device when every bucket takes a fused kernel (_GradClip), else torch's
        # clip_grad_norm_ over the bucket views before the update
        self._max_grad_norm = max_grad_norm
        self._grad_norm: Optional[torch.Tensor] = None
        self._clip: Optional[_GradClip] = None
        if (max_grad_norm is not None or clip_per_param) and self._device_update():
            self._clip = _GradClip(self, clip_per_param, max_grad_norm or 0.0)
        self._lamb = _LambNorms(self) if self._update is _LambUpdate and self._device_update() else None

    def _resync_replicas(self) -> None:
        """After a handled fault: every replica takes rank 0's parameters (and momentum) again."""
        w = self._allreducer.world
        if w.size == 1:
            return
        for b in self._buckets:
            if b.flat_param is not None:
                w.broadcast(b.flat_param, 0)
            else:
                for p in b.params:
                    w.broadcast(p.data, 0)
            for t in self._flat_state.get(b.index, {}).values():
                if torch.is_tensor(t):
                    w.broadcast(t, 0)

    @property
    def _okt_adam(self) -> bool:
        """True while the step runs the flat-bucket ``fused_adam`` kernel (derived from ``_update``, never set)."""
        return self._update is _AdamUpdate

    def refresh_lr(self) -> None:
        """Push the current per-group device scalars to the device (one tiny async H2D, only when changed).
        Never called while a stream is capturing: graph replays call it right before ``replay()``."""
        if self._lr_dev is None or self._update is None:
            return
        vals = [self._update.scalars(self, g) for g in self.param_groups]
        if vals == self._lr_last:
            return
        self._lr_ring = (self._lr_ring + 1) % len(self._lr_pin)
        pin = self._lr_pin[self._lr_ring]
        if self._lr_ev[self._lr_ring] is not None:          # the host may run many (graph-replayed) steps ahead:
            self._lr_ev[self._lr_ring].synchronize()        # never overwrite a staging slot whose copy is pending
        n = len(vals[0]) if vals else 0
        for gi, sc in enumerate(vals):
            for j, v in enumerate(sc):
                pin[gi * n + j] = v
        (self._hyper_dev if self._hyper_dev is not None else self._lr_dev).copy_(pin, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._lr_ev[self._lr_ring] = ev
        self._lr_last = vals

    def _lr_ptr(self, gi: int) -> int:
        return self._lr_dev.data_ptr() + 4 * self._update.n_scalars * gi

    def _maybe_refresh_lr(self) -> None:
        if self._lr_dev is not None and not torch.cuda.is_current_stream_capturing():
            self.refresh_lr()

    # ------------------------------------------------------------------ hooks
    def _make_hook(self, p):
        def hook(param):
            b = self._bucket_of[p]
            b.dirty = True
            if self.local:                        # accumulation micro-step: no communication (:78)
                return
            b.pending -= 1
            if b.pending == 0:
                self._launch_ready()
            elif b.index in self._packs:
                self._pack_early(b, p)
        return hook

    def _pack_early(self, b: Bucket, p) -> None:
        """Parameter ``p`` of bucket ``b`` has its gradient: pack the ready, unpacked gradients now if they are enough
        (``PackPlanner``), on the communication stream behind the work that produced them."""
        if b.packing is None:
            b.packing = (self._direct and not self.momentum_correction and self._ls is None
                         and self._allreducer.reads_sources(b.name) and self._allreducer.packs_early(b.name))
        if not b.packing:
            return
        planner = self._packs[b.index]
        ranges = planner.ready(self._pos_in_bucket[p])
        if ranges is None:
            return
        ptrs, offs, lens = [], [], []
        for q, o, v in sorted(zip(b.params, b.offsets, b.grad_views), key=lambda t: t[1]):
            g = q.grad
            if not any(lo <= o < hi for lo, hi in ranges) or g is None or g.numel() == 0:
                continue
            if (g.data_ptr() == v.data_ptr() or g.dtype != torch.float32 or not g.is_cuda or g.stride() != v.stride()
                    or g.data_ptr() % 16):
                raise RuntimeError("early pack: the gradient of %s cannot be read in place; set "
                                   "OkTopkConfig.early_pack=False" % self._parameter_names.get(q, "?"))
            ptrs.append(g.data_ptr())
            offs.append(o)
            lens.append(g.numel())
        if b.ahead is None:
            # the step's momentum buffers exist (not its first step) and the device lr is this step's (eager steps push
            # it here, ahead of step(); graph replays push it before the replay)
            b.ahead = b.index in self._ahead_stash and self._update.keys[0] in self._flat_state.get(b.index, {})
            if b.ahead:
                self._maybe_refresh_lr()
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        self._comm_stream.wait_event(ev)
        with torch.cuda.stream(self._comm_stream):
            self._allreducer.pack_segment(b.name, ranges, (ptrs, offs, lens), stream=self._comm_stream)
        if b.ahead:
            self._sgd_ahead(b, ranges, ev)

    def _sgd_ahead(self, b: Bucket, ranges, ev) -> None:
        """The zero-gradient SGD update of bucket ``b``'s ``ranges`` (those of the segment just enqueued), per param group,
        behind ``ev`` on the side stream; ``synchronize()`` joins it."""
        s_ = self._ahead_stream
        if s_ is not self._comm_stream:
            s_.wait_event(ev)
        sp, sm = self._ahead_stash[b.index]
        fs = self._flat_state[b.index]
        C = ext.require()
        for gi, s, e in b.group_slices:
            rs = _clip_ranges(ranges, s, e)
            if not rs:
                continue
            m, damp, wd, nest = _SGDUpdate.hyper(self, self.param_groups[gi])
            C.sgd_ahead(b.flat_param.data_ptr() + 4 * s, fs["momentum_buffer"].data_ptr() + 4 * s, sp.data_ptr() + 4 * s,
                        sm.data_ptr() + 4 * s if sm is not None else 0, e - s, rs, m, damp, wd, int(nest),
                        int(self._ahead_ctas), s_.cuda_stream, self._lr_ptr(gi))

    def _launch_ready(self) -> None:
        # strictly in bucket order on every rank: the fused kernels spin on peers' flags, so two
        # ranks must never enqueue two buckets in opposite orders.
        while self._next_launch < len(self._buckets) and self._buckets[self._next_launch].pending <= 0:
            self._launch(self._buckets[self._next_launch])
            self._next_launch += 1

    def _land_bucket(self, b: Bucket) -> None:
        """Copy the autograd-produced gradients of bucket ``b`` into the flat bucket with one kernel launch and re-point
        ``p.grad`` at the bucket views (what the user sees after ``synchronize()`` is the reduced gradient)."""
        srcs, offs, numels = [], [], []
        for p, o, v in zip(b.params, b.offsets, b.grad_views):
            g = p.grad
            if g is None:                         # no gradient in this step (unused parameter, or a conv bias folded
                srcs.append(0)                    # into a fused batch-norm): zero-filled by the same launch
                offs.append(o)
                numels.append(p.numel())
            elif g.data_ptr() == v.data_ptr():
                continue                          # already accumulated in place (gradients were never detached)
            elif g.dtype == torch.float32 and g.is_cuda and g.stride() == v.stride():
                srcs.append(g.data_ptr())
                offs.append(o)
                numels.append(g.numel())
            else:
                v.copy_(g)
            p.grad = v
        if srcs:
            ext.require().land_grads(srcs, offs, numels, b.grad.data_ptr(), torch.cuda.current_stream().cuda_stream)

    def _source_table(self, b: Bucket):
        """(pointers, offsets, lengths) of the autograd-produced gradients of bucket ``b``, for a reduction that reads them
        in place; ``p.grad`` is re-pointed at the bucket views (which receive the reduced gradient) and the source tensors
        are held on the bucket until ``synchronize()`` has made the current stream wait for the reduction.  None if a
        gradient cannot be read that way (already the bucket view, another dtype or layout, misaligned, too many
        tensors): the step then lands the gradients as before."""
        ptrs, offs, lens, held = [], [], [], []
        for p, o, v in zip(b.params, b.offsets, b.grad_views):
            g = p.grad
            if g is None or g.numel() == 0:       # no gradient in this step: its slice of the all-zero bucket is read
                continue
            if (g.data_ptr() == v.data_ptr() or g.dtype != torch.float32 or not g.is_cuda or g.stride() != v.stride()
                    or g.data_ptr() % 16):
                return None
            ptrs.append(g.data_ptr())
            offs.append(o)
            lens.append(g.numel())
            held.append(g)
        if len(ptrs) > ext.require().SRC_SEG_MAX:
            return None
        for p, v in zip(b.params, b.grad_views):
            p.grad = v
        b.held = held
        return ptrs, offs, lens

    def _launch(self, b: Bucket) -> None:
        if b.launched:
            return
        b.launched = True
        srcs = None
        if self._direct and not self.momentum_correction and self._allreducer.reads_sources(b.name):
            srcs = self._source_table(b)
        rest = None
        if b.index in self._packs and self._packs[b.index].segments:
            if srcs is None:
                raise RuntimeError("early pack: bucket %s was partly packed from its gradients but its last call cannot "
                                   "read them in place; set OkTopkConfig.early_pack=False" % b.name)
            rest = self._packs[b.index].rest()
        if srcs is None and self._land:
            self._land_bucket(b)
        if self.momentum_correction:
            self._apply_momentum_correction(b)
        if self._comm_stream is not None:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            self._comm_stream.wait_event(ev)
            with torch.cuda.stream(self._comm_stream):
                self._allreducer.reduce_bucket(b.name, b.grad, stream=self._comm_stream, srcs=srcs, scale=self._ls,
                                               pack_ranges=rest)
                b.event.record(self._comm_stream)
        else:
            self._allreducer.reduce_bucket(b.name, b.grad, srcs=srcs, scale=self._ls)

    def _apply_momentum_correction(self, b: Bucket) -> None:
        """``VGG/distributed_optimizer.py:81-88``: communicate the momentum-accumulated gradient."""
        fs = self._flat_state.setdefault(b.index, {})
        buf = fs.get("mc_buf")
        if buf is None:
            buf = fs["mc_buf"] = torch.zeros_like(b.grad)
        if b.grad.is_cuda and ext.available():
            ext.require().momentum_correct(b.grad.data_ptr(), buf.data_ptr(), b.numel, 0.9,
                                           torch.cuda.current_stream().cuda_stream)
        else:
            buf.mul_(0.9).add_(b.grad)
            b.grad.copy_(buf)

    # ------------------------------------------------------------------ loss scaling
    @property
    def momentum_correction(self) -> bool:
        return self._momentum_correction

    @momentum_correction.setter
    def momentum_correction(self, on: bool) -> None:
        if on and getattr(self, "_ls", None) is not None:
            raise ValueError("loss_scale cannot be combined with momentum_correction: the momentum buffer would absorb "
                             "the gradient of a skipped step")
        self._momentum_correction = bool(on)

    def scale_loss(self, loss: torch.Tensor) -> torch.Tensor:
        """``loss * scale`` with the scale read from device memory (no synchronisation, capturable).  Without a
        ``loss_scale`` the loss is returned as is."""
        if self._ls is None:
            return loss
        return loss * self._ls.scale()

    def loss_scale_state(self) -> Optional[Dict]:
        """``{scale, growth_tracker, skipped_steps}`` (a synchronous read: logging and tests), None without scaling."""
        if self._ls is None:
            return None
        st = self._ls.state()
        return {k: st[k] for k in ("scale", "growth_tracker", "skipped_steps")}

    def _scale_state_dict(self) -> Optional[Dict]:
        if self._ls is None:
            return None
        st = self._ls.state()
        st.pop("found_inf")
        return st

    def _load_scale_state(self, sd: Optional[Dict], adam_step: int) -> None:
        """A checkpoint without scale state starts from ``init_scale``."""
        if self._ls is None:
            return
        if sd is None:
            self._ls.reset(adam_step=adam_step)
        else:
            self._ls.reset(sd["scale"], sd["growth_tracker"], sd["skipped_steps"], sd.get("adam_step", adam_step))

    # ------------------------------------------------------------------ public API
    def synchronize(self) -> None:
        """Block (stream-wise) until every bucket holds its reduced gradient."""
        if self._synced:
            return
        for b in self._buckets:                   # flush buckets whose hooks did not all fire (unused params)
            b.pending = 0
        self._launch_ready()
        if self._comm_stream is not None:
            cur = torch.cuda.current_stream()
            for b in self._buckets:
                cur.wait_event(b.event)
            if any(b.ahead for b in self._buckets):
                cur.wait_stream(self._ahead_stream)
        for b in self._buckets:                   # the reductions' reads of the gradient tensors are ordered before
            b.held = None                         # anything the current stream does next: their memory may be reused
        self._synced = True

    def _after_step(self) -> None:
        for b in self._buckets:
            b.pending = len(b.params)
            b.launched = False
            if b.index in self._packs:
                self._packs[b.index].reset()
                b.packing = None
            b.ahead = None
        self._next_launch = 0
        self._synced = False
        self._allreducer.poll_faults()           # pinned host flag, no sync: a timed-out peer wait surfaces at once

    def _clear_buckets(self) -> None:
        """Re-establish the all-zero bucket that a reduction reading autograd's tensors expects."""
        if self._direct:
            with torch.no_grad():
                for b in self._buckets:
                    b.grad.zero_()

    def zero_grad(self, set_to_none: bool = False) -> None:  # noqa: ARG002 - views must survive
        if self._land:
            # detach the gradients from the bucket: the next backward hands every parameter a fresh tensor, which the
            # landing kernel copies in (the bucket itself is overwritten, never accumulated into: no memset either)
            for b in self._buckets:
                for p in b.params:
                    p.grad = None
                b.dirty = False
            return
        for b in self._buckets:
            if b.dirty:
                b.grad.zero_()
                b.dirty = False

    def stop(self) -> None:
        self._allreducer.stop()

    def add_train_epoch(self) -> None:
        self._allreducer.train_epoch += 1

    def get_current_density(self) -> float:
        return self._allreducer.get_current_density()

    def comm_stats(self) -> Dict:
        return self._allreducer.stats()

    def grad_norm(self) -> Optional[torch.Tensor]:
        """The gradient norm the last ``step()`` clipped with, as ``clip_grad_norm_`` returns it: a 0-dim tensor on the
        parameters' device, written by the step without a host synchronisation (BertAdam with ``clip_reduced`` on the
        device: one norm per parameter, in bucket order).  None before the first clipped step."""
        return self._grad_norm

    def check_faults(self) -> None:
        """Raise / call ``err_handler`` if a peer timed out inside a communication kernel (synchronous read)."""
        self._allreducer.check_faults()

    def close(self) -> None:
        for h in self._hook_handles:
            h.remove()
        self._hook_handles = []
        self._allreducer.close()

    # ------------------------------------------------------------------ fused updates
    def step(self, closure=None):
        """``synchronize()`` + parameter update (``VGG/distributed_optimizer.py:185-190``)."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        if not self.local:
            self.synchronize()
        if self._clip is None and self._max_grad_norm is not None:
            self._grad_norm = torch.nn.utils.clip_grad_norm_([p for g in self.param_groups for p in g["params"]],
                                                             self._max_grad_norm)
        # the fused kernels read the step verdict themselves; the torch update paths need it on the host
        host_skip = self._ls is not None and not self._device_update() and self._ls.found_host()
        if self._update is None:
            if not host_skip:
                super().step()
            for b in self._buckets:
                b.dirty = True
        else:
            self._maybe_refresh_lr()
            if self._hyper_dev is not None:
                ext.require().adam_scalars(self._ls.ptr, self._hyper_dev.data_ptr(), self._lr_dev.data_ptr(),
                                           len(self.param_groups), torch.cuda.current_stream().cuda_stream,
                                           lamb=int(self._update is _LambUpdate))
            if self._clip is not None:
                self._grad_norm = self._clip.run(self)
            with torch.no_grad():
                for b in self._buckets:
                    self._fused_update(b, host_skip)
            self.counter += 1
        if self._ls is not None:
            self._ls.update()
        self._after_step()
        return loss

    def _device_update(self) -> bool:
        """Every bucket is updated by a fused kernel (which reads the step verdict of loss scaling on the device)."""
        return self._update is not None and self._lr_dev is not None and all(
            b.grad.is_cuda and b.flat_param is not None for b in self._buckets)

    def _flat_buffers(self, b: Bucket) -> Dict[str, torch.Tensor]:
        """The bucket's flat state buffers, one per state key of the update, allocated zeroed on first use;
        ``self.state[p]`` holds views of them."""
        fs = self._flat_state.setdefault(b.index, {})
        for k in self._update.keys:
            if k not in fs:
                fs[k] = torch.zeros_like(b.grad)
                for p, v in zip(b.params, b.views(fs[k])):
                    self.state[p][k] = v
        return fs

    def _fused_update(self, b: Bucket, host_skip: bool = False) -> None:
        first = self._update.keys[0] not in self._flat_state.get(b.index, {})
        fs = self._flat_buffers(b)
        on_gpu = b.grad.is_cuda and b.flat_param is not None and ext.available()
        # after a landing step the next landing copy overwrites the whole bucket: it need not be cleared
        zero_grad = 0 if self._land and not self._direct else 1
        skip_ptr = self._ls.found_ptr if self._ls is not None else 0
        if b.ahead and on_gpu:
            self._sgd_tail(b, fs, zero_grad, skip_ptr)
            b.dirty = False
            return
        for gi, s, e in b.group_slices:
            def launch(fn, *hyper):
                clip = self._clip.ref(b, s) if self._clip is not None else {}
                fn(b.flat_param.data_ptr() + 4 * s, b.grad.data_ptr() + 4 * s,
                   *(fs[k].data_ptr() + 4 * s for k in self._update.keys), e - s, *hyper, zero_grad,
                   torch.cuda.current_stream().cuda_stream, self._lr_ptr(gi), self._allreducer.fault_ptr(b.name),
                   skip_ptr, **clip)
            if on_gpu or not host_skip:
                self._update.update(self, b, self.param_groups[gi], s, e, fs, first, launch if on_gpu else None)
            if not on_gpu:
                b.grad[s:e].zero_()
        b.dirty = False

    def _sgd_tail(self, b: Bucket, fs: Dict[str, torch.Tensor], zero_grad: int, skip_ptr: int) -> None:
        """The update of a bucket whose segments' ranges had ``_sgd_ahead``: one ``fused_sgd_tail`` per param group, which
        recomputes the elements the call wrote in those ranges and updates ``PackPlanner.rest()`` in full."""
        planner = self._packs[b.index]
        ahead = [r for seg in planner.segments for r in seg]
        rest = planner.rest()
        sp, sm = self._ahead_stash[b.index]
        C = ext.require()
        for gi, s, e in b.group_slices:
            m, damp, wd, nest = _SGDUpdate.hyper(self, self.param_groups[gi])
            C.fused_sgd_tail(b.flat_param.data_ptr() + 4 * s, b.grad.data_ptr() + 4 * s,
                             fs["momentum_buffer"].data_ptr() + 4 * s, sp.data_ptr() + 4 * s,
                             sm.data_ptr() + 4 * s if sm is not None else 0, e - s, _clip_ranges(ahead, s, e),
                             _clip_ranges(rest, s, e), m, damp, wd, int(nest), 0, zero_grad,
                             torch.cuda.current_stream().cuda_stream, self._lr_ptr(gi),
                             self._allreducer.fault_ptr(b.name), skip_ptr,
                             **(self._clip.ref(b, s) if self._clip is not None else {}))

    def _adopt_state(self, counter: Optional[int] = None) -> None:
        """Move per-parameter state (from ``load_state_dict`` or the wrapped optimizer) into the flat buffers.  A bucket
        gets buffers iff one of its parameters has state (zeros for those without): SGD's first step copies the update
        into a fresh momentum buffer.  The step count is ``counter``: given, or the per-parameter ``step`` of torch's
        format, which must then be equal.  Unequal step counts cannot share one bias correction: the optimizer then keeps
        the per-parameter state and uses torch's own ``step()`` from here on."""
        keys = self._update.keys
        have = {p for b in self._buckets for p in b.params if self.state.get(p, {}).get(keys[0]) is not None}
        if counter is None:
            steps = {float(self.state[p]["step"]) for p in have if "step" in self.state[p]}
            if len(steps) > 1:
                warnings.warn("DistributedOptimizer: the loaded %s state has unequal step counts per parameter %s; "
                              "using its own step() from now on" % (type(self).__name__, sorted(steps)))
                self._update = None
                self._clip = None                 # torch's step: the clip runs before it, in torch
                self._clear_buckets()
                self._direct = False              # torch's step reads the gradients from the landed bucket
                for b in self._buckets:
                    for k in keys:
                        self._flat_state.get(b.index, {}).pop(k, None)
                return
            counter = int(steps.pop()) if steps else 0
        self.counter = counter
        loaded = {(p, k): self.state[p][k] for p in have for k in keys}
        with torch.no_grad():
            for b in self._buckets:
                for p in b.params:
                    self.state.get(p, {}).pop("step", None)      # the step count is ``counter``
                if not any(p in have for p in b.params):
                    for k in keys:
                        self._flat_state.get(b.index, {}).pop(k, None)
                    continue
                fs = self._flat_buffers(b)          # (points state[p] at the views when it allocates them)
                for k in keys:
                    for p, v in zip(b.params, b.views(fs[k])):
                        if p in have:
                            v.copy_(loaded[p, k])
                        else:
                            v.zero_()
                        self.state[p][k] = v


def _clip_ranges(ranges, s: int, e: int):
    """Bucket element ranges -> their parts inside the param-group slice [s, e), relative to s and clipped to the slice's
    whole float4 vectors (its scalar tail is the tail kernel's, densely)."""
    top = 4 * ((e - s) // 4)
    out = []
    for lo, hi in ranges:
        lo, hi = max(lo - s, 0), min(hi - s, top)
        if lo < hi:
            out.append((lo, hi))
    return out


class _GradClip:
    """Gradient clipping on the device, between ``synchronize()`` and the fused update: one ``grad_sumsq`` per bucket
    (fp64 partial sums of squares, a fixed number per bucket, no atomics), one ``clip_coef`` that combines them in a
    fixed order into the norm and the factor, and the update kernels multiply the gradient by the factor as they read
    it.  Two launches per step more than an unclipped one-bucket step, no host synchronisation: a CUDA graph captures
    it.  After the reduction every rank holds the same bucket bits, so every rank computes the same factor.

    Global (``DistributedOptimizer(max_grad_norm=c)``): one norm over every bucket, each bucket one segment (its padding
    between parameters is zero), torch's ``clip_grad_norm_`` factor.  Per parameter (``BertAdam(clip_reduced=True)``):
    one segment, norm and factor per parameter, the bound ``max_grad_norm`` of its group read from the device scalars
    (``_BertAdamUpdate.scalars``); the update kernel finds a vector's factor from the segment ends of its group slice."""

    def __init__(self, opt, per_param: bool, max_norm: float):
        dev = opt._buckets[0].grad.device
        self.per_param, self.max_norm = per_param, float(max_norm)
        self.segs = None
        if per_param:
            self.segs = _SegTable(opt._buckets, dev)
            self.tables = self.segs.tables
            self.nseg, npart = self.segs.nseg, self.segs.npart
            self.seg_blk, self.ends = self.segs.blk, self.segs.ends
            self.seg_scal = _as_dev([gi * opt._update.n_scalars + 1 for gi in self.segs.group], dev)
        else:
            self.tables = []                      # (bucket, offsets, lengths, first partial)
            npart = 0
            for b in opt._buckets:
                self.tables.append((b, [0], [b.numel], npart))
                npart += max(1, -(-b.numel // ext.require().SUMSQ_CHUNK))
            self.nseg = 1
            self.seg_blk = self.seg_scal = self.ends = None
        self.partial = torch.zeros(npart, dtype=torch.float64, device=dev)
        self.norm = torch.zeros(self.nseg, dtype=torch.float32, device=dev)
        self.coef = torch.ones(self.nseg, dtype=torch.float32, device=dev)

    def run(self, opt) -> torch.Tensor:
        """Enqueue the norm and the factor on the current stream; returns the norm (0-dim, or one per parameter)."""
        C, stream = ext.require(), torch.cuda.current_stream().cuda_stream
        for b, offs, lens, p0 in self.tables:
            C.grad_sumsq(b.grad.data_ptr(), offs, lens, self.partial.data_ptr() + 8 * p0, stream)
        if self.per_param:
            C.clip_coef(self.partial.data_ptr(), self.partial.numel(), self.seg_blk.data_ptr(), self.seg_scal.data_ptr(),
                        self.nseg, opt._lr_dev.data_ptr(), 0.0, self.norm.data_ptr(), self.coef.data_ptr(), stream)
            return self.norm
        C.clip_coef(self.partial.data_ptr(), self.partial.numel(), 0, 0, 0, 0, self.max_norm, self.norm.data_ptr(),
                    self.coef.data_ptr(), stream)
        return self.norm[0]

    def ref(self, b: Bucket, s: int) -> Dict[str, int]:
        """The factor arguments of the update of bucket ``b``'s group slice starting at element ``s``."""
        if not self.per_param:
            return {"coef_ptr": self.coef.data_ptr()}
        t = self.segs.slices[b.index, s][0]
        return {"coef_ptr": self.coef.data_ptr() + 4 * t, "ends_ptr": self.ends.data_ptr() + 4 * t}


def _as_dev(values, dev) -> torch.Tensor:
    return torch.tensor(values, dtype=torch.int32).to(dev)


class _SegTable:
    """One segment per parameter tensor of every bucket, for the kernels that reduce over each parameter (the
    per-parameter clip, LAMB's norms).  Segments are numbered in bucket order, which is also group-slice order, and
    each gets the chunk partials [blk[t], blk[t + 1]) that a per-segment pass writes, one per SUMSQ_CHUNK elements
    (at least one).  On the device, int32: ``off`` (the segment's offset in its group slice), ``len``, ``blk`` and
    ``ends`` (the float4 vector of the group slice where the next segment starts, INT_MAX for a slice's last: the
    cursor the update kernels find a vector's segment with).  Host side: ``tables`` (bucket, offsets, lengths, first
    partial) for ``grad_sumsq``, ``group`` and ``params`` per segment, and ``slices``: (bucket index, group slice
    start) -> (first segment, segments, partials)."""

    def __init__(self, buckets: List[Bucket], dev: torch.device):
        chunk = ext.require().SUMSQ_CHUNK
        off, lens, blk, ends = [], [], [0], []
        self.group, self.params, self.tables = [], [], []
        self.slices: Dict[tuple, tuple] = {}
        for b in buckets:
            self.tables.append((b, list(b.offsets), [p.numel() for p in b.params], blk[-1]))
            for gi, s, e in b.group_slices:
                ts = [t for t, o in enumerate(b.offsets) if s <= o < e]
                self.slices[b.index, s] = (len(lens), len(ts), blk[-1])
                for j, t in enumerate(ts):
                    n = b.params[t].numel()
                    off.append(b.offsets[t] - s)
                    lens.append(n)
                    blk.append(blk[-1] + max(1, -(-n // chunk)))
                    ends.append((b.offsets[ts[j + 1]] - s) // 4 if j + 1 < len(ts) else 2 ** 31 - 1)
                    self.group.append(gi)
                    self.params.append(b.params[t])
                t0, nseg, p0 = self.slices[b.index, s]
                self.slices[b.index, s] = (t0, nseg, blk[-1] - p0)
        self.nseg, self.npart = len(lens), blk[-1]
        self.off, self.len, self.blk, self.ends = (_as_dev(v, dev) for v in (off, lens, blk, ends))


# ====================================================================================== fused update families
# What a fused flat-bucket update needs to know about one optimizer: the per-parameter state it keeps in flat buffers
# (``keys``), its device scalars per param group (``scalars``, ``n_scalars`` of them) and its update of one (bucket,
# param group) slice: the kernel through ``launch``, or, with ``launch`` None (no flat CUDA bucket or no extension, as on
# the CPU; SGD and BertAdam only), the same math in torch.
class _SGDUpdate:
    """``torch.optim.SGD``: weight decay, momentum, dampening, nesterov."""
    keys = ("momentum_buffer",)
    n_scalars = 1

    @staticmethod
    def scalars(opt, g):
        return (float(g["lr"]),)

    @staticmethod
    def hyper(opt, g):
        """(momentum, dampening, weight_decay, nesterov) of param group ``g``."""
        m = 0.0 if opt.momentum_correction else g.get("momentum", 0.0)   # momentum correction: applied before the call
        return m, g.get("dampening", 0.0), g.get("weight_decay", 0.0), bool(g.get("nesterov", False))

    @staticmethod
    def update(opt, b, g, s, e, fs, first, launch):
        lr = g["lr"]
        m, damp, wd, nest = _SGDUpdate.hyper(opt, g)
        if launch is not None:
            launch(ext.require().fused_sgd, m, damp, wd, int(nest), int(first))
            return
        gs, ms = b.grad[s:e], fs["momentum_buffer"][s:e]
        if b.flat_param is not None:
            _SGDUpdate.math(b.flat_param[s:e], gs, ms, lr, m, damp, wd, nest, first)
        else:
            for p, o in zip(b.params, b.offsets):
                if s <= o < e:
                    _SGDUpdate.math(p.data.view(-1), gs[o - s:o - s + p.numel()], ms[o - s:o - s + p.numel()],
                                    lr, m, damp, wd, nest, first)

    @staticmethod
    def math(p, g, mom, lr, m, damp, wd, nest, first) -> None:
        d = g.add(p, alpha=wd) if wd != 0 else g.clone()
        if m != 0:
            if first:
                mom.copy_(d)
            else:
                mom.mul_(m).add_(d, alpha=1 - damp)
            d = d.add(mom, alpha=m) if nest else mom
        p.add_(d, alpha=-lr)


class _AdamUpdate:
    """``torch.optim.Adam`` / ``AdamW`` built with ``fused=True`` (see ``_fused_adam_applies``): kernel only."""
    keys = ("exp_avg", "exp_avg_sq")
    n_scalars = 3

    @staticmethod
    def scalars(opt, g):
        if opt._hyper_dev is not None:            # loss scaling: the device knows t (csrc/scale.cu adam_scalars)
            return (float(g["lr"]), float(g["weight_decay"]), float(g["betas"][0]), float(g["betas"][1]))
        # torch's non-capturable Adam, in double: t = the step about to run
        lr, (b1, b2), t = float(g["lr"]), g["betas"], float(opt.counter + 1)
        return (1 - lr * g["weight_decay"], (lr / (1 - b1 ** t)) * -1, (1 - b2 ** t) ** 0.5)

    @staticmethod
    def update(opt, b, g, s, e, fs, first, launch):
        launch(ext.require().fused_adam, g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"],
               int(bool(g["decoupled_weight_decay"])))


class _BertAdamUpdate:
    """``BertAdam``: no bias correction, decoupled weight decay, the learning rate of its schedule.  Device scalars: the
    scheduled lr and the group's ``max_grad_norm`` (the bound of the per-parameter clip on the device)."""
    keys = ("next_m", "next_v")
    n_scalars = 2

    @staticmethod
    def scalars(opt, g):
        return (float(opt._scheduled_lr(g, opt.counter)), float(g["max_grad_norm"]))

    @staticmethod
    def update(opt, b, g, s, e, fs, first, launch):
        if opt.clip_reduced and g["max_grad_norm"] > 0 and opt._clip is None:     # the reference of the device clip
            for p, o in zip(b.params, b.offsets):
                if s <= o < e:
                    gv = b.grad[o:o + p.numel()]
                    nrm = float(gv.norm())
                    if nrm > g["max_grad_norm"]:
                        gv.mul_(g["max_grad_norm"] / (nrm + 1e-6))
        if launch is not None:
            launch(ext.require().fused_bert_adam, g["b1"], g["b2"], g["e"], g["weight_decay"])
            return
        lr = opt._scheduled_lr(g, opt.counter)
        gs, ms, vs = b.grad[s:e], fs["next_m"][s:e], fs["next_v"][s:e]
        ms.mul_(g["b1"]).add_(gs, alpha=1 - g["b1"])
        vs.mul_(g["b2"]).addcmul_(gs, gs, value=1 - g["b2"])
        upd = ms / (vs.sqrt() + g["e"])
        if b.flat_param is not None:
            ps = b.flat_param[s:e]
            if g["weight_decay"] > 0.0:
                upd += g["weight_decay"] * ps
            ps.add_(upd, alpha=-lr)
        else:
            for p, o in zip(b.params, b.offsets):
                if s <= o < e:
                    u = upd[o - s:o - s + p.numel()].view_as(p)
                    if g["weight_decay"] > 0.0:
                        u = u + g["weight_decay"] * p.data
                    p.data.add_(u, alpha=-lr)


class _LambUpdate:
    """``Lamb``: ``fused_lamb``'s three kernels per slice, or ``_lamb_param`` per parameter on the bucket's views.  Device
    scalars: {lr, weight_decay, 1 - beta1^t, 1 - beta2^t}; under loss scaling the device derives them from its step count
    (``adam_scalars`` with lamb=1) out of {lr, weight_decay, beta1, beta2}.  Betas of 0 stand for no bias correction:
    1 - 0^t = 1."""
    keys = ("exp_avg", "exp_avg_sq")
    n_scalars = 4

    @staticmethod
    def scalars(opt, g):
        b1, b2 = g["betas"] if g["bias_correction"] else (0.0, 0.0)
        if opt._hyper_dev is not None:
            return (float(g["lr"]), float(g["weight_decay"]), float(b1), float(b2))
        t = float(opt.counter + 1)
        return (float(g["lr"]), float(g["weight_decay"]), 1 - b1 ** t, 1 - b2 ** t)

    @staticmethod
    def update(opt, b, g, s, e, fs, first, launch):
        if launch is not None:
            n = opt._lamb
            t0, nseg, nblk = n.segs.slices[b.index, s]
            tab = [x.data_ptr() + 4 * t0 for x in (n.segs.off, n.segs.len, n.segs.blk, n.segs.ends)]
            launch(ext.require().fused_lamb, g["betas"][0], g["betas"][1], g["eps"], nseg, *tab, nblk,
                   n.partial[0].data_ptr(), n.partial[1].data_ptr(), n.norm[0].data_ptr() + 4 * t0,
                   n.norm[1].data_ptr() + 4 * t0, n.ratio.data_ptr() + 4 * t0)
            return
        t = opt.counter + 1
        for p, o, gv in zip(b.params, b.offsets, b.grad_views):
            if s <= o < e:
                _lamb_param(p.data, gv, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"], g, t)


class _LambNorms:
    """What ``fused_lamb`` keeps between its passes, allocated with the optimizer (never inside a captured step): the
    per-parameter segment table, the fp64 partial sums of w^2 and u^2 (``partial[0]`` / ``partial[1]``), and per
    parameter ||w||, ||u|| (``norm[0]`` / ``norm[1]``) and the trust ratio, in the table's segment order
    (``segs.params``) as of the last applied step."""

    def __init__(self, opt):
        dev = opt._buckets[0].grad.device
        self.segs = _SegTable(opt._buckets, dev)
        self.partial = torch.zeros(2, self.segs.npart, dtype=torch.float64, device=dev)
        self.norm = torch.zeros(2, self.segs.nseg, dtype=torch.float32, device=dev)
        self.ratio = torch.ones(self.segs.nseg, dtype=torch.float32, device=dev)


# ====================================================================================== DistributedOptimizer
class _DistributedOptimizerMixin(_BucketedComm):
    def state_dict(self):
        sd = super().state_dict()
        scale = self._scale_state_dict()
        if self._update is _AdamUpdate or self._update is _LambUpdate:
            # torch's Adam format: a float32 0-dim step, on the param's device for fused Adam, on the host for Lamb
            params = [p for g in self.param_groups for p in g["params"]]
            steps = scale["adam_step"] if scale is not None else self.counter     # skipped steps do not count
            for i, st in list(sd["state"].items()):
                dev = params[i].device if self._update is _AdamUpdate else "cpu"
                sd["state"][i] = dict(st, step=torch.tensor(float(steps), dtype=torch.float32, device=dev))
        sd["oktopk"] = self._allreducer.state_dict()
        if scale is not None:
            sd["loss_scale"] = scale
        return sd

    def load_state_dict(self, state_dict):
        state_dict = dict(state_dict)
        okt = state_dict.pop("oktopk", None)
        scale = state_dict.pop("loss_scale", None)
        super().load_state_dict(state_dict)
        if self._update is not None:
            self._adopt_state()
        self._load_scale_state(scale, getattr(self, "counter", 0))
        if okt is not None:
            self._allreducer.load_state_dict(okt)
        self._clear_buckets()


def DistributedOptimizer(optimizer: torch.optim.Optimizer, named_parameters=None, compression=NoneCompressor,
                         is_sparse: bool = False, err_handler=None, layerwise_times=None, sigma_scale: float = 2.5,
                         density: float = 0.1, norm_clip: Optional[float] = None, writer=None,
                         cfg: Optional[OkTopkConfig] = None, world: Optional[World] = None,
                         backend: Optional[str] = None, flatten_params: bool = True,
                         loss_scale: Optional[LossScale] = None, max_grad_norm: Optional[float] = None):
    """Wrap ``optimizer`` so that ``step()`` first allreduces the gradients with the chosen scheme.

    Horovod-style dynamic subclass of the user's optimizer class, as in the reference
    (``VGG/distributed_optimizer.py:203-207``).  ``compression`` may be a registry key, a compressor
    class (``compressors['oktopk']``) or an instance; ``cfg`` overrides the scalar arguments.
    ``loss_scale``: dynamic loss scaling for fp16 training (see ``LossScale``); back-propagate
    ``opt.scale_loss(loss)``.
    ``max_grad_norm``: clip the reduced gradient as ``synchronize(); clip_grad_norm_(params, max_grad_norm); step()``
    does, the norm over every parameter of the optimizer (``grad_norm()`` returns it).  With SGD or the fused Adam /
    AdamW or ``Lamb`` on flat CUDA buckets the clip runs on the device inside ``step()`` (the update kernels apply the
    factor; the bucket is not rescaled in place); otherwise ``step()`` calls ``clip_grad_norm_`` over the bucket views.
    A wrapped ``Lamb`` takes the fused LAMB kernels on flat CUDA buckets, its own per-parameter math elsewhere.
    """
    if max_grad_norm is not None and not float(max_grad_norm) > 0:
        raise ValueError("max_grad_norm must be a positive number, got %r" % (max_grad_norm,))
    base_cls = optimizer.__class__
    cls = type(base_cls.__name__, (_DistributedOptimizerMixin, base_cls), {})
    obj = cls.__new__(cls)
    base_cls.__init__(obj, optimizer.param_groups)
    obj.state.update(optimizer.state)
    ar = AllReducer(compression=compression, sparse=is_sparse, density=density, cfg=cfg, world=world,
                    backend=backend, err_callback=err_handler, layerwise_times=layerwise_times,
                    sigma_scale=sigma_scale, norm_clip=norm_clip, writer=writer)
    if isinstance(optimizer, torch.optim.SGD):
        obj._update = _SGDUpdate
    elif _fused_adam_applies(optimizer):
        obj._update = _AdamUpdate
    elif isinstance(optimizer, Lamb):
        obj._update = _LambUpdate
    else:
        obj._update = None                        # torch's own step()
    if obj._update is not None:
        obj.counter = 0                           # steps taken: Adam's bias correction (GraphedTrainStep keeps it too)
    obj._okt_setup(named_parameters, ar, flatten_params=flatten_params, loss_scale=loss_scale,
                   max_grad_norm=None if max_grad_norm is None else float(max_grad_norm))
    if obj._update is not None and obj.state:
        obj._adopt_state()
        obj._load_scale_state(None, obj.counter)
    return obj


def _fused_adam_applies(opt: torch.optim.Optimizer) -> bool:
    """A torch Adam / AdamW that asked for a fused kernel (``fused=True``) and whose options the flat-bucket kernel
    implements: it then runs ``fused_adam`` instead of torch's update.  Flat fp32 CUDA buckets are checked at setup."""
    if not isinstance(opt, torch.optim.Adam):
        return False
    for g in opt.param_groups:
        if g.get("fused") is not True or g.get("amsgrad") or g.get("maximize") or g.get("differentiable"):
            return False
        if torch.is_tensor(g["lr"]) or any(torch.is_tensor(b) for b in g["betas"]):
            return False
        if any(not p.is_cuda or p.dtype != torch.float32 for p in g["params"]):
            return False
    return True


def rank() -> int:
    return _world().rank


def size() -> int:
    return _world().size


def broadcast_parameters(model_or_params, root_rank: int = 0, world: Optional[World] = None) -> None:
    """One-time parameter sync (the reference pickles the whole ``state_dict`` through
    ``comm.bcast``, ``VGG/main_trainer.py:52-55``)."""
    w = world or _world()
    if w.size == 1:
        return
    if isinstance(model_or_params, torch.nn.Module):
        tensors = list(model_or_params.state_dict().values())
    else:
        tensors = [p.data if isinstance(p, torch.nn.Parameter) else p for p in model_or_params]
    for t in tensors:
        if torch.is_tensor(t):
            w.broadcast(t, root_rank)
    w.barrier()


# ====================================================================================== BertAdam
def warmup_cosine(x, warmup=0.002):
    if x < warmup:
        return x / warmup
    return 0.5 * (1.0 + math.cos(math.pi * x))


def warmup_constant(x, warmup=0.002):
    if x < warmup:
        return x / warmup
    return 1.0


def warmup_linear(x, warmup=0.002):
    if x < warmup:
        return x / warmup
    return max((x - 1.0) / (warmup - 1.0), 0.0)


def warmup_poly(x, warmup=0.002, degree=0.5):
    if x < warmup:
        return x / warmup
    return (1.0 - x) ** degree


SCHEDULES = {
    "warmup_cosine": warmup_cosine,
    "warmup_constant": warmup_constant,
    "warmup_linear": warmup_linear,
    "warmup_poly": warmup_poly,
}


def scheduled_lr(lr: float, step: int, t_total: int, warmup: float, schedule: str = "warmup_linear") -> float:
    """BertAdam's learning rate after ``step`` steps: ``lr`` times ``schedule`` at step / t_total, or ``lr`` itself
    when ``t_total`` is -1."""
    if t_total != -1:
        return lr * SCHEDULES[schedule](step / t_total, warmup)
    return lr


class BertAdam(_BucketedComm, torch.optim.Optimizer):
    """BERT's Adam (no bias correction, decoupled weight decay, warm-up schedules) with the sparse
    allreducer embedded -- ``BERT/bert/transformers/optimization.py:68-227``.

    ``max_grad_norm``: the reference calls ``clip_grad_norm_(p, ...)`` on the *local* ``p.grad`` and
    then applies the *reduced* gradient, so its clipping never affects the update (A.4-6).  Here
    ``clip_reduced=True`` clips the reduced per-parameter gradient for real; the default reproduces the
    reference's effective behaviour (no clipping).  On flat CUDA buckets that clip runs on the device (``_GradClip``:
    no host synchronisation, so the step can be captured in a CUDA graph), elsewhere in torch per parameter.
    """

    def __init__(self, params, lr=1e-3, warmup=-1, t_total=-1, schedule="warmup_linear", b1=0.9, b2=0.999, e=1e-6,
                 weight_decay=0.01, max_grad_norm=1.0, density=1.0, compressor="none", rank=-1, named_parameters=None,
                 cfg: Optional[OkTopkConfig] = None, world: Optional[World] = None, backend: Optional[str] = None,
                 clip_reduced: bool = False, flatten_params: bool = True, loss_scale: Optional[LossScale] = None,
                 **_ignored):
        if lr < 0.0:
            raise ValueError("Invalid learning rate: {} - should be >= 0.0".format(lr))
        if schedule not in SCHEDULES:
            raise ValueError("Invalid schedule parameter: {}".format(schedule))
        if not 0.0 <= warmup < 1.0 and not warmup == -1:
            raise ValueError("Invalid warmup: {} - should be in [0.0, 1.0[ or -1".format(warmup))
        if not 0.0 <= b1 < 1.0 or not 0.0 <= b2 < 1.0 or not e >= 0.0:
            raise ValueError("Invalid Adam hyper-parameters")
        defaults = dict(lr=lr, schedule=schedule, warmup=warmup, t_total=t_total, b1=b1, b2=b2, e=e,
                        weight_decay=weight_decay, max_grad_norm=max_grad_norm)
        torch.optim.Optimizer.__init__(self, params, defaults)
        self.rank = rank
        self.counter = 0                          # steps taken: the schedule's position and every parameter's step
        self.clip_reduced = clip_reduced
        self._update = _BertAdamUpdate
        base = cfg if cfg is not None else OkTopkConfig(
            warmup_iters=0, local_recompute_interval=128, global_recompute_interval=128, overselect_guard_loops=0,
            local_adapt_low=4 / 5, local_adapt_high=5 / 4, local_adapt_factor=1.025, global_adapt_low=4 / 5,
            global_adapt_high=5 / 4, global_adapt_inc=1.036, global_adapt_dec=1.025, balanced_allgather=True)
        ar = AllReducer(compression=compressor, sparse=(compressor != "none"), density=density,
                        cfg=base.replace(density=density), world=world, backend=backend)
        self._okt_setup(named_parameters, ar, flatten_params=flatten_params, loss_scale=loss_scale,
                        clip_per_param=clip_reduced)

    def get_lr(self) -> List[float]:
        out = []
        for g in self.param_groups:
            out.append(self._scheduled_lr(g, self.counter))
        return out if self.counter > 0 else [0]

    @staticmethod
    def _scheduled_lr(g: dict, step: int) -> float:
        return scheduled_lr(g["lr"], step, g["t_total"], g["warmup"], g["schedule"])

    def state_dict(self):
        sd = torch.optim.Optimizer.state_dict(self)
        for i, st in list(sd["state"].items()):
            sd["state"][i] = dict(st, step=self.counter)
        sd["oktopk"] = self._allreducer.state_dict()
        sd["counter"] = self.counter
        scale = self._scale_state_dict()
        if scale is not None:
            sd["loss_scale"] = scale
        return sd

    def load_state_dict(self, state_dict):
        state_dict = dict(state_dict)
        okt = state_dict.pop("oktopk", None)
        counter = state_dict.pop("counter", 0)
        scale = state_dict.pop("loss_scale", None)
        torch.optim.Optimizer.load_state_dict(self, state_dict)
        self._adopt_state(counter)
        self._load_scale_state(scale, counter)
        if okt is not None:
            self._allreducer.load_state_dict(okt)
        self._clear_buckets()


# ====================================================================================== LAMB
def _lamb_param(w: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, group: dict, t: int) -> None:
    """One LAMB step of parameter tensor ``w`` (in place, with its moments ``m`` and ``v``) at step ``t`` (1-based)."""
    b1, b2 = group["betas"]
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    bc1, bc2 = (1 - b1 ** t, 1 - b2 ** t) if group["bias_correction"] else (1.0, 1.0)
    u = (m / bc1).div_((v / bc2).sqrt_().add_(group["eps"]))
    wd = group["weight_decay"]
    if wd == 0:
        w.add_(u, alpha=-group["lr"])
        return
    u.add_(w, alpha=wd)
    wn, un = w.norm(), u.norm()
    r = torch.where((wn > 0) & (un > 0), wn / un, torch.ones_like(wn))       # the trust ratio, 1 for a zero norm
    w.sub_(u.mul_(r * group["lr"]))


class Lamb(torch.optim.Optimizer):
    """LAMB (You et al., "Large Batch Optimization for Deep Learning: Training BERT in 76 minutes"), as apex's
    ``FusedLAMB`` computes it with its defaults (``adam_w_mode=True``, ``grad_averaging=True``, ``use_nvlamb=False``)
    but without its global gradient clip.  For each parameter tensor w with gradient g at step t (1-based)::

        m = b1*m + (1-b1)*g;   v = b2*v + (1-b2)*g*g
        m_hat = m / (1 - b1^t);   v_hat = v / (1 - b2^t)          (bias_correction=False: m_hat = m, v_hat = v)
        u = m_hat / (sqrt(v_hat) + eps) + wd*w
        r = ||w|| / ||u||  if wd != 0 and both norms are > 0, else 1      (norms over the one tensor)
        w = w - lr * r * u

    This class runs that in torch ops, one parameter at a time (state ``exp_avg``, ``exp_avg_sq`` and ``step`` as in
    torch's Adam).  Wrapped in ``DistributedOptimizer`` on flat CUDA buckets it runs on the fused LAMB kernels, and
    ``DistributedOptimizer(..., max_grad_norm=c)`` adds the global clip of ``clip_grad_norm_`` before the step."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-6, weight_decay: float = 0.01,
                 bias_correction: bool = True):
        if torch.is_tensor(lr) or not lr >= 0.0:
            raise ValueError("Invalid learning rate: %r (a number >= 0)" % (lr,))
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid betas: %r" % (betas,))
        if not eps >= 0.0 or not weight_decay >= 0.0:
            raise ValueError("Invalid eps or weight_decay: %r, %r" % (eps, weight_decay))
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay,
                                      bias_correction=bool(bias_correction)))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["step"] += 1
                _lamb_param(p, p.grad, st["exp_avg"], st["exp_avg_sq"], group, int(st["step"]))
        return loss
