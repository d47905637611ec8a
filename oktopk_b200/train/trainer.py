"""Trainer (L1/L2): model + data + loss + LR schedule + evaluation + the S-SGD loop.

Capability parity with ``DLTrainer`` (``VGG/dl_trainer.py:105-796``) and ``robust_ssgd``
(``VGG/main_trainer.py:26-140``), and with the data-parallel branch of the BERT ``StageRuntime``
(``BERT/runtime.py:842-900``): per-workload optimizer defaults, warm-up/step LR schedules, gradient
accumulation through ``optimizer.local``, LSTM gradient clipping between ``synchronize()`` and
``step()``, periodic throughput logging, evaluation (top-1 / perplexity / greedy-CTC WER),
checkpoint save/resume that includes the sparse-allreduce state.
"""
from __future__ import annotations

import json
import math
import os
import time
from typing import Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import compression as _comp
from ..config import LossScale, OkTopkConfig, preset as _preset
from ..models import create_net
from ..models.bert import BertPreTrainingHeads
from ..ops.fused_ctc import ctc_loss
from ..ops.fused_xent import softmax_cross_entropy
from ..optimizer import BertAdam, DistributedOptimizer, Lamb, broadcast_parameters, scheduled_lr
from ..parallel.world import World, world as _world
from ..utils.logging import get_logger
from ..utils.metrics import MetricsWriter, PhaseTimers
from . import data as D

_DATASET_OF = {"lstman4": "an4", "lstm": "ptb", "bert": "wikipedia", "bert_base": "wikipedia", "mnistnet": "mnist",
               "alexnet": "imagenet", "resnet18": "imagenet", "resnet34": "imagenet", "resnet50": "imagenet",
               "resnet101": "imagenet", "resnet152": "imagenet"}


def preset_for(dnn: str) -> str:
    if dnn in ("lstman4", "lstm"):
        return "lstm_an4"
    if dnn.startswith("bert"):
        return "bert_base"
    return "vgg16"


class Trainer:
    def __init__(self, dnn: str = "vgg16", dataset: Optional[str] = None, data_dir: Optional[str] = None,
                 batch_size: int = 16, lr: float = 0.1, nsteps_update: int = 1, max_epochs: int = 1,
                 compressor: str = "oktopk", density: float = 0.001, compression: bool = True,
                 cfg: Optional[OkTopkConfig] = None, world: Optional[World] = None, device: Optional[torch.device] = None,
                 seed: int = 0, prefix: str = "run", log_dir: Optional[str] = None, num_workers: int = 0,
                 seq_len: int = 128, t_total: int = -1, warmup: float = -1, pretrain: Optional[str] = None,
                 norm_clip: Optional[float] = None, backend: Optional[str] = None, cuda_graph: bool = False,
                 model_kwargs: Optional[dict] = None, autocast: Optional[str] = None, loss_scale=None,
                 an4_pad_multiple: int = 0, fused_clip: bool = False, lamb: bool = False):
        """``an4_pad_multiple=m >= 1`` (AN4 only; 0, the default, is off): every training batch is staged into a
        ``data.PaddedAN4Batch`` with its frames padded up to a multiple of m and its lengths on the device, and with
        ``cuda_graph`` the steps are captured per padded length (``GraphedTrainStep``).  With the stock batch-norm the
        padded frames change one thing: those layers count them in their statistics, as they count the padding inside a
        batch.  With ``fuse_bn`` (``model_kwargs``) the statistics stop at the longest utterance and the padded batch
        gives the unpadded batch's loss and gradients to rounding.

        ``fused_clip`` (AN4 and PTB, the two workloads that clip the reduced gradient every step; off by default): the
        clip runs on the device inside the optimizer's step (``DistributedOptimizer(max_grad_norm=...)``): one norm pass
        and a factor that the fused update applies, instead of ``clip_grad_norm_`` between ``synchronize()`` and
        ``step()``.  The same factor as torch's up to the norm's rounding, no host synchronisation.

        ``lamb`` (BERT only; off by default): the optimizer is ``Lamb`` wrapped in ``DistributedOptimizer`` with the
        global clip ``max_grad_norm=1.0`` on the device, over BertAdam's two param groups (weight decay 0.01, none for
        biases and LayerNorm), its learning rate following BertAdam's warmup_linear schedule over ``t_total`` /
        ``warmup``, instead of ``BertAdam``."""
        self.world = world or _world()
        self.rank, self.nworkers = self.world.rank, self.world.size
        # The host side of a step is tiny tensor ops (collate 16 images, one pinned copy): on a many-core box an
        # unconstrained intra-op pool costs milliseconds of thread wake-ups per op.  torchrun already pins
        # OMP_NUM_THREADS=1 per rank; do the equivalent for a plain `python` launch.
        if "OMP_NUM_THREADS" not in os.environ:
            # GPU training: ONE intra-op thread.  The host ops of a step are tiny (collate 16 images, a 200 KB pinned copy);
            # split across an OpenMP team they cost team wake-ups / barrier spins, which on a busy or core-limited box took
            # the staging of one batch from a fraction of a millisecond to several
            want = 1 if torch.cuda.is_available() else 4
            if torch.get_num_threads() > want:
                torch.set_num_threads(want)
        self.dnn = dnn
        # the bound LSTM/main_trainer.py:94-99 clips the reduced gradient to, per model
        self.clip_norm = {"lstman4": 400.0, "lstm": 0.25}.get(dnn)
        if fused_clip and self.clip_norm is None:
            raise ValueError("fused_clip applies to lstman4 and lstm, the models that clip their gradient; not %s" % dnn)
        self.fused_clip = bool(fused_clip)
        if lamb and not dnn.startswith("bert"):
            raise ValueError("lamb applies to the BERT models; not %s" % dnn)
        self.lamb = bool(lamb)
        self.t_total, self.warmup = t_total, warmup
        self.dataset = (dataset or _DATASET_OF.get(dnn, "cifar10")).lower()
        if an4_pad_multiple < 0 or (an4_pad_multiple and self.dataset != "an4"):
            raise ValueError("an4_pad_multiple must be 0 (off) or, for the AN4 dataset, >= 1; got %r for %s"
                             % (an4_pad_multiple, self.dataset))
        self.an4_pad_multiple = int(an4_pad_multiple)
        self._an4_out_frames: Dict[int, int] = {}
        self.batch_size, self.lr, self.nsteps_update, self.max_epochs = batch_size, lr, nsteps_update, max_epochs
        self.device = device or (torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available()
                                 else torch.device("cpu"))
        self.logger = get_logger(self.rank, log_dir)
        self.writer = MetricsWriter(log_dir, self.rank)
        self.timers = PhaseTimers()
        torch.manual_seed(seed)
        self.seq_len = seq_len
        # ---- model ------------------------------------------------------------------------
        self.num_classes = D.DATASET_CLASSES.get(self.dataset, 10)
        net, self.ext = create_net(self.num_classes, dnn, **(model_kwargs or {}))
        # optional mixed precision (the reference's --fp16 is apex O3, off in every script; bf16 autocast here)
        self.autocast = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(autocast or "", None)
        # dynamic (or fixed) loss scaling, off by default: "dynamic", a number (fixed scale) or a LossScale
        self.loss_scale = LossScale.parse(loss_scale)
        self.net = net.to(self.device)
        self.is_bert = dnn.startswith("bert")
        # masked-LM heads whose overflow counter check_mlm_overflow() reads when their sparse_mlm switch is on
        self._mlm_heads = [m for m in self.net.modules() if isinstance(m, BertPreTrainingHeads)]
        # CNN zoo on the GPU: channels_last weights and activations.  cuDNN's TF32/fp32 convolution kernels are NHWC: with
        # NCHW tensors every convolution is bracketed by nchwToNhwc / nhwcToNchw transposes.  Numerics are unchanged (same kernels, no layout conversion).
        self.channels_last = (self.device.type == "cuda" and not self.is_bert and dnn not in ("lstman4", "lstm")
                              and os.environ.get("OKTOPK_CHANNELS_LAST", "1") == "1")
        if self.channels_last:
            self.net = self.net.to(memory_format=torch.channels_last)
        # cuDNN autotuning (opt-in, OKTOPK_CUDNN_BENCHMARK=1): slightly faster device-resident steps on VGG-16 but a
        # much slower end-to-end path, so it stays off by default.
        if (cuda_graph and self.channels_last and os.environ.get("OKTOPK_CUDNN_BENCHMARK", "0") == "1"):
            torch.backends.cudnn.benchmark = True
        if pretrain:
            self.load_checkpoint(pretrain, model_only=True)
        broadcast_parameters(self.net, 0, self.world)
        # ---- loss ---------------------------------------------------------------------------
        if self.dataset == "an4":
            self.criterion = nn.CTCLoss(blank=0, reduction="sum", zero_infinity=True)   # warpctc semantics: summed
        else:
            self.criterion = nn.CrossEntropyLoss()
        # ---- optimizer (VGG/dl_trainer.py:183-198; BERT/bert/main_bert.py:972-997) ----------------
        if cfg is None:
            cfg = _preset(preset_for(dnn), density=density)
        self.cfg = cfg.replace(compressor=compressor if compression else "none", sparse=compression and compressor != "none",
                               norm_clip=norm_clip)
        if backend:
            self.cfg = self.cfg.replace(backend=backend)
        if self.is_bert:
            no_decay = ("bias", "norm", "LayerNorm")
            named = list(self.net.named_parameters())
            groups = [{"params": [p for n, p in named if not any(nd in n for nd in no_decay)], "weight_decay": 0.01},
                      {"params": [p for n, p in named if any(nd in n for nd in no_decay)], "weight_decay": 0.0}]
            if self.lamb:
                self.optimizer = DistributedOptimizer(Lamb(groups, lr=lr), named_parameters=named,
                                                      compression=_comp.compressors[self.cfg.compressor],
                                                      is_sparse=self.cfg.sparse, density=self.cfg.density,
                                                      cfg=self.cfg, world=self.world, err_handler=self._err_handler,
                                                      loss_scale=self.loss_scale, max_grad_norm=1.0)
            else:
                self.optimizer = BertAdam(groups, lr=lr, warmup=warmup, t_total=t_total, density=self.cfg.density,
                                          compressor=self.cfg.compressor, rank=self.rank, named_parameters=named,
                                          cfg=self.cfg, world=self.world, loss_scale=self.loss_scale)
        else:
            if self.dataset == "ptb":
                base = torch.optim.SGD(self.net.parameters(), lr=lr, momentum=0.0, weight_decay=0.0)
            elif self.dataset == "imagenet":
                base = torch.optim.SGD(self.net.parameters(), lr=lr, momentum=0.9, weight_decay=5e-4)
            else:
                base = torch.optim.SGD(self.net.parameters(), lr=lr, momentum=0.9, weight_decay=1e-4)
            self.optimizer = DistributedOptimizer(base, named_parameters=self.net.named_parameters(),
                                                  compression=_comp.compressors[self.cfg.compressor],
                                                  is_sparse=self.cfg.sparse, cfg=self.cfg, world=self.world,
                                                  err_handler=self._err_handler, loss_scale=self.loss_scale,
                                                  max_grad_norm=self.clip_norm if self.fused_clip else None)
        # ---- data -----------------------------------------------------------------------------
        self.trainset = D.build_dataset(self.dataset, data_dir, train=True, seed=seed, seq=seq_len, batch_size=batch_size)
        self.loader, self.sampler = D.build_loader(self.trainset, self.dataset, batch_size, self.rank, self.nworkers,
                                                   train=True, num_workers=num_workers, seed=seed)
        self.prefetch = D.Prefetcher(self.loader, self.device, self.sampler)
        self.iters_per_epoch = max(len(self.loader), 1)
        self.testset = None
        self.train_epoch, self.train_iter = 0, 0
        self.loss_sum, self.loss_n, self.acc_sum = 0.0, 0, 0.0
        self.hidden = None
        self._loss_pin, self._loss_ev, self._loss_head, self._loss_hist = None, None, 0, []
        self.host_us = {"next": 0.0, "launch": 0.0, "stage_next": 0.0, "steps": 0}
        self.sparsities: List[float] = []
        self._iter_times: List[float] = []
        # whole-step CUDA graphs (graph_step: one input rule per kind of batch); unpadded AN4 batches vary in length
        self.graphed = None
        graph_ok = self.dataset != "an4" or self.an4_pad_multiple >= 1
        if cuda_graph and self.device.type == "cuda" and graph_ok and nsteps_update == 1:
            from .graph_step import GraphedTrainStep
            self.graphed = GraphedTrainStep(self)

    # ------------------------------------------------------------------ LR schedules
    def adjust_learning_rate(self) -> float:
        """``VGG/dl_trainer.py:507-563``."""
        e = self.train_epoch + (self.train_iter % self.iters_per_epoch) / float(self.iters_per_epoch)
        if self.is_bert and not self.lamb:
            return self.lr                                     # BertAdam schedules internally
        if self.is_bert:                                       # BertAdam's schedule at the optimizer's step count
            lr = scheduled_lr(self.lr, self.optimizer.counter, self.t_total, self.warmup)
        elif self.dnn == "lstman4":
            lr = self.lr / (1.01 ** self.train_epoch)           # /1.01 per epoch (:507-512)
        elif self.dnn == "lstm":
            # PTB step schedule (:514-529; the first boundary is 23+40 = 63 there, *after* the second one at 60, so the
            # 0.1x stage never happens: 1x until epoch 63, 0.01x until 80, 0.001x afterwards)
            ep = self.train_epoch
            lr = self.lr if ep < 63 else (self.lr * 0.01 if ep < 80 else self.lr * 0.001)
        else:
            # general schedule (:531-563): linear warm-up over 10 epochs from lr/nworkers, then 0.1x steps at
            # 81/122/155 (CIFAR-10 and the other small datasets), 30/60/80 (ImageNet), 24/60/80 (PTB models)
            warm = 10
            if e < warm and self.nworkers > 1:
                lr0 = self.lr / self.nworkers
                lr = lr0 + (self.lr - lr0) * e / warm
            else:
                bounds = {"imagenet": (30, 60, 80), "ptb": (24, 60, 80)}.get(self.dataset, (81, 122, 155))
                lr = self.lr
                for boundary in bounds:
                    if self.train_epoch >= boundary:
                        lr *= 0.1
        for g in self.optimizer.param_groups:
            g["lr"] = lr
        return lr

    # ------------------------------------------------------------------ one micro-step: forward + backward
    def stage_batch(self, batch):
        """The batch as a step takes it: with ``an4_pad_multiple`` an AN4 batch becomes a ``data.PaddedAN4Batch``
        (device ops only); anything else, or a batch already staged, is returned as it is."""
        if not self.an4_pad_multiple or isinstance(batch, D.PaddedAN4Batch):
            return batch
        return D.pad_an4_batch(batch, self.an4_pad_multiple, self.an4_out_frames)

    def an4_out_frames(self, frames: int) -> int:
        """The AN4 model's output frames for ``frames`` input frames (a host computation, cached)."""
        n = self._an4_out_frames.get(frames)
        if n is None:
            n = self._an4_out_frames[frames] = int(self.net.get_seq_lens(torch.tensor([frames]))[0])
        return n

    def _forward_loss(self, batch):
        if self.autocast is not None:
            with torch.autocast(self.device.type, dtype=self.autocast):
                return self._forward_loss_impl(batch)
        return self._forward_loss_impl(batch)

    def _forward_loss_impl(self, batch):
        if self.is_bert:
            ids, seg, mask, labels, nxt = batch
            return self.net(ids, seg, mask, labels, nxt), None
        if self.dataset == "an4":
            if isinstance(batch, D.PaddedAN4Batch):
                inputs, targets, tsizes = batch.inputs, batch.targets, batch.tsizes
                # device lengths wherever every layer is fused; the stock layers read them on the host
                dev = self.net.device_lengths_error(inputs.is_cuda, torch.is_autocast_enabled("cuda")) is None
                out, out_lens = self.net(inputs, batch.lengths, device_lengths=dev)
                if not (getattr(self.net, "fuse_ctc", False) and targets.is_cuda):
                    targets = targets[:batch.ntargets]     # the stock loss wants exactly the batch's targets
            else:
                inputs, targets, in_pct, tsizes = batch
                lengths = (in_pct * inputs.size(3)).int()
                out, out_lens = self.net(inputs, lengths)
            if getattr(self.net, "fuse_ctc", False):
                return ctc_loss(out.transpose(0, 1), targets, out_lens, tsizes) / inputs.size(0), None
            logp = F.log_softmax(out.transpose(0, 1), dim=-1)          # T x N x C
            # int64 device targets => torch's native CTC kernels (int32 host targets would route to cuDNN's CTC, which
            # has no zero_infinity handling and produced NaN gradients on synthetic utterances)
            loss = self.criterion(logp.float(), targets.to(logp.device).long(), out_lens.to(logp.device).long(),
                                  tsizes.to(logp.device).long()) / inputs.size(0)
            return loss, None
        if self.dataset == "ptb":
            x, y = batch
            x, y = x.t().contiguous(), y.t().contiguous()
            if self.hidden is None or self.hidden[0].size(1) != x.size(1):
                self.hidden = self.net.init_hidden(x.size(1), self.device)
            self.hidden = tuple(h.detach() for h in self.hidden)
            out, self.hidden = self.net(x, self.hidden)
            if getattr(self.net, "fuse_xent", False):
                return softmax_cross_entropy(out.view(-1, out.size(-1)), y.view(-1)), None
            return self.criterion(out.view(-1, out.size(-1)), y.view(-1)), None
        x, y = batch
        if self.channels_last and x.dim() == 4:
            x = x.contiguous(memory_format=torch.channels_last)
        out = self.net(x)
        return self.criterion(out, y), (out, y)

    def backward(self, loss: torch.Tensor) -> None:
        """Back-propagate ``loss`` times the optimizer's loss scale when scaling is on (read on the device: capturable)."""
        self.optimizer.scale_loss(loss).backward()

    def _forward_backward(self, batch) -> torch.Tensor:
        """Every eager step's and captured graph's body; it reads only ``_forward_loss`` and ``optimizer``."""
        loss, _ = self._forward_loss(batch)
        self.optimizer.scale_loss(loss).backward()
        return loss

    def train(self, num_of_iters: int = 1) -> float:
        """``DLTrainer.train`` (``VGG/dl_trainer.py:597-707``): forward+backward micro-steps; the
        communication happens inside backward (bucket hooks), the update in ``update_model``."""
        self.net.train()
        loss_val = 0.0
        for _ in range(num_of_iters):
            self.adjust_learning_rate()
            t0 = time.perf_counter()
            batch = self.stage_batch(self.prefetch.next(defer=True))
            self.timers.add("io", time.perf_counter() - t0)
            loss = self._forward_backward(batch)
            self.prefetch.advance()              # stage the next batch while the GPU works through this one
            self._last_loss = loss.detach()
            self._bookkeep_iter()
        return loss_val

    def last_loss(self) -> float:
        return float(self._last_loss)            # device -> host read (a synchronisation: use record_loss() in loops)

    # ---- asynchronous loss read-back: the step's loss is copied device -> pinned host memory on the compute stream
    #      without blocking the host; values are consumed when their copy has completed (or at flush time).  The host
    #      never stalls on the GPU, which is what lets it run ahead and keep the device busy (per-step float(loss)
    #      serialised host and device: e2e 0.67 scaling efficiency at 8 GPUs in round 1).
    _LOSS_RING = 64

    def record_loss(self) -> None:
        """Enqueue the D2H copy of the last step's loss (4 bytes) into a pinned ring slot."""
        t0 = time.perf_counter()
        self._record_loss()
        self.host_us["record_loss"] = self.host_us.get("record_loss", 0.0) + (time.perf_counter() - t0) * 1e6

    def _record_loss(self) -> None:
        if self.device.type != "cuda":
            self._loss_hist.append(float(self._last_loss))
            return
        if self._loss_pin is None:
            self._loss_pin = torch.zeros(self._LOSS_RING, dtype=torch.float32).pin_memory()
            self._loss_ev = [None] * self._LOSS_RING
        i = self._loss_head % self._LOSS_RING
        if self._loss_ev[i] is not None:                       # slot still holds an unread value: wait for it, keep it
            self._loss_ev[i].synchronize()
            self._loss_hist.append(float(self._loss_pin[i]))
        self._loss_pin[i:i + 1].copy_(self._last_loss.detach().reshape(1), non_blocking=True)
        ev = torch.cuda.Event(blocking=True)
        ev.record()
        self._loss_ev[i] = ev
        self._loss_head += 1

    def flush_losses(self) -> List[float]:
        """All recorded losses so far, in order (waits for the outstanding copies)."""
        if self._loss_pin is not None:
            n = min(self._loss_head, self._LOSS_RING)
            start = self._loss_head - n
            for j in range(start, self._loss_head):
                i = j % self._LOSS_RING
                if self._loss_ev[i] is not None:
                    self._loss_ev[i].synchronize()
                    self._loss_hist.append(float(self._loss_pin[i]))
                    self._loss_ev[i] = None
        self.check_mlm_overflow()
        out, self._loss_hist = self._loss_hist, []
        return out

    def check_mlm_overflow(self) -> None:
        """Raise ``RuntimeError`` if a masked-LM head with ``sparse_mlm`` on has left labelled rows past its capacity
        out of the loss.  Reads the head's device counter, so it waits for the work queued so far: call it where the
        host reads values back anyway (``flush_losses``, the logging points and the end of ``robust_ssgd``)."""
        for h in self._mlm_heads:
            if h.sparse_mlm:
                n = int(h.mlm_overflow)
                if n:
                    raise RuntimeError("the sparse masked-LM head left %d labelled rows out of the loss: more rows were "
                                       "labelled than its capacity of %g of the batch's tokens holds; raise "
                                       "--mlm-capacity (mlm_capacity; 1.0 never overflows)" % (n, h.mlm_capacity))

    def update_model(self) -> None:
        if self.clip_norm is not None and not self.fused_clip:     # clip the *reduced* gradient (fused_clip: in step())
            self.optimizer.synchronize()
            torch.nn.utils.clip_grad_norm_(self.net.parameters(), self.clip_norm)
        self.optimizer.step()

    def _bookkeep_iter(self) -> None:
        self.loss_n += 1
        if self.train_iter % self.iters_per_epoch == self.iters_per_epoch - 1:
            self.train_epoch += 1
            self.optimizer.add_train_epoch()
        self.train_iter += 1

    def step(self, batch) -> torch.Tensor:
        """One optimizer step on ``batch`` (device tensors), graphed when ``cuda_graph`` left the graph step enabled.
        Returns the device loss: the graph's static loss buffer, which the next replay overwrites, or the eager loss."""
        if self.nsteps_update > 1:
            raise ValueError("step() runs one micro-step per update: use train_step() with nsteps_update > 1")
        self.net.train()
        self.adjust_learning_rate()
        if self.graphed is not None and self.graphed.enabled:
            loss = self.graphed.step(batch)
        else:
            self.optimizer.zero_grad()
            loss = self._forward_backward(self.stage_batch(batch)).detach()
            self.update_model()
        self._bookkeep_iter()
        self._last_loss = loss
        return loss

    def train_step(self) -> None:
        """One optimizer update = ``nsteps_update`` micro-steps (``VGG/main_trainer.py:83-100``)."""
        if self.graphed is not None and self.graphed.enabled:
            t0 = time.perf_counter()
            self.net.train()
            self.adjust_learning_rate()
            batch = self.prefetch.next(defer=True)
            t1 = time.perf_counter()
            self._last_loss = self.graphed.step(batch)
            t2 = time.perf_counter()
            self.prefetch.advance()              # host-side staging of the next batch overlaps the replayed step
            self._bookkeep_iter()
            t3 = time.perf_counter()
            h = self.host_us                     # host-side cost of a step, by part (observability: is the host the limiter?)
            h["next"] += (t1 - t0) * 1e6; h["launch"] += (t2 - t1) * 1e6; h["stage_next"] += (t3 - t2) * 1e6; h["steps"] += 1
            return
        self.optimizer.zero_grad()
        for j in range(self.nsteps_update):
            self.optimizer.local = j < self.nsteps_update - 1
            self.train(1)
        self.update_model()

    # ------------------------------------------------------------------ evaluation
    @torch.no_grad()
    def test(self, epoch: int = 0, max_batches: int = 20) -> Dict[str, float]:
        """``DLTrainer.test`` (``VGG/dl_trainer.py:709-784``): top-1 / perplexity / greedy-CTC WER."""
        self.net.eval()
        if self.testset is None:
            self.testset = D.build_dataset(self.dataset, None, train=False, seed=1, seq=self.seq_len, batch_size=self.batch_size)
            self.testloader, _ = D.build_loader(self.testset, self.dataset, self.batch_size, 0, 1, train=False)
        tot_loss, correct, total, wer_num, wer_den = 0.0, 0, 0, 0, 0
        for bi, batch in enumerate(self.testloader):
            if bi >= max_batches:
                break
            batch = tuple(t.to(self.device) if torch.is_tensor(t) else t for t in batch)
            if self.dataset == "an4":
                from ..utils.decoder import GreedyDecoder, wer
                inputs, targets, in_pct, tsizes = batch
                out, out_lens = self.net(inputs, (in_pct * inputs.size(3)).int())
                dec = GreedyDecoder(self.ext["labels"])
                hyp = dec.decode(out.cpu(), out_lens.cpu())
                ref = dec.convert_targets(targets.cpu(), tsizes.cpu())
                for h, r in zip(hyp, ref):
                    wer_num += wer(h, r)
                    wer_den += max(len(r.split()), 1)
                total += inputs.size(0)
            else:
                loss, aux = self._forward_loss(batch)
                tot_loss += float(loss)
                if aux is not None:
                    out, y = aux
                    correct += int((out.argmax(1) == y).sum())
                    total += y.numel()
                else:
                    total += 1
        nb = max(min(len(self.testloader), max_batches), 1)
        res = {"epoch": epoch, "loss": tot_loss / nb}
        if self.dataset == "an4":
            res["wer"] = wer_num / max(wer_den, 1)
        elif self.dataset == "ptb":
            res["perplexity"] = math.exp(min(res["loss"], 50))
        elif not self.is_bert:
            res["top1"] = correct / max(total, 1)
        self.writer.add_scalars("test", res, epoch)
        self.net.train()
        return res

    # ------------------------------------------------------------------ elastic / failure hooks (SURVEY 5.3)
    def _err_handler(self, new_num_workers: int, new_rank: int) -> None:
        self.update_nworker(new_num_workers, new_rank)

    def update_nworker(self, nworkers: int, new_rank: int = -1) -> None:
        """Rebuild the sharded sampler for a resized world (``VGG/dl_trainer.py:472-493``)."""
        if new_rank >= 0:
            self.rank = new_rank
        self.nworkers = nworkers
        self.loader, self.sampler = D.build_loader(self.trainset, self.dataset, self.batch_size, self.rank, nworkers)
        self.prefetch.close()
        self.prefetch = D.Prefetcher(self.loader, self.device, self.sampler)
        self.iters_per_epoch = max(len(self.loader), 1)

    # ------------------------------------------------------------------ checkpoint / resume (SURVEY 5.4)
    def save_checkpoint(self, path: str, collective: bool = True) -> None:
        """``collective=False`` (signal handlers, per-rank interrupted state): this rank writes one self-contained file,
        no barrier.  Otherwise collective when world > 1: rank 0 writes the model / optimizer file; EVERY rank writes its own sparse-allreduce
        state (error-feedback residuals, thresholds, region edges, counters are per-rank quantities: restoring rank 0's
        residual on all ranks would duplicate its accumulated error and lose everybody else's) next to it as
        ``<path>.rank<r>``."""
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        opt_sd = self.optimizer.state_dict()
        sparse = opt_sd.get("oktopk")
        if not collective:
            torch.save({"state": self.net.state_dict(), "optimizer": opt_sd, "epoch": self.train_epoch,
                        "iter": self.train_iter, "dnn": self.dnn, "cfg": self.cfg.to_dict(), "world": self.nworkers}, path)
            return
        if self.nworkers > 1:
            torch.save({"oktopk": sparse, "rank": self.rank, "world": self.nworkers}, "%s.rank%d" % (path, self.rank))
        if self.rank == 0:
            torch.save({"state": self.net.state_dict(), "optimizer": opt_sd, "epoch": self.train_epoch,
                        "iter": self.train_iter, "dnn": self.dnn, "cfg": self.cfg.to_dict(), "world": self.nworkers}, path)
        if self.nworkers > 1:
            self.world.barrier()

    @staticmethod
    def _load_file(path: str):
        try:
            return torch.load(path, map_location="cpu", weights_only=True)     # tensors + plain containers only
        except Exception:  # noqa: BLE001 - checkpoints written by older versions may hold other picklables
            return torch.load(path, map_location="cpu", weights_only=False)

    def load_checkpoint(self, path: str, model_only: bool = False) -> None:
        ck = self._load_file(path)
        self.net.load_state_dict(ck["state"])
        if not model_only:
            opt_sd = dict(ck["optimizer"])
            mine = "%s.rank%d" % (path, self.rank)
            if os.path.isfile(mine):
                per = self._load_file(mine)
                if per.get("world") == self.nworkers and per.get("oktopk") is not None:
                    opt_sd["oktopk"] = per["oktopk"]                              # this rank's own residual / thresholds
            elif self.nworkers > 1 and self.rank != 0 and opt_sd.get("oktopk") is not None:
                # no per-rank file (single-file checkpoint): do not replicate rank 0's residual on the other ranks
                opt_sd["oktopk"] = {**opt_sd["oktopk"], "buckets": {
                    k: {**v, "residual": None} for k, v in opt_sd["oktopk"].get("buckets", {}).items()}}
            self.optimizer.load_state_dict(opt_sd)
            self.train_epoch, self.train_iter = ck.get("epoch", 0), ck.get("iter", 0)

    def close(self) -> None:
        self.prefetch.close()
        self.optimizer.close()
        self.writer.close()


def robust_ssgd(dnn: str, dataset: Optional[str], data_dir: Optional[str], nworkers: int, lr: float, batch_size: int,
                nsteps_update: int, max_epochs: int, compression: bool = False, compressor: str = "topk",
                nwpernode: int = 1, sigma_scale: float = 2.5, pretrain: Optional[str] = None, density: float = 0.01,
                prefix: Optional[str] = None, max_iters: Optional[int] = None, log_every: int = 20,
                checkpoint_dir: Optional[str] = None, **kw) -> Trainer:
    """The reference's training driver (``VGG/main_trainer.py:26-140``) on the CUDA engine."""
    w = _world()
    if torch.cuda.is_available():
        torch.cuda.set_device(w.rank % max(nwpernode if nwpernode > 1 else torch.cuda.device_count(), 1))
    tr = Trainer(dnn=dnn, dataset=dataset, data_dir=data_dir, batch_size=batch_size, lr=lr, nsteps_update=nsteps_update,
                 max_epochs=max_epochs, compressor=compressor, density=density, compression=compression,
                 pretrain=pretrain, prefix=prefix or "run", **kw)
    log = tr.logger
    done = 0
    t_last = time.perf_counter()
    for epoch in range(max_epochs):
        for i in range(tr.iters_per_epoch):
            tr.train_step()
            done += 1
            if done % log_every == 0:
                loss = tr.last_loss()
                tr.optimizer.check_faults()
                tr.check_mlm_overflow()
                dt = (time.perf_counter() - t_last) / log_every
                t_last = time.perf_counter()
                if w.rank == 0:
                    log.info("Time per iteration including communication: %f, Speed: %f images/s, current density: %f, loss %f",
                             dt, batch_size * nsteps_update / dt, tr.optimizer.get_current_density(), loss)
                    tr.writer.add_scalars("train", {"loss": loss, "iter_time": dt,
                                                    "samples_per_s": batch_size * nsteps_update * w.size / dt}, done)
            if max_iters is not None and done >= max_iters:
                break
        if checkpoint_dir:                       # collective: every rank saves its own sparse state
            tr.save_checkpoint(os.path.join(checkpoint_dir, "%s-rank0-epoch%d.pth" % (dnn, epoch)))
        if max_iters is not None and done >= max_iters:
            break
    tr.optimizer.stop()
    tr.check_mlm_overflow()
    return tr
