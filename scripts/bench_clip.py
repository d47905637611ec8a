#!/usr/bin/env python
"""Gradient clipping inside the optimizer step (``Trainer(fused_clip=True)``: ``grad_sumsq`` + ``clip_coef``, the factor
applied by the fused SGD update) against the stock ``synchronize(); clip_grad_norm_(); step()``.

    python scripts/bench_clip.py [--steps 30] [--runs 5] [--prof-steps 10]

Workloads, Ok-Topk at the bench densities:
  * AN4 (``bench.MODELS["lstman4"]``, 27.6 M parameters, bound 400), graphed, ``an4_pad_multiple=32``, ``fuse_lstm`` and
    ``fuse_ctc``, in fp32 and in bf16 with ``fuse_lstm_autocast``, on ``bench.make_batch`` i = 0..7;
  * PTB (66.0 M parameters, bound 0.25), bf16 with ``fuse_lstm`` and ``fuse_xent``, eager, on the synthetic stream.
1. ``--runs`` alternating runs of ``--steps`` steps per arm: median (range) ms/step from CUDA events.
2. A ``torch.profiler`` run of its own per arm (``--prof-steps`` steps): device time per step of the clip path, that is
   the clip's kernels (stock: every kernel ``clip_grad_norm_`` launches, measured on the live reduced gradient; fused:
   ``grad_sumsq`` and ``clip_coef``) plus the step's fused SGD update kernels, which read the factor.
Prints the card, its power limit and SM clock, before and after, and one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("OMP_NUM_THREADS", "1")

import bench  # noqa: E402  (make_batch, MODELS: the bench workload definition)
from scripts.bench_bf16 import _card  # noqa: E402

WORKLOADS = ("an4_fp32_graphed", "an4_bf16_graphed", "ptb_bf16_eager")


def _trainer(workload, fused_clip):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    if workload.startswith("an4"):
        dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
        bf16 = "bf16" in workload
        tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001,
                     cfg=okt.preset(preset, density=0.001, warmup_iters=2), t_total=100000, warmup=0.1, seed=0,
                     autocast="bf16" if bf16 else None, cuda_graph=True, an4_pad_multiple=32, fused_clip=fused_clip,
                     model_kwargs={"fuse_lstm": True, "fuse_lstm_autocast": bf16, "fuse_ctc": True})
        assert tr.graphed is not None and tr.graphed.enabled, tr.graphed.why_disabled
        return tr
    return Trainer(dnn="lstm", dataset="ptb", batch_size=20, lr=22, compressor="oktopk", density=0.02,
                   cfg=okt.preset("lstm_an4", density=0.02, warmup_iters=2), seed=0, autocast="bf16",
                   fused_clip=fused_clip, model_kwargs={"fuse_lstm": True, "fuse_xent": True})


class _Arm:
    def __init__(self, workload, fused_clip):
        self.tr, self.it = _trainer(workload, fused_clip), 0
        self.pool = None
        if workload.startswith("an4"):
            bs = bench.MODELS["lstman4"][2]
            self.pool = [tuple(t.cuda() for t in bench.make_batch("lstman4", i, 0, bs, 128)) for i in range(8)]

    def steps(self, n):
        tr = self.tr
        for _ in range(n):
            if self.pool is None:
                tr.train_step()
                continue
            tr.step(self.pool[self.it % len(self.pool)])
            self.it += 1


def _device_us(fn, n, match=None):
    """Device time per call of the kernels ``fn`` launches (those whose name contains one of ``match``), from a
    torch.profiler run of n calls."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    us = 0.0
    for e in p.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or e.name.startswith(("Memcpy", "Memset")):
            continue
        if match is None or any(m in e.name for m in match):
            us += getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)
    return us / n


def _clip_path_us(arm, fused, n):
    """Device µs per step of the clip path: the clip kernels on the live reduced gradient, plus the update kernels of
    whole steps (graphed steps replay without the profiler seeing their launches, so whole steps run eagerly here)."""
    import torch
    tr = arm.tr
    opt = tr.optimizer
    if arm.pool is not None:
        tr.graphed.enabled = False               # eager steps from here on: the profiler sees every launch
        arm.steps(2)
    opt.zero_grad()
    batch = tr.stage_batch(arm.pool[0]) if arm.pool is not None else tr.prefetch.next()
    loss, _ = tr._forward_loss(batch)
    tr.backward(loss)
    opt.synchronize()
    if fused:
        clip_us = _device_us(lambda: opt._clip.run(opt), n)
    else:
        clip_us = _device_us(lambda: torch.nn.utils.clip_grad_norm_(tr.net.parameters(), tr.clip_norm), n)
    opt.step()
    upd_us = _device_us(lambda: arm.steps(1), n, match=("fused_sgd",))
    return clip_us, upd_us


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--prof-steps", type=int, default=10)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip.py measures on a CUDA device; none is available")
    card0 = _card()
    print("card:", card0, flush=True)
    res = {}
    for w in a.workloads.split(","):
        arms = {"stock_clip": _Arm(w, False), "fused_clip": _Arm(w, True)}
        for arm in arms.values():
            arm.steps(20)                        # dense warm-up, first sparse steps, every graph captured
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(a.runs):                  # alternating runs
            for k, arm in arms.items():
                arm.steps(3)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                arm.steps(a.steps)
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) / a.steps)
        out = {}
        for k, arm in arms.items():
            assert all(torch.isfinite(p).all() for p in arm.tr.net.parameters()), (w, k)
            t = times[k]
            out[k] = {"ms_per_step": {"median": statistics.median(t), "min": min(t), "max": max(t)}}
        for k, arm in arms.items():
            clip_us, upd_us = _clip_path_us(arm, k == "fused_clip", a.prof_steps)
            out[k].update(clip_kernels_us=clip_us, update_kernels_us=upd_us, clip_path_us=clip_us + upd_us)
            arm.tr.close()
        res[w] = out
        for k, v in out.items():
            m = v["ms_per_step"]
            print("%-18s %-10s %7.3f ms/step (%.3f - %.3f)   clip path %7.1f us (clip %6.1f + update %6.1f)" % (
                w, k, m["median"], m["min"], m["max"], v["clip_path_us"], v["clip_kernels_us"],
                v["update_kernels_us"]), flush=True)
        del arms
        torch.cuda.empty_cache()
    card1 = _card()
    print("card after:", card1)
    print(json.dumps({"bench": "clip", "card_before": card0, "card_after": card1, "steps": a.steps, "runs": a.runs,
                      "results": res}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
