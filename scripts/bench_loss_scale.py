#!/usr/bin/env python
"""Step time of the VGG-16 Ok-Topk workload in fp32, under fp16 autocast without loss scaling, and under fp16 autocast
with dynamic loss scaling; and the ``unscale_check`` kernel alone on the VGG-16 bucket.

    python scripts/bench_loss_scale.py [--steps 200] [--warmup 20] [--runs 5] [--kernel-iters 200]

The workload is bench.py's (``bench.MODELS["vgg16"]``, ``bench.make_batch``, 16 images, the VGG-16 preset, Ok-Topk at
density 0.001, SGD) with whole-step CUDA graphs driven through ``GraphedTrainStep``; the dense warm-up is shortened to
``--dense-warmup`` steps so that only the sparse phase is timed.  Arms, alternated within every run:

  fp32         no autocast: bench.py's path;
  fp16         torch.autocast(fp16), no loss scaling (``--fp16`` alone);
  fp16_scaled  torch.autocast(fp16) with ``LossScale()`` (``--fp16 --loss-scale dynamic``).

Then ``unscale_check`` alone on one bucket of the VGG-16 size (14.73 M elements: reads and writes 8 B per element), timed
with CUDA events over ``--kernel-iters`` launches, against the 3.35 TB/s HBM3 figure of the H100 SXM data sheet.  Prints
the card, its power limit and SM clock.
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

HBM_BYTES_PER_S = 3.35e12


class _Shim:
    """The part of Trainer that GraphedTrainStep drives, with Trainer's autocast around the forward pass."""

    def __init__(self, net, opt, fp16):
        self.net, self.optimizer, self.fp16 = net, opt, fp16

    def _forward_loss(self, batch):
        import torch
        x, y = batch
        if self.fp16:
            with torch.autocast("cuda", torch.float16):
                return torch.nn.functional.cross_entropy(self.net(x), y), None
        return torch.nn.functional.cross_entropy(self.net(x), y), None

    def update_model(self):
        self.optimizer.step()


def _arm(kind, dnn, lr, cfg):
    import torch
    import oktopk_b200 as okt
    from oktopk_b200.models import create_net
    from oktopk_b200.train.graph_step import GraphedTrainStep
    torch.manual_seed(0)
    net, _ = create_net(10, dnn)
    net = net.cuda().to(memory_format=torch.channels_last)
    opt = okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=lr, momentum=0.9, weight_decay=1e-4),
                                   named_parameters=net.named_parameters(), compression=okt.compressors["oktopk"],
                                   is_sparse=True, cfg=cfg,
                                   loss_scale=okt.LossScale() if kind == "fp16_scaled" else None)
    return opt, GraphedTrainStep(_Shim(net, opt, kind != "fp32"))


def _unscale_check_us(n, iters):
    import torch
    import oktopk_b200 as okt
    from oktopk_b200.optimizer import _ScaleState
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.world import World
    eng = CudaBucketEngine(n, okt.OkTopkConfig(density=0.001), World(), name="bench")
    ls = _ScaleState(okt.LossScale(init_scale=1.0), torch.device("cuda"))       # inv_scale 1: values stay put
    eng.grad.normal_()
    for _ in range(20):
        eng.unscale_check(ls.ptr)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        eng.unscale_check(ls.ptr)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    eng.close()
    return us


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=8)
    p.add_argument("--kernel-iters", type=int, default=200)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_loss_scale.py needs a GPU", file=sys.stderr)
        return 2
    import oktopk_b200 as okt
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    dnn, _, bs, lr, preset = bench.MODELS["vgg16"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=a.dense_warmup)
    pool = []
    for i in range(4):
        x, y = bench.make_batch("vgg16", i, 0, bs, 128)
        pool.append((x.cuda().contiguous(memory_format=torch.channels_last), y.cuda()))
    arms = {k: _arm(k, dnn, lr, cfg) for k in ("fp32", "fp16", "fp16_scaled")}
    it = {k: 0 for k in arms}

    def run(k, n):
        gs = arms[k][1]
        for _ in range(n):
            gs.step(pool[it[k] % len(pool)])
            it[k] += 1

    for k in arms:
        run(k, a.dense_warmup + a.warmup)
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.runs):
        for k in arms:
            run(k, a.warmup)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(k, a.steps)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / a.steps)
    for k, (opt, gs) in arms.items():
        assert all(torch.isfinite(q).all() for b in opt._buckets for q in b.params), k
    numel = sum(b.numel for b in arms["fp32"][0]._buckets)
    scale_state = arms["fp16_scaled"][0].loss_scale_state()

    us = _unscale_check_us(numel, a.kernel_iters)
    nbytes = 8 * numel
    out = {"card": card, "card_after": _card(), "steps": a.steps, "runs": a.runs,
           "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                           for k, v in times.items()},
           "graphs": {k: {"enabled": gs.enabled, "captured": len(gs.graphs), "why_disabled": gs.why_disabled}
                      for k, (_, gs) in arms.items()},
           "loss_scale_state": scale_state,
           "unscale_check": {"numel": numel, "bytes": nbytes, "us": us, "bytes_per_s": nbytes / (us * 1e-6),
                             "floor_us_at_3.35TBps": nbytes / HBM_BYTES_PER_S * 1e6,
                             "share_of_hbm_peak": nbytes / HBM_BYTES_PER_S / (us * 1e-6)}}
    print("card", card)
    for k, v in out["ms_per_step"].items():
        print("%-12s ms/step median %.4f  range %.4f-%.4f  graph %s" % (k, v["median"], v["min"], v["max"],
                                                                       out["graphs"][k]["enabled"]))
    u = out["unscale_check"]
    print("unscale_check %d elements: %.1f us, %.2f TB/s, %.0f%% of 3.35 TB/s (floor %.1f us)" % (
        numel, u["us"], u["bytes_per_s"] / 1e12, 100 * u["share_of_hbm_peak"], u["floor_us_at_3.35TBps"]))
    print(json.dumps(out))
    for opt, _ in arms.values():
        opt.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
