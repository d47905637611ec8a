#!/usr/bin/env python
"""Step time of the VGG-16 Ok-Topk workload in fp32, under fp16 autocast with dynamic loss scaling on the stock and on
the fused batch-norm path, and under bf16 autocast fused; and the fused batch-norm kernels alone in fp32, bf16 and fp16.

    python scripts/bench_fp16.py [--steps 200] [--warmup 20] [--runs 5] [--kernel-iters 500]

The workload is bench.py's (``bench.MODELS["vgg16"]``, ``bench.make_batch``, 16 images, the VGG-16 preset, Ok-Topk at
density 0.001, SGD) with whole-step CUDA graphs driven through ``GraphedTrainStep``.  The dense warm-up is shortened to
``--dense-warmup`` steps: only the sparse phase is timed.  Arms, alternated within every run:

  fp32               no autocast, the fused fp32 batch-norm kernels: bench.py's path;
  fp16_scaled_stock  torch.autocast(fp16) + ``LossScale()`` with ``fuse_fp16=False``: stock BatchNorm2d, ReLU and
                     MaxPool2d in fp16 (``--fp16 --loss-scale dynamic``);
  fp16_scaled_fused  the same through the fp16 instantiation of the fused kernels (``... --fused-bn-fp16``);
  bf16_fused         torch.autocast(bf16) through the bf16 fused kernels, no loss scaling (``--bf16``).

Then ``bn_forward`` + ``bn_backward`` alone at the 13 VGG-16 layer shapes (16 images, the pool folded in where a block
ends) in fp32, bf16 and fp16, timed with CUDA events over ``--kernel-iters`` launches of each pair.  Prints the card,
its power limit and SM clock, before and after.
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
from scripts.bench_bf16 import VGG16_LAYERS, _card, _kernel_pair_us  # noqa: E402

ARMS = ("fp32", "fp16_scaled_stock", "fp16_scaled_fused", "bf16_fused")


class _Shim:
    """The part of Trainer that GraphedTrainStep drives, with Trainer's autocast around the forward pass (the loss
    scale, when the optimizer has one, is applied by GraphedTrainStep)."""

    def __init__(self, net, opt, dtype):
        self.net, self.optimizer, self.dtype = net, opt, dtype

    def _forward_loss(self, batch):
        import torch
        x, y = batch
        with torch.autocast("cuda", self.dtype or torch.float16, enabled=self.dtype is not None):
            return torch.nn.functional.cross_entropy(self.net(x), y), None

    def update_model(self):
        self.optimizer.step()


def _arm(kind, dnn, lr, cfg):
    import torch
    import oktopk_b200 as okt
    from oktopk_b200.models import create_net
    from oktopk_b200.train.graph_step import GraphedTrainStep
    torch.manual_seed(0)
    net, _ = create_net(10, dnn, fuse_fp16=kind == "fp16_scaled_fused")
    net = net.cuda().to(memory_format=torch.channels_last)
    scaled = kind.startswith("fp16_scaled")
    opt = okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=lr, momentum=0.9, weight_decay=1e-4),
                                   named_parameters=net.named_parameters(), compression=okt.compressors["oktopk"],
                                   is_sparse=True, cfg=cfg, loss_scale=okt.LossScale() if scaled else None)
    dtype = {"fp32": None, "bf16_fused": torch.bfloat16}.get(kind, torch.float16)
    return opt, GraphedTrainStep(_Shim(net, opt, dtype))


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=8)
    p.add_argument("--kernel-iters", type=int, default=500)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_fp16.py needs a GPU", file=sys.stderr)
        return 2
    import oktopk_b200 as okt
    from oktopk_b200.ops import ext
    C = ext.require()
    torch.cuda.set_device(0)
    card = _card()
    dnn, _, bs, lr, preset = bench.MODELS["vgg16"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=a.dense_warmup)
    pool = []
    for i in range(4):
        x, y = bench.make_batch("vgg16", i, 0, bs, 128)
        pool.append((x.cuda().contiguous(memory_format=torch.channels_last), y.cuda()))
    arms = {k: _arm(k, dnn, lr, cfg) for k in ARMS}
    it = {k: 0 for k in arms}

    def run(k, n):
        gs = arms[k][1]
        for _ in range(n):
            gs.step(pool[it[k] % len(pool)])
            it[k] += 1

    bn0 = ext.LAUNCH_COUNT.get("bn_forward", 0)
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
        assert gs.enabled, (k, gs.why_disabled)
    assert ext.LAUNCH_COUNT.get("bn_forward", 0) > bn0

    kern = []
    dts = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
    for shape, pooled in VGG16_LAYERS:
        r = {"shape": list(shape), "pool": pooled}
        for name, dt in dts.items():
            r[name + "_us"] = _kernel_pair_us(C, shape, pooled, dt, a.kernel_iters)
        kern.append(r)

    out = {"card": card, "card_after": _card(), "steps": a.steps, "runs": a.runs,
           "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                           for k, v in times.items()},
           "graphs": {k: {"enabled": gs.enabled, "captured": len(gs.graphs), "why_disabled": gs.why_disabled}
                      for k, (_, gs) in arms.items()},
           "loss_scale_state": {k: arms[k][0].loss_scale_state() for k in ARMS if k.startswith("fp16_scaled")},
           "bn_fwd_bwd_pair_us": kern,
           "bn_fwd_bwd_total_us": {n: sum(r[n + "_us"] for r in kern) for n in dts}}
    print("card", card)
    for k, v in out["ms_per_step"].items():
        print("%-18s ms/step median %.4f  range %.4f-%.4f  graph %s" % (k, v["median"], v["min"], v["max"],
                                                                         out["graphs"][k]["enabled"]))
    for r in kern:
        print("bn_forward+bn_backward %-18s pool=%d  fp32 %6.1f us  bf16 %6.1f us  fp16 %6.1f us" % (
            tuple(r["shape"]), r["pool"], r["fp32_us"], r["bf16_us"], r["fp16_us"]))
    t = out["bn_fwd_bwd_total_us"]
    print("13 layers: fp32 %.1f us, bf16 %.1f us, fp16 %.1f us" % (t["fp32"], t["bf16"], t["fp16"]))
    print("card after", out["card_after"])
    print(json.dumps(out))
    for opt, _ in arms.values():
        opt.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
