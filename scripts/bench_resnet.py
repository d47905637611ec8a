#!/usr/bin/env python
"""Step time of ResNet-20 on CIFAR shapes with the Ok-Topk workload of its launch config
(``scripts/exp_configs/resnet20.conf``: 32 images, the vgg16 preset, density 0.02, SGD lr 0.1, momentum 0.9, weight
decay 1e-4), on the stock batch-norm modules and through the fused batch-norm kernels with the residual add and ReLU
folded in (``create_net(..., fuse_bn=True)``, ``--fused-bn``); and the residual kernel pair alone.

    python scripts/bench_resnet.py [--steps 200] [--runs 5] [--kernel-iters 500]

Whole-step CUDA graphs through ``GraphedTrainStep``, the dense warm-up shortened to ``--dense-warmup`` steps (only the
sparse phase is timed), seeded synthetic batches.  Arms, alternated within every run:

  stock_fp32, fused_fp32   no autocast;
  stock_bf16, fused_bf16   torch.autocast(bf16).

Then, at the ResNet-20 layer shapes, ``bn_forward`` + ``bn_backward`` with a residual against the stock sequence they
replace (batch-norm, add, ReLU; threshold backward, batch-norm backward), each captured in a CUDA graph of
``--kernel-iters`` pairs and timed with CUDA events.  Prints the card, its power limit and SM clock, before and after,
and one JSON line.
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

from scripts.bench_bf16 import _card  # noqa: E402

ARMS = ("stock_fp32", "fused_fp32", "stock_bf16", "fused_bf16")
RESNET20_SHAPES = [(32, 16, 32, 32), (32, 32, 16, 16), (32, 64, 8, 8)]


class _Shim:
    """The part of Trainer that GraphedTrainStep drives, with Trainer's autocast around the forward pass."""

    def __init__(self, net, opt, dtype):
        self.net, self.optimizer, self.dtype = net, opt, dtype

    def _forward_loss(self, batch):
        import torch
        x, y = batch
        with torch.autocast("cuda", self.dtype or torch.bfloat16, enabled=self.dtype is not None):
            return torch.nn.functional.cross_entropy(self.net(x), y), None

    def update_model(self):
        self.optimizer.step()


def _arm(kind, dnn, classes, cfg):
    import torch
    import oktopk_b200 as okt
    from oktopk_b200.models import create_net
    from oktopk_b200.train.graph_step import GraphedTrainStep
    torch.manual_seed(0)
    net, _ = create_net(classes, dnn, fuse_bn=kind.startswith("fused"))
    net = net.cuda().to(memory_format=torch.channels_last)
    opt = okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4),
                                   named_parameters=net.named_parameters(), compression=okt.compressors["oktopk"],
                                   is_sparse=True, cfg=cfg)
    return opt, GraphedTrainStep(_Shim(net, opt, torch.bfloat16 if kind.endswith("bf16") else None))


def _batches(classes, side, n=4, bs=32):
    import torch
    out = []
    for i in range(n):
        g = torch.Generator().manual_seed(1234 + 977 * i)
        x = torch.randn(bs, 3, side, side, generator=g)
        y = torch.randint(0, classes, (bs,), generator=g)
        out.append((x.cuda().contiguous(memory_format=torch.channels_last), y.cuda()))
    return out


def _workload(dnn, classes, side, a):
    import torch
    import oktopk_b200 as okt
    from oktopk_b200.ops import ext
    steps = a.steps
    cfg = okt.preset("vgg16", density=0.02, warmup_iters=a.dense_warmup)
    pool = _batches(classes, side)
    arms = {k: _arm(k, dnn, classes, cfg) for k in ARMS}
    it = {k: 0 for k in arms}

    def run(k, n):
        gs = arms[k][1]
        for _ in range(n):
            gs.step(pool[it[k] % len(pool)])
            it[k] += 1

    warm = a.warmup
    bn0 = ext.LAUNCH_COUNT.get("bn_forward", 0)
    for k in arms:
        run(k, a.dense_warmup + warm)
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.runs):
        for k in arms:
            run(k, warm)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(k, steps)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / steps)
    for k, (opt, gs) in arms.items():
        assert all(torch.isfinite(q).all() for b in opt._buckets for q in b.params), k
        assert gs.enabled, (k, gs.why_disabled)
    assert ext.LAUNCH_COUNT.get("bn_forward", 0) > bn0
    out = {"steps": steps, "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                                           for k, v in times.items()},
           "graphs": {k: {"enabled": gs.enabled, "captured": len(gs.graphs)} for k, (_, gs) in arms.items()}}
    for opt, _ in arms.values():
        opt.close()
    del arms
    torch.cuda.empty_cache()
    return out


def _graph_us(fn, iters):
    """µs per call of ``fn``, captured ``iters`` times in one CUDA graph and replayed."""
    import torch
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (3 * iters)


def _kernel_pairs(C, shape, dtype, iters):
    """The residual bn_forward + bn_backward pair and the stock sequence it replaces, µs per pair."""
    import torch
    from oktopk_b200.ops.ext import DTYPE_CODE
    N, Ch, H, W = shape
    M = N * H * W
    cl = torch.channels_last
    x = torch.randn(shape, device="cuda").to(dtype).contiguous(memory_format=cl)
    r = torch.randn(shape, device="cuda").to(dtype).contiguous(memory_format=cl)
    dy = torch.randn(shape, device="cuda").to(dtype).contiguous(memory_format=cl)
    y, dx, dr = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    rows = C.bn_tile_rows(M, Ch)
    partial = torch.empty((M + rows - 1) // rows * 2 * Ch, device="cuda")
    gamma, beta = torch.ones(Ch, device="cuda"), torch.zeros(Ch, device="cuda")
    rm, rv = torch.zeros(Ch, device="cuda"), torch.ones(Ch, device="cuda")
    nbt = torch.zeros((), dtype=torch.long, device="cuda")
    stats, dgb = torch.empty(2 * Ch, device="cuda"), torch.empty(2 * Ch, device="cuda")
    flag = DTYPE_CODE[dtype]

    def fused():
        s = torch.cuda.current_stream().cuda_stream
        C.bn_forward(x.data_ptr(), y.data_ptr(), 0, partial.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 0,
                     stats.data_ptr(), stats.data_ptr() + 4 * Ch, rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(), 0.1, 1e-5,
                     1, M, Ch, 0, 1022, 0, s, flag, r.data_ptr())
        C.bn_backward(x.data_ptr(), dy.data_ptr(), 0, dx.data_ptr(), partial.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                      stats.data_ptr(), stats.data_ptr() + 4 * Ch, dgb.data_ptr(), dgb.data_ptr() + 4 * Ch, 1, M, Ch, 0,
                      1022, 0, s, flag, r.data_ptr(), dr.data_ptr())

    # the stock modules' forward and backward, as the block's  F.relu(bn(x) + r, inplace=True)  dispatches them
    xg, rg = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
    gg, bg = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)

    def stock():
        out = torch.nn.functional.relu(torch.nn.functional.batch_norm(xg, rm, rv, gg, bg, True, 0.1, 1e-5) + rg,
                                       inplace=True)
        torch.autograd.grad(out, (xg, rg, gg, bg), dy)

    return _graph_us(fused, iters), _graph_us(stock, iters)


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
        print("bench_resnet.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    C = ext.require()
    torch.cuda.set_device(0)
    card = _card()
    res = {"resnet20": _workload("resnet20", 10, 32, a)}
    kern = []
    for shape in RESNET20_SHAPES:
        row = {"shape": list(shape)}
        for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
            row[name + "_fused_us"], row[name + "_stock_us"] = _kernel_pairs(C, shape, dt, a.kernel_iters)
        kern.append(row)
    out = {"card": card, "card_after": _card(), "runs": a.runs, "workloads": res, "bn_residual_pair_us": kern}
    print("card", card)
    for dnn, w in res.items():
        for k, v in w["ms_per_step"].items():
            print("%-9s %-11s ms/step median %.4f  range %.4f-%.4f  graph %s" % (
                dnn, k, v["median"], v["min"], v["max"], w["graphs"][k]["enabled"]))
    for row in kern:
        print("residual bn pair %-16s fp32 fused %6.1f us stock %6.1f us | bf16 fused %6.1f us stock %6.1f us" % (
            tuple(row["shape"]), row["fp32_fused_us"], row["fp32_stock_us"], row["bf16_fused_us"], row["bf16_stock_us"]))
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
