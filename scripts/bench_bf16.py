#!/usr/bin/env python
"""Step time of the VGG-16 Ok-Topk workload in fp32 and under bf16 autocast, and the fused batch-norm kernels alone.

    python scripts/bench_bf16.py [--steps 200] [--warmup 20] [--runs 5] [--kernel-iters 500]

The workload is bench.py's (``bench.MODELS["vgg16"]``, ``bench.make_batch``, 16 images, the VGG-16 preset, Ok-Topk at
density 0.001, SGD) with whole-step CUDA graphs driven through ``GraphedTrainStep``.  The dense warm-up is shortened to
``--dense-warmup`` steps: only the sparse phase is timed.  Arms, alternated within every run:

  fp32        no autocast, the fused fp32 batch-norm kernels: bench.py's path;
  bf16_stock  torch.autocast(bf16) with ``net.fuse = False``: stock BatchNorm2d, ReLU and MaxPool2d in bf16;
  bf16_fused  torch.autocast(bf16) through the bf16 instantiation of the fused batch-norm kernels.

Then ``bn_forward`` + ``bn_backward`` alone at the 13 VGG-16 layer shapes (16 images, the pool folded in where a block
ends), fp32 against bf16, timed with CUDA events over ``--kernel-iters`` launches of each pair.  Prints the card, its
power limit and SM clock.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("OMP_NUM_THREADS", "1")

import bench  # noqa: E402  (make_batch, MODELS: the bench workload definition)

# the BN input of the 13 VGG-16 layers at 16 images, and whether a 2x2 max-pool follows (the last layer of a block)
VGG16_LAYERS = [((16, 64, 32, 32), False), ((16, 64, 32, 32), True),
                ((16, 128, 16, 16), False), ((16, 128, 16, 16), True),
                ((16, 256, 8, 8), False), ((16, 256, 8, 8), False), ((16, 256, 8, 8), True),
                ((16, 512, 4, 4), False), ((16, 512, 4, 4), False), ((16, 512, 4, 4), True),
                ((16, 512, 2, 2), False), ((16, 512, 2, 2), False), ((16, 512, 2, 2), True)]


class _Shim:
    """The part of Trainer that GraphedTrainStep drives, with Trainer's autocast around the forward pass."""

    def __init__(self, net, opt, autocast):
        self.net, self.optimizer, self.autocast = net, opt, autocast

    def _forward_loss(self, batch):
        import torch
        x, y = batch
        if self.autocast:
            with torch.autocast("cuda", torch.bfloat16):
                return torch.nn.functional.cross_entropy(self.net(x), y), None
        return torch.nn.functional.cross_entropy(self.net(x), y), None

    def update_model(self):
        self.optimizer.step()


def _card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = "nvidia-smi unavailable: %r" % (e,)
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")])) if "," in out else {"nvidia-smi": out}


def _arm(kind, dnn, lr, cfg):
    import torch
    import oktopk_b200 as okt
    from oktopk_b200.models import create_net
    from oktopk_b200.train.graph_step import GraphedTrainStep
    torch.manual_seed(0)
    net, _ = create_net(10, dnn)
    net = net.cuda().to(memory_format=torch.channels_last)
    net.fuse = kind != "bf16_stock"
    opt = okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=lr, momentum=0.9, weight_decay=1e-4),
                                   named_parameters=net.named_parameters(), compression=okt.compressors["oktopk"],
                                   is_sparse=True, cfg=cfg)
    return opt, GraphedTrainStep(_Shim(net, opt, kind != "fp32"))


def _kernel_pair_us(C, shape, pooled, dtype, iters):
    """bn_forward + bn_backward at one layer shape, µs per pair."""
    import torch
    N, Ch, H, W = shape
    M = N * H * W
    x = torch.randn(shape, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last)
    ys = (N, Ch, H // 2, W // 2) if pooled else shape
    y = torch.empty(ys, device="cuda", dtype=dtype).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(ys, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last)
    dx = torch.empty_like(x)
    arg = torch.empty(y.numel() if pooled else 1, dtype=torch.uint8, device="cuda")
    rows = C.bn_tile_rows(M, Ch)
    partial = torch.empty((M + rows - 1) // rows * 2 * Ch, device="cuda")
    gamma, beta = torch.ones(Ch, device="cuda"), torch.zeros(Ch, device="cuda")
    rm, rv = torch.zeros(Ch, device="cuda"), torch.ones(Ch, device="cuda")
    nbt = torch.zeros((), dtype=torch.long, device="cuda")
    stats, dgb = torch.empty(2 * Ch, device="cuda"), torch.empty(2 * Ch, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    from oktopk_b200.ops.ext import DTYPE_CODE
    flag = DTYPE_CODE[dtype]
    Wp = W if pooled else 0

    def pair():
        C.bn_forward(x.data_ptr(), y.data_ptr(), arg.data_ptr() if pooled else 0, partial.data_ptr(), gamma.data_ptr(),
                     beta.data_ptr(), 0, stats.data_ptr(), stats.data_ptr() + 4 * Ch, rm.data_ptr(), rv.data_ptr(),
                     nbt.data_ptr(), 0.1, 1e-5, 1, M, Ch, Wp, 1023, 0, s, flag)
        C.bn_backward(x.data_ptr(), dy.data_ptr(), arg.data_ptr() if pooled else 0, dx.data_ptr(), partial.data_ptr(),
                      gamma.data_ptr(), beta.data_ptr(), stats.data_ptr(), stats.data_ptr() + 4 * Ch, dgb.data_ptr(),
                      dgb.data_ptr() + 4 * Ch, 1, M, Ch, Wp, 1023, 0, s, flag)

    for _ in range(20):
        pair()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        pair()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


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
        print("bench_bf16.py needs a GPU", file=sys.stderr)
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
    arms = {k: _arm(k, dnn, lr, cfg) for k in ("fp32", "bf16_stock", "bf16_fused")}
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

    kern = []
    for shape, pooled in VGG16_LAYERS:
        f32 = _kernel_pair_us(C, shape, pooled, torch.float32, a.kernel_iters)
        b16 = _kernel_pair_us(C, shape, pooled, torch.bfloat16, a.kernel_iters)
        kern.append({"shape": list(shape), "pool": pooled, "fp32_us": f32, "bf16_us": b16})

    out = {"card": card, "card_after": _card(), "steps": a.steps, "runs": a.runs,
           "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                           for k, v in times.items()},
           "graphs": {k: {"enabled": gs.enabled, "captured": len(gs.graphs), "why_disabled": gs.why_disabled}
                      for k, (_, gs) in arms.items()},
           "bn_fwd_bwd_pair_us": kern,
           "bn_fwd_bwd_total_us": {"fp32": sum(r["fp32_us"] for r in kern), "bf16": sum(r["bf16_us"] for r in kern)}}
    print("card", card)
    for k, v in out["ms_per_step"].items():
        print("%-11s ms/step median %.4f  range %.4f-%.4f  graph %s" % (k, v["median"], v["min"], v["max"],
                                                                      out["graphs"][k]["enabled"]))
    for r in kern:
        print("bn_forward+bn_backward %-18s pool=%d  fp32 %6.1f us  bf16 %6.1f us" % (tuple(r["shape"]), r["pool"],
                                                                                     r["fp32_us"], r["bf16_us"]))
    print("13 layers: fp32 %.1f us, bf16 %.1f us" % (out["bn_fwd_bwd_total_us"]["fp32"], out["bn_fwd_bwd_total_us"]["bf16"]))
    print(json.dumps(out))
    for opt, _ in arms.values():
        opt.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
