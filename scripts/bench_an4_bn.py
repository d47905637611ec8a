#!/usr/bin/env python
"""The fused batch-norm of the AN4 DeepSpeech model (``fuse_bn``, ``ops/fused_frame_bn``) against the stock modules.

    python scripts/bench_an4_bn.py [--steps 30] [--runs 5] [--op-iters 200] [--conv-steps 300]

1. The op alone: the model's seven batch-norm sites (two conv blocks at F = 81 / 41, four ``_SeqBN`` sites and ``fc``'s
   BatchNorm1d, H = 800), forward + backward, N = 2 at T' = 48 / 123 / 198 output frames, fp32 and bf16: the stock glue
   (mask -> BatchNorm2d -> mask -> Hardtanh -> mask, reshape -> BatchNorm1d, device lengths) against the fused kernels.
   Per pass over all seven sites: the time from CUDA events around ``--op-iters`` passes (host launch cost included),
   median (range) of ``--runs`` alternating runs; and, in a ``torch.profiler`` run of its own, the kernels' device time
   and count.
2. The step: ``bench.MODELS["lstman4"]`` with ``fuse_lstm`` and ``fuse_ctc`` in every arm (and ``fuse_lstm_autocast``
   under bf16) on ``bench.make_batch`` i = 0..7 (108 to 396 frames), three arms: eager unpadded with the stock
   batch-norm, graphed at m = 32 with the stock batch-norm, graphed at m = 32 with ``fuse_bn``.  ``--runs`` alternating
   runs of ``--steps`` steps, median (range) ms/step.
3. Convergence: the same three arms (fp32) on one stream of mixed-length batches from ``SyntheticAN4`` (100 to 400
   frames, two utterances of different lengths per batch) under Ok-Topk for ``--conv-steps`` steps: the mean loss over
   each 50-step window.  Two controls: eager unpadded with ``fuse_bn``, and eager unpadded with the stock batch-norm
   started from parameters one ulp away (how far rounding alone moves this training).

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

ARMS = {"eager_stock_bn": (0, False, False), "graphed_m32_stock_bn": (32, True, False),
        "graphed_m32_fuse_bn": (32, True, True)}
CONTROLS = {"eager_fuse_bn": (0, False, True), "eager_stock_bn_one_ulp": (0, False, False, True)}


def _op_us(precision, T, iters, runs):
    import torch
    import torch.nn as nn
    from oktopk_b200.ops import fused_frame_bn as fb
    dt = torch.float32 if precision == "fp32" else torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(T)
    N = 2
    lens = torch.tensor([T, (7 * T) // 10], dtype=torch.int32, device="cuda")
    sites = [(1, (N, 32, 81, T), nn.BatchNorm2d(32)), (1, (N, 32, 41, T), nn.BatchNorm2d(32))]
    sites += [(0, (T, N, 800), nn.BatchNorm1d(800)) for _ in range(5)]
    data = []
    for conv, shape, bn in sites:
        x = torch.randn(shape, device="cuda", generator=g).to(dt).requires_grad_(True)
        data.append((conv, x, torch.randn(shape, device="cuda", generator=g).to(dt), bn.cuda()))

    def run(fused):
        for conv, x, dy, bn in data:
            if fused:
                y = (fb.conv_block_bn if conv else fb.seq_bn)(x, bn, lens)
            else:
                y = fb._stock_conv_block(x, bn, lens) if conv else fb._stock_seq(x, bn)
            torch.autograd.grad(y, [x, bn.weight, bn.bias], dy)

    arms = (("stock", False), ("fused", True))
    times = {name: [] for name, _ in arms}
    for _ in range(runs):                        # alternating runs
        for name, fused in arms:
            for _ in range(10):
                run(fused)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                run(fused)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1e3 / iters)
    out = {}
    for name, fused in arms:
        kern_us, kern_n = _kernel_time(lambda: run(fused), 20)
        out[name] = {"median": statistics.median(times[name]), "min": min(times[name]), "max": max(times[name]),
                     "kernel_us": kern_us, "kernels": kern_n}
    return out


def _kernel_time(fn, n):
    """Device time of the kernels ``fn`` launches, and their number, per call (a torch.profiler run of n calls)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    us = count = 0
    for e in p.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset")):
            us += getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)
            count += 1
    return us / n, count / n


class _Arm:
    """One trainer and its step counter; ``steps`` runs graphed steps where the trainer has a graph step, else eager."""

    def __init__(self, tr):
        self.tr, self.it = tr, 0

    def steps(self, pool, n):
        tr, loss = self.tr, None
        for _ in range(n):
            loss = tr.step(pool[self.it % len(pool)])
            self.it += 1
        return loss


def _arm(precision, m, graph, fuse_bn, one_ulp=False):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    autocast = None if precision == "fp32" else precision
    cfg = okt.preset(preset, density=0.001, warmup_iters=2)
    arm = _Arm(Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                       t_total=100000, warmup=0.1, seed=0, autocast=autocast, cuda_graph=graph, an4_pad_multiple=m,
                       model_kwargs={"fuse_lstm": True, "fuse_lstm_autocast": autocast is not None, "fuse_ctc": True,
                                     "fuse_bn": fuse_bn}))
    if graph:
        assert arm.tr.graphed is not None and arm.tr.graphed.enabled, arm.tr.graphed.why_disabled
    if one_ulp:                                  # every parameter one ulp up or down
        import torch
        g = torch.Generator(device="cuda").manual_seed(1)
        with torch.no_grad():
            for p in arm.tr.net.parameters():
                p.mul_(1 + 2.0 ** -23 * torch.randn(p.shape, device="cuda", generator=g).sign())
    return arm


def _steps(precision, a):
    import torch
    bs = bench.MODELS["lstman4"][2]
    pool = [tuple(t.cuda() for t in bench.make_batch("lstman4", i, 0, bs, 128)) for i in range(8)]
    arms = {k: _arm(precision, *v) for k, v in ARMS.items()}
    for arm in arms.values():
        arm.steps(pool, 2 + 2 * len(pool))
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.runs):
        for k, arm in arms.items():
            arm.steps(pool, 3)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arm.steps(pool, a.steps)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / a.steps)
    for arm in arms.values():
        assert all(torch.isfinite(p).all() for p in arm.tr.net.parameters())
        arm.tr.close()
    return {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for k, v in times.items()}


def _convergence(n_steps):
    import torch
    from oktopk_b200.train.data import SyntheticAN4, an4_collate
    bs = bench.MODELS["lstman4"][2]
    ds = SyntheticAN4(n=n_steps * bs, seed=11)
    stream = [tuple(t.cuda() for t in an4_collate([ds[i * bs + j] for j in range(bs)])) for i in range(n_steps)]
    out = {}
    for k, v in dict(ARMS, **CONTROLS).items():
        arm = _arm("fp32", *v)
        losses = []
        for b in stream:
            losses.append(arm.steps([b], 1).detach().clone())    # a graph's loss is overwritten by its next replay
        losses = torch.stack(losses).float().cpu()
        w = 50
        out[k] = {"window_mean_loss": [round(float(losses[i:i + w].mean()), 4) for i in range(0, len(losses), w)],
                  "final_loss": float(losses[-w:].mean()),
                  "fallbacks": dict(arm.tr.graphed.fallbacks) if arm.tr.graphed is not None else None}
        arm.tr.close()
    return out


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--op-iters", type=int, default=200)
    p.add_argument("--conv-steps", type=int, default=300)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_an4_bn.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    op = {prec: {"T%d" % T: _op_us(prec, T, a.op_iters, a.runs) for T in (48, 123, 198)} for prec in ("fp32", "bf16")}
    steps = {prec: _steps(prec, a) for prec in ("fp32", "bf16")}
    conv = _convergence(a.conv_steps)
    out = {"card": card, "card_after": _card(), "op_us": op, "ms_per_step": steps, "convergence": conv}
    print("card", card)
    for prec, r in op.items():
        for T, v in r.items():
            print("7 sites fwd+bwd %s %-4s " % (prec, T) + "  ".join(
                "%s %.1f us (%.1f-%.1f), kernels %.1f us in %.0f" % (k, r["median"], r["min"], r["max"], r["kernel_us"],
                                                                    r["kernels"]) for k, r in v.items()))
    for prec, r in steps.items():
        for k, v in r.items():
            print("lstman4 %s %-22s ms/step median %.3f  range %.3f-%.3f" % (prec, k, v["median"], v["min"], v["max"]))
    for k, v in conv.items():
        print("convergence %-22s %s  fallbacks %s" % (k, v["window_mean_loss"], v["fallbacks"]))
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
