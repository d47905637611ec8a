#!/usr/bin/env python
"""The fused look-ahead convolution + Hardtanh of the AN4 DeepSpeech model (``fuse_lookahead``,
``ops/fused_lookahead``) against the stock module.

    python scripts/bench_lookahead.py [--steps 30] [--runs 5] [--op-iters 200]

1. The op alone: H = 800, context 20, N = 2 at T' = 48 / 123 / 198 output frames, fp32 and bf16 (the stock module
   under bf16 autocast, as in the model), forward + backward: stock ``Lookahead`` -> ``Hardtanh`` against
   ``lookahead_hardtanh`` with the lengths on the device.  Per pass: the time from CUDA events around ``--op-iters``
   passes (host launch cost included), median (range) of ``--runs`` alternating runs; and, in a ``torch.profiler`` run
   of its own, the kernels' device time and count.
2. The step: ``bench.MODELS["lstman4"]`` graphed at m = 32 with ``fuse_lstm``, ``fuse_ctc`` and ``fuse_bn`` in every
   arm (and ``fuse_lstm_autocast`` under bf16) on ``bench.make_batch`` i = 0..7 (108 to 396 frames), the stock
   look-ahead against ``fuse_lookahead``.  ``--runs`` alternating runs of ``--steps`` steps, median (range) ms/step.

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
from scripts.bench_an4_bn import _Arm, _kernel_time  # noqa: E402
from scripts.bench_bf16 import _card  # noqa: E402

H, CONTEXT = 800, 20
ARMS = {"graphed_m32_stock_lookahead": False, "graphed_m32_fuse_lookahead": True}


def _op_us(precision, T, iters, runs):
    import torch
    import torch.nn as nn
    from oktopk_b200.models.deepspeech import Lookahead
    from oktopk_b200.ops.fused_lookahead import lookahead_hardtanh
    dt = torch.float32 if precision == "fp32" else torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(T)
    N = 2
    lens = torch.tensor([T, (7 * T) // 10], dtype=torch.int32, device="cuda")
    la = Lookahead(H, CONTEXT).cuda()
    stock = nn.Sequential(la, nn.Hardtanh(0, 20, inplace=True))
    x = (1.0 + torch.randn(T, N, H, device="cuda", generator=g)).to(dt)
    x = x.masked_fill(torch.arange(T, device="cuda").view(-1, 1, 1) >= lens.view(1, -1, 1), 0).requires_grad_(True)
    dy = torch.randn(T, N, H, device="cuda", generator=g).to(dt)

    def run(fused):
        with torch.autocast("cuda", dtype=dt, enabled=dt != torch.float32):
            y = lookahead_hardtanh(x, la.weight, lens) if fused else stock(x)
        torch.autograd.grad(y, [x, la.weight], dy.to(y.dtype))

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


def _arm(precision, fuse_lookahead):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    autocast = None if precision == "fp32" else precision
    cfg = okt.preset(preset, density=0.001, warmup_iters=2)
    arm = _Arm(Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                       t_total=100000, warmup=0.1, seed=0, autocast=autocast, cuda_graph=True, an4_pad_multiple=32,
                       model_kwargs={"fuse_lstm": True, "fuse_lstm_autocast": autocast is not None, "fuse_ctc": True,
                                     "fuse_bn": True, "fuse_lookahead": fuse_lookahead}))
    assert arm.tr.graphed is not None and arm.tr.graphed.enabled, arm.tr.graphed.why_disabled
    return arm


def _steps(precision, a):
    import torch
    bs = bench.MODELS["lstman4"][2]
    pool = [tuple(t.cuda() for t in bench.make_batch("lstman4", i, 0, bs, 128)) for i in range(8)]
    arms = {k: _arm(precision, v) for k, v in ARMS.items()}
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
        assert arm.tr.graphed.fallbacks == {"shapes": 0, "targets": 0}, arm.tr.graphed.fallbacks
        arm.tr.close()
    return {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for k, v in times.items()}


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--op-iters", type=int, default=200)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_lookahead.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    op = {prec: {"T%d" % T: _op_us(prec, T, a.op_iters, a.runs) for T in (48, 123, 198)} for prec in ("fp32", "bf16")}
    steps = {prec: _steps(prec, a) for prec in ("fp32", "bf16")}
    out = {"card": card, "card_after": _card(), "op_us": op, "ms_per_step": steps}
    print("card", card)
    for prec, r in op.items():
        for T, v in r.items():
            print("look-ahead fwd+bwd %s %-4s " % (prec, T) + "  ".join(
                "%s %.1f us (%.1f-%.1f), kernels %.1f us in %.0f" % (k, r["median"], r["min"], r["max"], r["kernel_us"],
                                                                    r["kernels"]) for k, r in v.items()))
    for prec, r in steps.items():
        for k, v in r.items():
            print("lstman4 %s %-28s ms/step median %.3f  range %.3f-%.3f" % (prec, k, v["median"], v["min"], v["max"]))
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
