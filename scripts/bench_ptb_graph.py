#!/usr/bin/env python
"""Whole-step CUDA graphs for the PTB language model (``Trainer(dnn="lstm", cuda_graph=True)``, ``--cuda-graph``) against
eager steps.

    python scripts/bench_ptb_graph.py [--steps 30] [--runs 5] [--prof-steps 10] [--dense-warmup 2]

The workload is ``scripts/bench_ptb.py``'s: ``Trainer`` on ``SyntheticPTB`` (N = 20, T = 35, the hidden state carried
across batches), SGD lr 22, gradient clip 0.25 on the device (``fused_clip``), Ok-Topk at density 0.02, the dense
warm-up shortened to ``--dense-warmup`` steps.  Arms, each eager and graphed:

  bf16_fused   bf16 autocast, ``fuse_lstm`` + ``fuse_xent``;
  fp16_fused   fp16 autocast with dynamic loss scaling, ``fuse_lstm`` + ``fuse_xent``;
  fp32_fused   ``fuse_lstm_fp32`` + ``fuse_xent``;
  fp32_stock   the stock cuDNN layer and loss in fp32 (cuDNN's RNN in TF32, torch's default).

1. ``--runs`` alternating runs of ``--steps`` steps per arm, timed with CUDA events: median (range) ms/step.  Before
   them each arm's peak allocated memory over construction and warm-up (every graph captured), above what was
   allocated before it, its graph count and the host time its captures took.
2. A ``torch.profiler`` run of its own per arm (``--prof-steps`` steps): device time per step (kernels, copies and
   memsets), host synchronisations per step (``cuda*Synchronize`` and synchronous ``cudaMemcpy`` calls), and
   host-to-device / device-to-host copies per step.
Prints the card, its power limit and SM clock before and after, and one JSON line.  Needs a GPU: there is no fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("OMP_NUM_THREADS", "1")

from scripts.bench_bf16 import _card  # noqa: E402

N, T = 20, 35
# arm -> (autocast, model_kwargs)
ARMS = {"bf16_fused": ("bf16", {"fuse_lstm": True, "fuse_xent": True}),
        "fp16_fused": ("fp16", {"fuse_lstm": True, "fuse_xent": True}),
        "fp32_fused": (None, {"fuse_lstm": True, "fuse_lstm_fp32": True, "fuse_xent": True}),
        "fp32_stock": (None, {})}
SYNCS = ("cudaDeviceSynchronize", "cudaStreamSynchronize", "cudaEventSynchronize", "cudaMemcpy")


def _trainer(autocast, model_kwargs, graph: bool, dense_warmup: int):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    cfg = okt.preset("lstm_an4", density=0.02, warmup_iters=dense_warmup)
    tr = Trainer(dnn="lstm", dataset="ptb", batch_size=N, lr=22.0, compressor="oktopk", density=0.02, cfg=cfg, seed=0,
                 autocast=autocast, loss_scale="dynamic" if autocast == "fp16" else None, fused_clip=True,
                 cuda_graph=graph, model_kwargs=model_kwargs)
    if graph:
        assert tr.graphed is not None and tr.graphed.enabled, tr.graphed.why_disabled
    return tr


class _Arm:
    def __init__(self, name, graph, pool, dense_warmup):
        autocast, kw = ARMS[name]
        self.tr, self.graph, self.pool, self.it = _trainer(autocast, kw, graph, dense_warmup), graph, pool, 0
        self.capture_s = 0.0
        if graph:                                # host time of every capture, the synchronisations around it included
            gs = self.tr.graphed
            capture = gs._capture

            def timed(key):
                import torch
                t0 = time.perf_counter()
                g = capture(key)
                torch.cuda.synchronize()
                self.capture_s += time.perf_counter() - t0
                return g
            gs._capture = timed

    def steps(self, n):
        for _ in range(n):
            self.tr.step(self.pool[self.it % len(self.pool)])
            self.it += 1


def _profile(arm, n) -> dict:
    """Per step: device time of kernels, copies and memsets; host synchronisations; H2D and D2H copies."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
        arm.steps(n)
        torch.cuda.synchronize()
    dev_us, syncs, h2d, d2h = 0.0, 0, 0, 0
    for e in p.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            dev_us += getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)
            h2d += "HtoD" in e.name
            d2h += "DtoH" in e.name
        elif e.name in SYNCS:
            syncs += 1
    syncs -= 1                                   # the synchronize that closes the profiled window
    return {"device_us": dev_us / n, "host_syncs": syncs / n, "h2d_copies": h2d / n, "d2h_copies": d2h / n}


def _pool():
    import torch
    from oktopk_b200.train.data import SyntheticPTB
    ds = SyntheticPTB(batch_size=N, num_steps=T)
    pool = []
    for b in range(8):                           # consecutive [N, T] batches, as the loader hands them over
        rows = [ds[b * N + i] for i in range(N)]
        pool.append((torch.stack([r[0] for r in rows]).cuda(), torch.stack([r[1] for r in rows]).cuda()))
    return pool


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--prof-steps", type=int, default=10)
    ap.add_argument("--dense-warmup", type=int, default=2)
    ap.add_argument("--arms", default=",".join(ARMS))
    a = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ptb_graph.py measures on a CUDA device; none is available")
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = False
    card0 = _card()
    print("card:", card0, flush=True)
    pool = _pool()
    arms, out = {}, {}
    for name in a.arms.split(","):
        for graph in (False, True):
            k = "%s_%s" % (name, "graphed" if graph else "eager")
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            arm = arms[k] = _Arm(name, graph, pool, a.dense_warmup)
            arm.steps(a.dense_warmup + 10)       # the dense warm-up, the first sparse steps, every graph captured
            torch.cuda.synchronize()
            out[k] = {"peak_allocated_mib": (torch.cuda.max_memory_allocated() - base) / 2 ** 20}
            if graph:
                gs = arm.tr.graphed
                assert gs.enabled, gs.why_disabled
                out[k].update(graphs=len(gs.graphs), capture_s=arm.capture_s, fallbacks=dict(gs.fallbacks))
    times = {k: [] for k in arms}
    for _ in range(a.runs):                      # alternating runs
        for k, arm in arms.items():
            arm.steps(a.warmup)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arm.steps(a.steps)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / a.steps)
    for k, arm in arms.items():
        assert all(torch.isfinite(p).all() for p in arm.tr.net.parameters()), k
        t = times[k]
        out[k]["ms_per_step"] = {"median": statistics.median(t), "min": min(t), "max": max(t), "runs": t}
        out[k]["last_loss"] = float(arm.tr._last_loss)
    for k, arm in arms.items():
        out[k]["profile"] = _profile(arm, a.prof_steps)
        if arm.graph:
            out[k]["graphs_after"] = len(arm.tr.graphed.graphs)
        arm.tr.close()
    card1 = _card()
    print("%-20s %26s %10s %8s %6s %6s %9s %7s %9s" % ("arm", "ms/step median (range)", "device us", "syncs",
                                                          "H2D", "D2H", "peak MiB", "graphs", "capture s"))
    for k, v in out.items():
        m, pr = v["ms_per_step"], v["profile"]
        print("%-20s %8.3f (%6.3f - %6.3f) %10.1f %8.1f %6.1f %6.1f %9.0f %7s %9s" % (
            k, m["median"], m["min"], m["max"], pr["device_us"], pr["host_syncs"], pr["h2d_copies"], pr["d2h_copies"],
            v["peak_allocated_mib"], v.get("graphs", "-"),
            "%.2f" % v["capture_s"] if "capture_s" in v else "-"), flush=True)
    print("card after:", card1)
    print(json.dumps({"bench": "ptb_graph", "card_before": card0, "card_after": card1, "steps": a.steps,
                      "runs": a.runs, "prof_steps": a.prof_steps, "dense_warmup": a.dense_warmup, "results": out}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
