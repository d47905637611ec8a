#!/usr/bin/env python
"""Whole-step CUDA graphs for the AN4 DeepSpeech model over padded batches (``Trainer(an4_pad_multiple=m)``,
``--an4-pad-multiple``) against today's best eager step.

    python scripts/bench_an4_graph.py [--steps 30] [--runs 5] [--profile-steps 10]

Every arm runs ``bench.MODELS["lstman4"]`` with ``fuse_lstm`` and ``fuse_ctc`` (and ``fuse_lstm_autocast`` under bf16)
on ``bench.make_batch`` for i = 0..7: 108 to 396 frames, six padded lengths at m = 32.  The dense warm-up is cut to 2
steps; the sparse phase is timed.

1. Three arms in fp32 and in bf16: eager unpadded (``an4_pad_multiple=0``), eager padded (m = 32) and graphed padded
   (m = 32, ``cuda_graph=True``).  After every arm has captured its graphs, ``--runs`` alternating runs of ``--steps``
   steps each, median (range) ms/step from CUDA events.
2. The graphed arm over m in {1, 16, 32, 64} (fp32), each m in a process of its own: ms/step (median of 3 runs),
   graphs captured, the time spent in the captures, and peak memory allocated (the process's, and the arm's own: less
   what the batch pool held before the trainer was built).
3. One layer (H = 800, N = 2, fp32), forward + backward on the device-lengths entry, µs per call: T' = 123 frames,
   the same utterances padded to 139 frames (the kernels stop at 123), and 139 frames that all run (what the padding
   would cost without the bound).
4. A ``torch.profiler`` run of its own per arm of (1) over ``--profile-steps`` steps: device time per step and
   device-to-host copies and host synchronisations per step.

Prints the card, its power limit and SM clock, before and after, and one JSON line.
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

import bench  # noqa: E402  (make_batch, MODELS: the bench workload definition)
from scripts.bench_bf16 import _card  # noqa: E402

PRECISIONS = ("fp32", "bf16")
SWEEP = (1, 16, 32, 64)


def _trainer(precision, m, graph):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    autocast = None if precision == "fp32" else precision
    cfg = okt.preset(preset, density=0.001, warmup_iters=2)
    return Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                   t_total=100000, warmup=0.1, seed=0, autocast=autocast, cuda_graph=graph, an4_pad_multiple=m,
                   model_kwargs={"fuse_lstm": True, "fuse_lstm_autocast": autocast is not None, "fuse_ctc": True})


class _Arm:
    def __init__(self, precision, m, graph):
        import torch
        torch.cuda.reset_peak_memory_stats()
        self.tr = _trainer(precision, m, graph)
        self.it = 0
        self.capture_s = 0.0
        gs = self.tr.graphed
        if graph:
            assert gs is not None and gs.enabled, gs and gs.why_disabled
            inner = gs._capture

            def timed(key):                      # the captures' wall time, synchronisations included
                t0 = time.perf_counter()
                g = inner(key)
                torch.cuda.synchronize()
                self.capture_s += time.perf_counter() - t0
                return g
            gs._capture = timed

    def steps(self, pool, n):
        tr = self.tr
        loss = None
        for _ in range(n):
            loss = tr.step(pool[self.it % len(pool)])
            self.it += 1
        return loss


def _pool():
    bs = bench.MODELS["lstman4"][2]
    return [tuple(t.cuda() for t in bench.make_batch("lstman4", i, 0, bs, 128)) for i in range(8)]


def _timed(arm, pool, n):
    import torch
    arm.steps(pool, 3)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    loss = arm.steps(pool, n)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, float(loss.detach())


def _arms(precision, a):
    import torch
    pool = _pool()
    spec = {"eager": (0, False), "eager_padded": (32, False), "graphed_padded": (32, True)}
    arms = {k: _Arm(precision, m, g) for k, (m, g) in spec.items()}
    for arm in arms.values():
        arm.steps(pool, 2 + 2 * len(pool))       # the dense warm-up, then every length of the pool twice (captures)
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    loss = {}
    for _ in range(a.runs):
        for k, arm in arms.items():
            t, loss[k] = _timed(arm, pool, a.steps)
            times[k].append(t)
    prof = {k: _profile(arm, pool, a.profile_steps) for k, arm in arms.items()}
    gs = arms["graphed_padded"].tr.graphed
    out = {"ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                           for k, v in times.items()},
           "last_loss": loss, "profile": prof, "graphs": len(gs.graphs), "fallbacks": dict(gs.fallbacks)}
    for arm in arms.values():
        assert all(torch.isfinite(p).all() for p in arm.tr.net.parameters())
        arm.tr.close()
    return out


def _sweep_one(m, steps):
    """The graphed fp32 arm at one m, in a process of its own: peak memory is this arm's alone.  ``arm_peak_mb`` is the
    peak minus what was allocated before the trainer existed (the batch pool)."""
    import torch
    pool = _pool()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    arm = _Arm("fp32", m, True)
    arm.steps(pool, 2 + 2 * len(pool))
    torch.cuda.synchronize()
    ts = [_timed(arm, pool, steps)[0] for _ in range(3)]
    gs = arm.tr.graphed
    peak = torch.cuda.max_memory_allocated()
    return {"ms_per_step": statistics.median(ts), "runs": ts, "graphs": len(gs.graphs),
            "padded_lengths": sorted({k[0][3] for k in gs.graphs}), "capture_s": arm.capture_s,
            "peak_mem_mb": peak / 2 ** 20, "arm_peak_mb": (peak - base) / 2 ** 20, "fallbacks": dict(gs.fallbacks)}


def _sweep(a):
    """Each m in a fresh process: a trainer's objects are frozen out of the cyclic collector once its graphs exist
    (``GraphedTrainStep.precapture_sparse``), so one that has run in this process is never freed here."""
    import subprocess
    out = {}
    for m in SWEEP:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--sweep-m", str(m), "--steps", str(a.steps)],
                           capture_output=True, text=True, check=True)
        out["m%d" % m] = json.loads(r.stdout.strip().splitlines()[-1])
    return out


def _layer_us(iters):
    """One fused layer forward + backward, µs per call, on the device-lengths entry."""
    import torch
    import torch.nn as nn
    from oktopk_b200.ops.fused_lstm import lstm_layer_device
    torch.manual_seed(0)
    rnn = nn.LSTM(800, 800).cuda()
    out = {}
    for name, T, L in (("T123", 123, 123), ("T139_len123", 139, 123), ("T139_len139", 139, 139)):
        x = torch.randn(T, 2, 800, device="cuda", requires_grad=True)
        dy = torch.randn(T, 2, 800, device="cuda")
        lens = torch.full((2,), L, dtype=torch.int32, device="cuda")

        def fn():
            torch.autograd.grad(lstm_layer_device(x, lens, rnn), [x] + list(rnn.parameters()), dy)
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) * 1e3 / iters
    return out


def _profile(arm, pool, n):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
        arm.steps(pool, n)
        torch.cuda.synchronize()
    total = 0.0
    d2h = syncs = 0
    for e in p.events():
        name = e.name
        dev_us = getattr(e, "device_time", None)
        if dev_us is None:
            dev_us = getattr(e, "cuda_time", 0.0)
        if e.device_type == torch.autograd.DeviceType.CUDA:
            if "Memcpy DtoH" in name:
                d2h += 1
            if not name.startswith("Memcpy") and not name.startswith("Memset"):
                total += dev_us
        elif name in ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaEventSynchronize"):
            syncs += 1
    # the closing synchronize() above is the profiler's, not the step's
    return {"kernel_us_per_step": total / n, "d2h_copies_per_step": d2h / n, "host_syncs_per_step": (syncs - 1) / n}


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--layer-iters", type=int, default=100)
    p.add_argument("--profile-steps", type=int, default=10)
    p.add_argument("--sweep-m", type=int, default=None, help=argparse.SUPPRESS)    # one sweep point (a child process)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_an4_graph.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    if a.sweep_m is not None:
        print(json.dumps(_sweep_one(a.sweep_m, a.steps)))
        return 0
    card = _card()
    steps = {prec: _arms(prec, a) for prec in PRECISIONS}
    sweep = _sweep(a)
    layer = _layer_us(a.layer_iters)
    out = {"card": card, "card_after": _card(), "lstman4": steps, "sweep_fp32": sweep, "layer_us": layer}
    print("card", card)
    for prec, r in steps.items():
        for k, v in r["ms_per_step"].items():
            pr = r["profile"][k]
            print("lstman4 %s %-14s ms/step median %.3f  range %.3f-%.3f  loss %.4f  device %.0f us/step  "
                  "D2H copies %.1f  syncs %.1f per step" % (prec, k, v["median"], v["min"], v["max"], r["last_loss"][k],
                                                           pr["kernel_us_per_step"], pr["d2h_copies_per_step"],
                                                           pr["host_syncs_per_step"]))
        print("lstman4 %s graphs %d fallbacks %s" % (prec, r["graphs"], r["fallbacks"]))
    for k, v in sweep.items():
        print("sweep fp32 %-3s ms/step %.3f  graphs %d  lengths %s  capture %.2f s  peak %.0f MB (arm %.0f MB)" % (
            k, v["ms_per_step"], v["graphs"], v["padded_lengths"], v["capture_s"], v["peak_mem_mb"], v["arm_peak_mb"]))
    print("one layer fwd+bwd us: %s" % {k: round(v, 1) for k, v in layer.items()})
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
