#!/usr/bin/env python
"""Step time of the VGG-16 Ok-Topk workload under three optimizers, and the ``fused_adam`` kernel on its own.

    python scripts/bench_adam.py [--steps 200] [--warmup 20] [--runs 5] [--kernel-iters 1000]

The workload is bench.py's (``bench.MODELS["vgg16"]``, ``bench.make_batch``, 16 images, the VGG-16 preset, Ok-Topk at
density 0.001) with whole-step CUDA graphs driven through ``GraphedTrainStep``.  The dense warm-up is shortened to
``--dense-warmup`` steps: only the sparse phase is timed.  Arms, alternated within every run:

  sgd          SGD(lr 0.1, momentum 0.9, weight decay 1e-4), as in bench.py;
  adamw        AdamW(fused=True) on the flat-bucket fused_adam path;
  adamw_torch  AdamW(fused=True) on the path every other optimizer takes: landing copy + torch's fused kernel, eager
               (torch's Adam refuses CUDA-graph capture unless capturable=True).

Then ``fused_adam`` alone on the VGG-16 bucket, timed with CUDA events over ``--kernel-iters`` launches, against the
28 B/element it must move (p, m, v read and written, g read).  Prints the card, its power limit and SM clock.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from unittest import mock

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("OMP_NUM_THREADS", "1")

import bench  # noqa: E402  (make_batch, MODELS: the bench workload definition)

BYTES_PER_ELEM = 28
HBM_TBPS = 3.35          # H100 SXM data sheet


class _Shim:
    """The part of Trainer that GraphedTrainStep drives."""

    def __init__(self, net, opt):
        self.net, self.optimizer = net, opt

    def _forward_loss(self, batch):
        import torch
        x, y = batch
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
    import oktopk_b200.optimizer as okt_opt
    from oktopk_b200.models import create_net
    from oktopk_b200.train.graph_step import GraphedTrainStep
    torch.manual_seed(0)
    net, _ = create_net(10, dnn)
    net = net.cuda().to(memory_format=torch.channels_last)
    if kind == "sgd":
        base = torch.optim.SGD(net.parameters(), lr=lr, momentum=0.9, weight_decay=1e-4)
    else:
        base = torch.optim.AdamW(net.parameters(), lr=1e-3, weight_decay=1e-2, fused=True)
    # adamw_torch: the gate refuses, as it does for any optimizer without a flat-bucket kernel
    gate = (lambda o: False) if kind == "adamw_torch" else okt_opt._fused_adam_applies
    with mock.patch.object(okt_opt, "_fused_adam_applies", gate):
        opt = okt.DistributedOptimizer(base, named_parameters=net.named_parameters(),
                                       compression=okt.compressors["oktopk"], is_sparse=True, cfg=cfg)
    assert bool(getattr(opt, "_okt_adam", False)) == (kind == "adamw"), kind
    return opt, GraphedTrainStep(_Shim(net, opt))


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=8)
    p.add_argument("--kernel-iters", type=int, default=1000)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_adam.py needs a GPU", file=sys.stderr)
        return 2
    import oktopk_b200 as okt
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    dnn, _, bs, lr, preset = bench.MODELS["vgg16"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=a.dense_warmup)
    pool = []
    for i in range(4):
        x, y = bench.make_batch("vgg16", i, 0, bs, 128)
        pool.append((x.cuda().contiguous(memory_format=torch.channels_last), y.cuda()))
    arms = {k: _arm(k, dnn, lr, cfg) for k in ("sgd", "adamw", "adamw_torch")}
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

    # fused_adam alone on a copy of the VGG-16 bucket; the gradient is the all-zero bucket of a sparse step
    opt = arms["adamw"][0]
    b = opt._buckets[0]
    n = b.numel
    pf = b.flat_param.clone()
    g = torch.zeros_like(pf)
    m, v = (opt._flat_state[b.index][k].clone() for k in ("exp_avg", "exp_avg_sq"))
    scal = torch.tensor([1 - 1e-3 * 1e-2, -1e-3 / (1 - 0.9 ** 100), (1 - 0.999 ** 100) ** 0.5], dtype=torch.float32,
                        device="cuda")
    C, st = ext.require(), torch.cuda.current_stream().cuda_stream

    def launch():
        C.fused_adam(pf.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, 0.9, 0.999, 1e-8, 1e-2, 1, 1, st,
                     scal.data_ptr())

    for _ in range(50):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.kernel_iters):
        launch()
    e1.record()
    torch.cuda.synchronize()
    k_us = e0.elapsed_time(e1) * 1e3 / a.kernel_iters
    k_tbps = BYTES_PER_ELEM * n / (k_us * 1e-6) / 1e12

    out = {"card": _card(), "steps": a.steps, "runs": a.runs,
           "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                           for k, v in times.items()},
           "graphs": {k: {"enabled": gs.enabled, "captured": len(gs.graphs), "why_disabled": gs.why_disabled}
                      for k, (_, gs) in arms.items()},
           "fused_adam": {"elements": n, "us": k_us, "TB_per_s": k_tbps, "bytes_per_elem": BYTES_PER_ELEM,
                          "floor_us_at_3.35TBps": BYTES_PER_ELEM * n / (HBM_TBPS * 1e12) * 1e6,
                          "share_of_3.35TBps": k_tbps / HBM_TBPS}}
    for k, v in out["ms_per_step"].items():
        print("%-12s ms/step median %.4f  range %.4f-%.4f  graph %s" % (k, v["median"], v["min"], v["max"],
                                                                       out["graphs"][k]["enabled"]))
    print("fused_adam on %d elements: %.1f us, %.2f TB/s at %d B/element (floor %.1f us at %.2f TB/s)"
          % (n, k_us, k_tbps, BYTES_PER_ELEM, out["fused_adam"]["floor_us_at_3.35TBps"], HBM_TBPS))
    print(json.dumps(out))
    for opt, _ in arms.values():
        opt.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
