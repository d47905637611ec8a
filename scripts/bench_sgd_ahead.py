#!/usr/bin/env python
"""The early SGD update on / off on ``bench.py``'s flagship configuration (VGG-16, 16 images, fp32, Ok-Topk at density
0.001, whole-step CUDA graphs), alternated within one process.

    python scripts/bench_sgd_ahead.py [--rounds 5] [--steps 200] [--warmup 20] [--out DIR] [--arm STREAM:CTAS ...]

Arms: ``off`` (``sgd_ahead=False``) and ``on`` (the defaults), plus one per ``--arm STREAM:CTAS``: the ahead pass on
at most CTAS CTAs, on the communication stream right behind the segment (``comm``) or on a side stream forked from the
segment's event (``side``).  All arms are built first (same seed, the preset's untimed dense warm-up, graphs captured),
then every round times ``--steps`` sparse steps of each arm with CUDA events, the arms' order reversed every other
round.  Prints (and writes to ``DIR/sgd_ahead.json``) the median and range of
ms/step per arm, the change of each arm against ``off``, the card's name, power limit and SM clock.
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
from scripts.bench_early_pack import card  # noqa: E402


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--out", default=None)
    p.add_argument("--arm", action="append", default=[], metavar="STREAM:CTAS")
    a = p.parse_args(argv)

    import gc
    import torch
    import oktopk_b200 as okt
    from oktopk_b200.ops import ext
    from oktopk_b200.train.trainer import Trainer

    assert torch.cuda.is_available(), "bench_sgd_ahead.py needs a GPU"
    w = okt.init()
    ext.require()
    dnn, dataset, bs, lr, preset = bench.MODELS["vgg16"]
    specs = {"off": (False, None, None), "on": (True, None, None)}
    for arm in a.arm:
        where, ctas = arm.split(":")
        assert where in ("comm", "side"), arm
        specs[arm] = (True, int(ctas), where == "comm")
    arms = {}
    for name, (on, ctas, comm) in specs.items():
        torch.manual_seed(0)
        cfg = okt.preset(preset, density=0.001, sgd_ahead=on)
        tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001,
                     compression=True, cfg=cfg, world=w, seq_len=128, t_total=100000, warmup=0.1, cuda_graph=True)
        tr.adjust_learning_rate = lambda: lr
        for g in tr.optimizer.param_groups:
            g["lr"] = lr
        if ctas is not None:
            tr.optimizer._ahead_ctas = ctas
        if comm:
            tr.optimizer._ahead_stream = tr.optimizer._comm_stream
        pool = [tuple(t.to(tr.device) for t in bench.make_batch("vgg16", i, w.rank, bs, 128)) for i in range(4)]
        arms[name] = {"tr": tr, "pool": pool, "it": 0, "ms": []}

    def step(arm):
        loss = arm["tr"].step(arm["pool"][arm["it"] % 4])
        arm["it"] += 1
        return loss

    for arm in arms.values():
        for _ in range(int(arm["tr"].optimizer._cfg.warmup_iters) + a.warmup):
            step(arm)
    torch.cuda.synchronize()
    gc.collect()
    gc.disable()
    for r in range(a.rounds):
        for name in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
            arm = arms[name]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                loss = step(arm)
            e1.record()
            torch.cuda.synchronize()
            arm["ms"].append(e0.elapsed_time(e1) / a.steps)
            arm["loss"] = float(loss)
    gc.enable()
    cfg = arms["on"]["tr"].optimizer._cfg
    res = {"card": card(), "rounds": a.rounds, "steps": a.steps, "defaults": {"early_pack_ctas": cfg.early_pack_ctas},
           "arms": {k: {"median_ms": statistics.median(v["ms"]), "min_ms": min(v["ms"]), "max_ms": max(v["ms"]),
                        "ms": v["ms"], "final_loss": v["loss"]} for k, v in arms.items()}}
    off = res["arms"]["off"]
    for k, v in res["arms"].items():
        if k != "off":
            v["change_pct"] = 100.0 * (v["median_ms"] / off["median_ms"] - 1.0)
            v["ranges_apart"] = v["max_ms"] < off["min_ms"] or off["max_ms"] < v["min_ms"]
    text = json.dumps(res)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "sgd_ahead.json"), "w") as f:
            f.write(text + "\n")
    for arm in arms.values():
        arm["tr"].close()
    okt.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
