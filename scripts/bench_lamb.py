#!/usr/bin/env python
"""BERT-base pre-training with LAMB (``Trainer(lamb=True)``, ``--lamb``) against BertAdam: step time, peak memory, the
update alone and a short convergence run.

    python scripts/bench_lamb.py [--steps 50] [--runs 5] [--update-iters 100] [--conv-steps 300]

The step workload is bench.py's BERT configuration (``bench.MODELS["bert"]``, ``bench.make_batch``: BERT-base, 8
sequences of 128 tokens, Ok-Topk at density 0.001) with whole-step CUDA graphs and ``fuse_ln``, ``fuse_xent`` and
``sparse_mlm`` in every arm.  Arms, alternated within every run: bertadam_fp32, lamb_fp32, bertadam_bf16, lamb_bf16.
Peak memory is each arm's peak allocation above what was allocated before it was built, through its warm-up.

The update alone: every bucket's fused update (``_fused_update``) of the fp32 arms, timed with CUDA events over
``--update-iters`` repetitions, and the rate against the bytes the update must move: 40 B per parameter for LAMB's three
passes, 28 B for BertAdam's one.

Convergence: ``--conv-steps`` graphed steps of the synthetic BERT stream in fp32 with each optimizer, the
mean loss per 50 steps.  Prints the card, its power limit and SM clock, before and after, and one JSON line.
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

ARMS = ("bertadam_fp32", "lamb_fp32", "bertadam_bf16", "lamb_bf16")
FUSED = {"fuse_ln": True, "fuse_xent": True, "sparse_mlm": True}


def _trainer(kind, dense_warmup, lr, t_total=100000):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, _, preset = bench.MODELS["bert"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=dense_warmup)
    tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                 seq_len=128, t_total=t_total, warmup=0.1, cuda_graph=True, seed=0,
                 autocast="bf16" if kind.endswith("bf16") else None, model_kwargs=dict(FUSED),
                 lamb=kind.startswith("lamb"))
    assert tr.graphed is not None
    return tr


def _lr(kind, a):
    return a.lamb_lr if kind.startswith("lamb") else bench.MODELS["bert"][3]


def _workload(a):
    import torch
    from oktopk_b200.ops import ext
    bs = bench.MODELS["bert"][2]
    pool = [tuple(t.cuda() for t in bench.make_batch("bert", i, 0, bs, 128)) for i in range(4)]
    arms, it, peak = {}, {}, {}

    def run(k, n):
        tr = arms[k]
        for _ in range(n):
            tr.step(pool[it[k] % len(pool)])
            it[k] += 1

    l0 = ext.LAUNCH_COUNT.get("fused_lamb", 0)
    for k in ARMS:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        arms[k], it[k] = _trainer(k, a.dense_warmup, _lr(k, a)), 0
        run(k, a.dense_warmup + a.warmup)
        torch.cuda.synchronize()
        peak[k] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    assert ext.LAUNCH_COUNT.get("fused_lamb", 0) > l0
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
    for k, tr in arms.items():
        assert tr.graphed.enabled, (k, tr.graphed.why_disabled)
        assert all(torch.isfinite(p).all() for p in tr.net.parameters()), k
    upd = {k: _update_us(arms[k], a.update_iters) for k in ("bertadam_fp32", "lamb_fp32")}
    out = {"steps": a.steps, "lr": {k: _lr(k, a) for k in ARMS},
           "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                           for k, v in times.items()},
           "peak_mib": peak, "graphs": {k: len(tr.graphed.graphs) for k, tr in arms.items()}, "update": upd}
    for tr in arms.values():
        tr.close()
    del arms
    torch.cuda.empty_cache()
    return out


def _update_us(tr, iters):
    """µs per step of the fused update of every bucket (nothing else), and its rate against the bytes it must move."""
    import torch
    opt = tr.optimizer
    params = sum(p.numel() for g in opt.param_groups for p in g["params"])
    per_elem = 40 if opt._update.__name__ == "_LambUpdate" else 28

    def once():
        with torch.no_grad():
            for b in opt._buckets:
                opt._fused_update(b)

    for _ in range(3):
        once()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        once()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    gb = per_elem * params / 1e9
    return {"us": us, "params": params, "bytes_per_param": per_elem, "gb_per_step": gb, "tb_per_s": gb / us * 1e3,
            "datasheet_floor_us": gb * 1e9 / 3.35e12 * 1e6}         # a computed figure at 3.35 TB/s, not a measurement


def _convergence(a):
    """Mean training loss per 50 steps over the trainer's own synthetic stream, graphed, fp32."""
    import torch
    out = {}
    for k in ("bertadam_fp32", "lamb_fp32"):
        tr = _trainer(k, 50, _lr(k, a), t_total=a.conv_steps)
        losses = []
        for _ in range(a.conv_steps):
            tr.train_step()
            losses.append(tr._last_loss.clone())
        torch.cuda.synchronize()
        vals = [float(x) for x in losses]
        out[k] = [statistics.fmean(vals[i:i + 50]) for i in range(0, len(vals), 50)]
        tr.close()
        del tr
        torch.cuda.empty_cache()
    return out


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=8)
    p.add_argument("--update-iters", type=int, default=100)
    p.add_argument("--conv-steps", type=int, default=300)
    p.add_argument("--lamb-lr", type=float, default=2e-3, help="LAMB's peak learning rate (BertAdam keeps bench.py's)")
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_lamb.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    res = _workload(a)
    conv = _convergence(a) if a.conv_steps > 0 else {}
    out = {"card": card, "card_after": _card(), "runs": a.runs, "bert_base": res, "convergence": conv}
    print("card", card)
    for k, v in res["ms_per_step"].items():
        print("bert_base %-13s ms/step median %.3f  range %.3f-%.3f  peak %.0f MiB" % (
            k, v["median"], v["min"], v["max"], res["peak_mib"][k]))
    for k, u in res["update"].items():
        print("update alone %-13s %.1f us/step  %.2f GB -> %.2f TB/s  (data-sheet floor %.0f us)" % (
            k, u["us"], u["gb_per_step"], u["tb_per_s"], u["datasheet_floor_us"]))
    for k, v in conv.items():
        print("convergence %-13s mean loss per 50 steps %s" % (k, " ".join("%.4f" % x for x in v)))
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
