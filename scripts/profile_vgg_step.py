#!/usr/bin/env python
"""Kernel-by-kernel timeline of one VGG-16 training step (``bench.py``'s flagship configuration), from ``torch.profiler``.

    python scripts/profile_vgg_step.py [--steps 20] [--warmup 20] [--out profiles/vgg_step] [--no-sgd-ahead]

Builds the workload as ``bench.py`` does (16 images, fp32, Ok-Topk at density 0.001, the preset's untimed dense warm-up,
whole-step CUDA graphs), replays ``--steps`` threshold-reuse sparse steps under the profiler and splits the trace into
steps at each SGD update (``fused_sgd_kernel``, or ``fused_sgd_tail_kernel`` after the early SGD update; ``--no-sgd-ahead``
turns that off).  It writes ``<out>/vgg_step.md`` and ``.json``:

* every kernel of the median-length step with its grid, block, duration and start offset within the step;
* per step: the step span, the Ok-Topk call and the *backward tail* -- the time from the end of layer 9's convolution
  backward (the last of layers 9 - 13's weight gradients; the start of layer 8's batch-norm backward) to the start of
  the Ok-Topk call, i.e. how long the bucket's big gradients sit finished while backward runs layers 8 -> 1;
* per step: the update kernel's and the early SGD update's (``sgd_ahead_kernel``) durations, and the backward span from
  the start of layer 13's batch-norm backward to the end of layer 1's;
* the grid sizes of the kernels in that tail.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("OMP_NUM_THREADS", "1")

import bench  # noqa: E402  (make_batch, MODELS: the bench workload definition)

N_CONV = 13          # VGG-16's convolution + batch-norm layers


def split_steps(kernels):
    """Kernel events sorted by start time -> lists of one step each (a step ends with its SGD update kernel)."""
    steps, cur = [], []
    for k in kernels:
        cur.append(k)
        if "fused_sgd_kernel" in k["name"] or "fused_sgd_tail_kernel" in k["name"]:
            steps.append(cur)
            cur = []
    return steps


def analyse(step):
    t0 = step[0]["ts"]
    okt = [k for k in step if "oktopk_fused_kernel" in k["name"]]
    bn_bwd = [k for k in step if "bn_bwd" in k["name"]]
    out = {"span_us": step[-1]["ts"] + step[-1]["dur"] - t0, "kernels": len(step)}
    out["update_us"] = step[-1]["dur"]
    ahead = [k for k in step if "sgd_ahead_kernel" in k["name"]]
    if ahead:
        out["ahead_us"] = sum(k["dur"] for k in ahead)
    if bn_bwd:
        out["backward_us"] = bn_bwd[-1]["ts"] + bn_bwd[-1]["dur"] - bn_bwd[0]["ts"]
    if okt:
        out["oktopk_us"] = okt[0]["dur"]
        out["oktopk_start_us"] = okt[0]["ts"] - t0
    # backward runs layers 13 -> 1: the 6th batch-norm backward is layer 8's, launched once conv 9's backward is done
    if okt and len(bn_bwd) == N_CONV:
        l8 = bn_bwd[N_CONV - 8]
        out["tail_start_us"] = l8["ts"] - t0
        out["tail_us"] = okt[0]["ts"] - l8["ts"]
        tail = [k for k in step if l8["ts"] <= k["ts"] < okt[0]["ts"]]
        out["tail_busy_us"] = sum(k["dur"] for k in tail)
        out["tail_grids"] = [(k["name"][:60], k["grid"], round(k["dur"], 1)) for k in tail]
    return out


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--out", default=os.path.join("profiles", "vgg_step"))
    p.add_argument("--no-sgd-ahead", action="store_true", help="OkTopkConfig.sgd_ahead=False")
    a = p.parse_args(argv)

    import torch
    from torch.profiler import ProfilerActivity, profile
    import oktopk_b200 as okt
    from oktopk_b200.ops import ext
    from oktopk_b200.train.trainer import Trainer

    assert torch.cuda.is_available(), "profile_vgg_step.py needs a GPU"
    w = okt.init()
    ext.require()
    dnn, dataset, bs, lr, preset = bench.MODELS["vgg16"]
    cfg = okt.preset(preset, density=0.001, sgd_ahead=not a.no_sgd_ahead)
    tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001,
                 compression=True, cfg=cfg, world=w, seq_len=128, t_total=100000, warmup=0.1, cuda_graph=True)
    tr.adjust_learning_rate = lambda: lr
    for g in tr.optimizer.param_groups:
        g["lr"] = lr
    pool = [tuple(t.to(tr.device) for t in bench.make_batch("vgg16", i, w.rank, bs, 128)) for i in range(4)]

    it = 0
    for _ in range(int(cfg.warmup_iters) + a.warmup):
        tr.step(pool[it % len(pool)])
        it += 1
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            tr.step(pool[it % len(pool)])
            it += 1
        torch.cuda.synchronize()
    fd, path = tempfile.mkstemp(suffix=".json")
    os.close(fd)
    prof.export_chrome_trace(path)
    with open(path) as f:
        trace = json.load(f)
    os.unlink(path)
    kernels = sorted(({"name": e["name"], "ts": float(e["ts"]), "dur": float(e["dur"]),
                       "grid": tuple(e.get("args", {}).get("grid", ())), "block": tuple(e.get("args", {}).get("block", ())),
                       "stream": e.get("args", {}).get("stream")}
                      for e in trace.get("traceEvents", []) if e.get("cat") == "kernel"), key=lambda k: k["ts"])
    steps = split_steps(kernels)[1:]                 # the first may be cut by the profiler's start
    info = [analyse(s) for s in steps]
    # exact-threshold steps (1 in tau) run the longer flavour of the call: report the threshold-reuse ones
    reuse = [(s, i) for s, i in zip(steps, info) if "oktopk_us" in i]
    med_ok = statistics.median(i["oktopk_us"] for _, i in reuse)
    reuse = [(s, i) for s, i in reuse if i["oktopk_us"] < 1.5 * med_ok]
    spans = sorted(reuse, key=lambda r: r[1]["span_us"])
    rep, rep_info = spans[len(spans) // 2]

    props = torch.cuda.get_device_properties(0)
    summ = {k: statistics.median(i[k] for _, i in reuse if k in i)
            for k in ("span_us", "oktopk_us", "oktopk_start_us", "tail_start_us", "tail_us", "tail_busy_us", "update_us",
                      "ahead_us", "backward_us")
            if any(k in i for _, i in reuse)}
    summ["steps"] = len(reuse)
    t0 = rep[0]["ts"]
    lines = ["# VGG-16 step timeline: 16 images, fp32, Ok-Topk 0.001, CUDA graph, 1 GPU (%s, %d SMs)\n"
             % (props.name, props.multi_processor_count),
             "Medians over %d threshold-reuse steps (us): %s\n" % (len(reuse), json.dumps({k: round(v, 1) for k, v in summ.items()})),
             "Backward tail = start of layer 8's batch-norm backward (conv 9's weight gradient done) -> start of the "
             "Ok-Topk call.\n",
             "## Median step, kernel by kernel\n",
             "| # | start us | dur us | grid | block | stream | kernel |", "|---|---|---|---|---|---|---|"]
    for n, k in enumerate(rep):
        lines.append("| %d | %.1f | %.1f | %s | %s | %s | `%s` |" % (n, k["ts"] - t0, k["dur"], k["grid"], k["block"],
                                                                   k["stream"], k["name"][:100]))
    text = "\n".join(lines) + "\n"
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "vgg_step.md"), "w") as f:
        f.write(text)
    with open(os.path.join(a.out, "vgg_step.json"), "w") as f:
        json.dump({"gpu": props.name, "summary": summ, "steps": [i for _, i in reuse],
                   "median_step": [dict(k, ts=k["ts"] - t0) for k in rep]}, f, indent=1)
    print(text)
    tr.close()
    okt.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
