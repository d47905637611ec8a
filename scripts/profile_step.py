#!/usr/bin/env python
"""Where the device time of one training step goes, by kernel family, measured with ``torch.profiler``.

    python scripts/profile_step.py [--model vgg16] [--steps 300] [--warmup 20] [--out profiles/step]

Builds the workload the way ``bench.py`` does (same trainer, preset, synthetic batches, the workload's untimed dense
warm-up, whole-step CUDA graphs), times ``--steps`` steps with CUDA events, then profiles the same number of steps in a
separate window and writes ``<out>/kernels_<model>.md`` (and ``.json``): kernel family, calls per step, device us per
step and share of the event-timed step.  Kernels inside a CUDA graph are traced one by one.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("OMP_NUM_THREADS", "1")

import bench  # noqa: E402  (make_batch, MODELS: the bench workload definition)

# (family, pattern on the demangled kernel name); first match wins
FAMILIES = [
    ("bn+relu+pool (bnrelu.cu)", r"okt::(bn_|maxpool2_)"),
    ("ok-topk allreduce", r"okt::(oktopk|gather|gtopk|dense_allreduce|kth_abs)"),
    ("gradient landing", r"okt::land"),
    ("fused update", r"okt::(fused_sgd|fused_bert_adam|fused_adam|momentum_correct|grad_sumsq|clip_coef)"),
    ("other okt::", r"okt::"),
    ("convolution (cuDNN)", r"(?i)conv|cudnn|xmma|implicit|wgrad|dgrad|fprop|winograd|fft"),
    ("gemm (cuBLAS)", r"(?i)gemm|cutlass|sm90_|ampere_|gemv"),
    ("aten elementwise/reduce", r"at::native|aten"),
]


def family(name: str) -> str:
    for fam, pat in FAMILIES:
        if re.search(pat, name):
            return fam
    return "other"


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--model", default="vgg16", choices=sorted(bench.MODELS))
    p.add_argument("--steps", type=int, default=300)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--out", default=os.path.join("profiles", "step"))
    p.add_argument("--no-graph", action="store_true", help="eager launches instead of whole-step CUDA graphs")
    a = p.parse_args(argv)

    import torch
    from torch.profiler import ProfilerActivity, profile
    import oktopk_b200 as okt
    from oktopk_b200.ops import ext
    from oktopk_b200.train.trainer import Trainer

    assert torch.cuda.is_available(), "profile_step.py needs a GPU"
    w = okt.init()
    ext.require()
    dnn, dataset, bs, lr, preset = bench.MODELS[a.model]
    cfg = okt.preset(preset, density=0.001)
    tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001,
                 compression=True, cfg=cfg, world=w, seq_len=128, t_total=100000, warmup=0.1, cuda_graph=not a.no_graph)
    if a.model == "vgg16":
        tr.adjust_learning_rate = lambda: lr
        for g in tr.optimizer.param_groups:
            g["lr"] = lr
    pool = [tuple(t.to(tr.device) for t in bench.make_batch(a.model, i, w.rank, bs, 128)) for i in range(4)]

    def step(i):
        tr.net.train()
        if tr.graphed is not None and tr.graphed.enabled:
            tr.adjust_learning_rate()
            loss = tr.graphed.step(pool[i % len(pool)])
            tr._bookkeep_iter()
            return loss
        tr.optimizer.zero_grad()
        loss, _ = tr._forward_loss(pool[i % len(pool)])
        loss.backward()
        tr.update_model()
        return loss

    it = 0
    for _ in range(int(cfg.warmup_iters) + a.warmup):
        step(it)
        it += 1
    torch.cuda.synchronize()

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        step(it)
        it += 1
    e1.record()
    torch.cuda.synchronize()
    step_us = e0.elapsed_time(e1) * 1e3 / a.steps

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step(it)
            it += 1
        torch.cuda.synchronize()

    per_kernel = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if ev.name.startswith(("Memcpy", "Memset")) or "memcpy" in ev.name.lower():
            continue
        k = per_kernel[ev.name]
        k[0] += 1
        k[1] += ev.time_range.elapsed_us()
    fams = collections.defaultdict(lambda: [0, 0.0])
    for name, (n, us) in per_kernel.items():
        f = fams[family(name)]
        f[0] += n
        f[1] += us
    dev_us = sum(v[1] for v in fams.values()) / a.steps

    props = torch.cuda.get_device_properties(0)
    rows = sorted(((f, n / a.steps, us / a.steps) for f, (n, us) in fams.items()), key=lambda r: -r[2])
    krows = sorted(((k, n / a.steps, us / a.steps) for k, (n, us) in per_kernel.items()), key=lambda r: -r[2])
    os.makedirs(a.out, exist_ok=True)
    tag = "kernels_%s%s" % (a.model, "_eager" if a.no_graph else "")
    lines = ["# Device time per step: %s, 1 GPU (%s), %s\n" % (a.model, props.name, "eager" if a.no_graph else "CUDA graph"),
             "%d steps traced with torch.profiler after %d timed with CUDA events.  Event-timed step: %.1f us.  "
             "Kernel time per step: %.1f us (the rest is idle time between kernels).\n" % (a.steps, a.steps, step_us, dev_us),
             "| kernel family | calls / step | device us / step | share of step |", "|---|---|---|---|"]
    lines += ["| %s | %.1f | %.1f | %.1f %% |" % (f, n, us, 100 * us / step_us) for f, n, us in rows]
    lines += ["", "| kernel | calls / step | device us / step | share of step |", "|---|---|---|---|"]
    lines += ["| `%s` | %.1f | %.1f | %.1f %% |" % (k[:110], n, us, 100 * us / step_us) for k, n, us in krows[:40]]
    text = "\n".join(lines) + "\n"
    with open(os.path.join(a.out, tag + ".md"), "w") as f:
        f.write(text)
    with open(os.path.join(a.out, tag + ".json"), "w") as f:
        json.dump({"gpu": props.name, "steps": a.steps, "step_us": step_us, "kernel_us": dev_us,
                   "families": {f: {"calls_per_step": n, "us_per_step": us} for f, n, us in rows},
                   "kernels": {k: {"calls_per_step": n, "us_per_step": us} for k, n, us in krows}}, f, indent=1)
    print(text)
    tr.close()
    okt.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
