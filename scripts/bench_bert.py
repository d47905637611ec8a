#!/usr/bin/env python
"""Step time of BERT-base with the fused dropout + residual add + LayerNorm kernels (``create_net(..., fuse_ln=True)``,
``--fused-ln``) against the stock ops, and the fused forward + backward alone.

    python scripts/bench_bert.py [--steps 50] [--runs 5] [--kernel-iters 200]

The workload is bench.py's BERT configuration (``bench.MODELS["bert"]``, ``bench.make_batch``: BERT-base, 8 sequences of
128 tokens, Ok-Topk at density 0.001, BertAdam) with whole-step CUDA graphs driven through ``GraphedTrainStep``.  The
dense warm-up is shortened to ``--dense-warmup`` steps: only the sparse phase is timed.  Arms, alternated within every
run:

  stock_fp32, fused_fp32   no autocast;
  stock_bf16, fused_bf16   torch.autocast(bf16): the linear layers hand the LayerNorm sites a bf16 ``a``.

Then, at (1024, 768) and (1024, 1024) with ``a`` in fp32 and in bf16 and p = 0.1, the fused forward + backward against the
stock dropout + add + layer_norm forward + backward, each captured ``--kernel-iters`` times in one CUDA graph and timed
with CUDA events.  Prints the card, its power limit and SM clock, before and after, and one JSON line.
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
from scripts.bench_resnet import _graph_us  # noqa: E402

ARMS = ("stock_fp32", "fused_fp32", "stock_bf16", "fused_bf16")
KERNEL_SHAPES = [(1024, 768), (1024, 1024)]


def _arm(kind, a):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["bert"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=a.dense_warmup)
    tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                 seq_len=128, t_total=100000, warmup=0.1, cuda_graph=True, seed=0,
                 autocast="bf16" if kind.endswith("bf16") else None,
                 model_kwargs={"fuse_ln": True} if kind.startswith("fused") else None)
    assert tr.graphed is not None
    return tr


def _workload(a):
    import torch
    from oktopk_b200.ops import ext
    bs = bench.MODELS["bert"][2]
    pool = [tuple(t.cuda() for t in bench.make_batch("bert", i, 0, bs, 128)) for i in range(4)]
    arms = {k: _arm(k, a) for k in ARMS}
    it = {k: 0 for k in arms}

    def run(k, n):
        tr = arms[k]
        for _ in range(n):
            tr.graphed.step(pool[it[k] % len(pool)])
            it[k] += 1

    ln0 = ext.LAUNCH_COUNT.get("ln_forward", 0)
    for k in arms:
        run(k, a.dense_warmup + a.warmup)
    torch.cuda.synchronize()
    assert ext.LAUNCH_COUNT.get("ln_forward", 0) > ln0
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
    losses = {}
    for k, tr in arms.items():
        assert tr.graphed.enabled, (k, tr.graphed.why_disabled)
        assert all(torch.isfinite(p).all() for p in tr.net.parameters()), k
        losses[k] = float(tr.graphed.static_loss)
    out = {"steps": a.steps, "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                                             for k, v in times.items()},
           "graphs": {k: {"enabled": tr.graphed.enabled, "captured": len(tr.graphed.graphs)} for k, tr in arms.items()},
           "last_loss": losses}
    for tr in arms.values():
        tr.close()
    del arms
    torch.cuda.empty_cache()
    return out


def _kernel_pair(shape, adtype, p, iters):
    """µs per forward + backward of the fused op and of the stock ops it replaces, at one shape."""
    import torch
    import torch.nn.functional as F
    from oktopk_b200.ops.fused_ln import residual_dropout_layer_norm
    R, H = shape
    ln = torch.nn.LayerNorm(H, eps=1e-12).cuda()
    x = torch.randn(R, H, device="cuda", requires_grad=True)
    a = torch.randn(R, H, device="cuda").to(adtype).requires_grad_(True)
    dy = torch.randn(R, H, device="cuda")
    params = (x, a, ln.weight, ln.bias)

    def fused():
        torch.autograd.grad(residual_dropout_layer_norm(x, a, ln, p), params, dy)

    def stock():
        torch.autograd.grad(ln(x + F.dropout(a, p, True)), params, dy)

    return _graph_us(fused, iters), _graph_us(stock, iters)


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=8)
    p.add_argument("--kernel-iters", type=int, default=200)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_bert.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    res = _workload(a)
    kern = []
    for shape in KERNEL_SHAPES:
        row = {"shape": list(shape), "p": 0.1}
        for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
            row[name + "_fused_us"], row[name + "_stock_us"] = _kernel_pair(shape, dt, 0.1, a.kernel_iters)
        kern.append(row)
    out = {"card": card, "card_after": _card(), "runs": a.runs, "bert_base": res, "ln_fwd_bwd_us": kern}
    print("card", card)
    for k, v in res["ms_per_step"].items():
        print("bert_base %-11s ms/step median %.3f  range %.3f-%.3f  graph %s" % (
            k, v["median"], v["min"], v["max"], res["graphs"][k]["enabled"]))
    for row in kern:
        print("dropout+add+LN fwd+bwd %-12s a fp32: fused %6.1f us stock %6.1f us | a bf16: fused %6.1f us stock %6.1f us"
              % (tuple(row["shape"]), row["fp32_fused_us"], row["fp32_stock_us"], row["bf16_fused_us"],
                 row["bf16_stock_us"]))
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
