#!/usr/bin/env python
"""Step time of BERT-base with the fused masked-LM softmax cross-entropy (``create_net(..., fuse_xent=True)``,
``--fused-xent``) against stock ``F.cross_entropy``, and the fused forward + backward alone.

    python scripts/bench_xent.py [--steps 50] [--runs 5] [--kernel-iters 50]

The workload is bench.py's BERT configuration (``bench.MODELS["bert"]``, ``bench.make_batch``: BERT-base, 8 sequences of
128 tokens, Ok-Topk at density 0.001, BertAdam) with whole-step CUDA graphs driven through ``GraphedTrainStep``, every arm
with ``fuse_ln=True`` so that the baseline is the fastest configuration without this op.  The dense warm-up is shortened
to ``--dense-warmup`` steps: only the sparse phase is timed.  Arms, alternated within every run:

  stock_fp32, fused_fp32   no autocast;
  stock_bf16, fused_bf16   torch.autocast(bf16): the decoder hands the loss bf16 logits.

Each arm's peak memory is ``torch.cuda.max_memory_allocated`` over its construction, dense warm-up and graph capture,
less what was allocated before it was built (the arms built earlier stay alive, so their memory is constant in it).

Then, at (1024, 30522) with ~11 % of the rows labelled (the share ``bench.make_batch`` masks), the fused forward + backward
against stock ``F.cross_entropy`` with autocast's dtype handling (the logits widened to fp32, the gradient narrowed back),
in fp32 and bf16, each captured ``--kernel-iters`` times in one CUDA graph and timed with CUDA events, with the fused op's
bytes (computed from the shapes) over its time.  Prints the card, its power limit and SM clock, before and after, and one
JSON line.
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
OP_SHAPE = (1024, 30522)
OP_LABELLED = 0.11


def _arm(kind, a):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["bert"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=a.dense_warmup)
    tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                 seq_len=128, t_total=100000, warmup=0.1, cuda_graph=True, seed=0,
                 autocast="bf16" if kind.endswith("bf16") else None,
                 model_kwargs={"fuse_ln": True, "fuse_xent": kind.startswith("fused")})
    assert tr.graphed is not None
    return tr


def _workload(a):
    import torch
    from oktopk_b200.ops import ext
    bs = bench.MODELS["bert"][2]
    pool = [tuple(t.cuda() for t in bench.make_batch("bert", i, 0, bs, 128)) for i in range(4)]
    arms, it, peak = {}, {}, {}

    def run(k, n):
        tr = arms[k]
        for _ in range(n):
            tr.graphed.step(pool[it[k] % len(pool)])
            it[k] += 1

    xe0 = ext.LAUNCH_COUNT.get("xent_forward", 0)
    for k in ARMS:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        arms[k], it[k] = _arm(k, a), 0
        run(k, a.dense_warmup + a.warmup)
        torch.cuda.synchronize()
        peak[k] = torch.cuda.max_memory_allocated() - base
    assert ext.LAUNCH_COUNT.get("xent_forward", 0) > xe0
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
           "last_loss": losses, "peak_mib": {k: v / 2 ** 20 for k, v in peak.items()}}
    for tr in arms.values():
        tr.close()
    del arms
    torch.cuda.empty_cache()
    return out


def _op_bytes(R, V, n_lab, esize):
    """HBM bytes the fused forward + backward needs: the labelled rows read twice, the gradient written once, the
    targets read three times, lse and the row losses written and read."""
    return 2 * n_lab * V * esize + R * V * esize + 3 * 8 * R + 4 * 4 * R


def _op_pair(dtype, iters):
    """µs per forward + backward of the fused op and of stock cross_entropy at OP_SHAPE, and the fused op's bytes."""
    import torch
    import torch.nn.functional as F
    from oktopk_b200.ops.fused_xent import softmax_cross_entropy
    R, V = OP_SHAPE
    g = torch.Generator("cuda").manual_seed(0)
    x = (torch.randn(R, V, device="cuda", generator=g) * 2).to(dtype).requires_grad_(True)
    t = torch.randint(0, V, (R,), device="cuda", generator=g)
    t[torch.rand(R, device="cuda", generator=g) >= OP_LABELLED] = -1
    n_lab = int((t != -1).sum())

    def fused():
        torch.autograd.grad(softmax_cross_entropy(x, t, ignore_index=-1), x)

    def stock():
        torch.autograd.grad(F.cross_entropy(x.float(), t, ignore_index=-1), x)

    fu, st = _graph_us(fused, iters), _graph_us(stock, iters)
    nbytes = _op_bytes(R, V, n_lab, x.element_size())
    return {"fused_us": fu, "stock_us": st, "labelled_rows": n_lab, "fused_bytes": nbytes,
            "fused_gb_per_s": nbytes / (fu * 1e-6) / 1e9}


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=8)
    p.add_argument("--kernel-iters", type=int, default=50)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_xent.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    res = _workload(a)
    op = {name: _op_pair(dt, a.kernel_iters) for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16))}
    out = {"card": card, "card_after": _card(), "runs": a.runs, "bert_base": res, "xent_fwd_bwd": op}
    print("card", card)
    for k, v in res["ms_per_step"].items():
        print("bert_base %-11s ms/step median %.3f  range %.3f-%.3f  last loss %.4f  peak %.0f MiB  graph %s" % (
            k, v["median"], v["min"], v["max"], res["last_loss"][k], res["peak_mib"][k], res["graphs"][k]["enabled"]))
    for name, r in op.items():
        print("xent fwd+bwd %s %s (%d labelled rows): fused %7.1f us (%.0f GB/s)  stock %7.1f us" % (
            OP_SHAPE, name, r["labelled_rows"], r["fused_us"], r["fused_gb_per_s"], r["stock_us"]))
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
