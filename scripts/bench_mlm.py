#!/usr/bin/env python
"""Step time of BERT-base with the masked-LM head on the labelled rows only (``create_net(..., sparse_mlm=True)``,
``--sparse-mlm``) against the head on every token row, and the head plus its loss alone.

    python scripts/bench_mlm.py [--steps 50] [--runs 5] [--kernel-iters 20]

The workload is bench.py's BERT configuration (``bench.MODELS["bert"]``, ``bench.make_batch``: BERT-base, 8 sequences of
128 tokens, Ok-Topk at density 0.001, BertAdam) with whole-step CUDA graphs driven through ``GraphedTrainStep``, every arm
with ``fuse_ln=True`` and ``fuse_xent=True``, so that the baseline is the fastest configuration without the gathered head.
The dense warm-up is shortened to ``--dense-warmup`` steps: only the sparse phase is timed.  Arms, alternated within
every run:

  stock_fp32, sparse_fp32   no autocast;
  stock_bf16, sparse_bf16   torch.autocast(bf16).

The sparse arms use the default capacity, 0.25 of the 1024 token rows = 256 rows.  Each arm's peak memory is
``torch.cuda.max_memory_allocated`` over its construction, dense warm-up and graph capture, less what was allocated
before it was built.  After the timed runs every sparse arm's overflow counter is read: it must be 0.

Then the MLM head + NSP head + fused loss alone, forward and backward (the gradients of the sequence output and of every
head parameter), at (1024, 768) -> 30522 with ~11 % of the rows labelled (``bench.make_batch``'s masking), stock against
the head gathered into M = 256 rows, in fp32 and bf16, each captured ``--kernel-iters`` times in one CUDA graph and timed
with CUDA events, with the GEMM FLOPs of each (computed from the shapes).  Prints the card, its power limit and SM clock,
before and after, and one JSON line.
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

ARMS = ("stock_fp32", "sparse_fp32", "stock_bf16", "sparse_bf16")
OP_ROWS, OP_H, OP_V, OP_M = 1024, 768, 30522, 256


def _arm(kind, a):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["bert"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=a.dense_warmup)
    tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                 seq_len=128, t_total=100000, warmup=0.1, cuda_graph=True, seed=0,
                 autocast="bf16" if kind.endswith("bf16") else None,
                 model_kwargs={"fuse_ln": True, "fuse_xent": True, "sparse_mlm": kind.startswith("sparse")})
    assert tr.graphed is not None
    return tr


def _workload(a):
    import torch
    from oktopk_b200.ops import ext
    bs = bench.MODELS["bert"][2]
    pool = [tuple(t.cuda() for t in bench.make_batch("bert", i, 0, bs, 128)) for i in range(4)]
    labelled = [int((b[3] != -1).sum()) for b in pool]
    arms, it, peak = {}, {}, {}

    def run(k, n):
        tr = arms[k]
        for _ in range(n):
            tr.graphed.step(pool[it[k] % len(pool)])
            it[k] += 1

    sel0 = ext.LAUNCH_COUNT.get("mlm_select", 0)
    for k in ARMS:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        arms[k], it[k] = _arm(k, a), 0
        run(k, a.dense_warmup + a.warmup)
        torch.cuda.synchronize()
        peak[k] = torch.cuda.max_memory_allocated() - base
    assert ext.LAUNCH_COUNT.get("mlm_select", 0) > sel0
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
        tr.check_mlm_overflow()
        losses[k] = float(tr.graphed.static_loss)
    out = {"steps": a.steps, "labelled_rows": labelled,
           "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                           for k, v in times.items()},
           "graphs": {k: {"enabled": tr.graphed.enabled, "captured": len(tr.graphed.graphs)} for k, tr in arms.items()},
           "last_loss": losses, "peak_mib": {k: v / 2 ** 20 for k, v in peak.items()}}
    for tr in arms.values():
        tr.close()
    del arms
    torch.cuda.empty_cache()
    return out


def _head_flops(rows):
    """GEMM FLOPs of the MLM head's forward + backward on ``rows`` rows: transform and decoder, each x W^T, dX and dW."""
    return 3 * 2 * rows * OP_H * (OP_H + OP_V)


def _head_pair(dtype, iters):
    """µs per forward + backward of the heads and the fused loss at (OP_ROWS, OP_H) -> OP_V, stock and gathered."""
    import torch
    from oktopk_b200.models.bert import BertConfig, BertPreTrainingHeads, PretrainingCriterion
    torch.manual_seed(0)
    heads = BertPreTrainingHeads(BertConfig()).cuda()
    crit = PretrainingCriterion(OP_V)
    crit.fuse_xent = True
    ids, seg, mask, labels, nxt = (t.cuda() for t in bench.make_batch("bert", 0, 0, 8, 128))
    seq = (torch.randn(8, 128, OP_H, device="cuda") * 0.5).requires_grad_(True)
    pooled = torch.randn(8, OP_H, device="cuda")
    params = list(heads.parameters())
    autocast = dtype != torch.float32

    def stock():
        with torch.autocast("cuda", dtype, enabled=autocast):
            scores, nsp = heads(seq, pooled)
            loss = crit(scores, nsp, labels, nxt)
        torch.autograd.grad(loss, [seq] + params)

    def sparse():
        with torch.autocast("cuda", dtype, enabled=autocast):
            scores, nsp, tgt = heads(seq, pooled, labels)
            loss = crit(scores, nsp, tgt, nxt)
        torch.autograd.grad(loss, [seq] + params)

    st = _graph_us(stock, iters)
    heads.sparse_mlm = True
    sp = _graph_us(sparse, iters)
    assert int(heads.mlm_overflow) == 0
    return {"stock_us": st, "sparse_us": sp, "labelled_rows": int((labels != -1).sum()), "M": OP_M,
            "stock_gemm_tflop_per_s": _head_flops(OP_ROWS) / (st * 1e-6) / 1e12,
            "sparse_gemm_tflop_per_s": _head_flops(OP_M) / (sp * 1e-6) / 1e12}


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=8)
    p.add_argument("--kernel-iters", type=int, default=20)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_mlm.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    res = _workload(a)
    head = {name: _head_pair(dt, a.kernel_iters) for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16))}
    out = {"card": card, "card_after": _card(), "runs": a.runs, "bert_base": res, "mlm_head_fwd_bwd": head}
    print("card", card)
    print("labelled rows per batch", res["labelled_rows"])
    for k, v in res["ms_per_step"].items():
        print("bert_base %-12s ms/step median %.3f  range %.3f-%.3f  last loss %.4f  peak %.0f MiB  graph %s" % (
            k, v["median"], v["min"], v["max"], res["last_loss"][k], res["peak_mib"][k], res["graphs"][k]["enabled"]))
    for name, r in head.items():
        print("mlm head + loss fwd+bwd (%d, %d) -> %d %s (%d labelled rows): stock %7.1f us (%.1f TFLOP/s)  "
              "gathered M=%d %7.1f us (%.1f TFLOP/s)" % (OP_ROWS, OP_H, OP_V, name, r["labelled_rows"], r["stock_us"],
                                                         r["stock_gemm_tflop_per_s"], r["M"], r["sparse_us"],
                                                         r["sparse_gemm_tflop_per_s"]))
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
