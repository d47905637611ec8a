#!/usr/bin/env python
"""Step time of BERT-base with the fused embedding block (``create_net(..., fuse_emb=True)``, ``--fused-emb``) against
the stock gathers, adds, LayerNorm and dropout, and the block alone.

    python scripts/bench_emb.py [--steps 50] [--runs 5] [--kernel-iters 20]

The workload is bench.py's BERT configuration (``bench.MODELS["bert"]``, ``bench.make_batch``: BERT-base, 8 sequences of
128 tokens, Ok-Topk at density 0.001, BertAdam) with whole-step CUDA graphs driven through ``GraphedTrainStep``, every arm
with ``fuse_ln``, ``fuse_xent`` and ``sparse_mlm`` on.  The dense warm-up is shortened to ``--dense-warmup`` steps: only
the sparse phase is timed.  Arms, alternated within every run:

  stock_fp32, fused_fp32   no autocast;
  stock_bf16, fused_bf16   torch.autocast(bf16).

Each arm's peak memory is ``torch.cuda.max_memory_allocated`` over its construction, dense warm-up and graph capture,
less what was allocated before it was built.

Then the block alone, forward and backward from the ids to the five parameter gradients with dropout 0.1, stock
(``BertEmbeddings`` with ``fuse_emb`` off) against fused, at (B, S, H) = (8, 128, 768) and (2, 512, 1024) with a
30522-row word table, captured ``--kernel-iters`` times in one CUDA graph and timed with CUDA events; the bytes the
fused pair must move at least (the word-table gradient written once, the tables' gathered rows and y / dy) give its
bandwidth.  Last, a ``torch.profiler`` run of its own per side at (8, 128, 768): every kernel of one forward + backward,
with its launches and device time per call.  Prints the card, its power limit and SM clock, before and after, and one
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
OP_SHAPES = ((8, 128, 768), (2, 512, 1024))
OP_P = 0.1
VOCAB = 30522


def _arm(kind, a):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["bert"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=a.dense_warmup)
    tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                 seq_len=128, t_total=100000, warmup=0.1, cuda_graph=True, seed=0,
                 autocast="bf16" if kind.endswith("bf16") else None,
                 model_kwargs={"fuse_ln": True, "fuse_xent": True, "sparse_mlm": True,
                               "fuse_emb": kind.startswith("fused")})
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

    launches = {}
    for k in ARMS:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        n0 = ext.LAUNCH_COUNT.get("emb_forward", 0)
        arms[k], it[k] = _arm(k, a), 0
        run(k, a.dense_warmup + a.warmup)
        torch.cuda.synchronize()
        peak[k] = torch.cuda.max_memory_allocated() - base
        launches[k] = ext.LAUNCH_COUNT.get("emb_forward", 0) - n0
        assert (launches[k] > 0) == k.startswith("fused"), (k, launches[k])
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
        assert int(tr.net.stages[0].embeddings.id_overflow) == 0, k
        tr.check_mlm_overflow()
        losses[k] = float(tr.graphed.static_loss)
    out = {"steps": a.steps, "emb_forward_launches_before_timing": launches,
           "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                           for k, v in times.items()},
           "graphs": {k: {"enabled": tr.graphed.enabled, "captured": len(tr.graphed.graphs)} for k, tr in arms.items()},
           "last_loss": losses, "peak_mib": {k: v / 2 ** 20 for k, v in peak.items()}}
    for tr in arms.values():
        tr.close()
    del arms
    torch.cuda.empty_cache()
    return out


def _block(shape, fused):
    """A BertEmbeddings of BERT-base's vocabulary at hidden size H in training mode, a batch of ids and dy, and the
    forward + backward closure from the ids to the five parameter gradients."""
    import torch
    from oktopk_b200.models.bert import BertConfig, BertEmbeddings
    from oktopk_b200.models import bert_synthetic_batch
    B, S, H = shape
    torch.manual_seed(0)
    emb = BertEmbeddings(BertConfig(hidden_size=H, hidden_dropout_prob=OP_P)).cuda().train()
    emb.fuse_emb = fused
    ids, seg, *_ = bert_synthetic_batch(B, S, device="cuda", generator=torch.Generator().manual_seed(1))
    dy = torch.randn(B, S, H, device="cuda")
    params = list(emb.parameters())

    def fn():
        torch.autograd.grad(emb(ids, seg), params, dy)

    return fn


def _op_bytes(B, S, H):
    """The fused pair's least traffic: the word-table gradient written once; forward the three gathered rows read and
    y written; backward dy read, the rows read again, de written and read back."""
    R = B * S
    return 4 * (VOCAB * H + 4 * R * H + 4 * R * H + 2 * R * H)


def _op_pair(shape, iters):
    st, fu = _graph_us(_block(shape, False), iters), _graph_us(_block(shape, True), iters)
    nbytes = _op_bytes(*shape)
    return {"stock_us": st, "fused_us": fu, "speedup": st / fu, "min_bytes": nbytes,
            "fused_gb_per_s": nbytes / (fu * 1e-6) / 1e9}


def _profile(shape, fused, n=5):
    """Every CUDA kernel of one forward + backward of the block: launches and device µs per call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn = _block(shape, fused)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    rows = {}
    for e in p.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = getattr(e, "device_time", None)
        if us is None:
            us = getattr(e, "cuda_time", 0.0)
        r = rows.setdefault(e.name, [0, 0.0])
        r[0] += 1
        r[1] += us
    kern = sorted(((k, c / n, t / n) for k, (c, t) in rows.items()), key=lambda x: -x[2])
    return {"kernels": [{"name": k, "launches": c, "us": t} for k, c, t in kern],
            "launches_per_call": sum(c for _, c, _ in kern), "device_us_per_call": sum(t for _, _, t in kern)}


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=8)
    p.add_argument("--kernel-iters", type=int, default=20)
    p.add_argument("--op-only", action="store_true", help="time the block alone, not the BERT step")
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_emb.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    res = None if a.op_only else _workload(a)
    op = {"%dx%dx%d" % shape: _op_pair(shape, a.kernel_iters) for shape in OP_SHAPES}
    prof = {side: _profile(OP_SHAPES[0], side == "fused") for side in ("stock", "fused")}
    out = {"card": card, "card_after": _card(), "runs": a.runs, "bert_base": res, "emb_fwd_bwd": op, "profile": prof}
    print("card", card)
    if res is not None:
        for k, v in res["ms_per_step"].items():
            print("bert_base %-11s ms/step median %.3f  range %.3f-%.3f  last loss %.4f  peak %.0f MiB  graph %s" % (
                k, v["median"], v["min"], v["max"], res["last_loss"][k], res["peak_mib"][k], res["graphs"][k]["enabled"]))
    for name, r in op.items():
        print("embedding block fwd+bwd %-11s stock %7.1f us  fused %7.1f us (%6.0f GB/s of the least traffic)  x%.2f" % (
            name, r["stock_us"], r["fused_us"], r["fused_gb_per_s"], r["speedup"]))
    for side, r in prof.items():
        print("profile %s %dx%dx%d: %.1f launches, %.1f us device time per forward + backward" % (
            side, *OP_SHAPES[0], r["launches_per_call"], r["device_us_per_call"]))
        for k in r["kernels"]:
            print("   %5.1f x %8.1f us  %s" % (k["launches"], k["us"], k["name"][:110]))
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
