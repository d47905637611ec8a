#!/usr/bin/env python
"""Step time of BERT-base with fused self-attention (``create_net(..., fuse_attn=True)``, ``--fused-attn``) against stock
``F.scaled_dot_product_attention``, and the attention op alone.

    python scripts/bench_attn.py [--steps 50] [--runs 5] [--kernel-iters 20]

The workload is bench.py's BERT configuration (``bench.MODELS["bert"]``, ``bench.make_batch``: BERT-base, 8 sequences of
128 tokens, Ok-Topk at density 0.001, BertAdam) with whole-step CUDA graphs driven through ``GraphedTrainStep``, every arm
with ``fuse_ln``, ``fuse_xent`` and ``sparse_mlm`` on, so that the baseline is the fastest configuration without fused
attention.  The dense warm-up is shortened to ``--dense-warmup`` steps: only the sparse phase is timed.  Arms, alternated
within every run:

  stock_fp32, fused_fp32   no autocast;
  stock_bf16, fused_bf16   torch.autocast(bf16).

Each arm's peak memory is ``torch.cuda.max_memory_allocated`` over its construction, dense warm-up and graph capture,
less what was allocated before it was built.

Then the op alone, forward and backward from the packed ``qkv`` to d(qkv) with the additive [B, 1, 1, S] padding mask
and dropout 0.1: stock (view, permute, SDPA, transpose, reshape and their backward) against ``self_attention``, at
(B, S, H, D) = (8, 128, 12, 64) and (2, 512, 16, 64), in fp32 and bf16, each captured ``--kernel-iters`` times in one
CUDA graph and timed with CUDA events, with the attention FLOPs computed from the shapes (forward 4 B H S^2 D, backward
2.5 times that: the five S x S products of the standard backward).  Prints the card, its power limit and SM clock,
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

ARMS = ("stock_fp32", "fused_fp32", "stock_bf16", "fused_bf16")
OP_SHAPES = ((8, 128, 12, 64), (2, 512, 16, 64))
OP_P = 0.1


def _arm(kind, a):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["bert"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=a.dense_warmup)
    tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                 seq_len=128, t_total=100000, warmup=0.1, cuda_graph=True, seed=0,
                 autocast="bf16" if kind.endswith("bf16") else None,
                 model_kwargs={"fuse_ln": True, "fuse_xent": True, "sparse_mlm": True,
                               "fuse_attn": kind.startswith("fused")})
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
        n0 = ext.LAUNCH_COUNT.get("attn_forward", 0)
        arms[k], it[k] = _arm(k, a), 0
        run(k, a.dense_warmup + a.warmup)
        torch.cuda.synchronize()
        peak[k] = torch.cuda.max_memory_allocated() - base
        launches[k] = ext.LAUNCH_COUNT.get("attn_forward", 0) - n0
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
        tr.check_mlm_overflow()
        losses[k] = float(tr.graphed.static_loss)
    out = {"steps": a.steps, "attn_forward_launches_before_timing": launches,
           "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                           for k, v in times.items()},
           "graphs": {k: {"enabled": tr.graphed.enabled, "captured": len(tr.graphed.graphs)} for k, tr in arms.items()},
           "last_loss": losses, "peak_mib": {k: v / 2 ** 20 for k, v in peak.items()}}
    for tr in arms.values():
        tr.close()
    del arms
    torch.cuda.empty_cache()
    return out


def _attn_flops(B, S, H, D):
    """Forward 4 B H S^2 D (QK^T and PV) plus backward 10 B H S^2 D (S, dP, dV, dQ, dK)."""
    return 14 * B * H * S * S * D


def _op_pair(shape, dtype, iters):
    """µs per forward + backward of the attention op, stock and fused, from qkv to d(qkv)."""
    import torch
    import torch.nn.functional as F
    from oktopk_b200.ops.fused_attn import self_attention
    B, S, H, D = shape
    g = torch.Generator("cuda").manual_seed(0)
    qkv = torch.randn(B, S, 3 * H * D, device="cuda", generator=g).to(dtype).requires_grad_(True)
    dout = torch.randn(B, S, H * D, device="cuda", generator=g).to(dtype)
    lengths = torch.randint(S // 2, S + 1, (B,), generator=torch.Generator().manual_seed(1)).cuda()
    mask = ((torch.arange(S, device="cuda")[None, :] >= lengths[:, None]).float() * -10000.0)[:, None, None, :]
    mask_t = mask.to(dtype)                     # stock SDPA needs the mask in the operands' type

    def stock():
        q, k, v = qkv.view(B, S, 3, H, D).permute(2, 0, 3, 1, 4)
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask_t, dropout_p=OP_P)
        o = o.transpose(1, 2).reshape(B, S, H * D)
        torch.autograd.grad(o, qkv, dout)

    def fused():
        torch.autograd.grad(self_attention(qkv, H, mask, OP_P), qkv, dout)

    st, fu = _graph_us(stock, iters), _graph_us(fused, iters)
    fl = _attn_flops(B, S, H, D)
    return {"stock_us": st, "fused_us": fu, "speedup": st / fu, "flop": fl,
            "stock_tflop_per_s": fl / (st * 1e-6) / 1e12, "fused_tflop_per_s": fl / (fu * 1e-6) / 1e12}


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=8)
    p.add_argument("--kernel-iters", type=int, default=20)
    p.add_argument("--op-only", action="store_true", help="time the op alone, not the BERT step")
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_attn.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    res = None if a.op_only else _workload(a)
    op = {"%dx%dx%dx%d_%s" % (*shape, name): _op_pair(shape, dt, a.kernel_iters)
          for shape in OP_SHAPES for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16))}
    out = {"card": card, "card_after": _card(), "runs": a.runs, "bert_base": res, "attn_fwd_bwd": op}
    print("card", card)
    if res is not None:
        for k, v in res["ms_per_step"].items():
            print("bert_base %-11s ms/step median %.3f  range %.3f-%.3f  last loss %.4f  peak %.0f MiB  graph %s" % (
                k, v["median"], v["min"], v["max"], res["last_loss"][k], res["peak_mib"][k], res["graphs"][k]["enabled"]))
    for name, r in op.items():
        print("attention fwd+bwd %-18s stock %8.1f us (%5.1f TFLOP/s)  fused %8.1f us (%5.1f TFLOP/s)  x%.2f" % (
            name, r["stock_us"], r["stock_tflop_per_s"], r["fused_us"], r["fused_tflop_per_s"], r["speedup"]))
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
