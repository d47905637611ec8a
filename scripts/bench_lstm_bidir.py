#!/usr/bin/env python
"""The fused LSTM recurrence on bidirectional layers (``bidirectional=True, fuse_lstm=True,
fuse_lstm_bidirectional=True``, ``--bidirectional --fused-lstm --fused-lstm-bidirectional``) against the stock
bidirectional layers.

    python scripts/bench_lstm_bidir.py [--steps 30] [--runs 5] [--op-iters 20]

The workload is bench.py's LSTM-AN4 configuration with the bidirectional network, as in ``scripts/bench_lstm.py``: 2
utterances (T' = 48 - 198 frames after the convolutions), the lstm_an4 preset, Ok-Topk at density 0.001, eager steps, the
dense warm-up shortened to ``--dense-warmup`` steps.  Two parts:

1. Step time of four arms: fp32 stock, fp32 fused, bf16 stock, bf16 fused (with ``fuse_lstm_autocast``).  The Trainers
   alternate ``--runs`` times, ``--steps`` steps each, timed with CUDA events; median (range) ms/step, each arm's last
   loss, and its peak allocated memory over construction and warm-up (all four batches of the pool), above what was
   allocated before it.
2. One ``BatchRNN`` (batch norm + ``nn.LSTM(800, 800)``) forward + backward at N = 2 and T' in {48, 123, 198}, both
   utterances of full length, fp32, eager, µs per call: the bidirectional layer stock and fused, and the fused
   one-direction layer, which gives the second direction's marginal cost.

Prints the card, its power limit and SM clock before and after, and one JSON line.  Needs a GPU: there is no fallback.
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

OP_T = (48, 123, 198)
# arm -> (autocast, fused)
ARMS = {"fp32_stock": (None, False), "fp32_fused": (None, True), "bf16_stock": ("bf16", False),
        "bf16_fused": ("bf16", True)}


def _trainer(autocast, fused: bool, dense_warmup: int):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=dense_warmup)
    return Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                   t_total=100000, warmup=0.1, seed=0, autocast=autocast,
                   model_kwargs={"bidirectional": True, "fuse_lstm": fused, "fuse_lstm_bidirectional": fused,
                                 "fuse_lstm_autocast": fused and autocast is not None})


def _step(tr, batch):
    tr.net.train()
    tr.optimizer.zero_grad()
    loss, _ = tr._forward_loss(batch)
    tr.backward(loss)
    tr.update_model()
    return loss


def _timed(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def step_times(a) -> dict:
    import torch
    from oktopk_b200.ops import ext
    bs = bench.MODELS["lstman4"][2]
    pool = [tuple(t.cuda() for t in bench.make_batch("lstman4", i, 0, bs, 128)) for i in range(4)]
    arms, it, last, peak = {}, {}, {}, {}

    def run(k, n):
        for _ in range(n):
            last[k] = _step(arms[k], pool[it[k] % len(pool)])
            it[k] += 1

    for k, (autocast, fused) in ARMS.items():
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        n0 = ext.LAUNCH_COUNT.get("lstm_forward", 0)
        arms[k], it[k] = _trainer(autocast, fused, a.dense_warmup), 0
        run(k, a.dense_warmup + max(a.warmup, len(pool)))
        torch.cuda.synchronize()
        peak[k] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        launches = ext.LAUNCH_COUNT.get("lstm_forward", 0) - n0
        assert (launches > 0) == fused, "%s: lstm_forward ran %d times" % (k, launches)
    times = {k: [] for k in arms}
    for _ in range(a.runs):
        for k in arms:
            run(k, a.warmup)
            times[k].append(_timed(lambda: run(k, 1), a.steps))
    losses = {k: float(v.detach()) for k, v in last.items()}
    for k, tr in arms.items():
        assert all(torch.isfinite(p).all() for p in tr.net.parameters()), k
        tr.close()
    del arms
    torch.cuda.empty_cache()
    return {"steps": a.steps, "last_loss": losses, "peak_allocated_mib": peak,
            "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                            for k, v in times.items()}}


def op_times(iters: int) -> dict:
    """µs per eager forward + backward; the three forms alternate in two rounds, the second is kept."""
    import torch
    from oktopk_b200.models.deepspeech import BatchRNN
    from oktopk_b200.ops import ext
    torch.manual_seed(0)
    forms = {"bidir_stock": BatchRNN(800, 800, bidirectional=True).cuda().train(),
             "bidir_fused": BatchRNN(800, 800, bidirectional=True, fuse=True, fuse_bidirectional=True).cuda().train(),
             "onedir_fused": BatchRNN(800, 800, fuse=True).cuda().train()}
    out = {}
    for T in OP_T:
        x32 = torch.randn(T, 2, 800, device="cuda")
        dy = torch.randn(T, 2, 800, device="cuda")
        lens = torch.full((2,), T, dtype=torch.int32)
        dev_lens = lens.cuda()                             # DeepSpeech copies the lengths once for all five layers
        res = {}
        for _ in range(2):
            for k, layer in forms.items():
                x = x32.detach().clone().requires_grad_(True)

                def call():
                    y = layer(x, lens, dev_lens)
                    torch.autograd.grad(y, [x] + list(layer.parameters()), dy)

                n0 = ext.LAUNCH_COUNT.get("lstm_forward", 0)
                for _ in range(3):
                    call()
                assert (ext.LAUNCH_COUNT.get("lstm_forward", 0) > n0) == (k != "bidir_stock"), k
                torch.cuda.synchronize()
                res[k] = _timed(call, iters) * 1e3
        out[T] = res
    return out


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=4)
    p.add_argument("--op-iters", type=int, default=20)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_lstm_bidir.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    steps = step_times(a)
    op = op_times(a.op_iters)
    res = {"card": card, "card_after": _card(), "runs": a.runs, "lstman4_bidirectional": steps,
           "batchrnn_fwd_bwd_us": op}
    print("card", card)
    for k, v in steps["ms_per_step"].items():
        print("lstman4 bidirectional %-10s ms/step median %.3f  range %.3f-%.3f  last loss %.4f  peak %.0f MiB" % (
            k, v["median"], v["min"], v["max"], steps["last_loss"][k], steps["peak_allocated_mib"][k]))
    for T, r in op.items():
        print("BatchRNN(800) fwd+bwd N=2 T'=%d us: %s" % (T, "  ".join("%s %.1f" % kv for kv in r.items())))
    print("card after", res["card_after"])
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
