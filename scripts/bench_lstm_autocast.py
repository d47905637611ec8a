#!/usr/bin/env python
"""The fused LSTM recurrence under bf16 / fp16 autocast (``fuse_lstm=True, fuse_lstm_autocast=True``,
``--fused-lstm --fused-lstm-autocast``) against the stock layers under the same autocast, and against the fp32 fused
path.

    python scripts/bench_lstm_autocast.py [--steps 30] [--runs 5] [--op-iters 20]

The workload is bench.py's LSTM-AN4 configuration, as in ``scripts/bench_lstm.py``: 2 utterances (T' = 48 - 198 frames
after the convolutions), the lstm_an4 preset, Ok-Topk at density 0.001, eager steps, the dense warm-up shortened to
``--dense-warmup`` steps.  fp16 arms run with dynamic loss scaling.  Three parts:

1. Step time of five arms: fp32 fused, bf16 stock, bf16 fused, fp16 stock, fp16 fused.  The Trainers alternate ``--runs``
   times, ``--steps`` steps each, timed with CUDA events; median (range) ms/step, each arm's last loss, and its peak
   allocated memory over construction and warm-up (all four batches of the pool), above what was allocated before it.
2. One ``BatchRNN`` (batch norm + ``nn.LSTM(800, 800)``) forward + backward at N = 2 and T' in {48, 123, 198}, both
   utterances of full length, in the same five forms, eager, µs per call; the input is in the autocast type, as the
   previous layer hands it over.
3. The PTB-sized layer, ``BatchRNN(1500, 1500)`` at N = 20, T = 35, under bf16 autocast, fused against stock (the fp32
   kernels cannot hold its W_hh in shared memory).

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
ARMS = {"fp32_fused": (None, True), "bf16_stock": ("bf16", False), "bf16_fused": ("bf16", True),
        "fp16_stock": ("fp16", False), "fp16_fused": ("fp16", True)}


def _trainer(autocast, fused: bool, dense_warmup: int):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=dense_warmup)
    return Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                   t_total=100000, warmup=0.1, seed=0, autocast=autocast,
                   loss_scale=okt.LossScale() if autocast == "fp16" else None,
                   model_kwargs={"fuse_lstm": fused, "fuse_lstm_autocast": fused and autocast is not None})


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
    arms, it, last, peak, launches = {}, {}, {}, {}, {}

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
        launches[k] = ext.LAUNCH_COUNT.get("lstm_forward", 0) - n0
        assert (launches[k] > 0) == fused, "%s: lstm_forward ran %d times" % (k, launches[k])
    times = {k: [] for k in arms}
    for _ in range(a.runs):
        for k in arms:
            run(k, a.warmup)
            times[k].append(_timed(lambda: run(k, 1), a.steps))
    losses = {k: float(v.detach()) for k, v in last.items()}
    scales = {k: tr.optimizer.loss_scale_state() for k, tr in arms.items() if tr.loss_scale is not None}
    for k, tr in arms.items():
        assert all(torch.isfinite(p).all() for p in tr.net.parameters()), k
        tr.close()
    del arms
    torch.cuda.empty_cache()
    return {"steps": a.steps, "last_loss": losses, "peak_allocated_mib": peak, "loss_scale": scales,
            "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                            for k, v in times.items()}}


def _layer_times(layer, x32, lens, dy32, forms, iters: int) -> dict:
    """µs per eager forward + backward of ``layer`` in each of ``forms``; two alternated rounds, the second is kept."""
    import torch
    dts = {None: None, "bf16": torch.bfloat16, "fp16": torch.float16}
    dev_lens = lens.cuda()                                 # DeepSpeech copies the lengths once for all five layers
    res = {}
    for _ in range(2):
        for k in forms:
            autocast, fused = ARMS[k]
            dt = dts[autocast]
            layer.fuse, layer.fuse_autocast = fused, fused and dt is not None
            x = x32.detach().to(dt or torch.float32).requires_grad_(True)
            dy = dy32.to(dt or torch.float32)

            def call():
                with torch.autocast("cuda", dtype=dt, enabled=dt is not None):
                    y = layer(x, lens, dev_lens)
                torch.autograd.grad(y, [x] + list(layer.parameters()), dy)

            for _ in range(3):
                call()
            torch.cuda.synchronize()
            res[k] = _timed(call, iters) * 1e3
    return res


def op_times(iters: int) -> dict:
    import torch
    from oktopk_b200.models.deepspeech import BatchRNN
    torch.manual_seed(0)
    layer = BatchRNN(800, 800).cuda().train()
    out = {}
    for T in OP_T:
        out[T] = _layer_times(layer, torch.randn(T, 2, 800, device="cuda"), torch.full((2,), T, dtype=torch.int32),
                              torch.randn(T, 2, 800, device="cuda"), list(ARMS), iters)
    return out


def ptb_layer_times(iters: int) -> dict:
    import torch
    from oktopk_b200.models.deepspeech import BatchRNN
    torch.manual_seed(0)
    T, N, H = 35, 20, 1500
    layer = BatchRNN(H, H).cuda().train()
    return _layer_times(layer, torch.randn(T, N, H, device="cuda"), torch.full((N,), T, dtype=torch.int32),
                        torch.randn(T, N, H, device="cuda"), ["bf16_stock", "bf16_fused"], iters)


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
        print("bench_lstm_autocast.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    steps = step_times(a)
    op = op_times(a.op_iters)
    ptb = ptb_layer_times(a.op_iters)
    res = {"card": card, "card_after": _card(), "runs": a.runs, "lstman4": steps, "batchrnn_fwd_bwd_us": op,
           "batchrnn_1500_n20_t35_us": ptb}
    print("card", card)
    for k, v in steps["ms_per_step"].items():
        print("lstman4 %-10s ms/step median %.3f  range %.3f-%.3f  last loss %.4f  peak %.0f MiB" % (
            k, v["median"], v["min"], v["max"], steps["last_loss"][k], steps["peak_allocated_mib"][k]))
    for T, r in op.items():
        print("BatchRNN(800) fwd+bwd N=2 T'=%d us: %s" % (T, "  ".join("%s %.1f" % kv for kv in r.items())))
    print("BatchRNN(1500) fwd+bwd N=20 T=35 us: %s" % "  ".join("%s %.1f" % kv for kv in ptb.items()))
    print("card after", res["card_after"])
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
