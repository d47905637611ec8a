#!/usr/bin/env python
"""The PTB language model's fused LSTM (``PTBLSTM(fuse_lstm=True, fuse_xent=True)``, ``--fused-lstm-lm --fused-xent``)
against the stock cuDNN layer under bf16 / fp16 autocast, and in fp32 (``fuse_lstm_fp32=True``,
``--fused-lstm-lm-fp32 --fused-xent``).

    python scripts/bench_ptb.py [--steps 20] [--runs 5] [--op-iters 20]

Four parts:

1. Step time on the PTB workload of ``scripts/exp_configs/lstm.conf``: ``Trainer`` on ``SyntheticPTB`` (N = 20, T = 35,
   the hidden state carried across batches), SGD lr 22, gradient clip 0.25, Ok-Topk at density 0.02, eager steps, the
   dense warm-up shortened to ``--dense-warmup`` steps.  Six arms: fp32 stock and fused, bf16 stock and fused, fp16
   (dynamic loss scaling) stock and fused.  The Trainers alternate ``--runs`` times, ``--steps`` steps each, timed with
   CUDA events; median (range) ms/step, each arm's last loss, and its peak allocated memory over construction and
   warm-up above what was allocated before it.  The fp32 arms run with torch's default TF32 switches, as the Trainer
   does: cuDNN's RNN in TF32, matmuls in fp32.
2. One ``nn.LSTM(1500, 1500)`` forward + backward at (T, N) = (35, 20) under bf16 with a non-zero (h0, c0), µs per
   call: stock, today's one-layer 16-bit kernels (``lstm_layer(..., autocast=True)``, which start from a zero state),
   and the stacked-layer kernels (``lstm_stack``).
3. The same layer in fp32: stock with ``cudnn.allow_tf32`` on (torch's default) and off, and the fp32 stacked-layer
   kernels (``lstm_stack(..., fp32=True)``), next to the bytes of W_hh their geometry reads from L2 per step.
4. µs per timestep and pass of each form, from the forward alone and forward + backward at T = 35 and T = 70.

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

from scripts.bench_bf16 import _card  # noqa: E402

N, T, H = 20, 35, 1500
# arm -> (autocast, fused)
ARMS = {"fp32_stock": (None, False), "fp32_fused": (None, True), "bf16_stock": ("bf16", False),
        "bf16_fused": ("bf16", True), "fp16_stock": ("fp16", False), "fp16_fused": ("fp16", True)}


def _trainer(autocast, fused: bool, dense_warmup: int):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    cfg = okt.preset("lstm_an4", density=0.02, warmup_iters=dense_warmup)
    return Trainer(dnn="lstm", dataset="ptb", batch_size=N, lr=22.0, compressor="oktopk", density=0.02, cfg=cfg,
                   norm_clip=0.25, seed=0, autocast=autocast,
                   loss_scale=okt.LossScale() if autocast == "fp16" else None,
                   model_kwargs={"fuse_lstm": fused, "fuse_xent": fused, "fuse_lstm_fp32": fused and autocast is None})


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


def _launches():
    from oktopk_b200.ops import ext
    return ext.LAUNCH_COUNT.get("lstm_seq_forward", 0)


def step_times(a) -> dict:
    import torch
    from oktopk_b200.train.data import SyntheticPTB
    ds = SyntheticPTB(batch_size=N, num_steps=T)
    pool = []
    for b in range(8):                                   # consecutive [N, T] batches, as the loader hands them over
        rows = [ds[b * N + i] for i in range(N)]
        pool.append((torch.stack([r[0] for r in rows]).cuda(), torch.stack([r[1] for r in rows]).cuda()))
    arms, it, last, peak = {}, {}, {}, {}

    def run(k, n):
        for _ in range(n):
            last[k] = _step(arms[k], pool[it[k] % len(pool)])
            it[k] += 1

    for k, (autocast, fused) in ARMS.items():
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        n0 = _launches()
        arms[k], it[k] = _trainer(autocast, fused, a.dense_warmup), 0
        run(k, a.dense_warmup + a.warmup)
        torch.cuda.synchronize()
        peak[k] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        assert (_launches() > n0) == fused, k
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


def _form_times(rnn, forms: dict, counter: dict, dt, iters: int) -> dict:
    """µs per eager call of each form of ``rnn`` at N = 20: the forward alone and forward + backward, at T = 35 and 70,
    under ``dt`` autocast (None: fp32); the forms alternate in two rounds and the second is kept.  A form is
    (fn(x), tf32), tf32 the ``cudnn.allow_tf32`` it runs with; ``counter[k]`` is the launch counter it must move."""
    import torch
    from oktopk_b200.ops import ext
    out = {}
    for t in (T, 2 * T):
        x32 = torch.randn(t, N, H, device="cuda")
        dy = torch.randn(t, N, H, device="cuda", dtype=dt or torch.float32)
        res = {}
        for _ in range(2):
            for k, (f, tf32) in forms.items():
                x = x32.detach().clone().requires_grad_(True)

                def fwd():
                    with torch.autocast("cuda", dtype=dt, enabled=dt is not None), torch.no_grad():
                        f(x)

                def fwd_bwd():
                    with torch.autocast("cuda", dtype=dt, enabled=dt is not None):
                        y = f(x)
                    torch.autograd.grad(y, [x] + list(rnn.parameters()), dy.to(y.dtype))

                old = torch.backends.cudnn.allow_tf32
                torch.backends.cudnn.allow_tf32 = tf32
                n0 = {c: ext.LAUNCH_COUNT.get(c, 0) for c in ("lstm_forward", "lstm_seq_forward")}
                for _ in range(3):
                    fwd_bwd()
                ran = {c for c in n0 if ext.LAUNCH_COUNT.get(c, 0) > n0[c]}
                assert ran == ({counter[k]} if counter[k] else set()), (k, ran)
                torch.cuda.synchronize()
                res[k] = {"fwd": _timed(fwd, iters) * 1e3, "fwd_bwd": _timed(fwd_bwd, iters) * 1e3}
                torch.backends.cudnn.allow_tf32 = old
        out[t] = res
    per_step = {}
    for k in forms:
        a, b = out[T][k], out[2 * T][k]
        f = (b["fwd"] - a["fwd"]) / T
        bw = ((b["fwd_bwd"] - b["fwd"]) - (a["fwd_bwd"] - a["fwd"])) / T
        per_step[k] = {"fwd": f, "bwd": bw}
    return {"us": out, "us_per_step": per_step}


def layer_times(iters: int) -> dict:
    """One nn.LSTM(1500, 1500) with a carried state under bf16 autocast: stock, the one-layer 16-bit kernels and the
    stacked-layer kernels."""
    import torch
    import torch.nn as nn
    from oktopk_b200.ops.fused_lstm import lstm_layer, lstm_stack
    torch.manual_seed(0)
    rnn = nn.LSTM(H, H).cuda().train()
    h0 = 0.5 * torch.randn(1, N, H, device="cuda")
    c0 = torch.randn(1, N, H, device="cuda")
    lens = {t: torch.full((N,), t, dtype=torch.int32) for t in (T, 2 * T)}
    forms = {"stock": (lambda x: rnn(x, (h0, c0))[0], True),
             "lstm_layer_16bit": (lambda x: lstm_layer(x, lens[x.size(0)], rnn, autocast=True), True),
             "lstm_stack": (lambda x: lstm_stack(x, (h0, c0), rnn, 0.0, True)[0], True)}
    counter = {"stock": None, "lstm_layer_16bit": "lstm_forward", "lstm_stack": "lstm_seq_forward"}
    return _form_times(rnn, forms, counter, torch.bfloat16, iters)


def layer_times_fp32(iters: int) -> dict:
    """The same layer in fp32: stock cuDNN with TF32 on (torch's default) and off, and the fp32 stacked-layer kernels,
    with the bytes of W_hh their geometry reads from L2 per step."""
    import torch
    import torch.nn as nn
    from oktopk_b200.ops.fused_lstm import lstm_seq_f32_geometry, lstm_stack
    torch.manual_seed(0)
    rnn = nn.LSTM(H, H).cuda().train()
    h0 = 0.5 * torch.randn(1, N, H, device="cuda")
    c0 = torch.randn(1, N, H, device="cuda")
    forms = {"fp32_stock_tf32": (lambda x: rnn(x, (h0, c0))[0], True),
             "fp32_stock": (lambda x: rnn(x, (h0, c0))[0], False),
             "fp32_fused": (lambda x: lstm_stack(x, (h0, c0), rnn, 0.0, True, fp32=True)[0], False)}
    counter = {"fp32_stock_tf32": None, "fp32_stock": None, "fp32_fused": "lstm_seq_forward"}
    res = _form_times(rnn, forms, counter, None, iters)
    p = torch.cuda.get_device_properties(0)
    res["geometry"] = lstm_seq_f32_geometry(H, N, p.multi_processor_count, p.shared_memory_per_block_optin)._asdict()
    return res


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=2)
    p.add_argument("--op-iters", type=int, default=20)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_ptb.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    torch.backends.cudnn.benchmark = False
    steps = step_times(a)
    layer = layer_times(a.op_iters)
    layer32 = layer_times_fp32(a.op_iters)
    res = {"card": card, "card_after": _card(), "runs": a.runs, "ptb_step": steps, "lstm1500_layer": layer,
           "lstm1500_layer_fp32": layer32}
    print("card", card)
    for k, v in steps["ms_per_step"].items():
        print("PTB %-10s ms/step median %.3f  range %.3f-%.3f  last loss %.4f  peak %.0f MiB" % (
            k, v["median"], v["min"], v["max"], steps["last_loss"][k], steps["peak_allocated_mib"][k]))
    for t, r in layer["us"].items():
        print("nn.LSTM(1500) bf16 N=20 T=%d us: %s" % (t, "  ".join(
            "%s fwd %.1f fwd+bwd %.1f" % (k, v["fwd"], v["fwd_bwd"]) for k, v in r.items())))
    print("us per timestep: %s" % "  ".join("%s fwd %.1f bwd %.1f" % (k, v["fwd"], v["bwd"])
                                            for k, v in layer["us_per_step"].items()))
    for t, r in layer32["us"].items():
        print("nn.LSTM(1500) fp32 N=20 T=%d us: %s" % (t, "  ".join(
            "%s fwd %.1f fwd+bwd %.1f" % (k, v["fwd"], v["fwd_bwd"]) for k, v in r.items())))
    g = layer32["geometry"]
    print("fp32 us per timestep: %s   (fused: W_hh from L2 per step fwd %.2f MB, bwd %.2f MB; rows on chip %d/%d fwd, "
          "%d/%d bwd)" % ("  ".join("%s fwd %.1f bwd %.1f" % (k, v["fwd"], v["bwd"])
                                   for k, v in layer32["us_per_step"].items()),
                         g["fwd_l2_bytes"] / 1e6, g["bwd_l2_bytes"] / 1e6, g["fwd_r_on"], 4 * g["units"],
                         g["bwd_r_on"], g["units"]))
    print("card after", res["card_after"])
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
