#!/usr/bin/env python
"""Where an LSTM-AN4 step spends its time, and the fused LSTM recurrence (``create_net(29, "lstman4", fuse_lstm=True)``,
``--fused-lstm``) against stock cuDNN.

    python scripts/bench_lstm.py [--out profiles/lstm] [--steps 30] [--runs 5] [--op-iters 20]

The workload is bench.py's LSTM-AN4 configuration (``bench.MODELS["lstman4"]``, ``bench.make_batch``: 2 utterances whose
lengths give T' = 48 - 198 frames after the convolutions, the lstm_an4 preset, Ok-Topk at density 0.001, SGD with the
reduced gradient clipped at 400).  AN4 steps are eager (their length varies), as in bench.py.  The dense warm-up is
shortened to ``--dense-warmup`` steps: only the sparse phase is timed.  Three parts:

1. ``profile_stock``: a ``torch.profiler`` trace of ``--profile-steps`` stock steps, written to ``<out>/``, and the
   device time of the recurrence in it: the kernels of cuDNN's RNN forward and backward ops and of the packing around
   them, against the time of all device-side activities (kernels, copies, memsets) of the profiled steps.
2. Step time, stock against fused: the two Trainers alternate ``--runs`` times, ``--steps`` steps each, timed with CUDA
   events; median (range) ms/step.
3. One ``BatchRNN`` (batch norm + ``nn.LSTM(800, 800)``) forward + backward at N = 2 and T' in {48, 123, 198}, both
   utterances of full length, stock cuDNN against the fused kernels, eager, µs per call (the lengths already on the
   device, as DeepSpeech hands them to its layers).

Prints the card, its power limit and SM clock before and after, and one JSON line.
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
# profiler op names of the recurrence on the stock path (cuDNN's fp32 RNN, both passes) and of the packing around it
RNN_OPS = ("aten::_cudnn_rnn", "aten::_cudnn_rnn_backward")
PACK_OPS = ("aten::_pack_padded_sequence", "aten::_pad_packed_sequence", "aten::_pack_padded_sequence_backward")


def _trainer(fused: bool, dense_warmup: int):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=dense_warmup)
    return Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                   t_total=100000, warmup=0.1, seed=0, model_kwargs={"fuse_lstm": fused})


def _pool(dev):
    bs = bench.MODELS["lstman4"][2]
    return [tuple(t.to(dev) for t in bench.make_batch("lstman4", i, 0, bs, 128)) for i in range(4)]


def _step(tr, batch):
    tr.net.train()
    tr.optimizer.zero_grad()
    loss, _ = tr._forward_loss(batch)
    loss.backward()
    tr.update_model()
    return loss


def _dev_us(evt) -> float:
    return float(getattr(evt, "device_time_total", None) or getattr(evt, "cuda_time_total", 0.0))


def _self_dev_us(evt) -> float:
    return float(getattr(evt, "self_device_time_total", None) or getattr(evt, "self_cuda_time_total", 0.0))


def profile_stock(out: str, dense_warmup: int = 4, warmup: int = 8, steps: int = 4) -> dict:
    """Profile ``steps`` stock steps (after ``dense_warmup + warmup`` unprofiled ones) and attribute device time."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(out, exist_ok=True)
    tr = _trainer(False, dense_warmup)
    pool = _pool(tr.device)
    for i in range(dense_warmup + warmup):
        _step(tr, pool[i % len(pool)])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            _step(tr, pool[i % len(pool)])
        torch.cuda.synchronize()
    trace = os.path.join(out, "lstman4_stock_step.pt.trace.json")
    prof.export_chrome_trace(trace)
    avg = prof.key_averages()
    # Device time is the device-side rows only (kernels, copies, memsets; no user annotations), as torch's own table sums
    # it: an aten op's row also carries its kernels' time as self device time, so summing every row counts it twice.
    # An op's device_time_total is the time of the kernels it launched.
    dev = [e for e in avg if e.device_type == DeviceType.CUDA and not getattr(e, "is_user_annotation", False)]
    total = sum(_self_dev_us(e) for e in dev)
    rnn = {e.key: _dev_us(e) / steps for e in avg if e.key in RNN_OPS}
    pack = {e.key: _dev_us(e) / steps for e in avg if e.key in PACK_OPS}
    top = sorted(dev, key=_self_dev_us, reverse=True)[:15]
    res = {"trace": trace, "steps": steps, "device_us_per_step": total / steps,
           "rnn_device_us_per_step": rnn, "pack_device_us_per_step": pack,
           "rnn_share_of_device_time": sum(rnn.values()) * steps / total if total else None,
           "device_activities_per_step": sum(e.count for e in dev) / steps,
           "top_device_us_per_step": {e.key: _self_dev_us(e) / steps for e in top}}
    tr.close()
    del tr
    torch.cuda.empty_cache()
    return res


def step_times(a) -> dict:
    import torch
    from oktopk_b200.ops import ext
    arms = {"stock": _trainer(False, a.dense_warmup), "fused": _trainer(True, a.dense_warmup)}
    pool = _pool(arms["stock"].device)
    it = {k: 0 for k in arms}
    last = {}

    def run(k, n):
        for _ in range(n):
            last[k] = _step(arms[k], pool[it[k] % len(pool)])
            it[k] += 1

    n0 = ext.LAUNCH_COUNT.get("lstm_forward", 0)
    for k in arms:
        run(k, a.dense_warmup + a.warmup)
    torch.cuda.synchronize()
    assert ext.LAUNCH_COUNT.get("lstm_forward", 0) > n0, "the fused arm did not run lstm_forward"
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
    losses = {k: float(v.detach()) for k, v in last.items()}
    for k, tr in arms.items():
        assert all(torch.isfinite(p).all() for p in tr.net.parameters()), k
        tr.close()
    del arms
    torch.cuda.empty_cache()
    return {"steps": a.steps, "last_loss": losses,
            "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                            for k, v in times.items()}}


def op_times(iters: int) -> dict:
    """µs per forward + backward of one BatchRNN(800, 800) at N = 2, stock and fused, eager."""
    import torch
    from oktopk_b200.models.deepspeech import BatchRNN
    torch.manual_seed(0)
    layer = BatchRNN(800, 800).cuda().train()
    out = {}
    for T in OP_T:
        x = torch.randn(T, 2, 800, device="cuda", requires_grad=True)
        lens = torch.full((2,), T, dtype=torch.int32)
        dev_lens = lens.cuda()                             # DeepSpeech copies the lengths once for all five layers
        dy = torch.randn(T, 2, 800, device="cuda")
        res = {}
        for fused in (False, True, False, True):            # alternated, the second round is kept
            layer.fuse = fused

            def call():
                torch.autograd.grad(layer(x, lens, dev_lens), [x] + list(layer.parameters()), dy)

            for _ in range(3):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            res["fused_us" if fused else "stock_us"] = e0.elapsed_time(e1) * 1e3 / iters
        out[T] = res
    return out


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--out", type=str, default=os.path.join(ROOT, "profiles", "lstm"))
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=4)
    p.add_argument("--profile-steps", type=int, default=4)
    p.add_argument("--op-iters", type=int, default=20)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_lstm.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    prof = profile_stock(a.out, a.dense_warmup, a.warmup, a.profile_steps)
    steps = step_times(a)
    op = op_times(a.op_iters)
    res = {"card": card, "card_after": _card(), "runs": a.runs, "profile_stock": prof, "lstman4": steps,
           "batchrnn_fwd_bwd": op}
    print("card", card)
    print("stock step profile: %.0f us device time per step, recurrence %s, packing %s (%.1f %% of device time), "
          "%.0f device activities per step" % (
              prof["device_us_per_step"], {k: round(v) for k, v in prof["rnn_device_us_per_step"].items()},
              {k: round(v) for k, v in prof["pack_device_us_per_step"].items()},
              100 * (prof["rnn_share_of_device_time"] or 0), prof["device_activities_per_step"]))
    for k, v in steps["ms_per_step"].items():
        print("lstman4 %-5s ms/step median %.3f  range %.3f-%.3f  last loss %.4f" % (
            k, v["median"], v["min"], v["max"], steps["last_loss"][k]))
    for T, r in op.items():
        print("BatchRNN(800) fwd+bwd N=2 T'=%d: stock %8.1f us  fused %8.1f us" % (T, r["stock_us"], r["fused_us"]))
    print("card after", res["card_after"])
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
