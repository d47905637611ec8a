#!/usr/bin/env python
"""The fused softmax + CTC loss (``ops/fused_ctc``, ``create_net(29, "lstman4", fuse_ctc=True)``, ``--fused-ctc``) against
DeepSpeech's stock loss (``log_softmax`` + ``.float()`` + ``nn.CTCLoss``), three ways.

    python scripts/bench_ctc.py [--steps 30] [--runs 5] [--op-iters 200] [--profile-steps 10]

1. The op alone, forward + backward, µs per call from CUDA events over ``--op-iters`` eager calls: N = 2 utterances,
   T' in {48, 123, 198} frames (bench.py's range), Ln in {8, 20, 33} labels (its transcript lengths), fp32 and bf16
   logits.  The inputs are what the trainer hands the loss: int32 targets and target lengths on the device, the input
   lengths on the host.
2. The LSTM-AN4 step (``bench.MODELS["lstman4"]``, ``bench.make_batch``), stock loss against fused loss, ``fuse_lstm=True``
   in both arms so that only the loss differs: ``--runs`` alternating runs of ``--steps`` steps, median (range) ms/step,
   in fp32 and in bf16 autocast with ``fuse_lstm_autocast``.  The dense warm-up is cut to 2 steps; the sparse phase is
   timed.
3. A ``torch.profiler`` run of its own per arm over ``--profile-steps`` steps: the loss's kernels' share of device time
   (kernels whose name holds "ctc" or "softmax"; the autocast casts in front of the stock loss are not counted) and the
   device-to-host copies and stream / device synchronisations per step.

Prints the card, its power limit and SM clock, before and after, and one JSON line.
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

PRECISIONS = ("fp32", "bf16")
OP_T = (48, 123, 198)
OP_L = (8, 20, 33)


def _op_us(dtype, T, L, iters):
    """µs per forward + backward, stock and fused, at N = 2 (both utterances T frames, L labels)."""
    import torch
    import torch.nn.functional as F
    from oktopk_b200.ops.fused_ctc import ctc_loss
    N, C = 2, 29
    g = torch.Generator("cuda").manual_seed(T * 100 + L)
    x = (torch.randn(T, N, C, device="cuda", generator=g) * 2).to(dtype).requires_grad_(True)
    targets = torch.randint(1, C, (N * L,), device="cuda", generator=g, dtype=torch.int32)
    tn = torch.full((N,), T, dtype=torch.int32)                  # host, as DeepSpeech returns it
    ln = torch.full((N,), L, dtype=torch.int32, device="cuda")

    def stock():
        logp = F.log_softmax(x, dim=-1)
        loss = F.ctc_loss(logp.float(), targets.long(), tn.to("cuda").long(), ln.long(), blank=0, reduction="sum",
                          zero_infinity=True)
        torch.autograd.grad(loss, x)

    def fused():
        torch.autograd.grad(ctc_loss(x, targets, tn, ln), x)

    out = {}
    for name, fn in (("stock", stock), ("fused", fused)):
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) * 1e3 / iters
    return out


def _trainer(precision, fuse):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    autocast = None if precision == "fp32" else precision
    cfg = okt.preset(preset, density=0.001, warmup_iters=2)
    return Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                   t_total=100000, warmup=0.1, seed=0, autocast=autocast,
                   model_kwargs={"fuse_lstm": True, "fuse_lstm_autocast": autocast is not None, "fuse_ctc": fuse})


def _steps(tr, pool, it, n):
    loss = None
    for _ in range(n):
        tr.net.train()
        tr.optimizer.zero_grad()
        loss, _ = tr._forward_loss(pool[it[0] % len(pool)])
        tr.backward(loss)
        tr.update_model()
        it[0] += 1
    return loss


def _step_times(precision, a):
    import torch
    bs = bench.MODELS["lstman4"][2]
    pool = [tuple(t.cuda() for t in bench.make_batch("lstman4", i, 0, bs, 128)) for i in range(8)]
    arms = {k: (_trainer(precision, k == "fused"), [0]) for k in ("stock", "fused")}
    for tr, it in arms.values():
        _steps(tr, pool, it, 2 + a.warmup)
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    loss = {}
    for _ in range(a.runs):
        for k, (tr, it) in arms.items():
            _steps(tr, pool, it, 3)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            loss[k] = _steps(tr, pool, it, a.steps)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / a.steps)
    prof = {k: _profile(tr, pool, it, a.profile_steps) for k, (tr, it) in arms.items()}
    for tr, _ in arms.values():
        assert all(torch.isfinite(p).all() for p in tr.net.parameters())
        tr.close()
    return {"ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                            for k, v in times.items()},
            "last_loss": {k: float(v) for k, v in loss.items()}, "profile": prof}


def _profile(tr, pool, it, n):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
        _steps(tr, pool, it, n)
        torch.cuda.synchronize()
    total = loss = 0.0
    d2h = syncs = 0
    for e in p.events():
        name = e.name
        dev_us = getattr(e, "device_time", None)
        if dev_us is None:
            dev_us = getattr(e, "cuda_time", 0.0)
        if e.device_type == torch.autograd.DeviceType.CUDA:
            if "Memcpy DtoH" in name:
                d2h += 1
            if not name.startswith("Memcpy") and not name.startswith("Memset"):
                total += dev_us
                if "ctc" in name.lower() or "softmax" in name.lower():
                    loss += dev_us
        elif name in ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaEventSynchronize"):
            syncs += 1
    return {"kernel_us_per_step": total / n, "loss_kernel_us_per_step": loss / n,
            "loss_share": loss / total if total else None, "d2h_copies_per_step": d2h / n,
            "host_syncs_per_step": syncs / n}


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--op-iters", type=int, default=200)
    p.add_argument("--profile-steps", type=int, default=10)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_ctc.py needs a GPU", file=sys.stderr)
        return 2
    from oktopk_b200.ops import ext
    ext.require()
    torch.cuda.set_device(0)
    card = _card()
    op = {}
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        op[name] = {"T%d_L%d" % (T, L): _op_us(dt, T, L, a.op_iters) for T in OP_T for L in OP_L}
    steps = {prec: _step_times(prec, a) for prec in PRECISIONS}
    out = {"card": card, "card_after": _card(), "op_us": op, "lstman4": steps}
    print("card", card)
    for name, rows in op.items():
        for k, r in rows.items():
            print("ctc fwd+bwd %s N=2 %-9s stock %7.1f us  fused %7.1f us" % (name, k, r["stock"], r["fused"]))
    for prec, r in steps.items():
        for k, v in r["ms_per_step"].items():
            pr = r["profile"][k]
            print("lstman4 %s %-5s ms/step median %.3f  range %.3f-%.3f  loss %.4f  loss kernels %.1f us/step "
                  "(%.1f %% of kernel time)  D2H copies %.1f  syncs %.1f per step" % (
                      prec, k, v["median"], v["min"], v["max"], r["last_loss"][k], pr["loss_kernel_us_per_step"],
                      100 * (pr["loss_share"] or 0), pr["d2h_copies_per_step"], pr["host_syncs_per_step"]))
    print("card after", out["card_after"])
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
