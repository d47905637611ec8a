#!/usr/bin/env python
"""The channel-sliced fused batch-norm kernels against the cooperative ones: per layer, and in the VGG-16 step.

    python scripts/bench_bn_sliced.py [--steps 200] [--warmup 20] [--runs 5] [--kernel-iters 200] [--check-steps 30]

Both kernel families live in csrc/bnrelu.cu.  A call with ``fused_bn.MAX_CTAS = 0`` takes the sliced kernels where
``bn_sliced(M, C, W)`` holds; ``MAX_CTAS = 1 << 30`` caps nothing and so runs the cooperative kernels exactly as they run
without the sliced ones.  Three parts, all in one process, the arms alternated within every round:

  1. kernel level: ``bn_forward`` + ``bn_backward`` at the 13 VGG-16 layer shapes (16 images, the pool folded in where a
     block ends), each pair captured ``--kernel-iters`` times in one CUDA graph and timed with CUDA events;
  2. step level: bench.py's VGG-16 workload (as scripts/bench_bf16.py builds it) with whole-step CUDA graphs, one
     optimizer and graph set per arm, in fp32 and under bf16 autocast;
  3. results: loss and updated parameters of the sliced and the cooperative arm after the same seeded steps, beside the
     difference between two cooperative arms (the step's own run-to-run difference).

Prints the card, its power limit and SM clock, then one JSON line.  Needs a GPU: without one it exits with an error.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]
os.environ.setdefault("OMP_NUM_THREADS", "1")

import bench  # noqa: E402  (make_batch, MODELS: the bench workload definition)
from bench_bf16 import VGG16_LAYERS, _arm, _card  # noqa: E402

COOPERATIVE = 1 << 30
CAP = {"sliced": 0, "coop": COOPERATIVE, "coop2": COOPERATIVE}


def _mmm(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def _pair_graph(C, shape, pooled, max_ctas, iters):
    """A CUDA graph of ``iters`` bn_forward + bn_backward pairs at one layer shape (fp32)."""
    import torch
    N, Ch, H, W = shape
    M = N * H * W
    cl = torch.channels_last
    x = torch.randn(shape, device="cuda").contiguous(memory_format=cl)
    ys = (N, Ch, H // 2, W // 2) if pooled else shape
    y = torch.empty(ys, device="cuda").contiguous(memory_format=cl)
    dy = torch.randn(ys, device="cuda").contiguous(memory_format=cl)
    dx = torch.empty_like(x)
    arg = torch.empty(y.numel() if pooled else 1, dtype=torch.uint8, device="cuda")
    rows = C.bn_tile_rows(M, Ch)
    partial = torch.empty((M + rows - 1) // rows * 2 * Ch, device="cuda")
    gamma, beta = torch.ones(Ch, device="cuda"), torch.zeros(Ch, device="cuda")
    rm, rv = torch.zeros(Ch, device="cuda"), torch.ones(Ch, device="cuda")
    nbt = torch.zeros((), dtype=torch.long, device="cuda")
    stats, dgb = torch.empty(2 * Ch, device="cuda"), torch.empty(2 * Ch, device="cuda")
    ap, Wp = arg.data_ptr() if pooled else 0, W if pooled else 0
    keep = (x, y, dy, dx, arg, partial, gamma, beta, rm, rv, nbt, stats, dgb)

    def pair(s):
        C.bn_forward(x.data_ptr(), y.data_ptr(), ap, partial.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 0,
                     stats.data_ptr(), stats.data_ptr() + 4 * Ch, rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(), 0.1, 1e-5, 1,
                     M, Ch, Wp, 1023, max_ctas, s, 0)
        C.bn_backward(x.data_ptr(), dy.data_ptr(), ap, dx.data_ptr(), partial.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                      stats.data_ptr(), stats.data_ptr() + 4 * Ch, dgb.data_ptr(), dgb.data_ptr() + 4 * Ch, 1, M, Ch, Wp,
                      1023, max_ctas, s, 0)

    for _ in range(3):
        pair(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(iters):
            pair(torch.cuda.current_stream().cuda_stream)
    return graph, keep


def _replay_us(graph, iters):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def main(argv=None) -> int:
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--runs", type=int, default=5)
    p.add_argument("--dense-warmup", type=int, default=8)
    p.add_argument("--kernel-iters", type=int, default=200)
    p.add_argument("--check-steps", type=int, default=30)
    a = p.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("bench_bn_sliced.py needs a GPU", file=sys.stderr)
        return 2
    import oktopk_b200 as okt
    from oktopk_b200.ops import ext, fused_bn
    C = ext.require()
    torch.cuda.set_device(0)
    card = _card()
    print("card", card)

    # 1. kernel level
    kern = []
    for shape, pooled in VGG16_LAYERS:
        N, Ch, H, W = shape
        sliced = bool(C.bn_sliced(N * H * W, Ch, W if pooled else 0))
        graphs = {k: _pair_graph(C, shape, pooled, CAP[k], a.kernel_iters) for k in ("sliced", "coop")}
        us = {k: [] for k in graphs}
        for k in graphs:
            _replay_us(graphs[k][0], a.kernel_iters)
        for _ in range(a.runs):
            for k in graphs:
                us[k].append(_replay_us(graphs[k][0], a.kernel_iters))
        kern.append({"shape": list(shape), "pool": pooled, "sliced": sliced, **{k: _mmm(v) for k, v in us.items()}})
        print("bn_forward+bn_backward %-18s pool=%d sliced=%d  default %6.2f us (%.2f-%.2f)  cooperative %6.2f us (%.2f-%.2f)"
              % (tuple(shape), pooled, sliced, *[kern[-1][k][m] for k in ("sliced", "coop") for m in ("median", "min", "max")]))
    tot = {k: sum(r[k]["median"] for r in kern) for k in ("sliced", "coop")}
    print("13 layers: default %.1f us, cooperative %.1f us" % (tot["sliced"], tot["coop"]))

    # 2. step level, 3. results
    dnn, _, bs, lr, preset = bench.MODELS["vgg16"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=a.dense_warmup)
    pool = []
    for i in range(4):
        x, y = bench.make_batch("vgg16", i, 0, bs, 128)
        pool.append((x.cuda().contiguous(memory_format=torch.channels_last), y.cuda()))
    names = [("fp32", "sliced"), ("fp32", "coop"), ("fp32", "coop2"), ("bf16_fused", "sliced"), ("bf16_fused", "coop")]
    arms = {n: _arm(n[0], dnn, lr, cfg) for n in names}
    it = {n: 0 for n in arms}
    loss = {}

    def run(n, steps):
        fused_bn.MAX_CTAS = CAP[n[1]]                # read at every call, so also while this arm's graphs are captured
        for _ in range(steps):
            loss[n] = arms[n][1].step(pool[it[n] % len(pool)])
            it[n] += 1
        fused_bn.MAX_CTAS = 0

    def params(n):
        return torch.cat([q.detach().float().flatten() for b in arms[n][0]._buckets for q in b.params])

    def diff(n, m):
        pa, pb = params(n), params(m)
        la, lb = (float(loss[k][0] if isinstance(loss[k], tuple) else loss[k]) for k in (n, m))
        return {"loss": [la, lb], "param_max_abs_diff": float((pa - pb).abs().max()), "param_max_abs": float(pa.abs().max()),
                "params_bitwise_equal": bool(torch.equal(pa, pb))}

    for n in arms:
        run(n, a.dense_warmup + a.check_steps)
    torch.cuda.synchronize()
    results = {"fp32 sliced vs cooperative": diff(names[0], names[1]), "fp32 cooperative vs cooperative": diff(names[1], names[2]),
               "bf16 sliced vs cooperative": diff(names[3], names[4])}
    for k, v in results.items():
        print("after %d steps, %s: %s" % (a.dense_warmup + a.check_steps, k, v))
    times = {n: [] for n in arms}
    for _ in range(a.runs):
        for n in arms:
            run(n, a.warmup)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(n, a.steps)
            e1.record()
            torch.cuda.synchronize()
            times[n].append(e0.elapsed_time(e1) / a.steps)
    for n, (opt, gs) in arms.items():
        assert all(torch.isfinite(q).all() for b in opt._buckets for q in b.params), n
        v = _mmm(times[n])
        print("%-10s %-6s ms/step median %.4f  range %.4f-%.4f  graph %s" % (*n, v["median"], v["min"], v["max"], gs.enabled))

    out = {"card": card, "card_after": _card(), "steps": a.steps, "runs": a.runs, "kernel_iters": a.kernel_iters,
           "bn_fwd_bwd_pair_us": kern, "bn_fwd_bwd_total_us": tot,
           "ms_per_step": {"%s %s" % n: {**_mmm(v), "runs": v} for n, v in times.items()},
           "graphs": {"%s %s" % n: {"enabled": gs.enabled, "captured": len(gs.graphs)} for n, (_, gs) in arms.items()},
           "results": results}
    print(json.dumps(out))
    for opt, _ in arms.values():
        opt.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
