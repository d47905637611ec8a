#!/usr/bin/env python
"""Where does an end-to-end step spend its host time?  (prefetch / step issue / loss read-back)"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import oktopk_b200 as okt  # noqa: E402
from oktopk_b200.train.trainer import Trainer  # noqa: E402

graph = "--no-graph" not in sys.argv
w = okt.init()
print("threads before Trainer:", torch.get_num_threads(), "OMP env:", os.environ.get("OMP_NUM_THREADS"))
cfg = okt.preset("vgg16", density=0.001, warmup_iters=0)
tr = Trainer(dnn="vgg16", dataset="cifar10", batch_size=16, lr=0.1, compressor="oktopk", density=0.001, cfg=cfg, world=w,
             cuda_graph=graph)
print("threads after Trainer:", torch.get_num_threads())
for _ in range(40):
    tr.train_step()
    tr.last_loss()
T = {"prefetch": 0.0, "issue": 0.0, "loss": 0.0}
N = 100
t_all = time.perf_counter()
for _ in range(N):
    t0 = time.perf_counter()
    batch = tr.prefetch.next()
    t1 = time.perf_counter()
    tr.step(batch)
    t2 = time.perf_counter()
    tr.last_loss()
    t3 = time.perf_counter()
    T["prefetch"] += t1 - t0
    T["issue"] += t2 - t1
    T["loss"] += t3 - t2
tot = time.perf_counter() - t_all
print("graph=%s  ms/step %.3f  " % (graph, tot / N * 1e3) + "  ".join("%s %.3f" % (k, v / N * 1e3) for k, v in T.items()))
tr.close()
