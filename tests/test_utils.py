"""Utilities: CTC decoder / WER, alpha-beta cost model + per-scheme volume formulas, metrics helpers, Prefetcher."""
import math

import pytest
import torch

from oktopk_b200.utils import perf_model as pm
from oktopk_b200.utils.decoder import GreedyDecoder, cer, levenshtein, wer
from oktopk_b200.utils.metrics import MetricsWriter, PhaseTimers, force_insert_item, sparsification_error


def test_edit_distances():
    assert levenshtein("kitten", "sitting") == 3
    assert levenshtein("", "abc") == 3 and levenshtein("abc", "abc") == 0
    assert wer("the cat sat", "the cat sat down") == 1
    assert wer("a b c", "x y z") == 3
    assert cer("hello world", "helo wrld") == 2


def test_greedy_ctc_decoder_collapses_repeats_and_blanks():
    labels = "_ab "
    dec = GreedyDecoder(labels, blank_index=0)
    # frames: a a _ a b b _ ' ' -> "aab "
    seq = [1, 1, 0, 1, 2, 2, 0, 3]
    probs = torch.zeros(1, len(seq), 4)
    for t, c in enumerate(seq):
        probs[0, t, c] = 1.0
    assert dec.decode(probs, torch.tensor([len(seq)])) == ["aab "]
    assert dec.decode(probs, torch.tensor([3])) == ["a"]
    assert dec.convert_targets(torch.tensor([1, 2, 3, 1]), torch.tensor([3, 1])) == ["ab ", "a"]


def test_volume_formulas_match_the_paper_table():
    n, k, P = 1_000_000, 1000, 8
    assert pm.volume_elems("dense", n, k, P) == pytest.approx(2 * n * 7 / 8)
    assert pm.volume_elems("topkA", n, k, P) == 2 * k * 7
    assert pm.volume_elems("gaussiank", n, k, P) == 2 * k * 7
    assert pm.volume_elems("topkSA", n, k, P) == pytest.approx(4 * k * 7 / 8)
    assert pm.volume_elems("gtopk", n, k, P) == 4 * k * 3
    assert pm.volume_elems("oktopk", n, k, P) == pytest.approx(6 * k * 7 / 8)
    with pytest.raises(KeyError):
        pm.volume_elems("nope", n, k, P)
    # the reference's hard-coded Ethernet tables (VGG/utils.py:62-83)
    assert pm.GBE[16] == (1.7e-3, 1.7e-8) and pm.TEN_GBE[16] == (1.4e-4, 2.0e-10)
    t_dense = pm.allreduce_time("dense", n, k, 16, pm.TEN_GBE)
    t_okt = pm.allreduce_time("oktopk", n, k, 16, pm.TEN_GBE)
    assert t_okt < t_dense
    r = pm.oktopk_roofline(134_217_728, 134_217, 8)
    assert r["floor_s"] == r["hbm_s"] and 6.2e-4 < r["hbm_s"] < 6.6e-4       # HBM-bound at density 0.001
    idx, val = pm.topk(__import__("numpy").array([0.1, -5.0, 3.0, 0.2]), 2)
    assert sorted(idx.tolist()) == [1, 2]


def test_metrics_helpers(tmp_path):
    d = {}
    force_insert_item(d, "a", 1.0)
    force_insert_item(d, "a", 2.0)
    assert d == {"a": [1.0, 2.0]}
    t = PhaseTimers()
    with t.cuda_range("phase"):
        sum(range(1000))
    t.add("io", 0.5)
    s = t.summary()
    assert s["io"] == 0.5 and s["phase"] >= 0.0 and t.summary() == {}
    w = MetricsWriter(str(tmp_path), rank=0)
    w.add_scalars("train", {"loss": 1.5}, 3)
    w.close()
    line = (tmp_path / "metrics.jsonl").read_text().strip()
    assert '"loss": 1.5' in line and '"step": 3' in line
    MetricsWriter(None).add_scalars("x", {"y": 1}, 0)              # no log dir: silently a no-op
    g = torch.randn(1000)
    e = sparsification_error(g, g.clone(), 1000)
    assert e["eps"] == 0.0 and e["nnz"] == int((g != 0).sum())
    assert sparsification_error(g, torch.zeros_like(g), 10)["eps"] > 0


def test_prefetcher_defer_and_advance_cpu():
    from oktopk_b200.train import data as D
    ds = D.build_dataset("mnist", None, train=True)
    loader, sampler = D.build_loader(ds, "mnist", 4, 0, 1, train=False)
    pf = D.Prefetcher(loader, torch.device("cpu"))
    ref = [b for _, b in zip(range(4), iter(loader))]
    b0 = pf.next(defer=True)
    assert pf.next_batch is None
    pf.advance()
    assert pf.next_batch is not None
    pf.advance()                                                  # idempotent until the batch is taken
    b1 = pf.next()
    b2 = pf.next(defer=True)
    b3 = pf.next()                                                # next() stages on demand if advance() was skipped
    for got, want in zip((b0, b1, b2, b3), ref):
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_profiling_flags_on_the_dist_path(tmp_path, monkeypatch, capsys):
    """settings.PROFILING_GRAD / PROFILING_NORM (VGG/allreducer.py:854-888,1361-1418; VGG/main_trainer.py:107-139):
    gradient / threshold snapshots at chosen iterations, and the (gtopk_norm, randk_norm, upbound, xnorm, dense_std)
    tuples saved per epoch."""
    import numpy as np
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.allreducer import AllReducer
    from oktopk_b200.utils import settings
    monkeypatch.setattr(settings, "PROFILING_GRAD", True)
    monkeypatch.setattr(settings, "PROFILING_NORM", True)
    monkeypatch.setattr(settings, "PREFIX", str(tmp_path))
    monkeypatch.setenv("OKTOPK_GRAD_DUMP_ITERS", "1-1")
    ar = AllReducer("topkA", True, 0.05, cfg=OkTopkConfig(density=0.05, compressor="topkA"))
    for it in range(3):
        g = torch.randn(2000, generator=torch.Generator().manual_seed(it))
        ar.run(g)
    out = capsys.readouterr().out
    assert "ok_gk_local_thrds" in out
    assert (tmp_path / "localgrad1_k100.npy").exists() and (tmp_path / "localthrds1_k100.npy").exists()
    assert len(ar._profiling_norms) == 3 and len(ar.profile_records) == 3
    gt, rk, ub, xn, sd = ar._profiling_norms[-1]
    assert 0 <= gt <= xn and rk <= xn + 1e-6 and ub < xn
    ar.save_profiling_norms(str(tmp_path), 0)
    arr = np.load(tmp_path / "gtopknorm-rank0-epoch0.npy")
    assert arr.shape == (3,) and ar._profiling_norms == []


def test_lr_schedule_boundaries_follow_the_reference():
    """ImageNet 30/60/80, PTB-LSTM 1x until epoch 63 then 0.01x / 0.001x (VGG/dl_trainer.py:514-563)."""
    from oktopk_b200.train.trainer import Trainer
    tr = Trainer(dnn="mnistnet", dataset="mnist", batch_size=4, lr=1.0, compressor="none", compression=False,
                 device=torch.device("cpu"))
    tr.dataset = "imagenet"
    lrs = {}
    for ep in (0, 29, 30, 59, 60, 80):
        tr.train_epoch, tr.train_iter = ep, ep * tr.iters_per_epoch
        lrs[ep] = tr.adjust_learning_rate()
    assert lrs[29] == pytest.approx(1.0) and lrs[30] == pytest.approx(0.1) and lrs[60] == pytest.approx(0.01) \
        and lrs[80] == pytest.approx(0.001)
    tr.dnn = "lstm"
    for ep, want in ((10, 1.0), (62, 1.0), (63, 0.01), (79, 0.01), (80, 0.001)):
        tr.train_epoch = ep
        assert tr.adjust_learning_rate() == pytest.approx(want), ep
    tr.close()


def test_graph_step_enumerates_every_call_plan_of_the_schedule():
    """GraphedTrainStep._sparse_flavours, keyed by the density and each engine's CallPlan: at P = 2 Ok-Topk's schedule
    has exactly three step flavours (threshold reuse, exact thresholds, exact + re-partition), at P = 1 two (a
    re-partition changes nothing there), and under the dense switch one; they are what precapture_sparse() captures up
    front."""
    from types import SimpleNamespace
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.state import CallPlan
    from oktopk_b200.train.graph_step import GraphedTrainStep
    cfg = OkTopkConfig(density=0.001, warmup_iters=512, local_recompute_interval=32, global_recompute_interval=32,
                       repartition_interval=64)
    eng = SimpleNamespace(host=SimpleNamespace(counter=600), P=2)
    opt = SimpleNamespace(_cfg=cfg, _buckets=[SimpleNamespace(name="b0")],
                          _allreducer=SimpleNamespace(_engines={"b0": eng}, compressor=SimpleNamespace(name="oktopk")),
                          get_current_density=lambda: 0.001)
    gs = GraphedTrainStep(SimpleNamespace(optimizer=opt))

    def flags(fl):
        assert all(k[0] == 0.001 and k[1].kind == "fused" for k in fl)
        return sorted((k[1].exact_local, k[1].exact_global, k[1].repartition) for k in fl)
    fl = gs._sparse_flavours()
    assert flags(fl) == [(False, False, False), (True, True, False), (True, True, True)]
    assert fl[(0.001, CallPlan("fused", True, True, True))] == 0
    assert gs._key([512 + 32])[1] == CallPlan("fused", True, True, False) and gs._key([100])[1] == CallPlan("dense")
    eng.P = 1
    fl = gs._sparse_flavours()
    assert flags(fl) == [(False, False, False), (True, True, False)]
    assert fl[(0.001, CallPlan("fused", True, True, False))] == 0
    eng.P = 2
    opt.get_current_density = lambda: 0.1                 # at or above dense_switch_density (0.05): every step is dense
    assert gs._sparse_flavours() == {(0.1, CallPlan("dense_switch")): 0}
    opt.get_current_density = lambda: 0.001
    opt._allreducer.compressor.name = "topkAopt"
    assert len(gs._sparse_flavours()) == 2
    opt._allreducer.compressor.name = "gtopk"
    assert len(gs._sparse_flavours()) == 1               # native tree kernel: one flavour, capturable


@pytest.mark.parametrize("P", [1, 2])
def test_plan_call_follows_the_schedule_of_every_scheme(P):
    """plan_call against the schedule written out here: dense warm-up, then Ok-Topk's exact local / exact global /
    re-partition iterations (re-partition only at P > 1), TopkAopt's exact-threshold iterations, and no flags for the
    other schemes; the dense switch takes the fused family only, at P > 1."""
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.state import CallPlan, plan_call, schedule_period
    cfg = OkTopkConfig(density=0.01, warmup_iters=5, local_recompute_interval=4, global_recompute_interval=6,
                       repartition_interval=8, topkaopt_recompute_interval=3, dense_switch_density=0.05)
    family = {"oktopk": "fused", "topkSA": "fused", "topkDSA": "fused", "gaussiankSA": "fused", "topkA": "gather",
              "topkA2": "gather", "topkAopt": "gather", "gaussiank": "gather", "gaussiankconcat": "gather",
              "gtopk": "tree"}
    for name, fam in family.items():
        period = {"oktopk": 24, "topkAopt": 3}.get(name, 1)
        assert schedule_period(cfg, name) == period
        for c in range(5 + 2 * 24):                      # two periods of the longest schedule
            it = c - 5
            if c < 5:
                want = CallPlan("dense")
            elif name == "oktopk":
                want = CallPlan("fused", it % 4 == 0, it % 6 == 0, P > 1 and it % 8 == 0)
            elif name == "topkAopt":
                want = CallPlan("gather", exact_local=it % 3 == 0)
            else:
                want = CallPlan(fam)
            assert plan_call(cfg, name, c, None, P) == want, (name, c)
            if c >= 5:
                assert plan_call(cfg, name, c + period, None, P) == want, (name, c)
        switched = plan_call(cfg, name, 5, 0.05, P)
        assert switched == (CallPlan("dense_switch") if fam == "fused" and P > 1 else plan_call(cfg, name, 5, None, P))
        assert plan_call(cfg.replace(dense_switch_density=0.0), name, 5, 0.5, P).kind == fam
        assert plan_call(cfg.replace(sparse=False), name, 5, None, P) == CallPlan("dense")
    assert plan_call(cfg, "none", 5, None, P) == plan_call(cfg, None, 5, None, P) == CallPlan("dense")
    with pytest.raises(KeyError):
        plan_call(cfg, "nosuchscheme", 5, None, P)


def test_bench_output_dump_is_seeded_and_bounded(tmp_path):
    """bench.py --dump-outputs: a model larger than the dump budget is represented by the same sample in every run, and
    the files stay under 64 MB."""
    from types import SimpleNamespace
    import bench
    torch.manual_seed(0)
    tr = SimpleNamespace(net=torch.nn.Linear(4096, 4096))              # 16.8 M parameters > DUMP_MAX_ELEMS
    a = bench.output_sample(tr, torch.tensor(2.5))
    b = bench.output_sample(tr, torch.tensor(2.5))
    assert a["params"].shape == (bench.DUMP_MAX_ELEMS,) and (a["params"] == b["params"]).all()
    assert a["params"].dtype == "float32" and float(a["loss"][0]) == 2.5
    bench.write_outputs(str(tmp_path / "out"), a)
    files = sorted((tmp_path / "out").iterdir())
    assert [f.name for f in files] == ["loss.npy", "params.npy"]
    assert sum(f.stat().st_size for f in files) <= 64 * 10 ** 6
