"""Single-process CPU tests: optimizer wrappers, model parameter counts, trainer/CLI/checkpoint plumbing."""
import copy
import math
import os

import pytest
import torch

import oktopk_b200 as okt
from oktopk_b200.optimizer import BertAdam, SCHEDULES, warmup_linear


def _mlp(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(12, 32), torch.nn.Tanh(), torch.nn.Linear(32, 4))


def _batch(it):
    g = torch.Generator().manual_seed(it)
    return torch.randn(16, 12, generator=g), torch.randint(0, 4, (16,), generator=g)


@pytest.mark.parametrize("nesterov", [False, True])
def test_dense_wrapper_equals_torch_sgd(nesterov):
    a, b = _mlp(), _mlp()
    kw = dict(lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=nesterov)
    ref = torch.optim.SGD(b.parameters(), **kw)
    opt = okt.DistributedOptimizer(torch.optim.SGD(a.parameters(), **kw), named_parameters=a.named_parameters(),
                                   compression=okt.compressors["none"], is_sparse=False)
    for it in range(6):
        x, y = _batch(it)
        opt.zero_grad(); ref.zero_grad()
        torch.nn.functional.cross_entropy(a(x), y).backward()
        torch.nn.functional.cross_entropy(b(x), y).backward()
        opt.step(); ref.step()
    for p, q in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)
    opt.close()


def test_gradient_accumulation_gate_and_synchronize():
    """``optimizer.local`` skips communication on accumulation micro-steps (VGG/distributed_optimizer.py:78,186);
    ``synchronize()`` exposes the reduced gradient in ``p.grad`` before ``step()`` (LSTM clipping path)."""
    a, b = _mlp(), _mlp()
    ref = torch.optim.SGD(b.parameters(), lr=0.1, momentum=0.9)
    opt = okt.DistributedOptimizer(torch.optim.SGD(a.parameters(), lr=0.1, momentum=0.9),
                                   named_parameters=a.named_parameters(), compression=okt.compressors["none"])
    for it in range(3):
        opt.zero_grad(); ref.zero_grad()
        for j in range(2):
            opt.local = j < 1
            x, y = _batch(10 * it + j)
            torch.nn.functional.cross_entropy(a(x), y).backward()
            torch.nn.functional.cross_entropy(b(x), y).backward()
        opt.synchronize()
        for p, q in zip(a.parameters(), b.parameters()):
            torch.testing.assert_close(p.grad, q.grad)
        torch.nn.utils.clip_grad_norm_(a.parameters(), 0.5)
        torch.nn.utils.clip_grad_norm_(b.parameters(), 0.5)
        opt.step(); ref.step()
    for p, q in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)
    opt.close()


def test_sparse_single_process_follows_error_feedback_topk():
    """P=1 Ok-Topk == SGD on the (strict) top-k of the error-compensated gradient."""
    a = _mlp()
    cfg = okt.OkTopkConfig(density=0.1, local_recompute_interval=1, global_recompute_interval=1)
    opt = okt.DistributedOptimizer(torch.optim.SGD(a.parameters(), lr=0.1), named_parameters=a.named_parameters(),
                                   compression=okt.compressors["oktopk"], is_sparse=True, cfg=cfg)
    x, y = _batch(0)
    opt.zero_grad()
    torch.nn.functional.cross_entropy(a(x), y).backward()
    opt.synchronize()
    st = opt.comm_stats()
    (name, s), = st.items()
    n = opt._buckets[0].numel                       # bucket length (parameters are aligned inside the flat buffer)
    nnz = sum(int((p.grad != 0).sum()) for p in a.parameters())
    assert s["mode"] == "oktopk" and 0 < nnz <= int(n * 0.1) + 1
    opt.step()
    assert opt.get_current_density() == pytest.approx(0.1)
    opt.add_train_epoch(); opt.stop(); opt.close()


def test_any_torch_optimizer_can_be_wrapped():
    a, b = _mlp(), _mlp()
    ref = torch.optim.Adam(b.parameters(), lr=1e-2)
    opt = okt.DistributedOptimizer(torch.optim.Adam(a.parameters(), lr=1e-2), named_parameters=a.named_parameters())
    assert type(opt).__name__ == "Adam" and isinstance(opt, torch.optim.Adam)
    for it in range(4):
        x, y = _batch(it)
        opt.zero_grad(); ref.zero_grad()
        torch.nn.functional.cross_entropy(a(x), y).backward()
        torch.nn.functional.cross_entropy(b(x), y).backward()
        opt.step(); ref.step()
    for p, q in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)
    with pytest.raises(ValueError):
        okt.DistributedOptimizer(torch.optim.SGD(a.parameters(), lr=0.1), named_parameters=list(a.parameters()))
    opt.close()


def test_bert_adam_math_and_schedules():
    """BertAdam: no bias correction, decoupled weight decay, warm-up schedule (optimization.py:173-225)."""
    a, b = _mlp(), _mlp()
    named = list(a.named_parameters())
    groups = [{"params": [p for n, p in named if "bias" not in n], "weight_decay": 0.01},
              {"params": [p for n, p in named if "bias" in n], "weight_decay": 0.0}]
    opt = BertAdam(groups, lr=1e-2, warmup=0.1, t_total=100, named_parameters=named, compressor="none", density=1.0)
    m = {p: torch.zeros_like(p) for p in b.parameters()}
    v = {p: torch.zeros_like(p) for p in b.parameters()}
    wd = {p: (0.0 if "bias" in n else 0.01) for n, p in b.named_parameters()}
    for it in range(5):
        x, y = _batch(it)
        opt.zero_grad()
        for p in b.parameters():
            p.grad = None
        torch.nn.functional.cross_entropy(a(x), y).backward()
        torch.nn.functional.cross_entropy(b(x), y).backward()
        lr = 1e-2 * warmup_linear(it / 100, 0.1)
        assert opt.get_lr()[0] == pytest.approx(lr if it > 0 else 0)
        opt.step()
        with torch.no_grad():
            for p in b.parameters():
                m[p].mul_(0.9).add_(p.grad, alpha=0.1)
                v[p].mul_(0.999).addcmul_(p.grad, p.grad, value=0.001)
                upd = m[p] / (v[p].sqrt() + 1e-6) + wd[p] * p
                p.add_(upd, alpha=-lr)
    for p, q in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)
    assert set(SCHEDULES) == {"warmup_cosine", "warmup_constant", "warmup_linear", "warmup_poly"}
    assert SCHEDULES["warmup_cosine"](0.5, 0.1) == pytest.approx(0.5 * (1 + math.cos(math.pi * 0.5)))
    assert SCHEDULES["warmup_poly"](0.75, 0.1) == pytest.approx(0.5)
    assert SCHEDULES["warmup_constant"](0.05, 0.1) == pytest.approx(0.5)
    with pytest.raises(ValueError):
        BertAdam(a.parameters(), lr=-1)
    opt.close()


def test_optimizer_state_dict_carries_sparse_state_and_resumes_bitwise():
    cfg = okt.OkTopkConfig(density=0.05, local_recompute_interval=3, global_recompute_interval=3)

    def make():
        net = _mlp()
        opt = okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9),
                                       named_parameters=net.named_parameters(), compression="oktopk", is_sparse=True, cfg=cfg)
        return net, opt

    def run(net, opt, its):
        for it in its:
            x, y = _batch(it)
            opt.zero_grad()
            torch.nn.functional.cross_entropy(net(x), y).backward()
            opt.step()

    a, oa = make()
    run(a, oa, range(4))
    sd_m, sd_o = a.state_dict(), oa.state_dict()
    bucket = next(iter(sd_o["oktopk"]["buckets"].values()))
    assert bucket["counter"] == 4 and bucket["residual"] is not None and bucket["local_thr"] > 0
    b, ob = make()
    b.load_state_dict(sd_m)
    ob.load_state_dict(sd_o)
    run(a, oa, range(4, 8))
    run(b, ob, range(4, 8))
    for p, q in zip(a.parameters(), b.parameters()):
        assert torch.equal(p, q)
    oa.close(); ob.close()


def _bert_adam(net):
    named = list(net.named_parameters())
    groups = [{"params": [p for n, p in named if "bias" not in n], "weight_decay": 0.01},
              {"params": [p for n, p in named if "bias" in n], "weight_decay": 0.0}]
    return BertAdam(groups, lr=1e-2, warmup=0.1, t_total=100, named_parameters=named, compressor="none", density=1.0)


def _train(net, opt, its, device="cpu"):
    for it in its:
        x, y = _batch(it)
        opt.zero_grad()
        torch.nn.functional.cross_entropy(net(x.to(device)), y.to(device)).backward()
        opt.step()


@pytest.mark.parametrize("device", ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)])
def test_bert_adam_state_dict_resumes_bitwise(device):
    """Every parameter's checkpointed step is the optimizer's step count; a fresh BertAdam resumes from the checkpoint
    bit for bit (moments, schedule position, flat-buffer aliasing)."""
    a = _mlp().to(device)
    oa = _bert_adam(a)
    _train(a, oa, range(4), device)
    sd = copy.deepcopy(oa.state_dict())
    assert sd["counter"] == 4 and sd["state"] and all(st["step"] == 4 for st in sd["state"].values())
    b = _mlp(seed=1).to(device)
    b.load_state_dict(a.state_dict())
    ob = _bert_adam(b)
    ob.load_state_dict(sd)
    assert ob.counter == 4 and all("step" not in ob.state[p] for p in b.parameters())
    _train(a, oa, range(4, 8), device)
    _train(b, ob, range(4, 8), device)
    for p, q in zip(a.parameters(), b.parameters()):
        assert torch.equal(p, q)
        assert torch.equal(oa.state[p]["next_m"], ob.state[q]["next_m"])
        assert torch.equal(oa.state[p]["next_v"], ob.state[q]["next_v"])
    assert all(st["step"] == 8 for st in ob.state_dict()["state"].values())
    oa.close(); ob.close()


def test_wrapped_sgd_state_dict_moves_to_and_from_torch_sgd():
    kw = dict(lr=0.1, momentum=0.9, weight_decay=1e-4)

    def wrap(net):
        return okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), **kw), named_parameters=net.named_parameters(),
                                        compression=okt.compressors["none"], is_sparse=False)

    def close(net_a, net_b):
        for p, q in zip(net_a.parameters(), net_b.parameters()):
            torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)

    # wrapper -> torch
    a = _mlp()
    opt = wrap(a)
    _train(a, opt, range(3))
    b = _mlp(seed=1)
    b.load_state_dict(a.state_dict())
    ref = torch.optim.SGD(b.parameters(), **kw)
    ref.load_state_dict(copy.deepcopy(opt.state_dict()))
    _train(a, opt, range(3, 6))
    _train(b, ref, range(3, 6))
    close(a, b)
    opt.close()
    # torch -> wrapper: the momentum lands in the flat buffer, and the next step is not a first step
    b = _mlp()
    ref = torch.optim.SGD(b.parameters(), **kw)
    _train(b, ref, range(3))
    a = _mlp(seed=1)
    a.load_state_dict(b.state_dict())
    opt = wrap(a)
    opt.load_state_dict(copy.deepcopy(ref.state_dict()))
    (bk,) = opt._buckets
    flat = opt._flat_state[bk.index]["momentum_buffer"]
    for p, q in zip(a.parameters(), b.parameters()):
        buf = opt.state[p]["momentum_buffer"]
        assert buf.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr()
        assert torch.equal(buf, ref.state[q]["momentum_buffer"])
    _train(a, opt, range(3, 6))
    _train(b, ref, range(3, 6))
    close(a, b)
    opt.close()


def test_momentum_correction_mode_runs():
    a = _mlp()
    opt = okt.DistributedOptimizer(torch.optim.SGD(a.parameters(), lr=0.1, momentum=0.9), named_parameters=a.named_parameters(),
                                   compression="oktopk", is_sparse=True, density=0.1)
    opt.momentum_correction = True
    for it in range(3):
        x, y = _batch(it)
        opt.zero_grad()
        torch.nn.functional.cross_entropy(a(x), y).backward()
        opt.step()
    assert all(torch.isfinite(p).all() for p in a.parameters())
    opt.close()


def test_functional_allreducer_single_process():
    ar = okt.AllReducer("oktopk", True, 0.01)
    g = torch.randn(10_000)
    ref = g.clone()
    out = ar.run(g)
    assert out is g
    k = 100
    thr = float(torch.topk(ref.abs(), k).values[-1])
    assert torch.equal(out != 0, ref.abs() > thr)
    from oktopk_b200.parallel.allreducer import dense_allreduce, gtopk_sparse_allreduce, topk_sparse_allreduce
    t = torch.randn(100)
    assert torch.equal(dense_allreduce(t.clone()), t)
    assert int((topk_sparse_allreduce(torch.randn(1000), 0.01) != 0).sum()) == 10
    assert int((gtopk_sparse_allreduce(torch.randn(1000), 0.01) != 0).sum()) <= 10


# --------------------------------------------------------------------------------------------- models
def test_reference_parameter_counts():
    """SURVEY 2.5: VGG-16 14,728,266 (54 tensors); lstman4 27,569,568 (40 tensors); BERT-base untied 133,547,324."""
    from oktopk_b200.models import create_net
    net, _ = create_net(10, "vgg16")
    ps = list(net.parameters())
    assert sum(p.numel() for p in ps) == 14_728_266 and len(ps) == 54
    assert max(p.numel() for p in ps) == 2_359_296
    net, ext = create_net(29, "lstman4")
    ps = list(net.parameters())
    assert sum(p.numel() for p in ps) == 27_569_568 and len(ps) == 40
    assert max(p.numel() for p in ps) == 4_198_400 and len(ext["labels"]) == 29
    with torch.device("meta"):
        from oktopk_b200.models.bert import bert_base
        net = bert_base(4)
    assert sum(p.numel() for p in net.parameters()) == 133_547_324


@pytest.mark.parametrize("dnn,shape,classes", [("resnet20", (2, 3, 32, 32), 10), ("preresnet110", (1, 3, 32, 32), 10),
                                               ("densenet100", (1, 3, 32, 32), 10), ("caffe_cifar", (2, 3, 32, 32), 10),
                                               ("mnistnet", (2, 1, 28, 28), 10), ("resnet18", (1, 3, 64, 64), 1000),
                                               ("vgg19", (1, 3, 32, 32), 10), ("resnext29", (1, 3, 32, 32), 10)])
def test_zoo_forward_shapes(dnn, shape, classes):
    from oktopk_b200.models import create_net
    net, _ = create_net(classes, dnn)
    net.eval()
    with torch.no_grad():
        out = net(torch.randn(*shape))
    assert out.shape == (shape[0], classes)


def test_deepspeech_and_ptb_forward():
    from oktopk_b200.models import create_net
    net, _ = create_net(29, "lstman4")
    net.eval()
    x = torch.randn(2, 1, 161, 60)
    out, lens = net(x, torch.tensor([60, 40]))
    assert out.shape[0] == 2 and out.shape[2] == 29 and int(lens[0]) == out.shape[1]
    ptb, _ = create_net(0, "lstm", vocab_size=100, batch_size=3)
    h = ptb.init_hidden(3, torch.device("cpu"))
    o, h = ptb(torch.randint(0, 100, (5, 3)), h)
    assert o.shape[-1] == 100


def test_bert_stage_modules_and_loss():
    """``--module models.bert12.depth=4`` style stage lists (BERT/bert/models/bert/depth=4/__init__.py:12-19)."""
    from oktopk_b200.models.bert import BertConfig, BertForPreTraining, build_stages, synthetic_batch
    cfg = BertConfig(vocab_size=2000, hidden_size=32, num_hidden_layers=4, num_attention_heads=4, intermediate_size=64,
                     max_position_embeddings=64)
    net = BertForPreTraining(cfg, depth=2)
    assert len(net.stages) == 2
    batch = synthetic_batch(3, 16, vocab=2000)
    loss = net(*batch)
    assert loss.dim() == 0 and torch.isfinite(loss)
    loss.backward()
    stages = build_stages(cfg, 4)
    assert len(stages) == 4
    # the decoder matrix is an untied copy (SURVEY A.4-10)
    dec = net.stages[-1].heads.decoder_weight
    emb = [p for n, p in net.named_parameters() if "word_embeddings" in n][0]
    assert dec.shape == emb.shape and dec.data_ptr() != emb.data_ptr()


# --------------------------------------------------------------------------------------------- trainer / CLI / checkpoint
def test_trainer_cpu_mnist_steps_and_checkpoint(tmp_path):
    from oktopk_b200.train.trainer import Trainer
    cfg = okt.preset("vgg16", density=0.05, warmup_iters=2, local_recompute_interval=2, global_recompute_interval=2)
    tr = Trainer(dnn="mnistnet", dataset="mnist", batch_size=8, lr=0.05, compressor="oktopk", density=0.05, cfg=cfg,
                 device=torch.device("cpu"), nsteps_update=2, log_dir=str(tmp_path / "logs"))
    for _ in range(4):
        tr.train_step()
    modes = [v["mode"] for v in tr.optimizer.comm_stats().values()]
    assert modes == ["oktopk"]
    l0 = tr.last_loss()
    assert math.isfinite(l0)
    ck = str(tmp_path / "ck" / "m.pth")
    tr.save_checkpoint(ck)
    res = tr.test(0, max_batches=2)
    assert 0.0 <= res["top1"] <= 1.0
    tr2 = Trainer(dnn="mnistnet", dataset="mnist", batch_size=8, lr=0.05, compressor="oktopk", density=0.05, cfg=cfg,
                  device=torch.device("cpu"), nsteps_update=2)
    tr2.load_checkpoint(ck)
    assert tr2.train_iter == tr.train_iter
    for p, q in zip(tr.net.parameters(), tr2.net.parameters()):
        assert torch.equal(p, q)
    sd = tr2.optimizer.state_dict()["oktopk"]["buckets"]
    assert next(iter(sd.values()))["counter"] == 4
    tr.update_nworker(1, 0)
    tr.close(); tr2.close()


def test_lr_schedules_match_reference_shapes():
    from oktopk_b200.train.trainer import Trainer
    tr = Trainer(dnn="mnistnet", dataset="mnist", batch_size=8, lr=0.1, compressor="none", compression=False,
                 device=torch.device("cpu"))
    tr.train_epoch = 0
    assert tr.adjust_learning_rate() == pytest.approx(0.1)       # single worker: no warm-up ramp
    for e, want in ((80, 0.1), (81, 0.01), (122, 0.001), (155, 0.0001)):
        tr.train_epoch = e
        assert tr.adjust_learning_rate() == pytest.approx(want)
    tr.nworkers = 4
    tr.train_epoch, tr.train_iter = 0, 0
    assert tr.adjust_learning_rate() == pytest.approx(0.1 / 4)   # 10-epoch linear warm-up from lr/P (dl_trainer.py:531-563)
    tr.train_epoch = 5
    assert tr.adjust_learning_rate() == pytest.approx(0.025 + 0.075 * 0.5)
    tr.dnn = "lstman4"
    tr.train_epoch = 2
    assert tr.adjust_learning_rate() == pytest.approx(0.1 / 1.01 ** 2)
    tr.close()


def test_cli_parser_flag_parity():
    from oktopk_b200.train.cli import build_parser
    p = build_parser()
    a = p.parse_args("--dnn vgg16 --dataset cifar10 --batch-size 16 --lr 0.1 --nsteps-update 1 --nworkers 16 --nwpernode 1 "
                     "--compression --compressor oktopk --density 0.02 --sigma-scale 2.5 --max-epochs 161 --data-dir /x".split())
    assert a.compression and a.compressor == "oktopk" and a.density == 0.02 and a.max_epochs == 161
    b = p.parse_args("--dnn bert_base --module models.bert12.depth=4 --train_batch_size 8 --max_seq_length 128 "
                     "--num_minibatches 1024 --gradient_accumulation_steps 1 --density 0.01 --compressor topkSA "
                     "--checkpoint_dir /tmp/x".split())
    assert b.batch_size == 8 and b.max_iters == 1024 and b.module.endswith("depth=4")
    for c in ("topkA", "topkAopt", "topkA2", "topkSA", "gtopk", "gaussiank", "gaussiankconcat", "gaussiankSA", "none"):
        assert p.parse_args(["--compressor", c]).compressor == c
    e = p.parse_args("--slot-factor 2 --overselect-cap 1.5 --dense-switch-density 0 --nvls off --comm-ctas 32 --norm-clip 5 "
                     "--trace /tmp/t".split())
    assert (e.slot_factor, e.overselect_cap, e.dense_switch_density, e.nvls, e.comm_ctas, e.norm_clip, e.trace) == \
        (2.0, 1.5, 0.0, "off", 32, 5.0, "/tmp/t")


def test_cli_end_to_end_on_cpu_with_engine_flags(tmp_path):
    """The CLI main() with the round-2 engine flags on the CPU/dist backend (one process)."""
    from oktopk_b200.train.cli import main
    rc = main(["--dnn", "mnistnet", "--dataset", "mnist", "--batch-size", "4", "--lr", "0.05", "--compression", "--compressor",
               "topkA", "--density", "0.02", "--max-iters", "3", "--norm-clip", "5", "--overselect-cap", "0", "--slot-factor", "2",
               "--dense-switch-density", "0", "--trace", str(tmp_path)])
    assert rc == 0
    assert any(f.startswith("trace_mnistnet_rank0") for f in os.listdir(tmp_path))


def test_robust_ssgd_driver_runs(tmp_path):
    from oktopk_b200.train.trainer import robust_ssgd
    tr = robust_ssgd("mnistnet", "mnist", None, 1, 0.05, 8, 1, 1, compression=True, compressor="gaussiank", density=0.05,
                     max_iters=3, log_every=1, checkpoint_dir=str(tmp_path), device=torch.device("cpu"))
    assert tr.train_iter == 3
    assert any(f.endswith(".pth") for f in os.listdir(tmp_path))


def test_signal_handler_saves_interrupted_state_and_resumes(tmp_path):
    """SURVEY 5.3: the reference defines SLURM signal handlers but never installs them; here they are live."""
    import signal
    from oktopk_b200.train.trainer import Trainer
    from oktopk_b200.utils import elastic
    tr = Trainer(dnn="mnistnet", dataset="mnist", batch_size=4, lr=0.05, compressor="oktopk", density=0.05,
                 device=torch.device("cpu"))
    tr.train_step()
    hit = []
    prev = elastic.install_signal_handlers(tr, str(tmp_path), exit_after=False, on_signal=hit.append)
    try:
        os.kill(os.getpid(), signal.SIGUSR1)
        assert hit == [signal.SIGUSR1] and os.path.exists(elastic.interrupted_path(str(tmp_path), 0))
        tr.train_step()
        assert elastic.resume_if_interrupted(tr, str(tmp_path)) and tr.train_iter == 1
        assert not elastic.resume_if_interrupted(tr, str(tmp_path))
        tr.optimizer.check_faults()                       # healthy: no-op
        elastic.shrink_world(tr, 1, 0)
    finally:
        for s, h in prev.items():
            signal.signal(s, h)
        tr.close()


def test_profiling_norm_records_sparsification_error(monkeypatch):
    """``settings.PROFILING_NORM``: relative error of the sparse result vs the true dense top-k (the paper's xi)."""
    from oktopk_b200.utils import settings
    monkeypatch.setattr(settings, "PROFILING_NORM", True)
    ar = okt.AllReducer("oktopk", True, 0.01)
    g = torch.randn(20_000)
    ar.run(g.clone())
    ar.run(torch.randn(20_000))
    assert len(ar.profile_records) == 2
    r = ar.profile_records[0]
    # P=1 exact iteration: the result is the strict top-k => only the k-th element is missing from the ideal set
    assert 0.0 <= r["eps"] < 0.05 and r["nnz"] == 199 and r["grad_norm"] > 0
