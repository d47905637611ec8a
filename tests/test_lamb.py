"""CPU tests of LAMB: ``okt.Lamb`` against a float64 implementation of its formula, the wrapped ``Lamb`` on the torch
flat-bucket path (no CUDA bucket) against the bare optimizer in a world of 1 and in a gloo world of 2, checkpoints in
both directions, the unequal-step fallback, and the ``--lamb`` switch with ``Trainer(lamb=True)``."""
import copy
import os
import sys
from unittest import mock

import pytest
import torch

from oktopk_b200.models import DNNS
from oktopk_b200.models.switches import BERTS, SWITCHES
from oktopk_b200.optimizer import Lamb
from oktopk_b200.train import cli

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from mp_util import run_distributed  # noqa: E402


def _lamb64(w, g, m, v, t, lr, b1, b2, eps, wd, bc):
    """One LAMB step in float64, written from the formula."""
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    mh, vh = (m / (1 - b1 ** t), v / (1 - b2 ** t)) if bc else (m, v)
    u = mh / (vh.sqrt() + eps) + wd * w
    wn, un = float(w.norm()), float(u.norm())
    r = wn / un if wd != 0 and wn > 0 and un > 0 else 1.0
    return w - lr * r * u, m, v, r


@pytest.mark.parametrize("bc", [True, False])
def test_step_against_float64_formula(bc):
    """Six steps over two groups (wd 0.01 and 0), with a zero-initialised weight (r = 1 on its first step) and a
    weight that is zero with a zero gradient on the first step (||u|| = 0, r = 1)."""
    gen = torch.Generator().manual_seed(3)
    shapes = [(33, 7), (5,), (16,), (3, 4), (9,)]
    params = [torch.nn.Parameter(torch.randn(s, generator=gen)) for s in shapes]
    with torch.no_grad():
        params[2].zero_()                         # zero weight, ordinary gradients: ||w|| = 0 on the first step
        params[3].zero_()                         # zero weight and a zero first gradient: u = 0
    hyper = dict(lr=2e-2, betas=(0.9, 0.99), eps=1e-6)
    opt = Lamb([{"params": params[:4], "weight_decay": 0.01}, {"params": params[4:], "weight_decay": 0.0}],
               bias_correction=bc, **hyper)
    wds = [0.01] * 4 + [0.0]
    ref = [(p.detach().double().clone(), torch.zeros(p.shape, dtype=torch.float64),
            torch.zeros(p.shape, dtype=torch.float64)) for p in params]
    ratios = []
    for t in range(1, 7):
        grads = [torch.randn(s, generator=gen) * 10 ** (i - 2) for i, s in enumerate(shapes)]
        if t == 1:
            grads[3].zero_()
        for p, g in zip(params, grads):
            p.grad = g.clone()
        opt.step()
        step_r = []
        for i, ((w, m, v), g) in enumerate(zip(ref, grads)):
            w, m, v, r = _lamb64(w, g.double(), m, v, t, hyper["lr"], 0.9, 0.99, 1e-6, wds[i], bc)
            ref[i] = (w, m, v)
            step_r.append(r)
        ratios.append(step_r)
        for p, (w, m, v) in zip(params, ref):
            torch.testing.assert_close(p.detach().double(), w, rtol=1e-5, atol=1e-6)
            for k, x in (("exp_avg", m), ("exp_avg_sq", v)):        # fp32 rounding, relative to the tensor's scale
                torch.testing.assert_close(opt.state[p][k].double(), x, rtol=1e-5,
                                           atol=1e-6 * float(x.abs().max()) + 1e-30)
    assert ratios[0][2] == 1.0 and ratios[0][3] == 1.0 and ratios[1][2] != 1.0     # the zero-norm cases, then not
    assert all(r[4] == 1.0 for r in ratios)                                      # wd == 0: no trust ratio
    assert all(float(opt.state[p]["step"]) == 6.0 for p in params)


def _net(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(20, 64), torch.nn.ReLU(), torch.nn.Linear(64, 5))


def _groups(net):
    return [{"params": [net[0].weight, net[2].weight], "weight_decay": 0.01},
            {"params": [net[0].bias, net[2].bias], "weight_decay": 0.0}]


def _batch(it, rank):
    g = torch.Generator().manual_seed(10 * it + rank)
    return torch.randn(8, 20, generator=g), torch.randint(0, 5, (8,), generator=g)


def _wrapped(net, max_grad_norm=None, **lamb):
    import oktopk_b200 as okt
    cfg = okt.OkTopkConfig(density=1.0, bucket_elems=300)             # several buckets
    return okt.DistributedOptimizer(Lamb(_groups(net), **dict(dict(lr=1e-2), **lamb)),
                                    named_parameters=net.named_parameters(), compression=okt.compressors["none"],
                                    cfg=cfg, max_grad_norm=max_grad_norm)


@pytest.mark.parametrize("bc", [True, False])
def test_wrapped_cpu_path_equals_bare_lamb(bc):
    from oktopk_b200.optimizer import _LambUpdate
    a, b = _net(), _net()
    opt, ref = _wrapped(a, bias_correction=bc), Lamb(_groups(b), lr=1e-2, bias_correction=bc)
    assert opt._update is _LambUpdate and opt._lamb is None and len(opt._buckets) >= 2
    for it in range(6):
        x, y = _batch(it, 0)
        for net, o in ((a, opt), (b, ref)):
            o.zero_grad()
            torch.nn.functional.cross_entropy(net(x), y).backward()
            o.step()
    for p, q in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-6, atol=1e-7)
        for k in ("exp_avg", "exp_avg_sq"):
            torch.testing.assert_close(opt.state[p][k], ref.state[q][k], rtol=1e-6, atol=1e-9)
    opt.close()


def test_wrapped_global_clip_equals_clip_then_bare_lamb():
    a, b = _net(), _net()
    opt, ref = _wrapped(a, max_grad_norm=0.05), Lamb(_groups(b), lr=1e-2)
    for it in range(4):
        x, y = _batch(it, 0)
        opt.zero_grad()
        torch.nn.functional.cross_entropy(a(x), y).backward()
        opt.step()
        ref.zero_grad()
        torch.nn.functional.cross_entropy(b(x), y).backward()
        assert float(torch.nn.utils.clip_grad_norm_(b.parameters(), 0.05)) > 0.05
        ref.step()
    for p, q in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-6, atol=1e-7)
    opt.close()


def _gloo_worker(rank, P, steps):
    net, ref = _net(), _net()
    opt = _wrapped(net)
    ref_opt = Lamb(_groups(ref), lr=1e-2)
    for it in range(steps):
        x, y = _batch(it, rank)
        opt.zero_grad()
        torch.nn.functional.cross_entropy(net(x), y).backward()
        opt.step()
        ref_opt.zero_grad()                       # the bare optimizer on the rank-averaged gradient
        tot = 0
        for r in range(P):
            xr, yr = _batch(it, r)
            tot = tot + torch.nn.functional.cross_entropy(ref(xr), yr) / P
        tot.backward()
        ref_opt.step()
    flat = torch.cat([p.detach().view(-1) for p in net.parameters()])
    refflat = torch.cat([p.detach().view(-1) for p in ref.parameters()])
    opt.close()
    return flat, refflat


def test_wrapped_gloo_world2_equals_bare_lamb_on_mean_gradient():
    out = run_distributed(_gloo_worker, 2, (5,), backend="gloo")
    assert torch.equal(out[0][0], out[1][0])
    torch.testing.assert_close(out[0][0], out[0][1], rtol=1e-5, atol=1e-6)


def _run(net, opt, its):
    for it in its:
        x, y = _batch(it, 0)
        opt.zero_grad()
        torch.nn.functional.cross_entropy(net(x), y).backward()
        opt.step()


@pytest.mark.parametrize("direction", ["wrapped_to_bare", "bare_to_wrapped"])
def test_state_dict_round_trip(direction):
    """Three steps on one side, its state_dict loaded into the other, three more steps: equal to six on one side."""
    a, b, c = _net(), _net(), _net()
    straight = Lamb(_groups(c), lr=1e-2)
    _run(c, straight, range(6))
    if direction == "wrapped_to_bare":
        first, second = _wrapped(a), Lamb(_groups(b), lr=1e-2)
    else:
        first, second = Lamb(_groups(a), lr=1e-2), None
    _run(a, first, range(3))
    sd = copy.deepcopy(first.state_dict())
    assert all(float(st["step"]) == 3.0 for st in sd["state"].values())
    with torch.no_grad():
        for p, q in zip(b.parameters(), a.parameters()):
            p.copy_(q)
    if second is None:
        second = _wrapped(b)
    second.load_state_dict(sd)
    _run(b, second, range(3, 6))
    for p, q in zip(b.parameters(), c.parameters()):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-6, atol=1e-7)
    for o in (first, second):
        if hasattr(o, "close"):
            o.close()


def test_unequal_step_counts_fall_back_to_lamb_step():
    import oktopk_b200 as okt
    net, ref = _net(), _net()
    bare = Lamb(_groups(net), lr=1e-2)
    _run(net, bare, range(2))
    bare.state[net[0].weight]["step"] += 1
    with pytest.warns(UserWarning, match="unequal step counts"):
        opt = okt.DistributedOptimizer(bare, named_parameters=net.named_parameters(),
                                       compression=okt.compressors["none"])
    assert opt._update is None
    _run(net, opt, range(2, 4))
    ref_opt = Lamb(_groups(ref), lr=1e-2)
    _run(ref, ref_opt, range(2))
    ref_opt.state[ref[0].weight]["step"] += 1
    _run(ref, ref_opt, range(2, 4))
    for p, q in zip(net.parameters(), ref.parameters()):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-6, atol=1e-7)
    opt.close()


# ------------------------------------------------------------------------------------------------ switch and trainer
def _check(argv):
    p = cli.build_parser()
    args = p.parse_args(argv)
    with mock.patch.object(p, "error", side_effect=SystemExit) as err:
        try:
            cli.check_switch_args(p, args)
        except SystemExit:
            return err.call_args[0][0]
    return cli.model_args(args)


def test_switch_entry_and_flag():
    sw = [s for s in SWITCHES if s.flag == "--lamb"]
    assert len(sw) == 1 and sw[0].keywords == () and sw[0].models == BERTS
    for dnn in DNNS:
        got = _check(["--dnn", dnn, "--lamb"])
        if dnn in BERTS:
            assert got == (dnn, {}), (dnn, got)          # a Trainer argument: no create_net keyword
        else:
            assert isinstance(got, str) and "--lamb" in got, (dnn, got)
    assert cli.build_parser().parse_args(["--dnn", "bert_base"]).lamb is False


def test_cli_passes_the_flag_to_the_trainer():
    seen = {}

    def fake(*a, **kw):
        seen.update(kw)
        raise SystemExit(0)
    for argv, want in ((["--dnn", "bert_base", "--lamb"], True), (["--dnn", "bert_base"], False)):
        seen.clear()
        with mock.patch("oktopk_b200.train.trainer.robust_ssgd", side_effect=fake):
            with pytest.raises(SystemExit):
                cli.main(argv + ["--backend", "dist"])
        assert seen["lamb"] is want


def test_trainer_refuses_lamb_off_bert():
    from oktopk_b200.train.trainer import Trainer
    with pytest.raises(ValueError, match="lamb"):
        Trainer(dnn="vgg16", dataset="cifar10", batch_size=2, compressor="none", compression=False,
                device=torch.device("cpu"), lamb=True)


def test_trainer_builds_wrapped_lamb_with_bertadam_groups_and_schedule():
    from oktopk_b200.models.bert import BertConfig
    from oktopk_b200.optimizer import _LambUpdate, scheduled_lr
    from oktopk_b200.train.trainer import Trainer
    tr = Trainer(dnn="bert_base", dataset="wikipedia", batch_size=2, lr=1e-3, compressor="none", compression=False,
                 device=torch.device("cpu"), seq_len=16, t_total=10, warmup=0.2, lamb=True,
                 model_kwargs={"config": BertConfig(num_hidden_layers=2, hidden_size=64, num_attention_heads=2,
                                                    intermediate_size=128), "depth": 2})
    opt = tr.optimizer
    assert isinstance(opt, Lamb) and opt._update is _LambUpdate and opt._max_grad_norm == 1.0
    assert [g["weight_decay"] for g in opt.param_groups] == [0.01, 0.0]
    names = {p: n for n, p in tr.net.named_parameters()}
    assert all(any(k in names[p] for k in ("bias", "norm", "LayerNorm")) for p in opt.param_groups[1]["params"])
    lrs = []
    for _ in range(3):
        lrs.append(tr.adjust_learning_rate())
        tr.train_step()
    assert lrs == [scheduled_lr(1e-3, i, 10, 0.2) for i in range(3)] and lrs[0] == 0.0 and lrs[1] < lrs[2]
    assert all(g["lr"] == lrs[-1] for g in opt.param_groups)
    tr.close()
