"""CPU tests of gradient clipping inside the optimizer step: the ``--fused-clip`` switch and ``Trainer(fused_clip=...)``,
and ``DistributedOptimizer(max_grad_norm=c)`` on the torch path (no flat CUDA bucket), which must match
``synchronize(); clip_grad_norm_(params, c); step()`` parameter for parameter, in a world of 1 and in a gloo world of 2."""
import os
import sys
from unittest import mock

import pytest
import torch

from oktopk_b200.models import DNNS
from oktopk_b200.train import cli

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from mp_util import run_distributed  # noqa: E402


def _check(argv):
    p = cli.build_parser()
    args = p.parse_args(argv)
    with mock.patch.object(p, "error", side_effect=SystemExit) as err:
        try:
            cli.check_switch_args(p, args)
        except SystemExit:
            return err.call_args[0][0]
    return cli.model_args(args)


def test_flag_accepted_on_the_two_clipping_models_only():
    for dnn in DNNS:
        got = _check(["--dnn", dnn, "--fused-clip"])
        if dnn in ("lstman4", "lstm"):
            assert got == (dnn, {}), (dnn, got)          # a Trainer argument: no create_net keyword
        else:
            assert isinstance(got, str) and "--fused-clip" in got, (dnn, got)
    assert cli.build_parser().parse_args(["--dnn", "lstm"]).fused_clip is False


def test_cli_passes_the_flag_to_the_trainer():
    seen = {}

    def fake(*a, **kw):
        seen.update(kw)
        raise SystemExit(0)
    with mock.patch("oktopk_b200.train.trainer.robust_ssgd", side_effect=fake):
        with pytest.raises(SystemExit):
            cli.main(["--dnn", "lstm", "--fused-clip", "--backend", "dist"])
    assert seen["fused_clip"] is True
    seen.clear()
    with mock.patch("oktopk_b200.train.trainer.robust_ssgd", side_effect=fake):
        with pytest.raises(SystemExit):
            cli.main(["--dnn", "lstman4", "--backend", "dist"])
    assert seen["fused_clip"] is False


def test_trainer_refuses_fused_clip_off_the_clipping_models():
    from oktopk_b200.train.trainer import Trainer
    with pytest.raises(ValueError, match="fused_clip"):
        Trainer(dnn="vgg16", dataset="cifar10", batch_size=2, compressor="none", compression=False,
                device=torch.device("cpu"), fused_clip=True)


def test_max_grad_norm_must_be_positive():
    from oktopk_b200.optimizer import DistributedOptimizer
    m = torch.nn.Linear(4, 2)
    for bad in (0.0, -1.0, float("nan")):
        with pytest.raises(ValueError, match="max_grad_norm"):
            DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters(),
                                 max_grad_norm=bad)


# ------------------------------------------------------------------------------------------- the torch path
SGD_CASES = {
    "plain": dict(momentum=0.0),
    "momentum": dict(momentum=0.9),
    "nesterov": dict(momentum=0.9, nesterov=True),
    "weight_decay": dict(momentum=0.9, weight_decay=1e-2),
    "dampening": dict(momentum=0.9, dampening=0.3, weight_decay=1e-3),
}


def _model(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.Tanh(), torch.nn.Linear(32, 4))


def _batch(it, rank):
    g = torch.Generator().manual_seed(17 * it + rank)
    return torch.randn(8, 16, generator=g) * 4, torch.randint(0, 4, (8,), generator=g)


def _run(rank, world, case, max_norm, fused):
    """Eight steps; ``fused``: ``DistributedOptimizer(max_grad_norm=...)`` and ``step()`` alone, else the trainer's
    stock sequence.  Returns the parameters, momentum buffers and the norms."""
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.optimizer import DistributedOptimizer
    from oktopk_b200.parallel.world import World
    model = _model()
    w = World() if world > 1 else None
    cfg = OkTopkConfig(compressor="none", backend="dist")
    opt = DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.1, **SGD_CASES[case]),
                               named_parameters=model.named_parameters(), cfg=cfg, world=w,
                               max_grad_norm=max_norm if fused else None)
    norms = []
    for it in range(8):
        opt.zero_grad()
        x, y = _batch(it, rank)
        torch.nn.functional.cross_entropy(model(x), y).backward()
        if fused:
            opt.step()
            norms.append(opt.grad_norm().clone())
        else:
            opt.synchronize()
            norms.append(torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm))
            opt.step()
    mom = [opt.state[p].get("momentum_buffer") for p in model.parameters()]
    return [p.detach().clone() for p in model.parameters()], [m.clone() for m in mom if m is not None], norms


def _assert_same(a, b):
    for x, y in zip(a[0] + a[1] + a[2], b[0] + b[1] + b[2]):
        assert torch.equal(x, y)


@pytest.mark.parametrize("case", sorted(SGD_CASES))
def test_sgd_max_grad_norm_matches_stock_clip_world_of_one(case):
    for max_norm in (0.05, 1e3):                    # clipping on every step; never clipping
        ref = _run(0, 1, case, max_norm, False)
        got = _run(0, 1, case, max_norm, True)
        _assert_same(got, ref)
        assert all(float(n) > 0.05 for n in got[2])


def _gloo_worker(rank, world, case):
    return [_run(rank, world, case, 0.05, fused) for fused in (False, True)]


@pytest.mark.parametrize("case", ["momentum", "dampening"])
def test_sgd_max_grad_norm_matches_stock_clip_gloo_world_of_two(case):
    got = run_distributed(_gloo_worker, 2, (case,), backend="gloo", timeout=240)
    for r in range(2):
        ref, fused = got[r]
        _assert_same(fused, ref)
        _assert_same(fused, got[0][1])               # the replicas agree
