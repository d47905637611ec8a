"""The AN4 DeepSpeech model's fused CTC loss switch on the CPU: ``create_net(29, "lstman4", fuse_ctc=True)`` is the stock
network (``state_dict`` keys and values), the Trainer's loss and gradients equal stock bit for bit on the CPU,
``net.fuse_ctc`` is a run-time switch, every fallback of ``ctc_loss`` calls exactly the stock expression, and the
``--fused-ctc`` flag."""
from unittest import mock

import pytest
import torch
import torch.nn.functional as F

from oktopk_b200.models import create_net
from oktopk_b200.ops import ext, fused_ctc
from oktopk_b200.train import cli


def _pair():
    torch.manual_seed(0)
    a, _ = create_net(29, "lstman4", fuse_ctc=True)
    torch.manual_seed(0)
    b, _ = create_net(29, "lstman4")
    return a, b


def test_fuse_ctc_keeps_the_stock_network():
    a, b = _pair()
    assert a.fuse_ctc is True and b.fuse_ctc is False
    assert list(a.state_dict()) == list(b.state_dict())
    for (k, va), vb in zip(a.state_dict().items(), b.state_dict().values()):
        assert torch.equal(va, vb), k
    assert not any("fuse" in k for k in a.state_dict())


def test_fuse_ctc_is_a_run_time_switch():
    a, _ = _pair()
    a.fuse_ctc = False
    assert a.fuse_ctc is False
    a.fuse_ctc = True
    assert a.fuse_ctc is True and a.fuse_lstm is False        # independent of fuse_lstm
    a.fuse_lstm = True
    assert a.fuse_ctc is True and a.fuse_lstm is True
    assert sum(1 for _ in a.buffers()) == sum(1 for _ in _pair()[1].buffers())


def test_trainer_loss_and_gradients_equal_stock_on_cpu():
    import bench
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, _ = bench.MODELS["lstman4"]
    batch = bench.make_batch("lstman4", 0, 0, bs, 128)
    res = []
    for fuse in (False, True):
        tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="none", compression=False,
                     t_total=100, warmup=0.1, seed=0, device=torch.device("cpu"), model_kwargs={"fuse_ctc": fuse})
        assert tr.device.type == "cpu" and tr.net.fuse_ctc is fuse
        tr.net.train()
        torch.manual_seed(3)
        loss, _ = tr._forward_loss(batch)
        loss.backward()
        res.append([loss.detach()] + [p.grad.clone() for p in tr.net.parameters()])
        tr.close()
    for x, y in zip(*res):
        assert torch.equal(x, y)


def _case(name):
    g = torch.Generator().manual_seed(5)
    T, N, C = 12, 3, 29
    x = torch.randn(T, N, C, generator=g)
    tn = torch.tensor([12, 9, 5], dtype=torch.int32)
    ln = torch.tensor([4, 3, 2], dtype=torch.int32)
    t = torch.randint(1, C, (9,), generator=g, dtype=torch.int32)
    if name == "2d_logits":
        x = x[:, 0]
    elif name == "fp64":
        x = x.double()
    elif name == "wide_c":
        x = torch.randn(T, N, 200, generator=g)
    elif name == "many_targets":
        ln = torch.tensor([1000, 1000, 48], dtype=torch.int32)
        tn = torch.tensor([T, T, T], dtype=torch.int32)
        x = torch.randn(T, N, C, generator=g)
        t = torch.randint(1, C, (2048,), generator=g, dtype=torch.int32)
    elif name == "padded_targets":
        t = torch.randint(1, C, (N, 4), generator=g)
    return x, t, tn, ln


@pytest.mark.parametrize("case", ["cpu", "no_extension", "2d_logits", "fp64", "wide_c", "many_targets",
                                  "padded_targets"])
def test_fallbacks_call_the_stock_expression(case):
    x, t, tn, ln = _case(case)
    if case == "2d_logits":                  # stock refuses 2-D log-probs with 1-D targets, and so does the fallback
        with mock.patch.object(fused_ctc.F, "ctc_loss", wraps=F.ctc_loss) as cl, pytest.raises(Exception):
            fused_ctc.ctc_loss(x, t, tn, ln)
        assert cl.call_count == 1
        return
    outs = []
    for fused in (True, False):
        xi = x.clone().requires_grad_(True)
        if fused:
            with mock.patch.object(fused_ctc.F, "ctc_loss", wraps=F.ctc_loss) as cl, \
                    mock.patch.object(fused_ctc.F, "log_softmax", wraps=F.log_softmax) as ls, \
                    mock.patch.object(ext, "available", return_value=case != "no_extension"):
                loss = fused_ctc.ctc_loss(xi, t, tn, ln)
            assert cl.call_count == 1 and ls.call_count == 1
            assert cl.call_args.kwargs == {"blank": 0, "reduction": "sum", "zero_infinity": True}
            assert ls.call_args.args[1] == -1
            assert [a.dtype for a in cl.call_args.args[1:]] == [torch.int64] * 3
            assert cl.call_args.args[0].dtype == torch.float32
        else:
            loss = F.ctc_loss(F.log_softmax(xi, -1).float(), t.long(), tn.long(), ln.long(), blank=0,
                              reduction="sum", zero_infinity=True)
        loss.backward()
        outs.append((loss.detach(), xi.grad))
    (la, ga), (lb, gb) = outs
    assert torch.equal(la, lb)
    assert torch.equal(ga, gb)


def test_cli_fused_ctc_flag():
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "lstman4", "--fused-ctc"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstman4", {"fuse_ctc": True})
    args = p.parse_args(["--dnn", "lstman4", "--fused-ctc", "--fused-lstm"])
    assert cli.model_args(args) == ("lstman4", {"fuse_lstm": True, "fuse_ctc": True})
    assert cli.model_args(p.parse_args(["--dnn", "lstman4"])) == ("lstman4", {})
    for bad in (["--dnn", "vgg16", "--fused-ctc"], ["--dnn", "lstm", "--fused-ctc"]):
        with pytest.raises(SystemExit):
            cli.main(bad)
