"""The AN4 DeepSpeech model's fused look-ahead switch on the CPU: ``create_net(29, "lstman4", fuse_lookahead=True)`` is
the stock network (outputs, gradients, parameters, ``state_dict`` keys), ``net.fuse_lookahead`` is a run-time switch,
the op falls back to the stock module, the bidirectional network refuses the switch, and the ``--fused-lookahead`` flag
maps to ``fuse_lookahead`` for lstman4 only."""
import pytest
import torch
import torch.nn as nn

from oktopk_b200.models import DNNS, create_net
from oktopk_b200.models.deepspeech import Lookahead
from oktopk_b200.models.switches import SWITCHES
from oktopk_b200.ops import fused_lookahead
from oktopk_b200.train import cli


def _pair(**kw):
    torch.manual_seed(0)
    a, _ = create_net(29, "lstman4", fuse_lookahead=True, **kw)
    torch.manual_seed(0)
    b, _ = create_net(29, "lstman4", **kw)
    return a, b


def test_the_switch_table_entry():
    (sw,) = [s for s in SWITCHES if s.flag == "--fused-lookahead"]
    assert sw.keywords == ("fuse_lookahead",) and sw.models == ("lstman4",)
    assert sw.needs == () and sw.precision is None and sw.type is None and sw.default is False


def test_fuse_lookahead_keeps_the_stock_network():
    a, b = _pair()
    assert a.fuse_lookahead is True and b.fuse_lookahead is False
    assert list(a.state_dict()) == list(b.state_dict())
    for (k, va), vb in zip(a.state_dict().items(), b.state_dict().values()):
        assert torch.equal(va, vb), k
    assert not any("fuse" in k for k in a.state_dict())
    assert [n for n, _ in a.named_parameters()] == [n for n, _ in b.named_parameters()]
    b.load_state_dict(a.state_dict())
    a.load_state_dict(b.state_dict())


@pytest.mark.parametrize("fuse_bn", [False, True])
def test_fuse_lookahead_on_the_cpu_is_the_stock_network(fuse_bn):
    a, b = _pair(fuse_bn=fuse_bn)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 1, 161, 60, generator=g)
    lens = torch.tensor([60, 41], dtype=torch.int32)
    w = torch.randn(2, 30, 29, generator=g)
    res = []
    for net in (a, b):
        net.train()
        out, out_lens = net(x, lens)
        (out * w).sum().backward()
        res.append([out, out_lens] + [p.grad for p in net.parameters()] + list(net.buffers()))
    for u, v in zip(*res):
        assert torch.equal(u, v)
    for net in (a, b):
        net.eval()
    with torch.no_grad():
        assert torch.equal(a(x, lens)[0], b(x, lens)[0])


def test_fuse_lookahead_is_a_run_time_switch():
    a, _ = _pair()
    a.fuse_lookahead = False
    assert a.fuse_lookahead is False
    a.fuse_lookahead = True
    assert a.fuse_lookahead is True and a.fuse_bn is False and a.fuse_lstm is False and a.fuse_ctc is False
    net = create_net(29, "lstman4")[0]
    assert net.fuse_lookahead is False and isinstance(net.lookahead[0], Lookahead)


def test_the_bidirectional_network_refuses_the_switch():
    with pytest.raises(ValueError, match="fuse_lookahead"):
        create_net(29, "lstman4", bidirectional=True, fuse_lookahead=True)
    net = create_net(29, "lstman4", bidirectional=True)[0]
    assert net.fuse_lookahead is False
    with pytest.raises(ValueError, match="fuse_lookahead"):
        net.fuse_lookahead = True
    net.fuse_lookahead = False                                   # off stays allowed


def test_the_op_falls_back_to_the_stock_module_on_the_cpu():
    torch.manual_seed(2)
    la = nn.Sequential(Lookahead(16, context=5), nn.Hardtanh(0, 20, inplace=True))
    with torch.no_grad():
        la[0].weight.mul_(30)                                    # both clamps in play
    x = torch.randn(9, 3, 16, requires_grad=True)
    lens = torch.tensor([9, 4, 6], dtype=torch.int32)
    y = fused_lookahead.lookahead_hardtanh(x, la[0].weight, lens)
    ref = la(x)
    assert torch.equal(y, ref)
    assert (ref == 0).any() and (ref == 20).any()
    dy = torch.randn_like(y)
    gx, gw = torch.autograd.grad(y, [x, la[0].weight], dy)
    rx, rw = torch.autograd.grad(ref, [x, la[0].weight], dy)
    assert torch.equal(gx, rx) and torch.equal(gw, rw)


@pytest.mark.parametrize("lens", [[9, 4], [[9, 4, 6]], [9.0, 4.0, 6.0], None], ids=["short", "2d", "float", "none"])
def test_the_op_refuses_lengths_that_are_not_one_per_utterance(lens):
    lens = None if lens is None else torch.tensor(lens)
    with pytest.raises(ValueError, match="lens"):
        fused_lookahead.lookahead_hardtanh(torch.randn(9, 3, 4), torch.randn(4, 3), lens)


def test_create_net_and_the_cli_flag():
    assert create_net(29, "lstman4", fuse_lookahead=True, fuse_bn=True)[0].fuse_lookahead is True
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "lstman4", "--fused-lookahead"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstman4", {"fuse_lookahead": True})
    args = p.parse_args(["--dnn", "lstman4", "--fused-lookahead", "--fused-bn", "--fused-lstm", "--fused-ctc",
                         "--an4-pad-multiple", "32"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstman4", {"fuse_lookahead": True, "fuse_bn": True, "fuse_lstm": True,
                                                "fuse_ctc": True})
    assert cli.model_args(p.parse_args(["--dnn", "lstman4"])) == ("lstman4", {})
    for bad in (["--dnn", "vgg16", "--fused-lookahead"], ["--dnn", "lstm", "--fused-lookahead"],
                ["--dnn", "bert_base", "--fused-lookahead"], ["--dnn", "resnet20", "--fused-lookahead"]):
        with pytest.raises(SystemExit):
            cli.main(bad)


def test_create_net_refuses_the_keyword_for_other_models():
    for dnn in (d for d in DNNS if d != "lstman4"):             # refused before anything is built
        with pytest.raises(ValueError, match="fuse_lookahead"):
            create_net(10, dnn, fuse_lookahead=True)
