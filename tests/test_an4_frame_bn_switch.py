"""The AN4 DeepSpeech model's fused batch-norm switch on the CPU: ``create_net(29, "lstman4", fuse_bn=True)`` is the
stock network (outputs, gradients, parameters, ``state_dict`` keys), ``net.fuse_bn`` is a run-time switch, the op's
fallbacks are the stock modules, and the ``--fused-bn`` flag maps to ``fuse_bn`` for lstman4 only."""
import pytest
import torch
import torch.nn as nn

from oktopk_b200.models import create_net
from oktopk_b200.ops import fused_frame_bn
from oktopk_b200.train import cli


def _pair(**kw):
    torch.manual_seed(0)
    a, _ = create_net(29, "lstman4", fuse_bn=True, **kw)
    torch.manual_seed(0)
    b, _ = create_net(29, "lstman4", **kw)
    return a, b


def test_fuse_bn_keeps_the_stock_network():
    a, b = _pair()
    assert a.fuse_bn is True and b.fuse_bn is False
    assert list(a.state_dict()) == list(b.state_dict())
    for (k, va), vb in zip(a.state_dict().items(), b.state_dict().values()):
        assert torch.equal(va, vb), k
    assert not any("fuse" in k for k in a.state_dict())
    assert [n for n, _ in a.named_parameters()] == [n for n, _ in b.named_parameters()]
    assert [n for n, _ in a.named_buffers()] == [n for n, _ in b.named_buffers()]


@pytest.mark.parametrize("bidirectional", [False, True])
def test_fuse_bn_on_the_cpu_is_the_stock_network(bidirectional):
    a, b = _pair(bidirectional=bidirectional)
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


def test_fuse_bn_is_a_run_time_switch():
    a, _ = _pair()
    a.fuse_bn = False
    assert a.fuse_bn is False
    a.fuse_bn = True
    assert a.fuse_bn is True and a.fuse_lstm is False and a.fuse_ctc is False
    a.fuse_lstm = True
    assert a.fuse_bn is True and a.fuse_lstm is True
    assert create_net(29, "lstman4")[0].fuse_bn is False


def test_the_ops_fall_back_to_the_stock_modules_on_the_cpu():
    torch.manual_seed(2)
    conv_bn = nn.BatchNorm2d(4)
    x = torch.randn(3, 4, 5, 9)
    lens = torch.tensor([9, 4, 6], dtype=torch.int32)
    ref_bn = nn.BatchNorm2d(4)
    t = torch.arange(9).view(1, 1, 1, -1)
    mask = t >= lens.view(-1, 1, 1, 1)
    ref = nn.Hardtanh(0, 20, inplace=True)(ref_bn(x.masked_fill(mask, 0)).masked_fill(mask, 0)).masked_fill(mask, 0)
    assert torch.equal(fused_frame_bn.conv_block_bn(x, conv_bn, lens), ref)
    assert torch.equal(conv_bn.running_var, ref_bn.running_var)
    seq = nn.BatchNorm1d(4)
    y = torch.randn(7, 3, 4)
    assert torch.equal(fused_frame_bn.seq_bn(y, seq, lens), nn.BatchNorm1d(4)(y.reshape(21, 4)).view(7, 3, 4))


def test_create_net_and_the_cli_flag():
    assert create_net(29, "lstman4", fuse_bn=True, fuse_lstm=True)[0].fuse_bn is True
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "lstman4", "--fused-bn"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstman4", {"fuse_bn": True})
    args = p.parse_args(["--dnn", "lstman4", "--fused-bn", "--fused-lstm", "--fused-ctc", "--an4-pad-multiple", "32"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstman4", {"fuse_bn": True, "fuse_lstm": True, "fuse_ctc": True})
    for bad in (["--dnn", "vgg16", "--fused-bn"], ["--dnn", "lstm", "--fused-bn"], ["--dnn", "bert_base", "--fused-bn"],
                ["--dnn", "resnet50", "--fused-bn"], ["--dnn", "resnet20", "--fp16", "--fused-bn-fp16"]):
        with pytest.raises(SystemExit):
            cli.main(bad)


@pytest.mark.parametrize("lens", [[9, 4], [[9, 4, 6]], [9.0, 4.0, 6.0], None], ids=["short", "2d", "float", "none"])
def test_the_ops_refuse_lengths_that_are_not_one_per_utterance(lens):
    lens = None if lens is None else torch.tensor(lens)
    with pytest.raises(ValueError, match="lens"):
        fused_frame_bn.conv_block_bn(torch.randn(3, 4, 5, 9), nn.BatchNorm2d(4), lens)
    with pytest.raises(ValueError, match="lens"):
        fused_frame_bn.seq_bn(torch.randn(9, 3, 4), nn.BatchNorm1d(4), lens)
