"""The fused LSTM's bidirectional switch on the CPU: the per-direction geometry the kernels are launched with (half the
SMs each), ``net.fuse_lstm_bidirectional`` sets every layer and changes nothing where the kernels do not run,
``create_net`` carries the keyword, and the ``--bidirectional`` / ``--fused-lstm-bidirectional`` flags."""
import pytest
import torch

from oktopk_b200.models import create_net, lstman4
from oktopk_b200.ops.fused_lstm import LstmGeometry, lstm_geometry
from oktopk_b200.train import cli

H100_SMS, H100_SMEM = 132, 232448
HALF = H100_SMS // 2


def _geom(H, N, u, fr, br, elem):
    w = 4 * elem * u * H
    return LstmGeometry(u, -(-H // u), fr, br, w + 4 * 5 * u * N + elem * H * fr, w + 4 * 2 * u * N + 4 * elem * H * br)


@pytest.mark.parametrize("elem,N,fr,br", [(4, 2, 2, 2), (4, 64, 15, 4), (2, 2, 2, 2), (2, 64, 64, 22)])
def test_h800_per_direction_geometry(elem, N, fr, br):
    """H = 800 on half of an H100's SMs: u = 13 on 62 CTAs per direction, 124 in all, with 166.4 KB of fp32 W_hh per CTA
    (83.2 KB in 16 bits)."""
    g = lstm_geometry(800, N, HALF, H100_SMEM, elem)
    assert g == _geom(800, N, 13, fr, br, elem)
    assert 2 * g.grid <= H100_SMS and max(g.fwd_smem, g.bwd_smem) <= H100_SMEM


@pytest.mark.parametrize("elem", [4, 2])
def test_h1500_does_not_fit_two_directions(elem):
    """u = 23 on 66 SMs: 552 KB of fp32 W_hh per CTA, 276 KB in 16 bits."""
    for N in (1, 20, 64):
        assert lstm_geometry(1500, N, HALF, H100_SMEM, elem) is None


def _pair(**kw):
    torch.manual_seed(0)
    a, _ = create_net(29, "lstman4", bidirectional=True, fuse_lstm=True, fuse_lstm_bidirectional=True, **kw)
    torch.manual_seed(0)
    b, _ = create_net(29, "lstman4", bidirectional=True, **kw)
    return a, b


def test_bidirectional_network_has_no_lookahead_and_the_same_keys():
    a, b = _pair()
    assert a.lookahead is None and all(m.rnn.bidirectional for m in a.rnns)
    assert list(a.state_dict()) == list(b.state_dict())
    assert [n for n, _ in a.named_parameters()] == [n for n, _ in b.named_parameters()]
    assert any(n.endswith("weight_hh_l0_reverse") for n, _ in a.named_parameters())


def test_property_sets_every_layer():
    a, b = _pair()
    assert a.fuse_lstm_bidirectional is True and all(m.fuse_bidirectional for m in a.rnns)
    assert b.fuse_lstm_bidirectional is False and not any(m.fuse_bidirectional for m in b.rnns)
    b.fuse_lstm_bidirectional = True
    assert b.fuse_lstm_bidirectional is True and all(m.fuse_bidirectional for m in b.rnns)
    assert b.fuse_lstm is False and b.fuse_lstm_autocast is False           # the switches are independent
    b.rnns[2].fuse_bidirectional = False
    assert b.fuse_lstm_bidirectional is False
    a.fuse_lstm_bidirectional = False
    assert a.fuse_lstm is True and not any(m.fuse_bidirectional for m in a.rnns)


def test_switch_on_cpu_is_the_stock_network():
    a, b = _pair(hidden_size=64, hidden_layers=3)
    a.fuse_lstm_autocast = True
    g = torch.Generator().manual_seed(1)
    x, lens = torch.randn(3, 1, 161, 90, generator=g), torch.tensor([90, 41, 67], dtype=torch.int32)
    outs = []
    for net in (a, b):
        net.train()
        o, _ = net(x, lens)
        o.square().sum().backward()
        outs.append([o.detach()] + [p.grad for p in net.parameters()])
    assert len(outs[0]) == len(outs[1])
    for va, vb in zip(*outs):
        assert torch.equal(va, vb)


def test_create_net_and_factory_carry_the_keyword():
    assert create_net(29, "lstman4", bidirectional=True, fuse_lstm_bidirectional=True)[0].fuse_lstm_bidirectional
    assert create_net(29, "lstman4", fuse_lstm=True)[0].fuse_lstm_bidirectional is False
    net = lstman4(hidden_size=16, hidden_layers=2, bidirectional=True, fuse_lstm=True, fuse_lstm_bidirectional=True)
    assert net.fuse_lstm is True and net.fuse_lstm_bidirectional is True and net.lookahead is None


def test_cli_bidirectional_flags(capsys):
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "lstman4", "--bidirectional"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstman4", {"bidirectional": True})
    args = p.parse_args(["--dnn", "lstman4", "--fused-lstm", "--bidirectional", "--fused-lstm-bidirectional"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstman4", {"fuse_lstm": True, "bidirectional": True,
                                                "fuse_lstm_bidirectional": True})
    args = p.parse_args(["--dnn", "lstman4", "--fused-lstm", "--bidirectional", "--fused-lstm-bidirectional",
                         "--fused-lstm-autocast", "--bf16"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args)[1] == {"fuse_lstm": True, "fuse_lstm_autocast": True, "bidirectional": True,
                                       "fuse_lstm_bidirectional": True}
    for bad, word in ((["--dnn", "vgg16", "--bidirectional"], "--bidirectional applies to lstman4"),
                      (["--dnn", "lstman4", "--bidirectional", "--fused-lstm-bidirectional"], "needs --fused-lstm"),
                      (["--dnn", "lstman4", "--fused-lstm", "--fused-lstm-bidirectional"], "needs --bidirectional")):
        with pytest.raises(SystemExit):
            cli.main(bad)
        assert word in capsys.readouterr().err
