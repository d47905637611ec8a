"""The fused LSTM's autocast switch on the CPU: the 16-bit geometry the kernels are launched with, ``net.fuse_lstm_autocast``
sets every layer and changes nothing where the kernels do not run, ``create_net`` carries the keyword, and the
``--fused-lstm-autocast`` flag."""
import pytest
import torch

from oktopk_b200.models import create_net, lstman4
from oktopk_b200.ops.fused_lstm import MAX_BATCH, LstmGeometry, lstm_geometry
from oktopk_b200.train import cli

H100_SMS, H100_SMEM = 132, 232448


def test_elem_4_is_the_four_argument_geometry():
    for H in (4, 128, 256, 800, 1024, 1500, 2048):
        for N in (1, 2, 20, 32, MAX_BATCH):
            for sms, smem in ((H100_SMS, H100_SMEM), (66, H100_SMEM), (108, 166912)):
                assert lstm_geometry(H, N, sms, smem, elem=4) == lstm_geometry(H, N, sms, smem), (H, N, sms)


def test_elem_2_reference_rows():
    # H = 800: 44.8 KB of W_hh per CTA; all 64 rows of h fit, dgates 28 rows at a time
    assert lstm_geometry(800, 64, H100_SMS, H100_SMEM, elem=2) == LstmGeometry(
        7, 115, 64, 28, 8 * 7 * 800 + 2 * 800 * 64 + 4 * 5 * 7 * 64, 8 * 7 * 800 + 8 * 800 * 28 + 4 * 2 * 7 * 64)
    # the PTB-sized layer: 144 KB of W_hh per CTA, which fp32 (288 KB) cannot hold
    assert lstm_geometry(1500, 20, H100_SMS, H100_SMEM, elem=2) == LstmGeometry(
        12, 125, 20, 7, 8 * 12 * 1500 + 2 * 1500 * 20 + 4 * 5 * 12 * 20, 8 * 12 * 1500 + 8 * 1500 * 7 + 4 * 2 * 12 * 20)
    assert lstm_geometry(1500, 20, H100_SMS, H100_SMEM, elem=4) is None
    for H, N in ((800, 2), (800, 64), (1500, 20), (128, 5)):
        g = lstm_geometry(H, N, H100_SMS, H100_SMEM, elem=2)
        assert max(g.fwd_smem, g.bwd_smem) <= H100_SMEM and g.grid <= H100_SMS
        assert g.fwd_smem % 4 == 0 and g.bwd_smem % 4 == 0


def test_elem_2_rejects_what_elem_4_rejects():
    assert lstm_geometry(802, 2, H100_SMS, H100_SMEM, elem=2) is None          # not a multiple of 4
    assert lstm_geometry(800, MAX_BATCH + 1, H100_SMS, H100_SMEM, elem=2) is None
    assert lstm_geometry(800, 0, H100_SMS, H100_SMEM, elem=2) is None
    assert lstm_geometry(800, 2, 20, H100_SMEM, elem=2) is None                # 40 units: 256 KB of W_hh per CTA
    assert lstm_geometry(800, 2, H100_SMS, H100_SMEM, elem=3) is None


def _pair():
    torch.manual_seed(0)
    a, _ = create_net(29, "lstman4", fuse_lstm=True, fuse_lstm_autocast=True)
    torch.manual_seed(0)
    b, _ = create_net(29, "lstman4")
    return a, b


def test_fuse_lstm_autocast_property_sets_every_layer():
    a, b = _pair()
    assert a.fuse_lstm_autocast is True and all(m.fuse_autocast for m in a.rnns)
    assert b.fuse_lstm_autocast is False and not any(m.fuse_autocast for m in b.rnns)
    b.fuse_lstm_autocast = True
    assert b.fuse_lstm_autocast is True and all(m.fuse_autocast for m in b.rnns)
    assert b.fuse_lstm is False                      # the two switches are independent
    b.rnns[3].fuse_autocast = False
    assert b.fuse_lstm_autocast is False
    a.fuse_lstm_autocast = False
    assert a.fuse_lstm is True and not any(m.fuse_autocast for m in a.rnns)
    assert list(a.state_dict()) == list(b.state_dict())
    assert [n for n, _ in a.named_parameters()] == [n for n, _ in b.named_parameters()]


def test_both_switches_on_cpu_are_the_stock_network():
    a, b = _pair()
    g = torch.Generator().manual_seed(1)
    x, lens = torch.randn(3, 1, 161, 90, generator=g), torch.tensor([90, 41, 67], dtype=torch.int32)
    outs = []
    for net in (a, b):
        net.train()
        o, _ = net(x, lens)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            o16, _ = net(x, lens)
        o.square().sum().backward()
        outs.append([o.detach(), o16.detach()] + [p.grad for p in net.parameters()])
    for va, vb in zip(*outs):
        assert torch.equal(va, vb)


def test_create_net_and_factory_carry_the_keyword():
    assert create_net(29, "lstman4", fuse_lstm_autocast=True)[0].fuse_lstm_autocast is True
    assert create_net(29, "lstman4", fuse_lstm=True)[0].fuse_lstm_autocast is False
    net = lstman4(hidden_size=16, hidden_layers=2, fuse_lstm=True, fuse_lstm_autocast=True)
    assert net.fuse_lstm is True and net.fuse_lstm_autocast is True


def test_cli_fused_lstm_autocast_flag(capsys):
    p = cli.build_parser()
    for prec in ("--bf16", "--fp16"):
        args = p.parse_args(["--dnn", "lstman4", "--fused-lstm", "--fused-lstm-autocast", prec])
        cli.check_switch_args(p, args)
        assert cli.model_args(args) == ("lstman4", {"fuse_lstm": True, "fuse_lstm_autocast": True})
    for bad, word in ((["--dnn", "lstman4", "--fused-lstm-autocast", "--bf16"], "needs --fused-lstm"),
                      (["--dnn", "lstman4", "--fused-lstm", "--fused-lstm-autocast"], "needs --bf16 or --fp16")):
        with pytest.raises(SystemExit):
            cli.main(bad)
        assert word in capsys.readouterr().err
