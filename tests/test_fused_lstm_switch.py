"""The AN4 DeepSpeech model's fused LSTM switch on the CPU: ``create_net(29, "lstman4", fuse_lstm=True)`` is the stock
network wherever the fused kernels do not run (outputs, gradients, ``state_dict`` keys, parameter order),
``net.fuse_lstm`` sets every layer, the geometry the kernels are launched with, and the ``--fused-lstm`` flag."""
import pytest
import torch

from oktopk_b200.models import create_net
from oktopk_b200.models.deepspeech import BatchRNN
from oktopk_b200.ops import fused_lstm
from oktopk_b200.ops.fused_lstm import lstm_geometry
from oktopk_b200.train import cli

H100_SMS, H100_SMEM = 132, 227 * 1024


def _pair():
    torch.manual_seed(0)
    a, _ = create_net(29, "lstman4", fuse_lstm=True)
    torch.manual_seed(0)
    b, _ = create_net(29, "lstman4")
    return a, b


def _utterances():
    g = torch.Generator().manual_seed(1)
    return torch.randn(3, 1, 161, 90, generator=g), torch.tensor([90, 41, 67], dtype=torch.int32)


def test_fuse_lstm_on_cpu_is_the_stock_network():
    a, b = _pair()
    assert a.fuse_lstm is True and b.fuse_lstm is False
    assert list(a.state_dict()) == list(b.state_dict())
    assert [n for n, _ in a.named_parameters()] == [n for n, _ in b.named_parameters()]
    for (k, va), vb in zip(a.state_dict().items(), b.state_dict().values()):
        assert torch.equal(va, vb), k
    x, lens = _utterances()
    a.eval(); b.eval()
    with torch.no_grad():
        (oa, la), (ob, lb) = a(x, lens), b(x, lens)
    assert torch.equal(oa, ob) and torch.equal(la, lb)
    a.train(); b.train()
    oa, _ = a(x, lens)
    ob, _ = b(x, lens)
    assert torch.equal(oa, ob)
    oa.square().sum().backward()
    ob.square().sum().backward()
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        assert torch.equal(pa.grad, pb.grad), n


def test_fuse_lstm_property_sets_every_layer():
    a, b = _pair()
    assert all(m.fuse for m in a.rnns) and not any(m.fuse for m in b.rnns)
    a.fuse_lstm = False
    assert a.fuse_lstm is False and not any(m.fuse for m in a.rnns)
    b.fuse_lstm = True
    assert b.fuse_lstm is True and all(m.fuse for m in b.rnns)
    b.rnns[2].fuse = False
    assert b.fuse_lstm is False
    assert not any("fuse" in k for k in a.state_dict())
    assert sum(1 for _ in a.buffers()) == sum(1 for _ in b.buffers())


@pytest.mark.parametrize("bidirectional", [False, True])
def test_lstm_layer_falls_back_to_the_stock_layer_on_cpu(bidirectional):
    torch.manual_seed(0)
    layer = BatchRNN(24, 16, bidirectional=bidirectional)
    x = torch.randn(9, 3, 24)
    lens = torch.tensor([9, 1, 5], dtype=torch.int32)
    layer.fuse = False
    ref = layer(x, lens)
    layer.fuse = True
    assert torch.equal(layer(x, lens), ref)
    assert torch.equal(fused_lstm.lstm_layer(x, lens, layer.rnn), fused_lstm.stock_layer(x, lens, layer.rnn))
    assert ref[5:, 2].abs().max() == 0 and ref[1:, 1].abs().max() == 0


def test_geometry_accepts_deepspeech_and_rejects_ptb():
    for n in (1, 2, 8, 16, 31, 32):
        g = lstm_geometry(800, n, H100_SMS, H100_SMEM)
        assert g is not None, n
        assert g.units == 7 and g.grid == 115 and g.grid <= H100_SMS
        assert 1 <= g.fwd_rows <= n and 1 <= g.bwd_rows <= n
        assert max(g.fwd_smem, g.bwd_smem) <= H100_SMEM
        assert g.fwd_smem == 4 * (4 * 7 * 800 + g.fwd_rows * 800 + 5 * 7 * n)
        assert g.bwd_smem == 4 * (4 * 7 * 800 + g.bwd_rows * 4 * 800 + 2 * 7 * n)
    assert lstm_geometry(800, 2, H100_SMS, H100_SMEM).fwd_rows == 2
    assert lstm_geometry(1500, 2, H100_SMS, H100_SMEM) is None        # the PTB model: 288 KB of W_hh per CTA
    assert lstm_geometry(800, fused_lstm.MAX_BATCH + 1, H100_SMS, H100_SMEM) is None
    assert lstm_geometry(802, 2, H100_SMS, H100_SMEM) is None          # not a multiple of 4
    assert lstm_geometry(800, 0, H100_SMS, H100_SMEM) is None
    assert lstm_geometry(800, 2, 66, H100_SMEM).units == 13           # fewer SMs: more units per CTA
    assert lstm_geometry(800, 2, 40, H100_SMEM) is None               # 20 units: 256 KB of W_hh per CTA
    small = lstm_geometry(128, 4, H100_SMS, H100_SMEM)
    assert small.units == 1 and small.grid == 128


def test_cli_fused_lstm_flag():
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "lstman4", "--fused-lstm"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstman4", {"fuse_lstm": True})
    args = p.parse_args(["--dnn", "lstman4"])
    assert cli.model_args(args) == ("lstman4", {})
    for bad in (["--dnn", "vgg16", "--fused-lstm"], ["--dnn", "lstm", "--fused-lstm"],
                ["--module", "models.bert12.depth=4", "--fused-lstm"]):
        with pytest.raises(SystemExit):
            cli.main(bad)
