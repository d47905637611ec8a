"""The PTB model's fused LSTM switch on the CPU: the stacked-layer kernels' geometry, ``PTBLSTM(fuse_lstm, fuse_xent)``
through ``create_net`` and ``Trainer``, unchanged ``state_dict`` keys, the stock fallback on the CPU, and the
``--fused-lstm-lm`` / ``--fused-xent`` flags for ``--dnn lstm``."""
from unittest import mock

import pytest
import torch
import torch.nn as nn

from oktopk_b200.models import PTBLSTM, create_net
from oktopk_b200.ops import fused_lstm
from oktopk_b200.ops.fused_lstm import MAX_BATCH, LstmSeqGeometry, lstm_seq_geometry
from oktopk_b200.train import cli

H100_SMS, H100_SMEM = 132, 232448


def test_ptb_layer_geometry():
    """H = 1500, N = 20: u = 12 on 125 CTAs.  Forward: 48 rows of W_hh and all 20 rows of h_{t-1}, 1512 elements apart
    (1500 padded to 1504, plus 8), one K split of the 2 x 6 tiles; backward: 12 columns of W_hh, 6008 apart, and 6 rows of
    dgates_{t+1} at a time, eight K splits of the 1 x 2 tiles."""
    g = lstm_seq_geometry(1500, 20, H100_SMS, H100_SMEM)
    fwd = 2 * (48 + 20) * 1512 + 4 * (1 * 20 * 48 + 48 * 20 + 12 * 20)
    bwd = 2 * (12 + 6) * 6008 + 4 * (8 * 6 * 12 + 2 * 12 * 20)
    assert g == LstmSeqGeometry(12, 125, 20, 6, fwd, bwd)
    assert fwd == 214272 and bwd == 220512
    assert 2 * (12 + 7) * 6008 + 4 * (8 * 7 * 12 + 2 * 12 * 20) > H100_SMEM          # a seventh row does not fit


@pytest.mark.parametrize("H,N", [(1500, 20), (800, 20), (800, MAX_BATCH), (64, 1), (64, 7), (1500, MAX_BATCH)])
def test_geometry_accepts(H, N):
    g = lstm_seq_geometry(H, N, H100_SMS, H100_SMEM)
    assert g is not None and g.grid <= H100_SMS and max(g.fwd_smem, g.bwd_smem) <= H100_SMEM
    assert 1 <= g.bwd_rows <= g.fwd_rows <= N and g.units * g.grid >= H > g.units * (g.grid - 1)


@pytest.mark.parametrize("H,N,sms", [(2000, 20, H100_SMS), (1500, 20, H100_SMS // 2), (1502, 20, H100_SMS),
                                     (0, 20, H100_SMS), (1500, 0, H100_SMS), (1500, MAX_BATCH + 1, H100_SMS),
                                     (800, 20, 0)])
def test_geometry_rejects(H, N, sms):
    """Too many units per CTA for the W_hh slice to fit (H = 2000; H = 1500 on half the SMs), H not a multiple of 4,
    and out-of-range sizes."""
    assert lstm_seq_geometry(H, N, sms, H100_SMEM) is None


def test_gate_reads_the_device_properties():
    """``_stack_ok`` sizes the layer on the tensor's device: with a CUDA tensor under bf16 autocast, an H100's properties
    accept the PTB layer and a device with half its shared memory rejects it."""
    rnn = nn.LSTM(1500, 1500, num_layers=2)
    x = mock.Mock(spec=torch.Tensor, is_cuda=True, dtype=torch.float32, device=torch.device("cpu"))
    x.dim.return_value = 3
    x.size.side_effect = lambda i: (35, 20, 1500)[i]
    for smem, ok in ((H100_SMEM, True), (H100_SMEM // 2, False)):
        props = mock.Mock(multi_processor_count=H100_SMS, shared_memory_per_block_optin=smem)
        with mock.patch.object(torch, "is_autocast_enabled", return_value=True), \
                mock.patch.object(torch, "get_autocast_dtype", return_value=torch.bfloat16), \
                mock.patch.object(fused_lstm.ext, "available", return_value=True), \
                mock.patch.object(torch.cuda, "get_device_properties", return_value=props):
            got = fused_lstm._stack_ok(x, None, rnn)
        assert (got is not None) is ok
        if ok:
            assert got == (lstm_seq_geometry(1500, 20, H100_SMS, H100_SMEM), torch.bfloat16)


def test_create_net_carries_both_keywords_and_keys_are_unchanged():
    torch.manual_seed(0)
    a, _ = create_net(1000, "lstm", vocab_size=1000, fuse_lstm=True, fuse_xent=True)
    torch.manual_seed(0)
    b, _ = create_net(1000, "lstm", vocab_size=1000)
    assert a.fuse_lstm is True and a.fuse_xent is True
    assert b.fuse_lstm is False and b.fuse_xent is False
    assert list(a.state_dict()) == list(b.state_dict())
    assert [n for n, _ in a.named_parameters()] == [n for n, _ in b.named_parameters()]
    assert all(torch.equal(u, v) for u, v in zip(a.state_dict().values(), b.state_dict().values()))
    b.fuse_lstm = True
    b.fuse_xent = True
    assert b.fuse_lstm and b.fuse_xent


def test_trainer_carries_both_keywords():
    from oktopk_b200.train.trainer import Trainer
    tr = Trainer(dnn="lstm", dataset="ptb", batch_size=2, lr=22, compressor="oktopk", density=0.02,
                 device=torch.device("cpu"), model_kwargs={"fuse_lstm": True, "fuse_xent": True})
    try:
        assert isinstance(tr.net, PTBLSTM) and tr.net.fuse_lstm is True and tr.net.fuse_xent is True
    finally:
        tr.close()


def test_cpu_is_exactly_the_stock_model():
    """On the CPU the switch runs ``nn.LSTM`` itself: the same output, state and gradients, bit for bit, in training
    (dropout between layers drawn by the module, under the same seed) and in eval."""
    torch.manual_seed(0)
    a = PTBLSTM(vocab_size=100, embedding_dim=32, num_layers=2, fuse_lstm=True)
    b = PTBLSTM(vocab_size=100, embedding_dim=32, num_layers=2)
    b.load_state_dict(a.state_dict())
    x = torch.randint(0, 100, (6, 3))
    hid = tuple(torch.randn(2, 3, 32) for _ in range(2))
    for train in (True, False):
        outs = []
        for m in (a, b):
            m.train(train)
            m.zero_grad()
            torch.manual_seed(5)
            out, (h, c) = m(x, hid)
            (out.square().sum() + h.sum() + c.sum()).backward()
            outs.append([out, h, c] + [p.grad for p in m.parameters()])
        for u, v in zip(*outs):
            assert torch.equal(u, v)


def test_lstm_stack_falls_back_to_the_module_off_the_gpu():
    rnn = nn.LSTM(8, 8, num_layers=3)
    x = torch.randn(4, 2, 8)
    with mock.patch.object(rnn, "forward", wraps=rnn.forward) as fwd:
        y, (h, c) = fused_lstm.lstm_stack(x, None, rnn, 0.0, False)
    assert fwd.call_count == 1 and h.shape == c.shape == (3, 2, 8)
    rnn64 = nn.LSTM(8, 8, num_layers=2).double()
    x64 = torch.randn(4, 2, 8, dtype=torch.float64)
    y, _ = fused_lstm.lstm_stack(x64, None, rnn64, 0.0, False)
    assert torch.equal(y, rnn64(x64)[0])


def test_cli_fused_lstm_lm_and_fused_xent_flags():
    p = cli.build_parser()
    for argv in (["--dnn", "lstm", "--bf16", "--fused-lstm-lm"], ["--dnn", "lstm", "--fp16", "--fused-lstm-lm"]):
        args = p.parse_args(argv)
        cli.check_switch_args(p, args)
        assert cli.model_args(args) == ("lstm", {"fuse_lstm": True})
    args = p.parse_args(["--dnn", "lstm", "--bf16", "--fused-lstm-lm", "--fused-xent"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstm", {"fuse_xent": True, "fuse_lstm": True})
    args = p.parse_args(["--dnn", "lstm", "--fused-xent"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstm", {"fuse_xent": True})
    for bad in (["--dnn", "lstm", "--fused-lstm-lm"],                              # no 16-bit autocast
                ["--dnn", "lstman4", "--bf16", "--fused-lstm-lm"],
                ["--dnn", "vgg16", "--fp16", "--fused-lstm-lm"],
                ["--dnn", "lstm", "--bf16", "--fused-lstm"],                        # --fused-lstm stays lstman4-only
                ["--dnn", "lstman4", "--fused-xent"]):
        with pytest.raises(SystemExit):
            cli.main(bad)
