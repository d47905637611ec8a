"""The PTB model's fp32 fused LSTM switch on the CPU: the fp32 stacked-layer kernels' geometry, the gate,
``PTBLSTM(fuse_lstm_fp32)`` through ``create_net`` and ``Trainer``, unchanged ``state_dict`` keys, the stock model on the
CPU, and the ``--fused-lstm-lm-fp32`` flag."""
from unittest import mock

import pytest
import torch
import torch.nn as nn

from oktopk_b200.models import PTBLSTM, create_net
from oktopk_b200.ops import fused_lstm
from oktopk_b200.ops.fused_lstm import MAX_BATCH, LstmSeqF32Geometry, lstm_seq_f32_geometry
from oktopk_b200.train import cli

H100_SMS, H100_SMEM = 132, 232448


def test_ptb_layer_geometry():
    """H = 1500, N = 20: u = 12 on 125 CTAs, 256-column chunks of the step operand in two buffers of 20 rows 260 floats
    apart.  Forward: rows of W_hh 1508 floats apart (1500 rounded up to 8, plus 4), 6 tiles of 8 weight rows, so two K
    splits; 29 of the 48 rows fit.  Backward: rows of W_hh^T 6004 apart, 2 tiles, eight K splits; 7 of 12 fit.  The
    other 19 and 5 rows of every CTA are read from L2 at each step: 19 x 1500 x 4 B and 5 x 6000 x 4 B per CTA."""
    g = lstm_seq_f32_geometry(1500, 20, H100_SMS, H100_SMEM)
    stage = 2 * 20 * 260
    fwd = 4 * (29 * 1508 + stage + 2 * 20 * 48 + 48 * 20 + 12 * 20)
    bwd = 4 * (7 * 6004 + stage + 8 * 20 * 12 + 2 * 12 * 20)
    assert g == LstmSeqF32Geometry(12, 125, 29, 256, 7, 256, fwd, bwd, 125 * 19 * 1500 * 4, 125 * 5 * 6000 * 4)
    assert fwd == 229008 and bwd == 219312
    assert fwd + 4 * 1508 > H100_SMEM and bwd + 4 * 6004 > H100_SMEM          # one more row fits in neither
    assert g.fwd_l2_bytes == 14_250_000 and g.bwd_l2_bytes == 15_000_000


@pytest.mark.parametrize("H,N", [(1500, 20), (800, 20), (800, MAX_BATCH), (64, 1), (64, 7), (1500, MAX_BATCH),
                                 (4224, 20)])
def test_geometry_accepts(H, N):
    g = lstm_seq_f32_geometry(H, N, H100_SMS, H100_SMEM)
    assert g is not None and g.grid <= H100_SMS and max(g.fwd_smem, g.bwd_smem) <= H100_SMEM
    assert 0 <= g.fwd_r_on <= 4 * g.units and 0 <= g.bwd_r_on <= g.units
    assert g.fwd_kc % 8 == 0 and g.bwd_kc % 8 == 0 and g.units * g.grid >= H > g.units * (g.grid - 1)


def test_small_layers_keep_all_weights_on_chip():
    for H, N in ((64, 7), (800, 20)):
        g = lstm_seq_f32_geometry(H, N, H100_SMS, H100_SMEM)
        assert g.fwd_r_on == 4 * g.units and g.bwd_r_on == g.units and g.fwd_l2_bytes == g.bwd_l2_bytes == 0


@pytest.mark.parametrize("H,N,sms,smem", [(4228, 20, H100_SMS, H100_SMEM), (1502, 20, H100_SMS, H100_SMEM),
                                          (0, 20, H100_SMS, H100_SMEM), (1500, 0, H100_SMS, H100_SMEM),
                                          (1500, MAX_BATCH + 1, H100_SMS, H100_SMEM), (800, 20, 0, H100_SMEM),
                                          (1500, 20, H100_SMS, 40000)])
def test_geometry_rejects(H, N, sms, smem):
    """More than 128 weight rows per CTA (H = 4228: u = 33), H not a multiple of 4, out-of-range sizes, and too little
    shared memory for the staged chunks alone."""
    assert lstm_seq_f32_geometry(H, N, sms, smem) is None


def _gate(rnn, smem, autocast=False, fp32=True):
    x = mock.Mock(spec=torch.Tensor, is_cuda=True, dtype=torch.float32, device=torch.device("cpu"))
    x.dim.return_value = 3
    x.size.side_effect = lambda i: (35, 20, 1500)[i]
    props = mock.Mock(multi_processor_count=H100_SMS, shared_memory_per_block_optin=smem)
    with mock.patch.object(torch, "is_autocast_enabled", return_value=autocast), \
            mock.patch.object(torch, "get_autocast_dtype", return_value=torch.bfloat16), \
            mock.patch.object(fused_lstm.ext, "available", return_value=True), \
            mock.patch.object(torch.cuda, "get_device_properties", return_value=props):
        return fused_lstm._stack_ok(x, None, rnn, fp32)


def test_gate_reads_the_device_properties():
    """With a CUDA fp32 tensor and ``fp32=True``, an H100's properties accept the PTB layer with the fp32 geometry, and
    a device with too little shared memory for the staged chunks rejects it.  Without ``fp32`` fp32 is not taken, and
    under autocast ``fp32`` changes nothing: the 16-bit geometry."""
    rnn = nn.LSTM(1500, 1500, num_layers=2)
    assert _gate(rnn, H100_SMEM) == (lstm_seq_f32_geometry(1500, 20, H100_SMS, H100_SMEM), torch.float32)
    assert _gate(rnn, 40000) is None
    assert _gate(rnn, H100_SMEM, fp32=False) is None
    assert _gate(rnn, H100_SMEM, autocast=True) == _gate(rnn, H100_SMEM, autocast=True, fp32=False) == (
        fused_lstm.lstm_seq_geometry(1500, 20, H100_SMS, H100_SMEM), torch.bfloat16)


def test_create_net_and_trainer_carry_the_keyword_and_keys_are_unchanged():
    from oktopk_b200.train.trainer import Trainer
    torch.manual_seed(0)
    a, _ = create_net(1000, "lstm", vocab_size=1000, fuse_lstm=True, fuse_lstm_fp32=True)
    torch.manual_seed(0)
    b, _ = create_net(1000, "lstm", vocab_size=1000)
    assert a.fuse_lstm is True and a.fuse_lstm_fp32 is True and b.fuse_lstm_fp32 is False
    assert list(a.state_dict()) == list(b.state_dict())
    assert [n for n, _ in a.named_parameters()] == [n for n, _ in b.named_parameters()]
    assert [n for n, _ in a.named_buffers()] == [n for n, _ in b.named_buffers()]
    assert all(torch.equal(u, v) for u, v in zip(a.state_dict().values(), b.state_dict().values()))
    tr = Trainer(dnn="lstm", dataset="ptb", batch_size=2, lr=22, compressor="oktopk", density=0.02,
                 device=torch.device("cpu"), model_kwargs={"fuse_lstm": True, "fuse_lstm_fp32": True})
    try:
        assert isinstance(tr.net, PTBLSTM) and tr.net.fuse_lstm is True and tr.net.fuse_lstm_fp32 is True
    finally:
        tr.close()


@pytest.mark.parametrize("flags", [(True, True), (False, True), (True, False)])
def test_cpu_is_exactly_the_stock_model(flags):
    """On the CPU the switches run ``nn.LSTM`` itself: the same output, state and gradients, bit for bit, in training
    (dropout between layers drawn by the module, under the same seed) and in eval."""
    torch.manual_seed(0)
    a = PTBLSTM(vocab_size=100, embedding_dim=32, num_layers=2, fuse_lstm=flags[0], fuse_lstm_fp32=flags[1])
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


def test_cli_fused_lstm_lm_fp32_flag():
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "lstm", "--fused-lstm-lm-fp32"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstm", {"fuse_lstm": True, "fuse_lstm_fp32": True})
    args = p.parse_args(["--dnn", "lstm", "--fused-lstm-lm-fp32", "--fused-xent"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("lstm", {"fuse_xent": True, "fuse_lstm": True, "fuse_lstm_fp32": True})
    args = p.parse_args(["--dnn", "lstm", "--bf16", "--fused-lstm-lm"])
    assert "fuse_lstm_fp32" not in cli.model_args(args)[1]
    for bad, msg in ((["--dnn", "lstm", "--bf16", "--fused-lstm-lm-fp32"], "use --fused-lstm-lm"),
                     (["--dnn", "lstm", "--fp16", "--fused-lstm-lm-fp32"], "use --fused-lstm-lm"),
                     (["--dnn", "lstman4", "--fused-lstm-lm-fp32"], "applies to lstm"),
                     (["--dnn", "vgg16", "--fused-lstm-lm-fp32"], "applies to lstm"),
                     (["--dnn", "lstm", "--fused-lstm-lm"], "needs --bf16 or --fp16")):
        args = p.parse_args(bad)
        with mock.patch.object(p, "error", side_effect=SystemExit) as err, pytest.raises(SystemExit):
            cli.check_switch_args(p, args)
        assert msg in err.call_args[0][0], (bad, err.call_args)
