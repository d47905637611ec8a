"""Padded AN4 batches on the CPU: ``data.pad_an4_batch``'s shapes, zero tails, lengths and target capacity, the
rounding of T_b, the Trainer's ``an4_pad_multiple`` (a padded step equals the unpadded one at m = 1 on the CPU), the
device-lengths errors of ``DeepSpeech.forward``, the ``--an4-pad-multiple`` flag, and padding's one effect on the stock
model: with the batch-norm statistics frozen, a batch padded to m = 32 gives the unpadded loss, logits and gradients."""
import pytest
import torch
import torch.nn as nn

from oktopk_b200.models import create_net
from oktopk_b200.train import cli
from oktopk_b200.train import data as D


def _batch(B=3, T=150, seed=0, tsizes=(12, 9, 5)):
    g = torch.Generator().manual_seed(seed)
    inputs = torch.randn(B, 1, 161, T, generator=g)
    in_pct = torch.tensor([1.0, 0.73, 0.41][:B])
    ts = torch.tensor(tsizes[:B], dtype=torch.int32)
    targets = torch.randint(1, 29, (int(ts.sum()),), generator=g, dtype=torch.int32)
    return inputs, targets, in_pct, ts


def _out_frames(T):
    return (T - 1) // 2 + 1


@pytest.mark.parametrize("T,m,Tb", [(150, 1, 150), (150, 16, 160), (160, 16, 160), (161, 32, 192), (1, 64, 64),
                                    (400, 64, 448)])
def test_padded_frames_round_up(T, m, Tb):
    assert D.an4_padded_frames(T, m) == Tb


@pytest.mark.parametrize("m", [1, 16, 32, 64])
def test_staging_shapes_zero_tails_and_lengths(m):
    inputs, targets, in_pct, tsizes = _batch()
    p = D.pad_an4_batch((inputs, targets, in_pct, tsizes), m, _out_frames)
    B, T = inputs.size(0), inputs.size(3)
    Tb = D.an4_padded_frames(T, m)
    assert p.inputs.shape == (B, 1, 161, Tb)
    assert torch.equal(p.inputs[..., :T], inputs) and torch.all(p.inputs[..., T:] == 0)
    assert p.lengths.dtype == torch.int32
    assert torch.equal(p.lengths, (in_pct * T).int())               # the eager formula on the unpadded T
    cap = min(B * _out_frames(Tb), 2047)
    assert p.targets.shape == (cap,) and p.targets.dtype == torch.int32
    n = targets.numel()
    assert p.ntargets == n and not p.over_capacity
    assert torch.equal(p.targets[:n], targets) and torch.all(p.targets[n:] == 0)
    assert torch.equal(p.tsizes, tsizes)


def test_lengths_are_clamped_into_the_tensor():
    inputs, targets, _, tsizes = _batch()
    p = D.pad_an4_batch((inputs, targets, torch.tensor([1.5, 0.0, 0.5]), tsizes), 32, _out_frames)
    assert p.lengths.tolist() == [150, 1, 75]


def test_capacity_is_capped_at_the_fused_ctc_limit_and_overflow_is_flagged():
    assert D.an4_target_capacity(64, 200) == 2047
    assert D.an4_target_capacity(2, 75) == 150
    inputs, _, in_pct, _ = _batch(B=2, T=20, tsizes=(9, 8))
    ts = torch.tensor([9, 8], dtype=torch.int32)                 # 17 targets, capacity 2 * 10 = 20
    p = D.pad_an4_batch((inputs, torch.ones(17, dtype=torch.int32), in_pct[:2], ts), 1, _out_frames)
    assert p.targets.numel() == 20 and not p.over_capacity
    ts = torch.tensor([12, 11], dtype=torch.int32)               # 23 > 20: kept as they are, flagged
    p = D.pad_an4_batch((inputs, torch.ones(23, dtype=torch.int32), in_pct[:2], ts), 1, _out_frames)
    assert p.targets.numel() == 23 and p.over_capacity and p.ntargets == 23


def test_model_output_frames_match_the_conv_formula():
    net, _ = create_net(29, "lstman4")
    for T in (1, 2, 99, 100, 150, 192, 400, 448):
        assert int(net.get_seq_lens(torch.tensor([T]))[0]) == _out_frames(T)


def test_device_lengths_errors():
    net, _ = create_net(29, "lstman4")
    assert "CUDA" in net.device_lengths_error(False)
    assert "fuse_lstm" in net.device_lengths_error(True)
    net.fuse_lstm = True
    assert net.device_lengths_error(True) is None
    assert "fuse_lstm_autocast" in net.device_lengths_error(True, autocast=True)
    net.fuse_lstm_autocast = True
    assert net.device_lengths_error(True, autocast=True) is None
    bi, _ = create_net(29, "lstman4", bidirectional=True, fuse_lstm=True)
    assert "fuse_lstm_bidirectional" in bi.device_lengths_error(True)
    with pytest.raises(RuntimeError, match="CUDA"):
        net(torch.zeros(1, 1, 161, 20), torch.tensor([20], dtype=torch.int32), device_lengths=True)


def _trainer(m, **kw):
    from oktopk_b200.train.trainer import Trainer
    return Trainer(dnn="lstman4", dataset="an4", batch_size=2, lr=0.001, compressor="none", compression=False,
                   t_total=100, warmup=0.1, seed=0, device=torch.device("cpu"), an4_pad_multiple=m, **kw)


def test_trainer_option_and_padded_step_on_cpu():
    import bench
    batch = bench.make_batch("lstman4", 0, 0, 2, 128)
    res = []
    for m in (0, 1):
        tr = _trainer(m, model_kwargs={"fuse_ctc": True})
        assert tr.an4_pad_multiple == m and tr.graphed is None
        staged = tr.stage_batch(batch)
        assert isinstance(staged, D.PaddedAN4Batch) == (m == 1)
        assert tr.stage_batch(staged) is staged
        tr.net.train()
        loss, _ = tr._forward_loss(staged)
        loss.backward()
        res.append([loss.detach()] + [p.grad.clone() for p in tr.net.parameters()])
        tr.close()
    for x, y in zip(*res):
        assert torch.equal(x, y)


def test_trainer_rejects_the_option_off_an4():
    from oktopk_b200.train.trainer import Trainer
    with pytest.raises(ValueError, match="an4_pad_multiple"):
        Trainer(dnn="vgg16", dataset="cifar10", batch_size=2, compressor="none", compression=False,
                device=torch.device("cpu"), an4_pad_multiple=32)
    with pytest.raises(ValueError, match="an4_pad_multiple"):
        _trainer(-1)


def test_cli_flag():
    parser = cli.build_parser()
    args = parser.parse_args(["--dnn", "lstman4", "--an4-pad-multiple", "32"])
    cli.check_switch_args(parser, args)
    assert args.an4_pad_multiple == 32
    assert parser.parse_args(["--dnn", "lstman4"]).an4_pad_multiple == 0
    for argv in (["--dnn", "vgg16", "--an4-pad-multiple", "32"], ["--dnn", "lstman4", "--an4-pad-multiple", "-1"]):
        args = parser.parse_args(argv)
        with pytest.raises(SystemExit):
            cli.check_switch_args(parser, args)


def _padded_against_unpadded(device, model_kwargs, frozen_bn):
    """One batch (108 frames, lengths 108 and 75) unpadded and staged at m = 32 (128 frames) through one model:
    ``[loss, logits at each utterance's valid frames, parameter gradients]`` for each.  ``frozen_bn``: the batch-norm
    layers run on their running statistics, the rest of the model in training mode."""
    import bench
    from oktopk_b200.train.trainer import Trainer
    tr = Trainer(dnn="lstman4", dataset="an4", batch_size=2, lr=0.001, compressor="none", compression=False,
                 t_total=100, warmup=0.1, seed=0, device=torch.device(device), an4_pad_multiple=32,
                 model_kwargs=model_kwargs)
    x, tg, _, ts = (t.to(device) for t in bench.make_batch("lstman4", 0, 0, 2, 128))
    batch = (x, tg, torch.tensor([1.0, 0.7], device=device), ts)
    staged = tr.stage_batch(batch)
    assert staged.inputs.size(3) == 128 and x.size(3) == 108
    net = tr.net.train()
    if frozen_bn:
        for m in net.modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                m.eval()
    params = [p for p in net.parameters()]
    res = []
    for b in (batch, staged):
        if b is batch:
            out, lens = net(x, (b[2] * x.size(3)).int())
        else:
            out, lens = net(b.inputs, b.lengths, device_lengths=b.inputs.is_cuda)
        lens = lens.tolist()
        loss, _ = tr._forward_loss(b)
        res.append([loss.detach()] + [out[n, :L].detach() for n, L in enumerate(lens)]
                   + list(torch.autograd.grad(loss, params)))
    assert lens == [54, 38]
    tr.close()
    return res


def _max_rel_err(a, b):
    return max(((x - y).abs().max() / y.abs().max().clamp_min(1e-30)).item() for x, y in zip(a, b))


def _check_padding_semantics(device, model_kwargs):
    """Padding changes the batch-norm statistics and nothing else: with them frozen, loss, valid-frame logits and
    every gradient agree with the unpadded batch to rounding (the convolutions and GEMMs run at other widths); with
    them live, the logits move far beyond that."""
    unpadded, padded = _padded_against_unpadded(device, model_kwargs, frozen_bn=True)
    assert _max_rel_err(padded[:3], unpadded[:3]) < 1e-4
    assert _max_rel_err(padded[3:], unpadded[3:]) < 1e-3
    unpadded, padded = _padded_against_unpadded(device, model_kwargs, frozen_bn=False)
    assert _max_rel_err(padded[1:3], unpadded[1:3]) > 1e-2


def test_padding_changes_only_the_batch_norm_statistics_on_cpu():
    _check_padding_semantics("cpu", {})
