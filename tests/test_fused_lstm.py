"""The persistent LSTM recurrence kernels (``csrc/lstm.cu``, ``ops/fused_lstm.py``) on the GPU: forward and all five
gradients against a float64 CPU ``nn.LSTM`` fed the same packed sequence, no worse than stock cuDNN (TF32 off) against the
same reference; unequal, unsorted lengths with exact zeros in the padding; bitwise determinism; every fallback is the
stock layer exactly; and the whole ``lstman4`` model and a few ``Trainer`` steps with ``fuse_lstm`` on."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oktopk_b200.models import create_net
from oktopk_b200.models.deepspeech import BatchRNN
from oktopk_b200.ops import ext, fused_lstm

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _launches():
    return ext.LAUNCH_COUNT.get("lstm_forward", 0), ext.LAUNCH_COUNT.get("lstm_backward", 0)


def _run(rnn, x, lens, dy, fn):
    """fn(x, lens, rnn) -> y; returns y and the gradients of (y * dy).sum() wrt x and the four parameters."""
    x = x.detach().clone().requires_grad_(True)
    for p in rnn.parameters():
        p.grad = None
    y = fn(x, lens, rnn)
    (y * dy.to(y.dtype)).sum().backward()
    return [y.detach(), x.grad, rnn.weight_ih_l0.grad, rnn.weight_hh_l0.grad, rnn.bias_ih_l0.grad, rnn.bias_hh_l0.grad]


def _three_ways(I, H, N, T, lens, seed=0):
    torch.manual_seed(seed)
    rnn = nn.LSTM(I, H).cuda()
    x = torch.randn(T, N, I, device="cuda")
    dy = torch.randn(T, N, H, device="cuda")
    lens = torch.tensor(lens, dtype=torch.int32)
    ref64 = copy.deepcopy(rnn).double().cpu()
    ref = _run(ref64, x.double().cpu(), lens, dy.double().cpu(), fused_lstm.stock_layer)
    stock = _run(rnn, x, lens, dy, fused_lstm.stock_layer)
    n0 = _launches()
    fused = _run(rnn, x, lens, dy, fused_lstm.lstm_layer)
    n1 = _launches()
    assert n1[0] == n0[0] + 1 and n1[1] == n0[1] + 1, "the fused kernels did not run"
    return ref, stock, fused


NAMES = ["y", "dx", "dW_ih", "dW_hh", "db_ih", "db_hh"]


def _check_vs_reference(ref, stock, fused):
    for name, r, s, f in zip(NAMES, ref, stock, fused):
        es = (s.cpu().double() - r).abs().max().item()
        ef = (f.cpu().double() - r).abs().max().item()
        floor = 1e-5 * max(1.0, r.abs().max().item())
        assert ef <= 2 * es + floor, (name, ef, es, floor)


@pytest.mark.parametrize("I,H,N,T", [(1312, 800, 2, 48), (1312, 800, 2, 198), (800, 800, 2, 48), (800, 800, 2, 198),
                                     (64, 128, 5, 30), (96, 256, 32, 20), (800, 800, 9, 25), (200, 4, 3, 12),
                                     (800, 800, 32, 40), (800, 800, fused_lstm.MAX_BATCH, 30)])
def test_forward_and_gradients_against_float64(I, H, N, T):
    lens = [T] + [max(1, T - 3 * i) for i in range(1, N)]
    _check_vs_reference(*_three_ways(I, H, N, T, lens))


@pytest.mark.parametrize("N,fwd_chunks,bwd_chunks", [(32, 1, 3), (fused_lstm.MAX_BATCH, 2, 7)])
def test_large_batches_stage_the_operand_in_chunks(N, fwd_chunks, bwd_chunks):
    """At H = 800 the backward kernel holds at most 11 rows of dgates and the forward kernel 41 rows of h at a time, so
    these batches take several staging passes per step (the shapes above check their results)."""
    g = fused_lstm._device_geometry(800, N, torch.device("cuda"))
    assert g is not None
    assert -(-N // g.fwd_rows) == fwd_chunks and -(-N // g.bwd_rows) == bwd_chunks, g


def test_unequal_unsorted_lengths_and_zero_padding():
    T = 40
    lens = [7, T, 1, T - 3, 12]
    ref, stock, fused = _three_ways(160, 800, len(lens), T, lens, seed=3)
    _check_vs_reference(ref, stock, fused)
    y, dx = fused[0], fused[1]
    for b, L in enumerate(lens):
        assert torch.all(y[L:, b] == 0) and torch.all(dx[L:, b] == 0), b
        assert y[:L, b].abs().max() > 0 and dx[:L, b].abs().max() > 0, b


def test_deterministic():
    torch.manual_seed(5)
    layer = BatchRNN(800, 800, fuse=True).cuda()
    x = torch.randn(123, 2, 800, device="cuda")
    lens = torch.tensor([123, 77], dtype=torch.int32)
    dy = torch.randn(123, 2, 800, device="cuda")
    outs = []
    for _ in range(2):
        xi = x.clone().requires_grad_(True)
        y = layer(xi, lens)
        grads = torch.autograd.grad(y, [xi] + list(layer.parameters()), dy)
        outs.append([y] + list(grads))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def _fallback_case(case):
    torch.manual_seed(7)
    I, H, N, T = 48, 64, 3, 10
    kw = {}
    dev, dtype = "cuda", torch.float32
    if case == "bidirectional":
        kw["bidirectional"] = True
    elif case == "ptb_hidden":
        I, H = 64, 1500
    elif case == "batch_over_limit":
        N = fused_lstm.MAX_BATCH + 1
    elif case == "cpu":
        dev = "cpu"
    elif case == "fp64":
        dtype = torch.float64
    layer = BatchRNN(I, H, **kw).to(dev, dtype)
    x = torch.randn(T, N, I, device=dev, dtype=dtype)
    lens = torch.randint(1, T + 1, (N,), dtype=torch.int32)
    lens[0] = T
    return layer, x, lens


@pytest.mark.parametrize("case", ["cpu", "autocast", "bidirectional", "ptb_hidden", "batch_over_limit", "fp64"])
def test_fallbacks_are_the_stock_layer(case):
    layer, x, lens = _fallback_case(case)
    outs = []
    for fuse in (False, True):
        layer.fuse = fuse
        for p in layer.parameters():
            p.grad = None
        xi = x.clone().requires_grad_(True)
        n0 = _launches()
        if case == "autocast":
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = layer(xi, lens)
        else:
            y = layer(xi, lens)
        y.float().square().sum().backward()
        assert _launches() == n0, case
        outs.append([y.detach(), xi.grad] + [p.grad for p in layer.parameters()])
    for a, b in zip(*outs):
        assert torch.equal(a, b), case


def _ctc_loss(out, targets, out_lens, tsizes):
    logp = F.log_softmax(out.transpose(0, 1), dim=-1)
    return F.ctc_loss(logp, targets, out_lens.long(), tsizes, blank=0, reduction="sum",
                      zero_infinity=True) / out.size(0)


def test_whole_model_against_float64():
    torch.manual_seed(0)
    net, _ = create_net(29, "lstman4")
    ref = copy.deepcopy(net).double()
    stock = net.cuda()
    fused = copy.deepcopy(stock)
    fused.fuse_lstm = True
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 1, 161, 400, generator=g)
    lens = torch.tensor([400, 290], dtype=torch.int32)
    tsizes = torch.tensor([20, 14])
    targets = torch.randint(1, 29, (int(tsizes.sum()),), generator=g)
    res = {}
    for name, m, dev, dt in (("ref", ref, "cpu", torch.float64), ("stock", stock, "cuda", torch.float32),
                             ("fused", fused, "cuda", torch.float32)):
        m.train()
        n0 = _launches()
        out, out_lens = m(x.to(dev, dt), lens)
        loss = _ctc_loss(out, targets.to(dev), out_lens.to(dev), tsizes.to(dev))
        loss.backward()
        ran = _launches() != n0
        assert ran == (name == "fused"), name
        res[name] = [out.detach().cpu().double(), loss.detach().cpu().double()] + \
                    [p.grad.detach().cpu().double() for p in m.parameters()]
    assert torch.isfinite(res["fused"][1])
    names = ["logits", "ctc"] + [n for n, _ in net.named_parameters()]
    for i, name in enumerate(names):
        r = res["ref"][i]
        es = (res["stock"][i] - r).abs().max().item()
        ef = (res["fused"][i] - r).abs().max().item()
        floor = 1e-5 * max(1.0, r.abs().max().item())
        assert ef <= 2 * es + floor, (name, ef, es, floor)


def test_trainer_steps_follow_stock():
    import bench
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    losses = {}
    for fuse in (False, True):
        cfg = okt.preset(preset, density=0.001, warmup_iters=2)
        tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                     t_total=100000, warmup=0.1, seed=0, model_kwargs={"fuse_lstm": fuse})
        assert tr.net.fuse_lstm is fuse
        seq = []
        n0 = _launches()
        for i in range(5):
            batch = tuple(t.to(tr.device) for t in bench.make_batch("lstman4", i, 0, bs, 128))
            tr.net.train()
            tr.optimizer.zero_grad()
            loss, _ = tr._forward_loss(batch)
            loss.backward()
            tr.update_model()
            seq.append(float(loss))
        assert (_launches() != n0) == fuse
        assert all(torch.isfinite(p).all() for p in tr.net.parameters())
        tr.close()
        losses[fuse] = seq
    for a, b in zip(losses[False], losses[True]):
        assert b == pytest.approx(a, rel=2e-2), losses
