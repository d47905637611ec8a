"""Bidirectional layers on the persistent LSTM recurrence kernels (``lstm_layer(..., bidirectional=True)``) on the GPU:
each half of a two-direction launch is bit for bit the one-direction kernel (the reverse half on each utterance reversed
within its length); forward and all nine gradients against a float64 CPU ``nn.LSTM(bidirectional=True)``, no worse
than the stock layer, in fp32 and under bf16 / fp16 autocast; zero padding and determinism; every fallback is the stock
layer exactly; fp16 overflow in the reverse direction; the whole bidirectional ``lstman4`` model and a few ``Trainer``
steps."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oktopk_b200.models import create_net
from oktopk_b200.models.deepspeech import BatchRNN
from oktopk_b200.ops import ext, fused_lstm
from oktopk_b200.ops.ext import DTYPE_CODE

pytestmark = pytest.mark.gpu

DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
NAMES = ["y", "dx", "dW_ih", "dW_hh", "db_ih", "db_hh", "dW_ih_rev", "dW_hh_rev", "db_ih_rev", "db_hh_rev"]


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _launches():
    return ext.LAUNCH_COUNT.get("lstm_forward", 0), ext.LAUNCH_COUNT.get("lstm_backward", 0)


# ---------------------------------------------------------------- the extension entry points, called directly
def _forward(gx, whh, lens):
    """gx [dirs, T, N, 4H]; whh: one W_hh per direction.  One launch."""
    C = ext.require()
    dirs, T, N = gx.size(0), gx.size(1), gx.size(2)
    H = whh[0].size(1)
    geom = fused_lstm._device_geometry(H, N, gx.device, gx.element_size(), dirs)
    y = torch.empty(dirs, T, N, H, device="cuda", dtype=gx.dtype)
    gates = torch.empty(dirs, T, N, 4 * H, device="cuda")
    cs = torch.empty(dirs, T, N, H, device="cuda")
    bar = torch.zeros(dirs, dtype=torch.int64, device="cuda")
    C.lstm_forward(gx.data_ptr(), whh[0].data_ptr(), lens.data_ptr(), y.data_ptr(), gates.data_ptr(), cs.data_ptr(),
                   bar.data_ptr(), T, N, H, geom.units, geom.fwd_rows, torch.cuda.current_stream().cuda_stream,
                   DTYPE_CODE[gx.dtype], whh[1].data_ptr() if dirs == 2 else 0)
    return y, gates, cs


def _backward(dy, gates, cs, whh, lens):
    """dy [T, N, H], the same for every direction; gates, cs [dirs, T, N, .].  One launch."""
    C = ext.require()
    dirs = gates.size(0)
    T, N, H = dy.shape
    geom = fused_lstm._device_geometry(H, N, dy.device, dy.element_size(), dirs)
    dg = torch.empty(dirs, T, N, 4 * H, device="cuda", dtype=dy.dtype)
    bar = torch.zeros(dirs, dtype=torch.int64, device="cuda")
    C.lstm_backward(dy.data_ptr(), gates.data_ptr(), cs.data_ptr(), whh[0].data_ptr(), lens.data_ptr(), dg.data_ptr(),
                    bar.data_ptr(), T, N, H, geom.units, geom.bwd_rows, torch.cuda.current_stream().cuda_stream,
                    DTYPE_CODE[dy.dtype], whh[1].data_ptr() if dirs == 2 else 0)
    return dg


def _flip(a, lens):
    """Each utterance n of the time-major a [T, N, K] reversed within its length lens[n]; the padding stays in place.
    Its own inverse."""
    T, N = a.size(0), a.size(1)
    t = torch.arange(T, device=a.device).view(T, 1)
    L = lens.to(a.device).long().view(1, N)
    idx = torch.where(t < L, L - 1 - t, t)
    return a.gather(0, idx.view(T, N, 1).expand_as(a))


EXACT = [(1, 23, [23]), (2, 23, [9, 23]), (33, 23, None), (64, 23, None), (2, 1, [1, 1]), (5, 1, [1] * 5)]


def _lengths(N, T, lens):
    if lens is not None:
        return lens
    g = torch.Generator().manual_seed(N)
    out = torch.randint(1, T + 1, (N,), generator=g)
    out[N // 3], out[N // 2] = 1, T                             # unsorted, with the extremes
    return out.tolist()


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("N,T,lens", EXACT)
def test_each_direction_is_the_one_direction_kernel(dt, N, T, lens):
    dt = DTYPES[dt]
    H = 800
    torch.manual_seed(N + T)
    lens = torch.tensor(_lengths(N, T, lens), dtype=torch.int32, device="cuda")
    gx = (2 * torch.randn(2, T, N, 4 * H, device="cuda")).to(dt)
    whh = [(torch.randn(4 * H, H, device="cuda") / H ** 0.5).to(dt) for _ in range(2)]
    dy = torch.randn(T, N, H, device="cuda").to(dt)
    n0 = _launches()
    y, gates, cs = _forward(gx, whh, lens)
    dg = _backward(dy, gates, cs, whh, lens)
    assert _launches() == (n0[0] + 1, n0[1] + 1)

    yf, gf, cf = _forward(gx[:1].contiguous(), whh[:1], lens)
    dgf = _backward(dy, gf, cf, whh[:1], lens)
    assert torch.equal(y[0], yf[0]) and torch.equal(gates[0], gf[0]) and torch.equal(cs[0], cf[0])
    assert torch.equal(dg[0], dgf[0])

    yr, gr, cr = _forward(_flip(gx[1], lens).unsqueeze(0).contiguous(), whh[1:], lens)
    dgr = _backward(_flip(dy, lens).contiguous(), gr, cr, whh[1:], lens)
    assert torch.equal(y[1], _flip(yr[0], lens)) and torch.equal(gates[1], _flip(gr[0], lens))
    assert torch.equal(cs[1], _flip(cr[0], lens))
    assert torch.equal(dg[1], _flip(dgr[0], lens))

    assert y[1].float().abs().max() > 0 and dg[1].float().abs().max() > 0
    for b, L in enumerate(lens.tolist()):
        for tsr in (y[1], gates[1], cs[1], dg[1]):
            assert torch.all(tsr[L:, b] == 0), b


def test_entry_points_check_the_reverse_w_hh():
    C = ext.require()
    H, N, T = 64, 2, 3
    gx = torch.zeros(2, T, N, 4 * H, device="cuda")
    whh = torch.zeros(2, 4 * H * H + 4, device="cuda")
    y, cs = torch.empty(2, T, N, H, device="cuda"), torch.empty(2, T, N, H, device="cuda")
    gates = torch.empty(2, T, N, 4 * H, device="cuda")
    lens = torch.full((N,), T, dtype=torch.int32, device="cuda")
    bar = torch.zeros(2, dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match="aligned"):
        C.lstm_forward(gx.data_ptr(), whh[0].data_ptr(), lens.data_ptr(), y.data_ptr(), gates.data_ptr(),
                       cs.data_ptr(), bar.data_ptr(), T, N, H, 1, 1, torch.cuda.current_stream().cuda_stream, 0,
                       whh[1].data_ptr() + 4)
    with pytest.raises(RuntimeError, match="bar"):
        C.lstm_forward(gx.data_ptr(), whh[0].data_ptr(), lens.data_ptr(), y.data_ptr(), gates.data_ptr(),
                       cs.data_ptr(), bar.data_ptr() + 4, T, N, H, 1, 1, torch.cuda.current_stream().cuda_stream, 0,
                       whh[1].data_ptr())


# ---------------------------------------------------------------- against float64
def _fused(dt):
    def fn(x, lens, rnn):
        return fused_lstm.lstm_layer(x, lens, rnn, autocast=dt is not None, bidirectional=True)
    return fn


def _run(rnn, x, lens, dy, fn, dt=None):
    """fn(x, lens, rnn) -> y, under ``dt`` autocast when given; y and the gradients of (y * dy).sum() wrt x and the
    eight parameters."""
    x = x.detach().clone().requires_grad_(True)
    for p in rnn.parameters():
        p.grad = None
    with torch.autocast("cuda", dtype=dt, enabled=dt is not None):
        y = fn(x, lens, rnn)
    y.backward(dy.to(y.dtype))
    return [y.detach(), x.grad] + [p.grad for p in rnn.parameters()]


def _three_ways(I, H, N, T, lens, dt, seed=0):
    """dt None: fp32."""
    torch.manual_seed(seed)
    rnn = nn.LSTM(I, H, bidirectional=True).cuda()
    x = torch.randn(T, N, I, device="cuda")
    dy = torch.randn(T, N, H, device="cuda")
    lens = torch.tensor(lens, dtype=torch.int32)
    ref = _run(copy.deepcopy(rnn).double().cpu(), x.double().cpu(), lens, dy.double().cpu(), fused_lstm.stock_layer)
    n0 = _launches()
    stock = _run(rnn, x, lens, dy, fused_lstm.stock_layer, dt)
    assert _launches() == n0
    fused = _run(rnn, x, lens, dy, _fused(dt), dt)
    assert _launches() == (n0[0] + 1, n0[1] + 1), "the fused kernels did not run"
    return ref, stock, fused


def _check_vs_reference(ref, stock, fused, dt, names=NAMES):
    """err_fused <= 2 err_stock + floor: in fp32 (dt None) the floor is 1e-5 of the reference's largest magnitude, as in
    test_fused_lstm; in 16 bits 2 ulps of dt there, as in test_fused_lstm_autocast (both at 1 for smaller tensors)."""
    bad = []
    for name, r, s, f in zip(names, ref, stock, fused):
        es = (s.cpu().double() - r).abs().max().item()
        ef = (f.cpu().double() - r).abs().max().item()
        floor = (1e-5 if dt is None else 2 * torch.finfo(dt).eps) * max(1.0, r.abs().max().item())
        if not ef <= 2 * es + floor:
            bad.append((name, ef, es, floor))
    assert not bad, bad


SHAPES = [(1312, 800, 2, 48), (1312, 800, 2, 198), (800, 800, 2, 48), (800, 800, 2, 198), (64, 128, 5, 30),
          (200, 4, 3, 12), (96, 256, 33, 20)]


@pytest.mark.parametrize("dt,I,H,N,T", [(d,) + s for d in DTYPES for s in SHAPES]
                         + [("fp32", 800, 800, fused_lstm.MAX_BATCH, 30)])
def test_forward_and_gradients_against_float64(dt, I, H, N, T):
    dt = None if dt == "fp32" else DTYPES[dt]
    lens = [max(1, T - 3 * i) for i in range(N)]
    lens[-1], lens[0] = lens[0], lens[-1]                  # unsorted
    ref, stock, fused = _three_ways(I, H, N, T, lens, dt)
    _check_vs_reference(ref, stock, fused, dt)
    assert fused[0].dtype == (dt or torch.float32)
    assert all(g.dtype == torch.float32 for g in fused[1:])
    assert len({g.data_ptr() for g in fused[2:]}) == 8          # eight gradients, none aliased


def test_zero_padding_and_determinism():
    T = 40
    lens = [7, T, 1, T - 3, 12]
    ref, stock, fused = _three_ways(160, 800, len(lens), T, lens, None, seed=3)
    _check_vs_reference(ref, stock, fused, None)
    y, dx = fused[0], fused[1]
    for b, L in enumerate(lens):
        assert torch.all(y[L:, b] == 0) and torch.all(dx[L:, b] == 0), b
        assert y[:L, b].abs().max() > 0 and dx[:L, b].abs().max() > 0, b

    torch.manual_seed(5)
    layer = BatchRNN(800, 800, bidirectional=True, fuse=True, fuse_bidirectional=True).cuda()
    x = torch.randn(123, 2, 800, device="cuda")
    lens = torch.tensor([77, 123], dtype=torch.int32)
    dy = torch.randn(123, 2, 800, device="cuda")
    outs = []
    for _ in range(2):
        xi = x.clone().requires_grad_(True)
        n0 = _launches()
        y = layer(xi, lens)
        grads = torch.autograd.grad(y, [xi] + list(layer.parameters()), dy)
        assert _launches() == (n0[0] + 1, n0[1] + 1)
        outs.append([y] + list(grads))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ---------------------------------------------------------------- fallbacks
def _fallback_case(case):
    torch.manual_seed(7)
    I, H, N, T = 48, 64, 3, 10
    dev, dtype = "cuda", torch.float32
    if case == "ptb_hidden":
        I, H = 64, 1500
    elif case == "batch_over_limit":
        N = fused_lstm.MAX_BATCH + 1
    elif case == "cpu":
        dev = "cpu"
    elif case == "fp64":
        dtype = torch.float64
    layer = BatchRNN(I, H, bidirectional=True).to(dev, dtype)
    x = torch.randn(T, N, I, device=dev, dtype=dtype)
    lens = torch.randint(1, T + 1, (N,), dtype=torch.int32)
    lens[0] = T
    return layer, x, lens


@pytest.mark.parametrize("case", ["switch_off", "cpu", "fp64", "batch_over_limit", "ptb_hidden"])
def test_fallbacks_are_the_stock_layer(case):
    """``ptb_hidden``: H = 1500 needs 552 KB of fp32 W_hh per CTA on half the SMs, so both directions go stock rather
    than being split into two launches."""
    layer, x, lens = _fallback_case(case)
    outs = []
    for fuse in (False, True):
        layer.fuse = fuse
        layer.fuse_bidirectional = fuse and case != "switch_off"
        for p in layer.parameters():
            p.grad = None
        xi = x.clone().requires_grad_(True)
        n0 = _launches()
        y = layer(xi, lens)
        y.square().sum().backward()
        assert _launches() == n0, case
        outs.append([y.detach(), xi.grad] + [p.grad for p in layer.parameters()])
    for a, b in zip(*outs):
        assert torch.equal(a, b), case


# ---------------------------------------------------------------- fp16 range
def test_fp16_overflow_in_the_reverse_direction_reaches_dgates_as_inf():
    """Only the reverse direction saturates (forget gate open, the carried dc grows by about dy / 2 a step, dy = 60000):
    its dgates pass 65504 and must be stored as inf, so that its weight gradients are non-finite and loss scaling skips
    the step.  The forward direction, with its forget gate shut, stays finite."""
    I, H, N, T = 16, 8, 2, 12
    rnn = nn.LSTM(I, H, bidirectional=True).cuda()
    with torch.no_grad():
        for p in rnn.parameters():
            p.zero_()
        rnn.bias_ih_l0[H:2 * H] = -10.0
        rnn.bias_ih_l0_reverse[H:2 * H] = 10.0
        rnn.bias_ih_l0_reverse[2 * H:3 * H] = 0.05
    torch.manual_seed(0)
    x = 0.01 * torch.randn(T, N, I, device="cuda")          # keeps the forward direction's fp16 dW_ih GEMM in range
    dy = torch.full((T, N, H), 60000.0, device="cuda")
    lens = torch.full((N,), T, dtype=torch.int32)
    n0 = _launches()
    out = _run(rnn, x, lens, dy, _fused(torch.float16), torch.float16)
    assert _launches() == (n0[0] + 1, n0[1] + 1)
    assert torch.isfinite(out[0]).all()
    for name, g in zip(NAMES[2:], out[2:]):
        assert torch.isfinite(g).all() == (not name.endswith("_rev")), name


# ---------------------------------------------------------------- whole model, trainer
def _ctc_loss(out, targets, out_lens, tsizes):
    logp = F.log_softmax(out.transpose(0, 1), dim=-1)
    return F.ctc_loss(logp, targets, out_lens.long(), tsizes, blank=0, reduction="sum",
                      zero_infinity=True) / out.size(0)


def test_whole_model_against_float64():
    torch.manual_seed(0)
    net, _ = create_net(29, "lstman4", bidirectional=True)
    ref = copy.deepcopy(net).double()
    stock = net.cuda()
    fused = copy.deepcopy(stock)
    fused.fuse_lstm = fused.fuse_lstm_bidirectional = True
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 1, 161, 400, generator=g)
    lens = torch.tensor([290, 400], dtype=torch.int32)
    tsizes = torch.tensor([14, 20])
    targets = torch.randint(1, 29, (int(tsizes.sum()),), generator=g)
    res = {}
    for name, m, dev, dt in (("ref", ref, "cpu", torch.float64), ("stock", stock, "cuda", torch.float32),
                             ("fused", fused, "cuda", torch.float32)):
        m.train()
        n0 = _launches()
        out, out_lens = m(x.to(dev, dt), lens)
        loss = _ctc_loss(out, targets.to(dev), out_lens.to(dev), tsizes.to(dev))
        loss.backward()
        n1 = _launches()
        assert (n1[0] - n0[0], n1[1] - n0[1]) == ((5, 5) if name == "fused" else (0, 0)), name
        res[name] = [out.detach().cpu().double(), loss.detach().cpu().double()] + \
                    [p.grad.detach().cpu().double() for p in m.parameters()]
    assert torch.isfinite(res["fused"][1])
    names = ["logits", "ctc"] + [n for n, _ in net.named_parameters()]
    _check_vs_reference(res["ref"], res["stock"], res["fused"], None, names)


def test_trainer_steps_follow_stock():
    import bench
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    losses = {}
    for fuse in (False, True):
        cfg = okt.preset(preset, density=0.001, warmup_iters=2)
        tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                     t_total=100000, warmup=0.1, seed=0,
                     model_kwargs={"bidirectional": True, "fuse_lstm": fuse, "fuse_lstm_bidirectional": fuse})
        assert tr.net.lookahead is None and tr.net.fuse_lstm_bidirectional is fuse
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
        n1 = _launches()
        assert (n1[0] - n0[0], n1[1] - n0[1]) == ((25, 25) if fuse else (0, 0))
        assert all(torch.isfinite(p).all() for p in tr.net.parameters())
        tr.close()
        losses[fuse] = seq
    for a, b in zip(losses[False], losses[True]):
        assert b == pytest.approx(a, rel=2e-2), losses
