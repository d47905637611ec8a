"""The 16-bit forms of the persistent LSTM recurrence kernels (``lstm_layer(..., autocast=True)`` under bf16 / fp16
autocast) on the GPU: a 16-bit launch is the fp32 kernel on the widened operands, rounded; y and the gradients follow a
torch loop that rounds at the kernels' rounding points; forward and all five gradients against a float64 CPU ``nn.LSTM``,
no worse than stock cuDNN under the same autocast; lengths, dtypes, determinism; fp16 overflow and subnormals; the gate;
the whole ``lstman4`` model and a few ``Trainer`` steps."""
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

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
NAMES = ["y", "dx", "dW_ih", "dW_hh", "db_ih", "db_hh"]


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _launches():
    return ext.LAUNCH_COUNT.get("lstm_forward", 0), ext.LAUNCH_COUNT.get("lstm_backward", 0)


def _fused(x, lens, rnn):
    return fused_lstm.lstm_layer(x, lens, rnn, autocast=True)


def _run(rnn, x, lens, dy, fn, dt=None):
    """fn(x, lens, rnn) -> y, under ``dt`` autocast when given; returns y and the gradients of (y * dy).sum() wrt x and
    the four parameters."""
    x = x.detach().clone().requires_grad_(True)
    for p in rnn.parameters():
        p.grad = None
    with torch.autocast("cuda", dtype=dt, enabled=dt is not None):
        y = fn(x, lens, rnn)
    y.backward(dy.to(y.dtype))
    return [y.detach(), x.grad, rnn.weight_ih_l0.grad, rnn.weight_hh_l0.grad, rnn.bias_ih_l0.grad, rnn.bias_hh_l0.grad]


# ---------------------------------------------------------------- the extension entry points, called directly
def _forward(gx, whh, lens, elem):
    C = ext.require()
    T, N, H = gx.size(0), gx.size(1), whh.size(1)
    geom = fused_lstm._device_geometry(H, N, gx.device, elem)
    y = torch.empty(T, N, H, device="cuda", dtype=gx.dtype)
    gates = torch.empty(T, N, 4 * H, device="cuda")
    cs = torch.empty(T, N, H, device="cuda")
    bar = torch.zeros(1, dtype=torch.int64, device="cuda")
    C.lstm_forward(gx.data_ptr(), whh.data_ptr(), lens.data_ptr(), y.data_ptr(), gates.data_ptr(), cs.data_ptr(),
                   bar.data_ptr(), T, N, H, geom.units, geom.fwd_rows, torch.cuda.current_stream().cuda_stream,
                   DTYPE_CODE[gx.dtype])
    return y, gates, cs


def _backward(dy, gates, cs, whh, lens, elem):
    C = ext.require()
    T, N, H = dy.shape
    geom = fused_lstm._device_geometry(H, N, dy.device, elem)
    dg = torch.empty(T, N, 4 * H, device="cuda", dtype=dy.dtype)
    bar = torch.zeros(1, dtype=torch.int64, device="cuda")
    C.lstm_backward(dy.data_ptr(), gates.data_ptr(), cs.data_ptr(), whh.data_ptr(), lens.data_ptr(), dg.data_ptr(),
                    bar.data_ptr(), T, N, H, geom.units, geom.bwd_rows, torch.cuda.current_stream().cuda_stream,
                    DTYPE_CODE[dy.dtype])
    return dg


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,N", [(800, 2), (128, 5)])
def test_one_step_is_the_fp32_kernel_on_widened_operands(dt, H, N):
    """T = 1: nothing a 16-bit launch rounded is read back, so its y and dgates are the fp32 launch's on the widened gx,
    W_hh and dy, rounded to nearest even, and the fp32 gates and c it saves are the fp32 launch's, all bit for bit."""
    dt = DTYPES[dt]
    torch.manual_seed(1)
    gx = (2 * torch.randn(1, N, 4 * H, device="cuda")).to(dt)
    whh = (torch.randn(4 * H, H, device="cuda") / H ** 0.5).to(dt)
    dy = torch.randn(1, N, H, device="cuda").to(dt)
    lens = torch.ones(N, dtype=torch.int32, device="cuda")
    y16, gates16, cs16 = _forward(gx, whh, lens, 2)
    y32, gates32, cs32 = _forward(gx.float(), whh.float(), lens, 4)
    assert y16.dtype == dt and torch.equal(y16, y32.to(dt))
    assert torch.equal(gates16, gates32) and torch.equal(cs16, cs32)
    dg16 = _backward(dy, gates16, cs16, whh, lens, 2)
    dg32 = _backward(dy.float(), gates32, cs32, whh.float(), lens, 4)
    assert dg16.dtype == dt and torch.equal(dg16, dg32.to(dt))
    assert y16.float().abs().max() > 0 and dg16.float().abs().max() > 0


# ---------------------------------------------------------------- a torch loop with the kernels' rounding points
def _emulate(rnn, x, lens, dy, dt):
    """The 16-bit path in fp32 torch ops, one timestep at a time, rounding to ``dt`` where the kernels do: W_hh, gx, y
    (read back as h_{t-1}), dy and dgates (read back at step t - 1); gates, c, dc and all sums in fp32.  The GEMMs
    outside the recurrence are the ones ``_LstmLayer`` runs, in ``dt``."""
    T, N, I = x.shape
    H = rnn.hidden_size
    lens = lens.to("cuda")
    xs, wi, wh = x.to(dt), rnn.weight_ih_l0.detach().to(dt), rnn.weight_hh_l0.detach().to(dt).float()
    b = (rnn.bias_ih_l0 + rnn.bias_hh_l0).detach().to(dt)
    gx = torch.addmm(b, xs.reshape(T * N, I), wi.t()).view(T, N, 4 * H).float()
    h = torch.zeros(N, H, device="cuda")
    c = torch.zeros(N, H, device="cuda")
    ys, gs, cs = [], [], []
    for t in range(T):
        on = (t < lens).view(N, 1)
        a = gx[t] + h @ wh.t()
        i, f, g, o = a.chunk(4, 1)
        i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
        c = torch.where(on, f * c + i * g, torch.zeros_like(c))
        h = torch.where(on, o * torch.tanh(c), torch.zeros_like(c)).to(dt).float()
        ys.append(h); gs.append((i, f, g, o)); cs.append(c)
    dgn = torch.zeros(N, 4 * H, device="cuda")
    dcn = torch.zeros(N, H, device="cuda")
    dgs = [None] * T
    dy = dy.to(dt).float()
    for t in range(T - 1, -1, -1):
        on = (t < lens).view(N, 1)
        i, f, g, o = gs[t]
        tc = torch.tanh(cs[t])
        cp = cs[t - 1] if t > 0 else torch.zeros_like(tc)
        dh = dy[t] + dgn @ wh
        dc = dh * o * (1 - tc * tc) + dcn
        dg = torch.cat([dc * g * i * (1 - i), dc * cp * f * (1 - f), dc * i * (1 - g * g), dh * tc * o * (1 - o)], 1)
        dgn = torch.where(on, dg, torch.zeros_like(dg)).to(dt).float()
        dcn = torch.where(on, dc * f, torch.zeros_like(dc))
        dgs[t] = dgn
    y = torch.stack(ys).to(dt)
    dg = torch.stack(dgs).to(dt)
    g2 = dg.view(T * N, 4 * H)
    dx = (g2 @ wi).view(T, N, I).to(x.dtype)
    dw_ih = (g2.t() @ xs.reshape(T * N, I)).float()
    dw_hh = (dg[1:].reshape(-1, 4 * H).t() @ y[:-1].reshape(-1, H)).float()
    db = g2.sum(0, dtype=torch.float32)
    return [y, dx, dw_ih, dw_hh, db, db]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("I,H,N,T", [(64, 128, 5, 48), (800, 800, 2, 48), (96, 256, 32, 20)])
def test_follows_the_rounding_point_emulation(dt, I, H, N, T):
    """Tolerance: 4 ulps of ``dt`` at each tensor's largest magnitude.  The loop's matmuls add in another order than the
    kernels, so a sum near a rounding boundary of y_t or dgates_t may round the other way (1 ulp of that element), and
    that difference is carried through the remaining steps and the GEMMs; a missing or misplaced rounding point, or
    a 16-bit cell state, would show as errors that grow with T well past this."""
    dt = DTYPES[dt]
    torch.manual_seed(2)
    rnn = nn.LSTM(I, H).cuda()
    x = torch.randn(T, N, I, device="cuda")
    dy = torch.randn(T, N, H, device="cuda")
    lens = torch.tensor([T] + [max(1, T - 5 * i) for i in range(1, N)], dtype=torch.int32)
    n0 = _launches()
    got = _run(rnn, x, lens, dy, _fused, dt)
    assert _launches() == (n0[0] + 1, n0[1] + 1)
    want = _emulate(rnn, x, lens, dy, dt)
    bad = []
    for name, a, b in zip(NAMES, got, want):
        tol = 4 * torch.finfo(dt).eps * b.float().abs().max().item()
        err = (a.float() - b.float()).abs().max().item()
        if not err <= tol:
            bad.append((name, err, tol))
    assert not bad, bad


# ---------------------------------------------------------------- against float64
def _three_ways(I, H, N, T, lens, dt, seed=0):
    torch.manual_seed(seed)
    rnn = nn.LSTM(I, H).cuda()
    x = torch.randn(T, N, I, device="cuda")
    dy = torch.randn(T, N, H, device="cuda")
    lens = torch.tensor(lens, dtype=torch.int32)
    ref64 = copy.deepcopy(rnn).double().cpu()
    ref = _run(ref64, x.double().cpu(), lens, dy.double().cpu(), fused_lstm.stock_layer)
    n0 = _launches()
    stock = _run(rnn, x, lens, dy, fused_lstm.stock_layer, dt)
    assert _launches() == n0
    fused = _run(rnn, x, lens, dy, _fused, dt)
    assert _launches() == (n0[0] + 1, n0[1] + 1), "the fused kernels did not run"
    return ref, stock, fused


def _check_vs_reference(ref, stock, fused, dt, names=NAMES):
    """err_fused <= 2 err_stock + floor, the floor being 2 ulps of ``dt`` (eps: 2^-7 in bf16, 2^-10 in fp16) at the
    reference tensor's largest magnitude (at 1 for smaller tensors): every tensor here passes through at least one
    rounding to ``dt`` on either path, so below that the two errors are rounding noise and their ratio says nothing."""
    bad = []
    for name, r, s, f in zip(names, ref, stock, fused):
        es = (s.cpu().double() - r).abs().max().item()
        ef = (f.cpu().double() - r).abs().max().item()
        floor = 2 * torch.finfo(dt).eps * max(1.0, r.abs().max().item())
        if not ef <= 2 * es + floor:
            bad.append((name, ef, es, floor))
    assert not bad, bad


SHAPES = [(1312, 800, 2, 48), (800, 800, 2, 198), (96, 256, 32, 20), (800, 800, fused_lstm.MAX_BATCH, 30),
          (200, 4, 3, 12)]


@pytest.mark.parametrize("dt,I,H,N,T", [(d,) + s for d in DTYPES for s in SHAPES] + [("bf16", 64, 1500, 20, 35)])
def test_forward_and_gradients_against_float64(dt, I, H, N, T):
    """The last shape is the PTB-sized layer, whose W_hh slice fits in shared memory only in 16 bits."""
    dt = DTYPES[dt]
    lens = [T] + [max(1, T - 3 * i) for i in range(1, N)]
    _check_vs_reference(*_three_ways(I, H, N, T, lens, dt), dt)


@pytest.mark.parametrize("dt", DTYPES)
def test_lengths_dtypes_and_determinism(dt):
    dt = DTYPES[dt]
    T = 40
    lens = [7, T, 1, T - 3, 12]
    ref, stock, fused = _three_ways(160, 800, len(lens), T, lens, dt, seed=3)
    _check_vs_reference(ref, stock, fused, dt)
    y, dx = fused[0], fused[1]
    for b, L in enumerate(lens):
        assert torch.all(y[L:, b] == 0) and torch.all(dx[L:, b] == 0), b
        assert y[:L, b].abs().max() > 0 and dx[:L, b].abs().max() > 0, b
    assert y.dtype == dt and dx.dtype == torch.float32
    assert all(g.dtype == torch.float32 for g in fused[2:])
    # the gradients' types are the stock layer's; its y is float16 under either autocast type (torch 2.11)
    assert [t.dtype for t in fused[1:]] == [t.dtype for t in stock[1:]]

    torch.manual_seed(5)
    layer = BatchRNN(800, 800, fuse=True, fuse_autocast=True).cuda()
    x = torch.randn(123, 2, 800, device="cuda").to(dt)           # what the previous layer hands over under autocast
    lens = torch.tensor([123, 77], dtype=torch.int32)
    dy = torch.randn(123, 2, 800, device="cuda").to(dt)
    outs = []
    for _ in range(2):
        xi = x.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=dt):
            y = layer(xi, lens)
        grads = torch.autograd.grad(y, [xi] + list(layer.parameters()), dy)
        outs.append([y] + list(grads))
    assert outs[0][0].dtype == dt and outs[0][1].dtype == dt
    assert all(g.dtype == torch.float32 for g in outs[0][2:])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ---------------------------------------------------------------- fp16 range
def _saturated_layer(I, H):
    """W = 0, forget gate open (f ~ 1), i = o = 1/2, g ~ 0.05 so that c stays small: the carried dc grows by about dy / 2
    a step, and the cell input's dgate is about half of it."""
    rnn = nn.LSTM(I, H).cuda()
    with torch.no_grad():
        for p in rnn.parameters():
            p.zero_()
        rnn.bias_ih_l0[H:2 * H] = 10.0
        rnn.bias_ih_l0[2 * H:3 * H] = 0.05
    return rnn


def test_fp16_overflowing_dgate_is_not_saturated():
    """dy = 60000 at every step: dgates exceed 65504 after a few steps of carried dc.  They must be stored as inf, so that
    the weight gradients are non-finite and dynamic loss scaling skips the step, not as the largest finite fp16."""
    I, H, N, T = 16, 8, 2, 12
    rnn = _saturated_layer(I, H)
    torch.manual_seed(0)
    x = torch.randn(T, N, I, device="cuda")
    dy = torch.full((T, N, H), 60000.0, device="cuda")
    lens = torch.full((N,), T, dtype=torch.int32)
    n0 = _launches()
    out = _run(rnn, x, lens, dy, _fused, torch.float16)
    assert _launches() == (n0[0] + 1, n0[1] + 1)
    assert torch.isfinite(out[0]).all()
    for name, g in zip(NAMES[2:], out[2:]):
        assert not torch.isfinite(g).all(), name


def test_fp16_subnormal_dgates_are_kept():
    """dy = 7 * 2^-24, gates as in ``_saturated_layer``: every dgate of the cell input is a few 2^-24, far below fp16's
    smallest normal (2^-14), and must be stored as a subnormal, not flushed to 0."""
    H, N, T = 8, 2, 4
    gx = torch.zeros(T, N, 4 * H, device="cuda")
    gx[..., H:2 * H] = 10.0
    gx[..., 2 * H:3 * H] = 0.05
    gx = gx.half()
    whh = torch.zeros(4 * H, H, device="cuda", dtype=torch.float16)
    lens = torch.full((N,), T, dtype=torch.int32, device="cuda")
    y, gates, cs = _forward(gx, whh, lens, 2)
    dy = torch.full((T, N, H), 7 * 2.0 ** -24, device="cuda", dtype=torch.float16)
    assert (dy != 0).all()
    dg = _backward(dy, gates, cs, whh, lens, 2)
    dgg = dg[..., 2 * H:3 * H].float()
    assert (dgg != 0).all() and dgg.abs().max() < 2.0 ** -14, (dgg.min().item(), dgg.max().item())


# ---------------------------------------------------------------- the gate
def _layer_case(case):
    torch.manual_seed(7)
    I, H, N, T = 48, 64, 3, 10
    kw, dtype = {}, torch.float32
    if case == "bidirectional":
        kw["bidirectional"] = True
    elif case == "batch_over_limit":
        N = fused_lstm.MAX_BATCH + 1
    elif case == "fp64":
        dtype = torch.float64
    layer = BatchRNN(I, H, **kw).cuda().to(dtype)
    x = torch.randn(T, N, I, device="cuda", dtype=dtype)
    lens = torch.randint(1, T + 1, (N,), dtype=torch.int32)
    lens[0] = T
    return layer, x, lens


def _layer_run(layer, x, lens, dt):
    for p in layer.parameters():
        p.grad = None
    xi = x.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=dt, enabled=dt is not None):
        y = layer(xi, lens)
    y.float().square().sum().backward()
    return [y.detach(), xi.grad] + [p.grad for p in layer.parameters()]


def test_gate_takes_the_kernels_under_autocast_with_both_switches():
    layer, x, lens = _layer_case("native")
    layer.fuse = layer.fuse_autocast = True
    for dt in DTYPES.values():
        n0 = _launches()
        out = _layer_run(layer, x, lens, dt)
        assert _launches() == (n0[0] + 1, n0[1] + 1), dt
        assert out[0].dtype == dt
    layer.fuse_autocast = False
    n0 = _launches()
    _layer_run(layer, x, lens, torch.bfloat16)
    assert _launches() == n0


@pytest.mark.parametrize("case", ["fp64", "bidirectional", "batch_over_limit"])
def test_gate_falls_back_to_the_stock_layer(case):
    layer, x, lens = _layer_case(case)
    outs = []
    for fuse in (False, True):
        layer.fuse = layer.fuse_autocast = fuse
        n0 = _launches()
        outs.append(_layer_run(layer, x, lens, torch.bfloat16))
        assert _launches() == n0, case
    for a, b in zip(*outs):
        assert torch.equal(a, b), case


def test_autocast_off_is_the_fp32_fused_layer():
    layer, x, lens = _layer_case("native")
    layer.fuse = True
    outs = []
    for on in (False, True):
        layer.fuse_autocast = on
        n0 = _launches()
        outs.append(_layer_run(layer, x, lens, None))
        assert _launches() == (n0[0] + 1, n0[1] + 1)
    for a, b in zip(*outs):
        assert a.dtype == torch.float32 and torch.equal(a, b)


# ---------------------------------------------------------------- whole model, trainer
def _ctc_loss(out, targets, out_lens, tsizes):
    logp = F.log_softmax(out.transpose(0, 1), dim=-1)
    return F.ctc_loss(logp.float(), targets, out_lens.long(), tsizes, blank=0, reduction="sum",
                      zero_infinity=True) / out.size(0)


def test_whole_model_against_float64():
    dt = torch.bfloat16
    torch.manual_seed(0)
    net, _ = create_net(29, "lstman4")
    ref = copy.deepcopy(net).double()
    stock = net.cuda()
    fused = copy.deepcopy(stock)
    fused.fuse_lstm = fused.fuse_lstm_autocast = True
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 1, 161, 400, generator=g)
    lens = torch.tensor([400, 290], dtype=torch.int32)
    tsizes = torch.tensor([20, 14])
    targets = torch.randint(1, 29, (int(tsizes.sum()),), generator=g)
    res = {}
    for name, m, dev, xdt in (("ref", ref, "cpu", torch.float64), ("stock", stock, "cuda", torch.float32),
                              ("fused", fused, "cuda", torch.float32)):
        m.train()
        n0 = _launches()
        with torch.autocast("cuda", dtype=dt, enabled=dev == "cuda"):
            out, out_lens = m(x.to(dev, xdt), lens)
            loss = _ctc_loss(out, targets.to(dev), out_lens.to(dev), tsizes.to(dev))
        loss.backward()
        n1 = _launches()
        assert (n1[0] - n0[0], n1[1] - n0[1]) == ((5, 5) if name == "fused" else (0, 0)), name
        res[name] = [out.detach().cpu().double(), loss.detach().cpu().double()] + \
                    [p.grad.detach().cpu().double() for p in m.parameters()]
    assert torch.isfinite(res["fused"][1])
    assert all(p.grad.dtype == torch.float32 for p in fused.parameters())
    names = ["logits", "ctc"] + [n for n, _ in net.named_parameters()]
    _check_vs_reference(res["ref"], res["stock"], res["fused"], dt, names)


@pytest.mark.parametrize("autocast", ["bf16", "fp16"])
def test_trainer_steps_follow_stock(autocast):
    """Five steps on the bench's AN4 batches, stock against fused under the same autocast (fp16 with dynamic loss
    scaling).  The two arms see the same batches from the same initial parameters and differ by 16-bit rounding in five
    stacked layers, so their losses agree to a few bf16 ulps (2^-7) of the loss, not bitwise: 5 %, where the fp32 pair is
    held to 2 %."""
    import bench
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    losses = {}
    for fuse in (False, True):
        cfg = okt.preset(preset, density=0.001, warmup_iters=2)
        tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                     t_total=100000, warmup=0.1, seed=0, autocast=autocast,
                     loss_scale=okt.LossScale() if autocast == "fp16" else None,
                     model_kwargs={"fuse_lstm": fuse, "fuse_lstm_autocast": fuse})
        assert tr.net.fuse_lstm is fuse and tr.net.fuse_lstm_autocast is fuse
        seq = []
        n0 = _launches()
        for i in range(5):
            batch = tuple(t.to(tr.device) for t in bench.make_batch("lstman4", i, 0, bs, 128))
            tr.net.train()
            tr.optimizer.zero_grad()
            loss, _ = tr._forward_loss(batch)
            tr.backward(loss)
            tr.update_model()
            seq.append(float(loss))
        n1 = _launches()
        assert (n1[0] - n0[0], n1[1] - n0[1]) == ((25, 25) if fuse else (0, 0))
        assert all(torch.isfinite(p).all() for p in tr.net.parameters())
        tr.close()
        losses[fuse] = seq
    for a, b in zip(losses[False], losses[True]):
        assert b == pytest.approx(a, rel=5e-2), losses
