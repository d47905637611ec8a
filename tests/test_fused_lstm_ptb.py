"""The stacked-layer LSTM kernels (``lstm_stack``, the PTB model's ``fuse_lstm``) on the GPU under bf16 / fp16 autocast:
y, the carried-out state and every gradient, the initial state's included, against a float64 CPU ``nn.LSTM``, no worse
than stock cuDNN under the same autocast; determinism; null upstream state gradients; fp16 overflow; dropout between
layers; the PTB model and truncated-BPTT ``Trainer`` steps; the fallbacks."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oktopk_b200.models import create_net
from oktopk_b200.ops import ext, fused_lstm

pytestmark = pytest.mark.gpu

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _launches():
    return ext.LAUNCH_COUNT.get("lstm_seq_forward", 0), ext.LAUNCH_COUNT.get("lstm_seq_backward", 0)


def _stock(x, hx, rnn):
    return rnn(x, hx)


def _fused(x, hx, rnn):
    return fused_lstm.lstm_stack(x, hx, rnn, rnn.dropout, rnn.training)


def _run(rnn, x, hx, up, fn, dt=None):
    """fn(x, hx, rnn) -> (y, (h_n, c_n)) under ``dt`` autocast when given; returns y, h_n, c_n and the gradients of
    sum(y dy) + sum(h_n dh_n) + sum(c_n dc_n) wrt x, h0, c0 and every parameter (``up`` = (dy, dh_n, dc_n), an entry
    None leaves that output out of the sum)."""
    x = x.detach().clone().requires_grad_(True)
    hx = tuple(h.detach().clone().requires_grad_(True) for h in hx)
    for p in rnn.parameters():
        p.grad = None
    with torch.autocast("cuda", dtype=dt, enabled=dt is not None):
        y, (hn, cn) = fn(x, hx, rnn)
    loss = sum((o.double() * u.to(o.device).double()).sum() for o, u in zip((y, hn, cn), up) if u is not None)
    loss.backward()
    return [y.detach(), hn.detach(), cn.detach(), x.grad, hx[0].grad, hx[1].grad] + [p.grad for p in rnn.parameters()]


def _names(rnn):
    return ["y", "h_n", "c_n", "dx", "dh0", "dc0"] + ["d" + n for n, _ in rnn.named_parameters()]


def _check_vs_reference(ref, stock, fused, dt, names):
    """err_fused <= 2 err_stock + 2 ulps of ``dt`` (eps 2^-7 in bf16, 2^-10 in fp16) at the reference tensor's largest
    magnitude (at 1 for smaller tensors), as for the single-layer 16-bit kernels."""
    bad = []
    for name, r, s, f in zip(names, ref, stock, fused):
        r = r.double()
        es = (s.cpu().double() - r).abs().max().item()
        ef = (f.cpu().double() - r).abs().max().item()
        floor = 2 * torch.finfo(dt).eps * max(1.0, r.abs().max().item())
        if not ef <= 2 * es + floor:
            bad.append((name, ef, es, floor))
    assert not bad, bad


def _case(H, N, T, L, seed=0, dropout=0.0):
    torch.manual_seed(seed)
    rnn = nn.LSTM(H, H, num_layers=L, dropout=dropout).cuda()
    x = torch.randn(T, N, H, device="cuda")
    hx = (0.5 * torch.randn(L, N, H, device="cuda"), torch.randn(L, N, H, device="cuda"))
    up = (torch.randn(T, N, H, device="cuda"), torch.randn(L, N, H, device="cuda"), torch.randn(L, N, H, device="cuda"))
    return rnn, x, hx, up


SHAPES = [(1500, 20, 35, 2), (64, 1, 1, 1), (64, 7, 9, 3), (800, 64, 12, 1)]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,N,T,L", SHAPES)
def test_stack_against_float64(dt, H, N, T, L):
    dt = DTYPES[dt]
    rnn, x, hx, up = _case(H, N, T, L)
    ref64 = copy.deepcopy(rnn).double().cpu()
    ref = _run(ref64, x.double().cpu(), tuple(h.double().cpu() for h in hx), tuple(u.cpu() for u in up), _stock)
    n0 = _launches()
    stock = _run(rnn, x, hx, up, _stock, dt)
    assert _launches() == n0
    fused = _run(rnn, x, hx, up, _fused, dt)
    assert _launches() == (n0[0] + L, n0[1] + L), "the stacked-layer kernels did not run"
    assert fused[0].dtype == dt and fused[1].dtype == dt and fused[2].dtype == torch.float32
    assert fused[0].shape == (T, N, H) and fused[1].shape == fused[2].shape == (L, N, H)
    assert all(g.dtype == torch.float32 for g in fused[3:])
    _check_vs_reference(ref, stock, fused, dt, _names(rnn))


@pytest.mark.parametrize("dt", DTYPES)
def test_deterministic_and_null_state_gradients(dt):
    """Two runs are bitwise equal.  With no gradient on h_n and c_n the backward kernel gets null dh_n / dc_n, which
    must equal passing zeros."""
    dt = DTYPES[dt]
    rnn, x, hx, up = _case(1500, 20, 35, 2, seed=1)
    a = _run(rnn, x, hx, up, _fused, dt)
    b = _run(rnn, x, hx, up, _fused, dt)
    for name, u, v in zip(_names(rnn), a, b):
        assert torch.equal(u, v), name
    null = _run(rnn, x, hx, (up[0], None, None), _fused, dt)
    zero = _run(rnn, x, hx, (up[0], torch.zeros_like(up[1]), torch.zeros_like(up[2])), _fused, dt)
    for name, u, v in zip(_names(rnn), null, zero):
        assert torch.equal(u, v), name


def test_fp16_overflowing_dgate_arrives_as_inf():
    """W = 0, forget gate open, i = o = 1/2, g ~ 0.05, c0 = 1, one timestep, and an upstream dc_n of 1e7: the input
    gate's dgate (dc g i (1 - i), about 1.2e5) and the cell input's (dc i (1 - g^2), about 5e6) exceed 65504 and must be
    stored as inf, not as the largest finite fp16, so that the gradients are non-finite and dynamic loss scaling skips
    the step; the forget gate's (dc c0 f (1 - f), about 450) and the output gate's stay finite.  (One step: at the next
    one the recurrent product would turn inf into NaN, 0 x inf, as in any LSTM.)"""
    H, N, T = 8, 2, 1
    rnn = nn.LSTM(H, H).cuda()
    with torch.no_grad():
        for p in rnn.parameters():
            p.zero_()
        rnn.bias_ih_l0[H:2 * H] = 10.0
        rnn.bias_ih_l0[2 * H:3 * H] = 0.05
    torch.manual_seed(0)
    x = torch.randn(T, N, H, device="cuda")
    hx = (torch.zeros(1, N, H, device="cuda"), torch.ones(1, N, H, device="cuda"))
    up = (torch.ones(T, N, H, device="cuda"), None, torch.full((1, N, H), 1e7, device="cuda"))
    n0 = _launches()
    out = _run(rnn, x, hx, up, _fused, torch.float16)
    assert _launches() == (n0[0] + 1, n0[1] + 1)
    assert torch.isfinite(out[0]).all()
    db = out[8]                                         # sum over the rows of dgates: [i, f, g, o] blocks of H
    assert torch.all(db[:H] == float("inf")) and torch.all(db[2 * H:3 * H] == float("inf")), db
    assert torch.isfinite(db[H:2 * H]).all() and torch.isfinite(db[3 * H:]).all(), db
    assert not torch.isfinite(out[6]).all()             # dW_ih


def test_dropout_between_layers_is_the_single_layer_reference():
    """Training with p = 0.5 between layers: the fused stack equals single-layer stock LSTMs with the same F.dropout
    calls under the same seed, and a float64 reference with the same masks, within the tolerance above.  (p = 0.5 keeps
    the kept elements' scale, 2, exact in 16 bits, so the masks can be replayed on ones.)"""
    dt = torch.bfloat16
    H, N, T, L, p = 256, 20, 16, 3, 0.5
    rnn, x, hx, up = _case(H, N, T, L, seed=2, dropout=p)
    rnn.train()
    layers = []
    for layer in range(L):
        m = nn.LSTM(H, H).cuda()
        for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
            getattr(m, n + "_l0").data.copy_(getattr(rnn, "%s_l%d" % (n, layer)).data)
        layers.append(m)

    def single_layers(xi, hxi, _rnn, masks=None):
        hs, cs = [], []
        for layer, m in enumerate(layers):
            if layer > 0:
                xi = xi * masks[layer - 1] if masks is not None else F.dropout(xi.to(dt), p, True)
            xi, (h, c) = m(xi, (hxi[0][layer:layer + 1], hxi[1][layer:layer + 1]))
            hs.append(h)
            cs.append(c)
        return xi, (torch.cat(hs), torch.cat(cs))

    torch.manual_seed(11)
    masks = [F.dropout(torch.ones(T, N, H, device="cuda", dtype=dt), p, True) for _ in range(L - 1)]
    torch.manual_seed(11)
    n0 = _launches()
    fused = _run(rnn, x, hx, up, _fused, dt)
    assert _launches() == (n0[0] + L, n0[1] + L)
    # the stock and float64 arms take their parameter gradients on `layers`, the fused one on `rnn`, in the same order
    torch.manual_seed(11)
    stock = _run(rnn, x, hx, up, single_layers, dt)[:6] + _layer_grads(layers)
    for m in layers:
        m.double().cpu()
        m.zero_grad(set_to_none=True)
    ref = _run(rnn, x.double().cpu(), tuple(h.double().cpu() for h in hx), tuple(u.cpu() for u in up),
               lambda xi, hxi, r: single_layers(xi, hxi, r, [m.double().cpu() for m in masks]))[:6] + _layer_grads(layers)
    _check_vs_reference(ref, stock, fused, dt, _names(rnn))
    assert all(0.3 < float((mk == 0).float().mean()) < 0.7 for mk in masks)


def _layer_grads(layers):
    return [getattr(m, n + "_l0").grad for m in layers for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]


def test_ptb_model_against_float64():
    """``PTBLSTM(fuse_lstm=True)`` with dropout 0 under bf16 and fp16 autocast: loss and every parameter gradient."""
    torch.manual_seed(0)
    net, _ = create_net(10000, "lstm")
    net.dropout.p = 0.0
    net.lstm.dropout = 0.0
    g = torch.Generator().manual_seed(3)
    x = torch.randint(0, 10000, (35, 20), generator=g)
    y = torch.randint(0, 10000, (35, 20), generator=g)
    hid = tuple(0.3 * torch.randn(2, 20, 1500, generator=g) for _ in range(2))
    ref = copy.deepcopy(net).double()
    out, _ = ref(x, tuple(h.double() for h in hid))
    loss = F.cross_entropy(out.view(-1, 10000), y.view(-1))
    loss.backward()
    res_ref = [loss.detach()] + [p.grad for p in ref.parameters()]
    names = ["loss"] + [n for n, _ in net.named_parameters()]
    for dt in DTYPES.values():
        res = {}
        for fuse in (False, True):
            m = copy.deepcopy(net).cuda()
            m.fuse_lstm = fuse
            n0 = _launches()
            with torch.autocast("cuda", dtype=dt):
                out, (hn, cn) = m(x.cuda(), tuple(h.cuda() for h in hid))
                loss = F.cross_entropy(out.view(-1, 10000), y.cuda().view(-1))
            loss.backward()
            assert _launches() == ((n0[0] + 2, n0[1] + 2) if fuse else n0)
            res[fuse] = [loss.detach()] + [p.grad for p in m.parameters()]
            assert all(p.grad.dtype == torch.float32 for p in m.parameters())
        _check_vs_reference(res_ref, res[False], res[True], dt, names)


@pytest.mark.parametrize("autocast", ["bf16", "fp16"])
def test_trainer_bptt_steps_follow_stock(autocast):
    """Three truncated-BPTT steps through ``Trainer`` on the synthetic PTB stream, the hidden state carried across
    batches, stock against fused (``fuse_lstm`` + ``fuse_xent``) under the same autocast (fp16 with dynamic loss scaling),
    dropout off so that both arms compute the same function.  The arms differ by 16-bit rounding in two stacked layers
    carried over 105 timesteps, so their losses agree to a few ulps of the loss, not bitwise: 5 %, as for the AN4
    model's fused 16-bit layers."""
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    losses = {}
    for fuse in (False, True):
        cfg = okt.preset("lstm_an4", density=0.02, warmup_iters=2)
        tr = Trainer(dnn="lstm", dataset="ptb", batch_size=20, lr=22, compressor="oktopk", density=0.02, cfg=cfg,
                     norm_clip=0.25, seed=0, autocast=autocast,
                     loss_scale=okt.LossScale() if autocast == "fp16" else None,
                     model_kwargs={"fuse_lstm": fuse, "fuse_xent": fuse})
        assert tr.net.fuse_lstm is fuse and tr.net.fuse_xent is fuse
        tr.net.dropout.p = 0.0
        tr.net.lstm.dropout = 0.0
        n0 = _launches()
        x0 = ext.LAUNCH_COUNT.get("xent_forward", 0)
        seq = []
        for _ in range(3):
            tr.train_step()
            seq.append(float(tr.last_loss()))
        assert (_launches() == (n0[0] + 6, n0[1] + 6)) is fuse
        assert (ext.LAUNCH_COUNT.get("xent_forward", 0) > x0) is fuse
        if fuse:
            assert tr.hidden[0].dtype == DTYPES[autocast] and tr.hidden[1].dtype == torch.float32
        losses[fuse] = seq
        tr.close()
    for a, b in zip(losses[False], losses[True]):
        assert abs(a - b) <= 0.05 * abs(a), losses


# ---------------------------------------------------------------- fallbacks
@pytest.mark.parametrize("case", ["fp32", "fp64", "too_large", "bidirectional"])
def test_fallbacks_are_exactly_stock(case):
    torch.manual_seed(4)
    H, N, T, L, dt, dtype, kw = 64, 3, 5, 2, torch.bfloat16, torch.float32, {}
    if case == "fp32":
        dt = None
    elif case == "fp64":
        dtype = torch.float64
    elif case == "too_large":
        H = 2000                                        # 64 rows of W_hh at 2008 elements: 257 KB per CTA
    elif case == "bidirectional":
        kw["bidirectional"] = True
    rnn = nn.LSTM(H, H, num_layers=L, **kw).cuda().to(dtype)
    D = 2 if case == "bidirectional" else 1
    x = torch.randn(T, N, H, device="cuda", dtype=dtype)
    hx = tuple(torch.randn(D * L, N, H, device="cuda", dtype=dtype) for _ in range(2))
    up = (torch.randn(T, N, D * H, device="cuda"), torch.randn(D * L, N, H, device="cuda"),
          torch.randn(D * L, N, H, device="cuda"))
    a = _run(rnn, x, hx, up, _stock, dt)
    n0 = _launches()
    b = _run(rnn, x, hx, up, _fused, dt)
    assert _launches() == n0, case
    for u, v in zip(a, b):
        assert u.dtype == v.dtype and torch.equal(u, v), case


def test_switch_off_is_the_stock_model():
    torch.manual_seed(0)
    net, _ = create_net(1000, "lstm", vocab_size=1000)
    net = net.cuda().eval()
    x = torch.randint(0, 1000, (7, 4), device="cuda")
    hid = net.init_hidden(4, "cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        a, ha = net(x, hid)
        net.fuse_lstm = True
        n0 = _launches()
        b, hb = net(x, hid)
        assert _launches()[0] == n0[0] + 2
        net.fuse_lstm = False
        c, hc = net(x, hid)
    assert torch.equal(a, c) and all(torch.equal(u, v) for u, v in zip(ha, hc))
    assert (a.float() - b.float()).abs().max() < 0.05
