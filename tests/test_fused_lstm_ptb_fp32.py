"""The fp32 stacked-layer LSTM kernels (``lstm_stack(..., fp32=True)``, the PTB model's ``fuse_lstm_fp32``) on the GPU:
y, the carried-out state and every gradient, the initial state's included, against a float64 CPU ``nn.LSTM``, no worse
than stock fp32 cuDNN (TF32 off); shapes whose W_hh fits on chip and shapes that stream part of it from L2;
determinism; null upstream state gradients; the PTB model and truncated-BPTT ``Trainer`` steps; the fallbacks."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oktopk_b200.models import create_net
from oktopk_b200.ops import ext, fused_lstm

pytestmark = pytest.mark.gpu

# fp32 ulps of slack on top of twice stock's error, at the reference tensor's largest magnitude (at 1 for smaller
# tensors): the two sum in different orders, and a tensor stock gets exactly right would otherwise allow no rounding.
FLOOR_ULPS = 8


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
    return fused_lstm.lstm_stack(x, hx, rnn, rnn.dropout, rnn.training, fp32=True)


def _run(rnn, x, hx, up, fn, dt=None):
    """fn(x, hx, rnn) -> (y, (h_n, c_n)), under ``dt`` autocast when given; returns y, h_n, c_n and the gradients of
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


def _check_vs_reference(ref, stock, fused, names):
    """err_fused <= 2 err_stock + FLOOR_ULPS fp32 ulps at the reference tensor's scale."""
    bad = []
    for name, r, s, f in zip(names, ref, stock, fused):
        r = r.double()
        es = (s.cpu().double() - r).abs().max().item()
        ef = (f.cpu().double() - r).abs().max().item()
        floor = FLOOR_ULPS * torch.finfo(torch.float32).eps * max(1.0, r.abs().max().item())
        if not ef <= 2 * es + floor:
            bad.append((name, ef, es, floor))
    assert not bad, bad


def _case(H, N, T, L, seed=0):
    torch.manual_seed(seed)
    rnn = nn.LSTM(H, H, num_layers=L).cuda()
    x = torch.randn(T, N, H, device="cuda")
    hx = (0.5 * torch.randn(L, N, H, device="cuda"), torch.randn(L, N, H, device="cuda"))
    up = (torch.randn(T, N, H, device="cuda"), torch.randn(L, N, H, device="cuda"), torch.randn(L, N, H, device="cuda"))
    return rnn, x, hx, up


# (1500, 20): the PTB layer, 29 of 48 forward and 7 of 12 backward weight rows on chip, the rest from L2 (also at T = 1,
# where the backward pass has no step product); (64, 7): all of W_hh on chip; (800, 64): streams, four M tiles.
SHAPES = [(1500, 20, 35, 2), (1500, 20, 1, 1), (64, 7, 9, 3), (800, 64, 12, 1)]


def test_shapes_cover_on_chip_and_streamed_weights():
    p = torch.cuda.get_device_properties(0)
    geoms = {(H, N): fused_lstm.lstm_seq_f32_geometry(H, N, p.multi_processor_count, p.shared_memory_per_block_optin)
             for H, N, _, _ in SHAPES}
    assert all(g is not None for g in geoms.values())
    assert any(g.fwd_l2_bytes == 0 and g.bwd_l2_bytes == 0 for g in geoms.values())
    assert any(g.fwd_l2_bytes > 0 and g.bwd_l2_bytes > 0 for g in geoms.values())


@pytest.mark.parametrize("H,N,T,L", SHAPES)
def test_stack_against_float64(H, N, T, L):
    rnn, x, hx, up = _case(H, N, T, L)
    ref64 = copy.deepcopy(rnn).double().cpu()
    ref = _run(ref64, x.double().cpu(), tuple(h.double().cpu() for h in hx), tuple(u.cpu() for u in up), _stock)
    n0 = _launches()
    stock = _run(rnn, x, hx, up, _stock)
    assert _launches() == n0
    fused = _run(rnn, x, hx, up, _fused)
    assert _launches() == (n0[0] + L, n0[1] + L), "the fp32 stacked-layer kernels did not run"
    assert all(t.dtype == torch.float32 for t in fused)
    assert fused[0].shape == (T, N, H) and fused[1].shape == fused[2].shape == (L, N, H)
    _check_vs_reference(ref, stock, fused, _names(rnn))


def test_deterministic_and_null_state_gradients():
    """Two runs are bitwise equal.  With no gradient on h_n and c_n the backward kernel gets null dh_n / dc_n, which
    must equal passing zeros."""
    rnn, x, hx, up = _case(1500, 20, 35, 2, seed=1)
    a = _run(rnn, x, hx, up, _fused)
    b = _run(rnn, x, hx, up, _fused)
    for name, u, v in zip(_names(rnn), a, b):
        assert torch.equal(u, v), name
    n0 = _launches()
    null = _run(rnn, x, hx, (up[0], None, None), _fused)
    assert _launches() == (n0[0] + 2, n0[1] + 2)
    zero = _run(rnn, x, hx, (up[0], torch.zeros_like(up[1]), torch.zeros_like(up[2])), _fused)
    for name, u, v in zip(_names(rnn), null, zero):
        assert torch.equal(u, v), name


def test_ptb_model_against_float64():
    """``PTBLSTM(fuse_lstm=True, fuse_lstm_fp32=True)`` with dropout 0 in fp32: loss and every parameter gradient."""
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
    res = {}
    for fuse in (False, True):
        m = copy.deepcopy(net).cuda()
        m.fuse_lstm = m.fuse_lstm_fp32 = fuse
        n0 = _launches()
        out, (hn, cn) = m(x.cuda(), tuple(h.cuda() for h in hid))
        loss = F.cross_entropy(out.view(-1, 10000), y.cuda().view(-1))
        loss.backward()
        assert _launches() == ((n0[0] + 2, n0[1] + 2) if fuse else n0)
        assert hn.dtype == cn.dtype == torch.float32
        res[fuse] = [loss.detach()] + [p.grad for p in m.parameters()]
    _check_vs_reference(res_ref, res[False], res[True], names)


def test_trainer_bptt_steps_follow_stock():
    """Three truncated-BPTT steps through ``Trainer`` on the synthetic PTB stream, the hidden state carried across
    batches, stock fp32 cuDNN against the fused fp32 layers, dropout off so that both arms compute the same function.
    Both are fp32-accurate (3xTF32 here, TF32 off for cuDNN), so they differ only by summation order, about 1e-6 relative
    per layer output, which SGD at lr 22 and Ok-Topk's selection over three steps amplify but not past 1e-3 of the loss:
    fifty times tighter than the 16-bit arms' 5 %."""
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    losses = {}
    for fuse in (False, True):
        cfg = okt.preset("lstm_an4", density=0.02, warmup_iters=2)
        tr = Trainer(dnn="lstm", dataset="ptb", batch_size=20, lr=22, compressor="oktopk", density=0.02, cfg=cfg,
                     norm_clip=0.25, seed=0, model_kwargs={"fuse_lstm": fuse, "fuse_lstm_fp32": fuse})
        assert tr.net.fuse_lstm is fuse and tr.net.fuse_lstm_fp32 is fuse
        tr.net.dropout.p = 0.0
        tr.net.lstm.dropout = 0.0
        n0 = _launches()
        seq = []
        for _ in range(3):
            tr.train_step()
            seq.append(float(tr.last_loss()))
        assert (_launches() == (n0[0] + 6, n0[1] + 6)) is fuse
        assert tr.hidden[0].dtype == tr.hidden[1].dtype == torch.float32
        losses[fuse] = seq
        tr.close()
    for a, b in zip(losses[False], losses[True]):
        assert abs(a - b) <= 1e-3 * abs(a), losses


# ---------------------------------------------------------------- fallbacks
@pytest.mark.parametrize("case", ["cpu", "fp64", "rejected_shape", "bidirectional", "autocast"])
def test_fallbacks_are_exactly_stock(case):
    """Everything off the fp32 path returns what it returned before: ``rnn(x, hx)`` itself, bit for bit, and under
    autocast (where the 16-bit kernels run) exactly what ``fp32=False`` returns."""
    torch.manual_seed(4)
    H, N, T, L, dt, dtype, dev, kw = 64, 3, 5, 2, None, torch.float32, "cuda", {}
    if case == "cpu":
        dev = "cpu"
    elif case == "fp64":
        dtype = torch.float64
    elif case == "rejected_shape":
        H = 66                                          # not a multiple of 4
    elif case == "bidirectional":
        kw["bidirectional"] = True
    elif case == "autocast":
        dt = torch.bfloat16
    rnn = nn.LSTM(H, H, num_layers=L, **kw).to(dev, dtype)
    D = 2 if case == "bidirectional" else 1
    x = torch.randn(T, N, H, device=dev, dtype=dtype)
    hx = tuple(torch.randn(D * L, N, H, device=dev, dtype=dtype) for _ in range(2))
    up = (torch.randn(T, N, D * H, device=dev), torch.randn(D * L, N, H, device=dev),
          torch.randn(D * L, N, H, device=dev))

    def plain(xi, hxi, r):
        return fused_lstm.lstm_stack(xi, hxi, r, r.dropout, r.training)

    n0 = _launches()
    a = _run(rnn, x, hx, up, plain if case == "autocast" else _stock, dt)
    n1 = _launches()
    b = _run(rnn, x, hx, up, _fused, dt)
    assert _launches() == (n1[0] + n1[0] - n0[0], n1[1] + n1[1] - n0[1]), case
    assert (n1 != n0) is (case == "autocast"), case
    for u, v in zip(a, b):
        assert u.dtype == v.dtype and torch.equal(u, v), case
