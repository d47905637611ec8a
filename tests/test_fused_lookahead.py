"""The fused look-ahead convolution + Hardtanh of the AN4 DeepSpeech model (``ops/fused_lookahead``,
``csrc/lookahead.cu``) on the GPU:

1. width invariance: a launch at a padded width ``T_b`` equals a launch on the tensor cropped to ``Tm`` frames bit for
   bit (y, dx, dW), and writes exact +0 after ``Tm`` and past each length;
2. against a float64 evaluation of the formula at the model's shapes, within twice the stock module's error; dW
   bitwise reproducible; Hardtanh's strict mask at and beyond its bounds; non-finite fp16 gradients reaching dW and dx
   as through the stock module; the fallbacks;
3. the model with ``fuse_lookahead``: one eager step gives the stock model's loss and gradients to rounding, state
   dicts interchange, the bidirectional network refuses it;
4. a graphed padded trainer follows an eager padded one bit for bit;
5. one launch per pass."""

import pytest
import torch
import torch.nn as nn

from oktopk_b200.models.deepspeech import Lookahead
from oktopk_b200.ops import ext, fused_lookahead
from oktopk_b200.ops.ext import DTYPE_CODE

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
DT_IDS = ["fp32", "bf16", "fp16"]
H, CONTEXT = 800, 20


@pytest.fixture(autouse=True)
def _deterministic_convs():
    old = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = old


def _bits(t):
    t = t.detach().contiguous()
    return t.view({8: torch.int64, 4: torch.int32, 2: torch.int16}[t.element_size()])


def _launch(x, dy, lens, w):
    """Both kernels, the backward pass on the forward pass's y; y, dx and dW start as NaN, so every element they hold
    was written."""
    C_ = ext.require()
    Tb, N, Hx = x.shape
    K = w.size(1)
    stream = torch.cuda.current_stream().cuda_stream
    y = torch.full_like(x, float("nan"))
    dx = torch.full_like(x, float("nan"))
    dw = torch.full_like(w, float("nan"))
    C_.lookahead_forward(x.data_ptr(), w.data_ptr(), lens.data_ptr(), y.data_ptr(), N, Hx, Tb, K, DTYPE_CODE[x.dtype],
                         stream)
    C_.lookahead_backward(x.data_ptr(), y.data_ptr(), dy.data_ptr(), w.data_ptr(), lens.data_ptr(), dx.data_ptr(),
                          dw.data_ptr(), N, Hx, Tb, K, DTYPE_CODE[x.dtype], stream)
    return {"y": y, "dx": dx, "dw": dw}


def _lengths(N, Tm, mixed, g):
    if not mixed or N == 1:
        return torch.full((N,), Tm, dtype=torch.int32, device="cuda")
    lens = torch.randint(1, Tm + 1, (N,), generator=g, device="cuda", dtype=torch.int32)
    lens[N // 2] = Tm
    return lens


def _past(T, lens):
    """[T, N, 1]: the frames at or past each utterance's length."""
    return torch.arange(T, device="cuda").view(-1, 1, 1) >= lens.view(1, -1, 1)


# -------------------------------------------------------------------------------------------- 1. width invariance
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("N", [1, 2, 5, 32])
@pytest.mark.parametrize("tm", ["Tb", "Tb-1", "9", "1"])
@pytest.mark.parametrize("mixed", [False, True], ids=["equal", "mixed"])
def test_a_padded_launch_equals_the_cropped_launch(dt, N, tm, mixed):
    """Tm = 9 and 1 are shorter than the 21 taps."""
    g = torch.Generator(device="cuda").manual_seed(7)
    Tb = 64
    Tm = {"Tb": Tb, "Tb-1": Tb - 1, "9": 9, "1": 1}[tm]
    lens = _lengths(N, Tm, mixed, g)
    w = 2 * torch.rand(H, CONTEXT + 1, device="cuda", generator=g) - 1
    x = (1.0 + 4.0 * torch.randn(Tb, N, H, device="cuda", generator=g)).to(dt)       # both clamps in play
    dy = torch.randn(Tb, N, H, device="cuda", generator=g).to(dt)
    past = _past(Tb, lens)
    x = x.masked_fill(past, float("nan"))                        # frames past a length are never read
    dy = dy.masked_fill(past, float("nan"))
    pad = _launch(x, dy, lens, w)
    cut = _launch(x[:Tm].contiguous(), dy[:Tm].contiguous(), lens, w)
    assert torch.isfinite(pad["dw"]).all()
    assert torch.equal(_bits(pad["dw"]), _bits(cut["dw"]))
    if Tm > CONTEXT:
        y = cut["y"].float()
        assert (y[~past[:Tm].expand_as(y)] == 0).any() and (y == 20).any()
    for k in ("y", "dx"):
        assert torch.isfinite(cut[k].float()).all(), k
        assert torch.equal(_bits(pad[k][:Tm]), _bits(cut[k])), k
        outside = past.expand_as(pad[k]).clone()
        outside[Tm:] = True
        assert torch.equal(_bits(pad[k])[outside], torch.zeros_like(_bits(pad[k])[outside])), k     # +0


# --------------------------------------------------------------------------------------------- 2. against float64
def _reference(x, dy, lens, w):
    """The formula in float64; returns y, dx, dW and z."""
    x, dy, w = x.double(), dy.double(), w.double()
    T, N, Hx = x.shape
    K = w.size(1)
    Tm = min(int(lens.max()), T)
    valid = ~_past(T, lens.clamp(max=Tm)).expand_as(x)
    xv = torch.where(valid, x, 0.0)
    xp = torch.cat([xv, xv.new_zeros(K - 1, N, Hx)])
    z = sum(w[:, k] * xp[k:k + T] for k in range(K))
    y = torch.where(valid, z.clamp(0, 20), 0.0)
    dz = torch.where(valid & (z > 0) & (z < 20), dy, 0.0)
    dzp = torch.cat([dz.new_zeros(K - 1, N, Hx), dz])
    dx = torch.where(valid, sum(w[:, k] * dzp[K - 1 - k:K - 1 - k + T] for k in range(K)), 0.0)
    dw = torch.stack([(xp[k:k + T] * dz).sum((0, 1)) for k in range(K)], 1)
    return {"y": y, "dx": dx, "dw": dw, "z": z, "valid": valid}


def _stock(x, dy, w, dt):
    """The model's stock module, under autocast for a 16-bit x as in the model."""
    la = Lookahead(w.size(0), w.size(1) - 1).cuda()
    with torch.no_grad():
        la.weight.copy_(w)
    mod = nn.Sequential(la, nn.Hardtanh(0, 20, inplace=True))
    xi = x.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=dt, enabled=dt != torch.float32):
        y = mod(xi)
    y.backward(dy.to(y.dtype))
    return {"y": y.detach(), "dx": xi.grad, "dw": la.weight.grad}


def _fused(x, dy, w, lens, dt):
    wi = w.clone().requires_grad_(True)
    xi = x.clone().requires_grad_(True)
    n0 = (ext.LAUNCH_COUNT.get("lookahead_forward", 0), ext.LAUNCH_COUNT.get("lookahead_backward", 0))
    with torch.autocast("cuda", dtype=dt, enabled=dt != torch.float32):
        y = fused_lookahead.lookahead_hardtanh(xi, wi, lens)
    y.backward(dy)
    assert (ext.LAUNCH_COUNT.get("lookahead_forward", 0), ext.LAUNCH_COUNT.get("lookahead_backward", 0)) == \
        (n0[0] + 1, n0[1] + 1)
    assert y.dtype == x.dtype and xi.grad.dtype == x.dtype and wi.grad.dtype == torch.float32
    return {"y": y.detach(), "dx": xi.grad, "dw": wi.grad}


def _err(a, ref, where=None):
    d = (a.double() - ref).abs()
    return (d[where] if where is not None else d).max().item()


SHAPES = [(2, 48), (2, 123), (2, 198)]


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("N,T", SHAPES, ids=["N%d-T%d" % s for s in SHAPES])
def test_against_float64_within_twice_stock(dt, N, T):
    """x is zero past each length, as the LSTM layers leave it; dy is zeroed where z is within rounding of a clamp, so
    that the strict mask takes the same branch in every precision and the comparison measures rounding only."""
    g = torch.Generator(device="cuda").manual_seed(N * 1000 + T)
    lens = torch.randint(1, T + 1, (N,), generator=g, device="cuda", dtype=torch.int32)
    lens[0] = T
    stdv = 1.0 / (CONTEXT + 1) ** 0.5
    w = (2 * torch.rand(H, CONTEXT + 1, device="cuda", generator=g) - 1) * stdv * 8
    past = _past(T, lens)
    x = (2.0 + 3.0 * torch.randn(T, N, H, device="cuda", generator=g)).to(dt).masked_fill(past, 0)
    ref0 = _reference(x, x, lens, w)
    near = ((ref0["z"].abs() < 0.25) | ((ref0["z"] - 20).abs() < 0.25)) if dt != torch.float32 else \
        ((ref0["z"].abs() < 1e-3) | ((ref0["z"] - 20).abs() < 1e-3))
    dy = torch.randn(T, N, H, device="cuda", generator=g).masked_fill(near, 0).to(dt)
    ref = _reference(x, dy, lens, w)
    assert (ref["y"][ref["valid"]] == 0).any() and (ref["y"] == 20).any()
    stock = _stock(x, dy, w, dt)
    fused = _fused(x, dy, w, lens, dt)
    valid = ref["valid"]
    for k, where in (("y", None), ("dx", valid), ("dw", None)):
        floor = ref[k].abs().max().item() * 2.0 ** -23
        es, ef = _err(stock[k], ref[k], where), _err(fused[k], ref[k], where)
        assert ef <= 2 * max(es, floor), (k, ef, es, floor)
    assert torch.equal(_bits(fused["dx"])[~valid], torch.zeros_like(_bits(fused["dx"])[~valid]))      # +0
    again = _fused(x, dy, w, lens, dt)
    for k in ("y", "dx", "dw"):
        assert torch.equal(_bits(again[k]), _bits(fused[k])), k


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_the_hardtanh_mask_is_torchs_strict_mask(dt):
    """Taps (1, 0): z = x exactly, at -1, -0, 0, 0.5, 19.5, 20, 21 and 1e4; 37 channels, a partial slice."""
    Hs = 37
    vals = torch.tensor([-1.0, -0.0, 0.0, 0.5, 19.5, 20.0, 21.0, 1e4], device="cuda")
    T, N = vals.numel(), 3
    x = vals.view(-1, 1, 1).expand(T, N, Hs).to(dt).contiguous()
    w = torch.zeros(Hs, 2, device="cuda")
    w[:, 0] = 1
    lens = torch.full((N,), T, dtype=torch.int32, device="cuda")
    dy = torch.randn(T, N, Hs, device="cuda").to(dt)
    out = _launch(x, dy, lens, w)
    xr = x.float().clone().requires_grad_(True)
    yr = nn.functional.hardtanh(xr, 0, 20)
    (gr,) = torch.autograd.grad(yr, xr, dy.float())
    assert torch.equal(_bits(out["y"]), _bits(yr.detach().to(dt).abs()))          # -0 comes out as +0
    assert torch.equal(out["dx"].float(), gr)
    mask = (x.float() > 0) & (x.float() < 20)
    assert mask.sum() == 2 * N * Hs
    ref_dw0 = (x.double() * torch.where(mask, dy.double(), 0.0)).sum((0, 1))
    assert torch.allclose(out["dw"][:, 0].double(), ref_dw0, rtol=1e-6, atol=0)


def test_non_finite_fp16_gradients_reach_dw_and_dx_as_through_the_stock_module():
    """inf / -inf / NaN in dy on valid frames: where the mask lets them through they reach dW (through the zeros past
    the length too) and dx as in the stock module under fp16 autocast; where it blocks them they reach nothing."""
    g = torch.Generator(device="cuda").manual_seed(11)
    T, N, Hs = 40, 2, 64
    lens = torch.tensor([40, 29], dtype=torch.int32, device="cuda")
    w = (2 * torch.rand(Hs, CONTEXT + 1, device="cuda", generator=g) - 1) * 0.3
    x = (1.0 + 3.0 * torch.randn(T, N, Hs, device="cuda", generator=g)).half().masked_fill(_past(T, lens), 0)
    dy = (0.01 * torch.randn(T, N, Hs, device="cuda", generator=g)).half()
    y = _fused(x, torch.zeros_like(dy), w, lens, torch.float16)["y"]
    passes = (y > 0) & (y < 20) & ~_past(T, lens)
    blocks = ~passes & ~_past(T, lens)
    for h, (v, i) in enumerate([(float("inf"), 0), (float("-inf"), -1), (float("nan"), 5), (float("inf"), -3)]):
        t, n = (int(j) for j in torch.nonzero(passes[:, :, h])[i])
        dy[t, n, h] = v
    bt, bn, bh = (int(i[0]) for i in torch.nonzero(blocks[:, :, 10:]).T)
    dy[bt, bn, bh + 10] = float("inf")                           # blocked: reaches nothing
    stock = _stock(x, dy, w, torch.float16)
    fused = _fused(x, dy, w, lens, torch.float16)
    valid = ~_past(T, lens).expand_as(x)
    for k, a, b in (("dw", fused["dw"], stock["dw"]), ("dx", fused["dx"][valid], stock["dx"][valid])):
        for cls in (torch.isnan, torch.isposinf, torch.isneginf):
            assert torch.equal(cls(a), cls(b.to(a.dtype))), (k, cls.__name__)
        assert not torch.isfinite(a).all(), k
    assert torch.isfinite(fused["dw"][bh + 10]).all() and torch.isfinite(fused["dw"][4:]).all()


@pytest.mark.parametrize("case", ["cpu", "fp64", "noncontiguous", "taps_over_the_cap"])
def test_fallbacks_are_the_stock_module(case):
    g = torch.Generator(device="cuda").manual_seed(5)
    T, N, Hs, context = 12, 3, 16, 4
    x = 4 * torch.randn(T, N, Hs, device="cuda", generator=g)
    w = torch.randn(Hs, context + 1, device="cuda", generator=g)
    lens = torch.tensor([12, 7, 3], dtype=torch.int32, device="cuda")
    if case == "cpu":
        x, w, lens = x.cpu(), w.cpu(), lens.cpu()
    elif case == "fp64":
        x = x.double()
        w = w.double()
    elif case == "noncontiguous":
        x = (4 * torch.randn(T, Hs, N, device="cuda", generator=g)).transpose(1, 2)
    else:
        assert fused_lookahead.max_taps() == 32
        w = torch.randn(Hs, 33, device="cuda", generator=g)
    xi, wi = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    n0 = ext.LAUNCH_COUNT.get("lookahead_forward", 0), ext.LAUNCH_COUNT.get("lookahead_backward", 0)
    y = fused_lookahead.lookahead_hardtanh(xi, wi, lens)
    dy = torch.randn_like(y)
    gx, gw = torch.autograd.grad(y, [xi, wi], dy)
    assert (ext.LAUNCH_COUNT.get("lookahead_forward", 0), ext.LAUNCH_COUNT.get("lookahead_backward", 0)) == n0
    la = Lookahead(Hs, w.size(1) - 1).to(device=x.device, dtype=x.dtype)
    with torch.no_grad():
        la.weight.copy_(w)
    xr = x.clone().requires_grad_(True)
    yr = nn.Sequential(la, nn.Hardtanh(0, 20, inplace=True))(xr)
    rx, rw = torch.autograd.grad(yr, [xr, la.weight], dy)
    assert torch.equal(y, yr) and torch.equal(gx, rx) and torch.equal(gw, rw)


# ------------------------------------------------------------------------------------------------------ 3. the model
def _max_rel(a, b, floor=0.0):
    return ((a.double() - b.double()).abs().max() / max(b.double().abs().max().item(), floor, 1e-30)).item()


@pytest.mark.parametrize("kw", [{}, {"fuse_lstm": True, "fuse_bn": True}], ids=["stock_layers", "fused_layers"])
def test_one_eager_step_gives_the_stock_loss_and_gradients(kw, monkeypatch):
    """Loss within 1e-5, every parameter gradient within 1e-4 of the largest gradient of its tensor (or 1e-3 of the
    network's largest: the conv biases in front of a batch-norm cancel to rounding noise)."""
    from oktopk_b200.models import create_net
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    torch.manual_seed(0)
    fused = create_net(29, "lstman4", fuse_lookahead=True, **kw)[0].cuda().train()
    stock = create_net(29, "lstman4", **kw)[0].cuda().train()
    stock.load_state_dict(fused.state_dict())                    # the state dicts interchange
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(2, 1, 161, 120, device="cuda", generator=g)
    lens = torch.tensor([120, 83], dtype=torch.int32)
    wt = torch.randn(2, 60, 29, device="cuda", generator=g)
    res = []
    for net in (stock, fused):
        n0 = ext.LAUNCH_COUNT.get("lookahead_forward", 0), ext.LAUNCH_COUNT.get("lookahead_backward", 0)
        out, out_lens = net(x, lens)
        loss = (out.log_softmax(-1) * wt).sum()
        grads = torch.autograd.grad(loss, list(net.parameters()))
        n1 = ext.LAUNCH_COUNT.get("lookahead_forward", 0), ext.LAUNCH_COUNT.get("lookahead_backward", 0)
        assert n1 == ((n0[0] + 1, n0[1] + 1) if net is fused else n0)
        res.append((loss.detach(), out.detach(), grads, [b.clone() for b in net.buffers()]))
    (ls, os_, gs, bs), (lf, of, gf, bf) = res
    assert _max_rel(lf, ls) < 1e-5
    assert _max_rel(of, os_) < 1e-4
    floor = 1e-3 * max(g_.abs().max().item() for g_ in gs)
    errs = {n: _max_rel(a, b, floor) for (n, _), a, b in zip(stock.named_parameters(), gf, gs)}
    assert max(errs.values()) < 1e-4, errs
    for a, b in zip(bf, bs):
        assert torch.allclose(a.double(), b.double(), rtol=1e-4, atol=1e-6)
    fused.load_state_dict(stock.state_dict())
    fused.eval()
    stock.eval()
    with torch.no_grad():
        assert _max_rel(fused(x, lens)[0], stock(x, lens)[0]) < 1e-4


def test_the_bidirectional_network_refuses_fuse_lookahead():
    from oktopk_b200.models import create_net
    with pytest.raises(ValueError, match="fuse_lookahead"):
        create_net(29, "lstman4", bidirectional=True, fuse_lookahead=True)


# ------------------------------------------------------------------------------------------------- 4. the trainers
KW = {"fuse_lstm": True, "fuse_ctc": True, "fuse_bn": True, "fuse_lookahead": True}


def _trainer(m, graph, autocast=None, loss_scale=None, model_kwargs=KW):
    import bench
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=5)
    return Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, density=0.001, cfg=cfg, compressor="oktopk",
                   t_total=100000, warmup=0.1, seed=0, cuda_graph=graph, an4_pad_multiple=m,
                   autocast=autocast, loss_scale=loss_scale, model_kwargs=dict(model_kwargs))


def _mixed_batches(n, bs=2):
    from oktopk_b200.train.data import SyntheticAN4, an4_collate
    ds = SyntheticAN4(n=n * bs, seed=3)
    return [tuple(t.cuda() for t in an4_collate([ds[i * bs + j] for j in range(bs)])) for i in range(n)]


@pytest.mark.parametrize("mode", ["fp32", "bf16", "fp16"])
def test_graphed_padded_follows_eager_padded(mode):
    kw = dict(autocast={"bf16": "bf16", "fp16": "fp16"}.get(mode),
              loss_scale="dynamic" if mode == "fp16" else None,
              model_kwargs=dict(KW, fuse_lstm_autocast=True) if mode in ("bf16", "fp16") else KW)
    pool = _mixed_batches(4)
    eager, graphed = _trainer(32, False, **kw), _trainer(32, True, **kw)
    gs = graphed.graphed
    assert gs.enabled, gs.why_disabled
    assert eager.net.fuse_lookahead and graphed.net.fuse_lookahead
    n0 = ext.LAUNCH_COUNT.get("lookahead_forward", 0)
    for it in range(16):
        b = pool[it % len(pool)]
        la = eager.step(b)
        lb = graphed.step(b)
        assert torch.equal(_bits(la), _bits(lb)), (mode, it)
    assert ext.LAUNCH_COUNT.get("lookahead_forward", 0) > n0
    torch.cuda.synchronize()
    n_graphs = len(gs.graphs)
    torch.cuda.set_sync_debug_mode("error")
    try:
        for b in pool:
            graphed.step(b)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for b in pool:
        eager.step(b)
    torch.cuda.synchronize()
    assert len(gs.graphs) == n_graphs
    for pa, pb in zip(eager.net.parameters(), graphed.net.parameters()):
        assert torch.equal(_bits(pa), _bits(pb))
    for ba, bb in zip(eager.net.buffers(), graphed.net.buffers()):
        assert torch.equal(ba, bb)
    assert gs.fallbacks == {"shapes": 0, "targets": 0}
    for tr in (eager, graphed):
        tr.close()


# ----------------------------------------------------------------------------------------------- 5. launch counts
@pytest.mark.parametrize("device_lengths", [False, True])
def test_one_launch_per_pass(device_lengths):
    from oktopk_b200.models import create_net
    net = create_net(29, "lstman4", **KW)[0].cuda().train()
    x = torch.randn(2, 1, 161, 120, device="cuda")
    lens = torch.tensor([120, 90], dtype=torch.int32)
    if device_lengths:
        lens = lens.cuda()
    f0, b0 = ext.LAUNCH_COUNT.get("lookahead_forward", 0), ext.LAUNCH_COUNT.get("lookahead_backward", 0)
    out, _ = net(x, lens, device_lengths=device_lengths)
    assert ext.LAUNCH_COUNT.get("lookahead_forward", 0) == f0 + 1
    out.float().square().sum().backward()
    assert ext.LAUNCH_COUNT.get("lookahead_backward", 0) == b0 + 1
    assert torch.isfinite(net.lookahead[0].weight.grad).all()
