"""fp16 activations through the fused batch-norm kernels of csrc/bnrelu.cu (opt-in: ``fp16=True`` in ops/fused_bn.py,
``VGG(fuse_fp16=True)``): bit for bit the fp32 kernels on the widened input with y and dx rounded to fp16, including
fp16's range (overflow to inf, subnormals, non-finite inputs); torch's own fp16 batch-norm within fp16 rounding; a whole
VGG-16 step under fp16 autocast; dynamic loss scaling through the fused path, eager and in whole-step CUDA graphs,
and an overflow produced inside the fused backward reaching the optimizer's check.  The CPU tests cover the switch."""
import copy
from unittest import mock

import pytest
import torch

gpu = pytest.mark.gpu

# the BN input of the 13 VGG-16 layers at 16 images (2, 2, 3, 3, 3 layers per block; the last of a block is pooled)
VGG_SHAPES = [(16, 64, 32, 32), (16, 128, 16, 16), (16, 256, 8, 8), (16, 512, 4, 4), (16, 512, 2, 2)]
FALLBACK = (3, 20, 6, 10)           # tiles are not whole pairs of image rows: the pool cannot be folded in
F16_MIN_NORMAL = 2.0 ** -14


def _bn(C, seed):
    torch.manual_seed(seed)
    bn = torch.nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        bn.weight.normal_(1.0, 0.3); bn.bias.normal_(0.0, 0.5)
        bn.running_mean.normal_(0.0, 0.1); bn.running_var.uniform_(0.5, 1.5)
    return bn


def _inputs(shape, seed, pooled, dy_scale=1.0):
    g = torch.Generator("cuda").manual_seed(seed)
    N, C, H, W = shape
    x = (torch.randn(shape, device="cuda", generator=g) * 1.7 + 0.3).half().contiguous(memory_format=torch.channels_last)
    cbias = torch.randn(C, device="cuda", generator=g) * 0.2
    dshape = (N, C, H // 2, W // 2) if pooled else shape
    dy = (torch.randn(dshape, device="cuda", generator=g) * dy_scale).half().contiguous(memory_format=torch.channels_last)
    return x, cbias, dy


def _run_fused(x, bn, cbias, pool, dy, fp16=True):
    from oktopk_b200.ops.fused_bn import bias_bn_relu
    xa = x.detach().clone().requires_grad_(True)
    y = bias_bn_relu(xa, bn, cbias, True, pool, fp16=fp16)
    y.backward(dy)
    return y, xa.grad, bn.weight.grad, bn.bias.grad


def _same(a, b):
    """Equal up to the NaN bits: the same NaN positions, every other element (infinities included) equal."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0), b.masked_fill(nb, 0))


def _fused_pair(shape, pooled, seed, x=None, dy=None, bn_init=None, nan_ok=False):
    """The fp16 kernels and the fp32 kernels on x.float() / dy.float(): y, dx bitwise (y32, dx32).half(); dgamma, dbeta,
    the running statistics and the batch counter bitwise."""
    pool = torch.nn.MaxPool2d(2, 2) if pooled else None
    x0, cbias, dy0 = _inputs(shape, seed, pooled)
    x = x0 if x is None else x
    dy = dy0 if dy is None else dy
    bn16, bn32 = _bn(shape[1], seed), _bn(shape[1], seed)
    if bn_init is not None:
        bn_init(bn16); bn_init(bn32)
    y, dx, dg, db = _run_fused(x, bn16, cbias, pool, dy)
    y32, dx32, dg32, db32 = _run_fused(x.float(), bn32, cbias, pool, dy.float())
    assert y.dtype == dx.dtype == torch.float16 and dg.dtype == db.dtype == torch.float32
    assert y.is_contiguous(memory_format=torch.channels_last) and dx.is_contiguous(memory_format=torch.channels_last)
    eq = _same if nan_ok else torch.equal
    assert eq(y, y32.half())
    assert eq(dx, dx32.half())
    assert eq(dg, dg32) and eq(db, db32)
    assert eq(bn16.running_mean, bn32.running_mean) and eq(bn16.running_var, bn32.running_var)
    assert int(bn16.num_batches_tracked) == int(bn32.num_batches_tracked) == 1
    return y, dx, dg, db, bn16


# ------------------------------------------------------------------------------------------ 1. against the fp32 kernel
@gpu
@pytest.mark.parametrize("pooled", [False, True])
@pytest.mark.parametrize("shape", VGG_SHAPES)
def test_fp16_kernel_is_fp32_kernel_on_widened_input(shape, pooled):
    """The fp16 kernels compute exactly what the fp32 kernels compute on x.float() / dy.float(), with y and dx rounded
    to fp16: the same bits, and the same fp32 dgamma, dbeta and running statistics; one launch per pass, no pool."""
    from oktopk_b200.ops import ext
    n0 = {k: ext.LAUNCH_COUNT.get(k, 0) for k in ("bn_forward", "bn_backward", "maxpool2_fwd", "maxpool2_bwd")}
    _fused_pair(shape, pooled, 5)
    d = {k: ext.LAUNCH_COUNT.get(k, 0) - v for k, v in n0.items()}
    assert d == {"bn_forward": 2, "bn_backward": 2, "maxpool2_fwd": 0, "maxpool2_bwd": 0}, d


@gpu
def test_fp16_kernel_fallback_shape():
    """A shape whose pool cannot be folded in: the fp16 batch-norm is still bitwise the fp32 one, and the pool then runs
    on torch's MaxPool2d in fp16 (the standalone pool kernels are fp32 only)."""
    from oktopk_b200.ops import ext
    from oktopk_b200.ops.fused_bn import _pool_fusable
    _fused_pair(FALLBACK, False, 5)
    pool = torch.nn.MaxPool2d(2, 2)
    x, cbias, dy = _inputs(FALLBACK, 9, True)
    assert not _pool_fusable(x, pool)
    bn16, bn32 = _bn(FALLBACK[1], 9), _bn(FALLBACK[1], 9)
    n0 = {k: ext.LAUNCH_COUNT.get(k, 0) for k in ("bn_forward", "maxpool2_fwd")}
    y, dx, dg, db = _run_fused(x, bn16, cbias, pool, dy)
    assert {k: ext.LAUNCH_COUNT.get(k, 0) - v for k, v in n0.items()} == {"bn_forward": 1, "maxpool2_fwd": 0}
    y32, *_ = _run_fused(x.float(), bn32, cbias, pool, dy.float())
    assert y.dtype == dx.dtype == torch.float16
    assert torch.equal(y, y32.half())                 # rounding is monotonic: the max of the rounded is the rounded max
    assert torch.equal(bn16.running_mean, bn32.running_mean) and torch.equal(bn16.running_var, bn32.running_var)


@gpu
@pytest.mark.parametrize("shape,pooled", [((16, 64, 32, 32), True), ((16, 512, 2, 2), True), ((128, 64, 32, 32), True),
                                          ((2, 1032, 3, 3), False)])
def test_fp16_capped_grid(shape, pooled, monkeypatch):
    """A grid smaller than the tile count (tiles read again from global memory, tiles too large to hold, more than one
    column tile): bitwise the fp32 kernels, and bitwise the uncapped fp16 grid."""
    from oktopk_b200.ops import fused_bn
    ref = _fused_pair(shape, pooled, 3)
    monkeypatch.setattr(fused_bn, "MAX_CTAS", 5)
    got = _fused_pair(shape, pooled, 3)
    for a, b in zip(ref[:4], got[:4]):
        assert torch.equal(a, b)
    assert torch.equal(ref[4].running_mean, got[4].running_mean) and torch.equal(ref[4].running_var, got[4].running_var)


# ------------------------------------------------------------------------------------------ 2. fp16's range
@gpu
@pytest.mark.parametrize("pooled", [False, True])
def test_fp16_overflow_is_inf_where_the_rounded_fp32_result_is(pooled):
    """Large gamma on some channels, near-constant input on others: some y and some dx round past 65504.  They are
    stored as inf exactly where (fp32 kernel).half() is inf (no saturation), and every other bit matches."""
    shape = (16, 128, 16, 16)
    C = shape[1]
    x, _, _ = _inputs(shape, 11, pooled)
    g = torch.Generator("cuda").manual_seed(10)
    x = x.clone()
    x[:, C // 2:C // 2 + 8] = (5.0 + 0.02 * torch.randn(shape[0], 8, *shape[2:], device="cuda", generator=g)).half()

    def init(bn):
        with torch.no_grad():
            bn.weight[:C // 4] = 3.0e4                  # |y| = gamma |xhat| past 65504 beyond ~2.2 standard deviations
            bn.weight[C // 2:C // 2 + 8] = 400.0        # a = gamma / std ~ 2e4: dx overflows, y stays finite

    _, _, dy = _inputs(shape, 12, pooled, dy_scale=4.0)
    y, dx, dg, db, _ = _fused_pair(shape, pooled, 11, x=x, dy=dy, bn_init=init)
    for t in (y, dx):
        assert not torch.isnan(t).any()
        assert 0 < int(torch.isinf(t).sum()) < t.numel() // 4, int(torch.isinf(t).sum())
    assert bool((y.float() >= 0).all())                 # +inf only, after the ReLU
    assert bool(torch.isinf(dx).flatten(2).any(2)[:, C // 2:C // 2 + 8].any())
    assert torch.isfinite(dg).all() and torch.isfinite(db).all()


@gpu
@pytest.mark.parametrize("pooled", [False, True])
def test_fp16_subnormals_are_kept(pooled):
    """A tiny dy (itself largely fp16-subnormal) puts a sizeable fraction of dx below 2^-14, and a tiny gamma does the
    same to y on a quarter of the channels: the subnormals are stored, not flushed, bit for bit (fp32 kernel).half()."""
    shape = (16, 128, 16, 16)
    C = shape[1]
    _, _, dy = _inputs(shape, 13, pooled, dy_scale=2.0 ** -16)
    assert float((dy != 0).float().mean()) > 0.9

    def init(bn):
        with torch.no_grad():
            bn.weight[:C // 4] = 2.0 ** -16
            bn.bias[:C // 4] = 0.0

    y, dx, *_ = _fused_pair(shape, pooled, 13, dy=dy, bn_init=init)

    def sub(t):
        return float(((t != 0) & (t.float().abs() < F16_MIN_NORMAL)).float().mean())

    assert sub(dx) > 0.1, sub(dx)
    assert sub(y[:, :C // 4]) > 0.25, sub(y[:, :C // 4])


@gpu
@pytest.mark.parametrize("pooled", [False, True])
@pytest.mark.parametrize("where", ["x", "dy"])
def test_fp16_non_finite_inputs_propagate_as_in_fp32(where, pooled):
    """inf, -inf and NaN planted in x (single elements) or dy (one image plane each, so that the ReLU cannot mask them
    all): the fp16 kernels propagate them exactly as the fp32 kernels do on the widened input -- into dx, dgamma /
    dbeta and, from x, the running statistics -- with the same non-finite positions and every other element equal.
    (The forward's ReLU, fmaxf, turns a NaN pre-activation into 0 in both.)"""
    shape = (16, 128, 16, 16)
    x, _, dy = _inputs(shape, 15, pooled)
    t = (x if where == "x" else dy).clone()
    at = (slice(1, 2), slice(2, 3)) if where == "x" else (slice(None), slice(None))
    t[(3, 5) + at] = float("inf")
    t[(7, 40) + at] = float("-inf")
    t[(1, 77) + at] = float("nan")
    if where == "x":
        x = t.contiguous(memory_format=torch.channels_last)
    else:
        dy = t.contiguous(memory_format=torch.channels_last)
    y, dx, dg, db, bn = _fused_pair(shape, pooled, 15, x=x, dy=dy, nan_ok=True)
    assert not torch.isfinite(dx).all() and not torch.isfinite(dg).all()
    assert torch.isfinite(dx[:, :5]).all() and torch.isfinite(dg[:5]).all()      # untouched channels stay finite
    if where == "x":                  # NaN statistics: the ReLU mask is all-zero there, so dbeta stays 0
        assert not torch.isfinite(bn.running_mean).all() and torch.isfinite(bn.running_mean[:5]).all()
    else:
        assert not torch.isfinite(db).all()
        assert torch.isfinite(y).all() and torch.isfinite(bn.running_var).all()


# ------------------------------------------------------------------------------------------ 3. against torch's fp16 path
def _fp16_ulp(t):
    """One fp16 ulp at |t| (fp32 result; 2^-24 for zero and subnormals)."""
    a = t.float().abs()
    e = torch.frexp(a)[1]
    ulp = torch.ldexp(torch.ones_like(a), (e - 11).clamp(min=-24))
    return torch.where(a == 0, torch.full_like(a, 2.0 ** -24), ulp)


def _tied_windows(ypre):
    """Pooled positions whose 2x2 window has its (positive) fp16 maximum more than once: there torch's arg-max (the
    first of the rounded values) and the fused kernel's (that of the fp32 values) may differ."""
    N, C, H, W = ypre.shape
    w = ypre.float().reshape(N, C, H // 2, 2, W // 2, 2)
    m = w.amax(dim=(3, 5), keepdim=True)
    return (((w == m).sum(dim=(3, 5), keepdim=True) > 1) & (m > 0)).reshape(N, C, H // 2, W // 2)


@gpu
@pytest.mark.parametrize("pooled", [False, True])
@pytest.mark.parametrize("shape", VGG_SHAPES + [FALLBACK])
def test_fp16_matches_torch_autocast(shape, pooled):
    """Against stock BatchNorm2d -> ReLU [-> MaxPool2d] under torch.autocast(fp16) on the same fp16 input: y within one
    fp16 ulp, statistics and dgamma / dbeta at the fp32 tolerances, dx within one ulp up to a few elements at a ReLU
    boundary.  The pooled gradient is zero at windows whose rounded maximum is tied."""
    from oktopk_b200.ops.fused_bn import bias_bn_relu
    pool = torch.nn.MaxPool2d(2, 2) if pooled else None
    x, _, dy = _inputs(shape, 17, pooled)
    bn_f, bn_t = _bn(shape[1], 17), _bn(shape[1], 17)
    xf = x.detach().clone().requires_grad_(True)
    xt = x.detach().clone().requires_grad_(True)
    with torch.autocast("cuda", torch.float16):
        y = bias_bn_relu(xf, bn_f, None, True, pool, fp16=True)
        ypre = torch.relu(bn_t(xt))
        yt = pool(ypre) if pooled else ypre
    if pooled:
        tied = _tied_windows(ypre)
        assert int(tied.sum()) <= tied.numel() // 10
        dy = dy.masked_fill(tied, 0).contiguous(memory_format=torch.channels_last)
    y.backward(dy)
    yt.backward(dy)
    dx, dg, db = xf.grad, bn_f.weight.grad, bn_f.bias.grad
    assert yt.dtype == y.dtype == dx.dtype == torch.float16 and y.shape == yt.shape
    assert int(bn_f.num_batches_tracked) == int(bn_t.num_batches_tracked) == 1
    diff = (y.float() - yt.float()).abs()
    assert bool((diff <= _fp16_ulp(torch.maximum(y.float().abs(), yt.float().abs())) + 2e-5).all()), float(diff.max())
    torch.testing.assert_close(bn_f.running_mean, bn_t.running_mean, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(bn_f.running_var, bn_t.running_var, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(dg, bn_t.weight.grad, rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(db, bn_t.bias.grad, rtol=2e-3, atol=2e-3)
    ddx = (dx.float() - xt.grad.float()).abs()
    bad = int((ddx > _fp16_ulp(torch.maximum(dx.float().abs(), xt.grad.float().abs())) + 1e-5).sum())
    assert bad <= max(4, dx.numel() // 20000), bad


# ------------------------------------------------------------------------------------------ 4. whole model
def _vgg(**kw):
    from oktopk_b200.models import create_net
    torch.manual_seed(0)
    net, _ = create_net(10, "vgg16", **kw)
    return net.cuda().to(memory_format=torch.channels_last)


def _grads(net, x, y, autocast, scale=1024.0):
    """Gradients of a loss scaled by ``scale`` (a power of two: exact), unscaled again, as loss scaling does."""
    net.zero_grad(set_to_none=True)
    with torch.autocast("cuda", torch.float16, enabled=autocast):
        loss = torch.nn.functional.cross_entropy(net(x), y)
    (loss * scale).backward()
    return {n: None if p.grad is None else p.grad / scale for n, p in net.named_parameters()}


@gpu
def test_vgg16_fp16_autocast_step():
    """One VGG-16 forward/backward under fp16 autocast with ``fuse_fp16=True``: 13 bn_forward and 13 bn_backward
    launches, no standalone pool, no stock batch-norm; each gradient no further from the fp32 one than stock fp16's.
    With ``fuse_fp16=False`` the same step launches no kernel of the package."""
    from oktopk_b200.ops import ext
    torch.backends.cudnn.deterministic = True
    ref = _vgg()
    fused = _vgg(fuse_fp16=True)
    stock = copy.deepcopy(ref)
    stock.fuse = False
    assert fused.fuse and fused.fuse_fp16 and not ref.fuse_fp16
    g = torch.Generator("cuda").manual_seed(1)
    x = torch.randn(16, 3, 32, 32, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (16,), device="cuda", generator=g)
    g32 = _grads(ref, x, y, False)
    n0 = {k: ext.LAUNCH_COUNT.get(k, 0) for k in ("bn_forward", "bn_backward", "maxpool2_fwd", "maxpool2_bwd")}

    def no_stock_bn(*a, **k):
        raise AssertionError("stock BatchNorm2d.forward ran on the fused path")

    with mock.patch.object(torch.nn.BatchNorm2d, "forward", no_stock_bn):
        gf = _grads(fused, x, y, True)
    d = {k: ext.LAUNCH_COUNT.get(k, 0) - v for k, v in n0.items()}
    assert d == {"bn_forward": 13, "bn_backward": 13, "maxpool2_fwd": 0, "maxpool2_bwd": 0}, d
    gs = _grads(stock, x, y, True)
    checked = 0
    for n, a in gf.items():
        if a is None:                       # conv bias ahead of a batch-norm: no gradient (see ops/fused_bn.py)
            assert n.startswith("features.") and n.endswith(".bias"), n
            continue
        assert a.dtype == torch.float32 and torch.isfinite(a).all(), n
        ref_norm = float(g32[n].norm())
        ef = float((a - g32[n]).norm()) / ref_norm
        es = float((gs[n] - g32[n]).norm()) / ref_norm
        assert ef <= 1.5 * es + 1e-3, (n, ef, es)
        checked += 1
    assert checked == 2 * 13 + 13 + 2         # conv weights, BN weight and bias, fc weight and bias

    off = copy.deepcopy(ref)                  # fuse on, fuse_fp16 off: today's fp16 behaviour
    assert off.fuse and not off.fuse_fp16
    n0 = ext.LAUNCH_COUNT["total"]
    _grads(off, x, y, True)
    assert ext.LAUNCH_COUNT["total"] == n0


# ------------------------------------------------------------------------------------------ 5. loss scaling
def _trainer(graph, loss_scale, warmup_iters, lr=0.05):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    return Trainer(dnn="vgg16", dataset="cifar10", batch_size=16, lr=lr, compressor="oktopk", density=0.001,
                   cfg=okt.preset("vgg16", density=0.001, warmup_iters=warmup_iters), autocast="fp16",
                   loss_scale=loss_scale, model_kwargs={"fuse_fp16": True}, cuda_graph=graph, seed=0)


def _eager_step(tr, batch):
    tr.optimizer.zero_grad()
    loss, _ = tr._forward_loss(batch)
    tr.backward(loss)
    tr.update_model()


def _count_graph_work(gs):
    """Per captured graph, the fused batch-norm and unscale_check launches it recorded; and the number of eager steps."""
    from oktopk_b200.ops import ext
    names = ("bn_forward", "bn_backward", "unscale_check")
    rec = {"captures": [], "eager": 0}
    capture, eager = gs._capture, gs._eager

    def counted_capture(key):
        n0 = {k: ext.LAUNCH_COUNT.get(k, 0) for k in names}
        g = capture(key)
        if g is not None:
            rec["captures"].append({k: ext.LAUNCH_COUNT.get(k, 0) - v for k, v in n0.items()})
        return g

    def counted_eager(batch):
        rec["eager"] += 1
        return eager(batch)

    gs._capture, gs._eager = counted_capture, counted_eager
    return rec


@gpu
def test_trainer_fp16_fused_loss_scaled_cuda_graph_matches_eager():
    """Trainer(autocast="fp16", loss_scale=LossScale(), fuse_fp16=True) on VGG-16 Ok-Topk: graph-replayed steps over the
    dense-to-sparse transition and 36 sparse steps give the parameters, buffers and loss-scale history of the same
    steps run eagerly, bit for bit; every captured graph holds the 13 + 13 fused batch-norm launches."""
    from oktopk_b200.config import LossScale
    torch.backends.cudnn.deterministic = True
    tg, te = _trainer(True, LossScale(), 4), _trainer(False, LossScale(), 4)
    assert tg.graphed is not None and te.graphed is None and tg.net.fuse_fp16 and te.net.fuse_fp16
    rec = _count_graph_work(tg.graphed)
    g = torch.Generator("cuda").manual_seed(2)
    batches = [(torch.randn(16, 3, 32, 32, device="cuda", generator=g).contiguous(memory_format=torch.channels_last),
                torch.randint(0, 10, (16,), device="cuda", generator=g)) for _ in range(4)]
    hist = {True: [], False: []}
    steps = 4 + 36
    for it in range(steps):
        batch = batches[it % len(batches)]
        tg.graphed.step(batch)
        _eager_step(te, batch)
        hist[True].append(tg.optimizer.loss_scale_state())
        hist[False].append(te.optimizer.loss_scale_state())
    torch.cuda.synchronize()
    assert tg.graphed.enabled, tg.graphed.why_disabled
    assert len(tg.graphed.graphs) >= 2 and rec["captures"]
    assert steps - rec["eager"] >= 30, rec["eager"]           # the rest were replays
    for c in rec["captures"]:
        assert c["bn_forward"] == 13 and c["bn_backward"] == 13 and c["unscale_check"] >= 1, c
    assert hist[True] == hist[False]
    assert any(h["growth_tracker"] > 0 for h in hist[True])    # steps were applied
    for (n, a), b in zip(tg.net.named_parameters(), te.net.parameters()):
        assert torch.isfinite(a).all(), n
        assert torch.equal(a, b), n
    for (n, a), b in zip(tg.net.named_buffers(), te.net.buffers()):
        assert torch.equal(a, b), n
    tg.close()
    te.close()


@gpu
def test_vgg16_fp16_fused_graphed_overflow_skips_until_the_first_applied_step():
    """The same workload through the fused fp16 kernels with LossScale(2^40): every overflowing step, eager or replayed,
    leaves parameters, momentum and residual bitwise unchanged and halves the scale, until the scale comes down to
    applied steps; graphed and eager runs agree, and the replay loop adds no host synchronisation."""
    from oktopk_b200.config import LossScale
    from oktopk_b200.ops import ext
    torch.backends.cudnn.deterministic = True
    runs = {}
    for graph in (False, True):
        tr = _trainer(graph, LossScale(init_scale=2.0 ** 40), 0, lr=0.01)
        tr.net.train()
        opt = tr.optimizer
        assert len(opt._buckets) == 1
        batch = tuple(t.cuda() for t in next(iter(tr.loader)))
        eng = opt._allreducer._engines[opt._buckets[0].name]
        hist, applied = [], 0
        n_bn = ext.LAUNCH_COUNT.get("bn_backward", 0)
        for i in range(48):
            snap = ([p.detach().clone() for p in tr.net.parameters()],
                    [t.clone() for fs in opt._flat_state.values() for t in fs.values()], eng.residual.clone())
            scale_before = opt.loss_scale_state()["scale"]
            if graph and i >= 4:                  # replays only: the first graphed step captured every flavour
                torch.cuda.set_sync_debug_mode("error")
            try:
                tr.graphed.step(batch) if graph else _eager_step(tr, batch)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            st = opt.loss_scale_state()
            skipped = st["scale"] < scale_before
            if skipped:
                assert st["scale"] == scale_before / 2
                assert all(torch.equal(a, p) for a, p in zip(snap[0], tr.net.parameters()))
                assert all(torch.equal(a, b) for a, b in zip(snap[1], [t for fs in opt._flat_state.values()
                                                                          for t in fs.values()]))
                assert torch.equal(snap[2], eng.residual)
            else:
                applied += 1
            hist.append((skipped, st["scale"]))
            if applied == 3:
                break
        assert ext.LAUNCH_COUNT.get("bn_backward", 0) - n_bn >= 13
        if graph:
            assert tr.graphed.enabled, tr.graphed.why_disabled
        runs[graph] = (hist, [p.detach().clone() for p in tr.net.parameters()])
        tr.close()
    hist, params = runs[True]
    assert hist[0][0], "2^40 must overflow the fp16 backward"
    assert sum(not h[0] for h in hist) == 3, "the scale must come down to applied steps"
    assert hist == runs[False][0]
    for a, b in zip(params, runs[False][1]):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def _conv_bn_grad(gamma, dy_scale):
    """Conv -> fused fp16 BN -> ReLU under fp16 autocast, backward from a finite dy: (y, dy, the BN input's gradient,
    the fp32 conv-weight gradient)."""
    from oktopk_b200.ops.fused_bn import bias_bn_relu
    torch.manual_seed(21)
    conv = torch.nn.Conv2d(16, 32, 3, padding=1).cuda().to(memory_format=torch.channels_last)
    bn = torch.nn.BatchNorm2d(32).cuda()
    with torch.no_grad():
        bn.weight.fill_(gamma)
    g = torch.Generator("cuda").manual_seed(22)
    x = torch.randn(8, 16, 8, 8, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    with torch.autocast("cuda", torch.float16):
        z = torch.nn.functional.conv2d(x, conv.weight, None, 1, 1)
        z.retain_grad()
        y = bias_bn_relu(z, bn, conv.bias, True, None, fp16=True)
    dy = (torch.randn(y.shape, device="cuda", generator=g) * dy_scale).half().contiguous(memory_format=torch.channels_last)
    y.backward(dy)
    return y, dy, z.grad, conv.weight.grad


@gpu
def test_overflow_inside_fused_backward_sets_the_step_verdict():
    """dy is finite, but the fused backward's dx = a (dy - ...) rounds past 65504: the inf it stores reaches the conv
    weight gradient, and ``unscale_check`` on that gradient sets the step verdict.  The same layer with a small gamma
    stays finite and leaves the verdict clear."""
    from oktopk_b200.config import LossScale, OkTopkConfig
    from oktopk_b200.optimizer import _ScaleState
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.world import World
    verdicts = {}
    for gamma in (1.0, 2000.0):
        y, dy, dz, gw = _conv_bn_grad(gamma, 30.0)
        assert torch.isfinite(dy).all() and torch.isfinite(y).all() and gw.dtype == torch.float32
        overflow = gamma > 1.0
        assert bool(torch.isinf(dz).any()) == overflow
        assert bool(torch.isfinite(gw).all()) != overflow
        n = gw.numel()
        eng = CudaBucketEngine(n, OkTopkConfig(density=0.01), World(), name="t")
        ls = _ScaleState(LossScale(init_scale=2.0 ** 10), torch.device("cuda"))
        eng.unscale_check(ls.ptr, srcs=([gw.data_ptr()], [0], [n]))
        torch.cuda.synchronize()
        verdicts[gamma] = ls.state()["found_inf"]
        eng.close()
    assert verdicts == {1.0: 0, 2000.0: 1}, verdicts


# ------------------------------------------------------------------------------------------ 6. the switch (CPU)
def test_create_net_forwards_fuse_fp16():
    from oktopk_b200.models import create_net
    assert create_net(10, "vgg16", fuse_fp16=True)[0].fuse_fp16 is True
    assert create_net(10, "vgg11", fuse_fp16=True)[0].fuse_fp16 is True
    assert create_net(10, "vgg16")[0].fuse_fp16 is False


def test_cli_fused_bn_fp16_reaches_model_kwargs():
    from oktopk_b200.train import cli
    p = cli.build_parser()
    assert cli.model_args(p.parse_args(["--fp16", "--fused-bn-fp16"])) == ("vgg16", {"fuse_fp16": True})
    assert cli.model_args(p.parse_args(["--fp16"])) == ("vgg16", {})
    with pytest.raises(SystemExit):
        cli.main(["--fused-bn-fp16"])                 # meaningless without --fp16


@pytest.mark.parametrize("autocast", [None, torch.bfloat16, torch.float16])
def test_dtype_gate_changes_only_fp16(autocast, monkeypatch):
    """``fp16=False`` accepts exactly what the kernels accepted before fp16 existed (fp32 / bf16, autocast off or bf16);
    ``fp16=True`` adds fp16 activations (autocast off or fp16) and fp32 input under fp16 autocast, and nothing else."""
    from oktopk_b200.ops import fused_bn
    monkeypatch.setattr(torch, "is_autocast_enabled", lambda *a: autocast is not None)
    monkeypatch.setattr(torch, "get_autocast_dtype", lambda *a: autocast or torch.float16)
    for dt in (torch.float32, torch.bfloat16, torch.float16, torch.float64):
        x = torch.empty(1, dtype=dt)
        before = dt in (torch.float32, torch.bfloat16) and autocast in (None, torch.bfloat16)
        assert fused_bn._dtype_ok(x) == fused_bn._dtype_ok(x, fp16=False) == before, (dt, autocast)
        opted = (dt == torch.float16 and autocast in (None, torch.float16)) or (dt == torch.float32
                                                                                and autocast == torch.float16)
        assert fused_bn._dtype_ok(x, fp16=True) == (before or opted), (dt, autocast)
