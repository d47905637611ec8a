"""bf16 activations through the fused batch-norm kernels of csrc/bnrelu.cu: bit for bit the fp32 kernels on the widened
input with y and dx rounded, torch's own bf16 batch-norm within bf16 rounding, a whole VGG-16 step under bf16 autocast,
the dtype gate, and whole-step CUDA graphs under bf16 autocast."""
import copy
from unittest import mock

import pytest
import torch

pytestmark = pytest.mark.gpu

# the BN input of the 13 VGG-16 layers at 16 images (2, 2, 3, 3, 3 layers per block; the last of a block is pooled)
VGG_SHAPES = [(16, 64, 32, 32), (16, 128, 16, 16), (16, 256, 8, 8), (16, 512, 4, 4), (16, 512, 2, 2)]
FALLBACK = (3, 20, 6, 10)           # tiles are not whole pairs of image rows: the pool cannot be folded in


def _bn(C, seed):
    torch.manual_seed(seed)
    bn = torch.nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        bn.weight.normal_(1.0, 0.3); bn.bias.normal_(0.0, 0.5)
        bn.running_mean.normal_(0.0, 0.1); bn.running_var.uniform_(0.5, 1.5)
    return bn


def _inputs(shape, seed, pooled):
    g = torch.Generator("cuda").manual_seed(seed)
    N, C, H, W = shape
    x = (torch.randn(shape, device="cuda", generator=g) * 1.7 + 0.3).bfloat16().contiguous(memory_format=torch.channels_last)
    cbias = torch.randn(C, device="cuda", generator=g) * 0.2
    dshape = (N, C, H // 2, W // 2) if pooled else shape
    dy = torch.randn(dshape, device="cuda", generator=g).bfloat16().contiguous(memory_format=torch.channels_last)
    return x, cbias, dy


def _run_fused(x, bn, cbias, pool, dy):
    from oktopk_b200.ops.fused_bn import bias_bn_relu
    xa = x.detach().clone().requires_grad_(True)
    y = bias_bn_relu(xa, bn, cbias, True, pool)
    y.backward(dy)
    return y, xa.grad, bn.weight.grad, bn.bias.grad


def _bitwise_against_fp32(shape, pooled, seed=5):
    pool = torch.nn.MaxPool2d(2, 2) if pooled else None
    x, cbias, dy = _inputs(shape, seed, pooled)
    bn16, bn32 = _bn(shape[1], seed), _bn(shape[1], seed)
    y, dx, dg, db = _run_fused(x, bn16, cbias, pool, dy)
    y32, dx32, dg32, db32 = _run_fused(x.float(), bn32, cbias, pool, dy.float())
    assert y.dtype == dx.dtype == torch.bfloat16 and dg.dtype == db.dtype == torch.float32
    assert y.is_contiguous(memory_format=torch.channels_last) and dx.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(y, y32.bfloat16())
    assert torch.equal(dx, dx32.bfloat16())
    assert torch.equal(dg, dg32) and torch.equal(db, db32)
    assert torch.equal(bn16.running_mean, bn32.running_mean) and torch.equal(bn16.running_var, bn32.running_var)
    assert int(bn16.num_batches_tracked) == int(bn32.num_batches_tracked) == 1
    return y, dx, dg, db, bn16


# ------------------------------------------------------------------------------------------ 1. against the fp32 kernel
@pytest.mark.parametrize("pooled", [False, True])
@pytest.mark.parametrize("shape", VGG_SHAPES)
def test_bf16_kernel_is_fp32_kernel_on_widened_input(shape, pooled):
    """The bf16 kernels compute exactly what the fp32 kernels compute on x.float() / dy.float(), with y and dx rounded
    to bf16: the same bits, and the same fp32 dgamma, dbeta and running statistics."""
    from oktopk_b200.ops import ext
    n0 = {k: ext.LAUNCH_COUNT.get(k, 0) for k in ("bn_forward", "bn_backward", "maxpool2_fwd")}
    _bitwise_against_fp32(shape, pooled)
    d = {k: ext.LAUNCH_COUNT.get(k, 0) - v for k, v in n0.items()}
    assert d == {"bn_forward": 2, "bn_backward": 2, "maxpool2_fwd": 0}, d


def test_bf16_kernel_fallback_shape():
    """A shape whose pool cannot be folded in: the bf16 batch-norm is still bitwise the fp32 one, and the pool then runs
    on torch's MaxPool2d in bf16 (the standalone pool kernels are fp32 only)."""
    from oktopk_b200.ops import ext
    from oktopk_b200.ops.fused_bn import _pool_fusable
    _bitwise_against_fp32(FALLBACK, False)
    pool = torch.nn.MaxPool2d(2, 2)
    x, cbias, dy = _inputs(FALLBACK, 9, True)
    assert not _pool_fusable(x, pool)
    bn16, bn32 = _bn(FALLBACK[1], 9), _bn(FALLBACK[1], 9)
    n0 = ext.LAUNCH_COUNT.get("maxpool2_fwd", 0)
    y, dx, dg, db = _run_fused(x, bn16, cbias, pool, dy)
    assert ext.LAUNCH_COUNT.get("maxpool2_fwd", 0) == n0
    y32, *_ = _run_fused(x.float(), bn32, cbias, pool, dy.float())
    assert y.dtype == dx.dtype == torch.bfloat16
    assert torch.equal(y, y32.bfloat16())             # rounding is monotonic: the max of the rounded is the rounded max
    assert torch.equal(bn16.running_mean, bn32.running_mean) and torch.equal(bn16.running_var, bn32.running_var)


@pytest.mark.parametrize("shape,pooled", [((16, 64, 32, 32), True), ((16, 512, 2, 2), True), ((128, 64, 32, 32), True),
                                          ((2, 1032, 3, 3), False)])
def test_bf16_capped_grid(shape, pooled, monkeypatch):
    """A grid smaller than the tile count (tiles read again from global memory, tiles too large to hold, more than one
    column tile): bitwise the fp32 kernels, and bitwise the uncapped bf16 grid."""
    from oktopk_b200.ops import fused_bn
    ref = _bitwise_against_fp32(shape, pooled, seed=3)
    monkeypatch.setattr(fused_bn, "MAX_CTAS", 5)
    got = _bitwise_against_fp32(shape, pooled, seed=3)
    for a, b in zip(ref[:4], got[:4]):
        assert torch.equal(a, b)
    assert torch.equal(ref[4].running_mean, got[4].running_mean) and torch.equal(ref[4].running_var, got[4].running_var)


# ------------------------------------------------------------------------------------------ 2. against torch's bf16 path
def _bf16_ulp(t):
    """One bf16 ulp at |t| (fp32 result; 2^-133 for zero, the smallest subnormal step)."""
    a = t.float().abs()
    e = torch.frexp(a)[1]
    ulp = torch.ldexp(torch.ones_like(a), (e - 8).clamp(min=-133))
    return torch.where(a == 0, torch.full_like(a, 2.0 ** -133), ulp)


def _tied_windows(ypre):
    """Pooled positions whose 2x2 window has its (positive) bf16 maximum more than once.  There torch's arg-max (the
    first of the rounded values) and the fused kernel's (that of the fp32 values) may differ: the pooled gradient then
    reaches a different element."""
    N, C, H, W = ypre.shape
    w = ypre.float().reshape(N, C, H // 2, 2, W // 2, 2)
    m = w.amax(dim=(3, 5), keepdim=True)
    return (((w == m).sum(dim=(3, 5), keepdim=True) > 1) & (m > 0)).reshape(N, C, H // 2, W // 2)


@pytest.mark.parametrize("pooled", [False, True])
@pytest.mark.parametrize("shape", VGG_SHAPES + [FALLBACK])
def test_bf16_matches_torch_autocast(shape, pooled):
    """Against stock BatchNorm2d -> ReLU [-> MaxPool2d] under torch.autocast(bf16) on the same bf16 input: y within one
    bf16 ulp, statistics and dgamma / dbeta at the fp32 tolerances, dx within one ulp up to a few elements at a ReLU
    boundary.  The pooled gradient is zero at windows whose rounded maximum is tied (their arg-max is a matter of
    rounding: see _tied_windows)."""
    from oktopk_b200.ops.fused_bn import bias_bn_relu
    pool = torch.nn.MaxPool2d(2, 2) if pooled else None
    x, _, dy = _inputs(shape, 17, pooled)
    bn_f, bn_t = _bn(shape[1], 17), _bn(shape[1], 17)
    xf = x.detach().clone().requires_grad_(True)
    xt = x.detach().clone().requires_grad_(True)
    with torch.autocast("cuda", torch.bfloat16):
        y = bias_bn_relu(xf, bn_f, None, True, pool)
        ypre = torch.relu(bn_t(xt))
        yt = pool(ypre) if pooled else ypre
    if pooled:
        tied = _tied_windows(ypre)
        assert int(tied.sum()) <= tied.numel() // 10
        dy = dy.masked_fill(tied, 0).contiguous(memory_format=torch.channels_last)
    y.backward(dy)
    yt.backward(dy)
    dx, dg, db = xf.grad, bn_f.weight.grad, bn_f.bias.grad
    assert yt.dtype == y.dtype == torch.bfloat16 and y.shape == yt.shape
    diff = (y.float() - yt.float()).abs()
    assert bool((diff <= _bf16_ulp(torch.maximum(y.float().abs(), yt.float().abs())) + 2e-5).all()), float(diff.max())
    torch.testing.assert_close(bn_f.running_mean, bn_t.running_mean, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(bn_f.running_var, bn_t.running_var, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(dg, bn_t.weight.grad, rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(db, bn_t.bias.grad, rtol=2e-3, atol=2e-3)
    bad = int((~torch.isclose(dx.float(), xt.grad.float(), rtol=2.0 ** -7, atol=2e-4)).sum())
    assert bad <= max(4, dx.numel() // 20000), bad


# ------------------------------------------------------------------------------------------ 3. whole model
def _vgg_pair():
    from oktopk_b200.models import create_net
    torch.manual_seed(0)
    net, _ = create_net(10, "vgg16")
    net = net.cuda().to(memory_format=torch.channels_last)
    return net


def _grads(net, x, y, autocast):
    net.zero_grad(set_to_none=True)
    if autocast:
        with torch.autocast("cuda", torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(net(x), y)
    else:
        loss = torch.nn.functional.cross_entropy(net(x), y)
    loss.backward()
    return {n: p.grad for n, p in net.named_parameters()}


def test_vgg16_bf16_autocast_step():
    """One VGG-16 forward/backward under bf16 autocast through the fused kernels: 13 bn_forward and 13 bn_backward
    launches, no standalone pool, no stock batch-norm; each gradient no further from the fp32 one than stock bf16's."""
    from oktopk_b200.ops import ext
    torch.backends.cudnn.deterministic = True
    ref = _vgg_pair()
    fused, stock = copy.deepcopy(ref), copy.deepcopy(ref)
    stock.fuse = False
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
            assert n.startswith("features.") and n.endswith(".bias") and g32[n] is None, n
            continue
        assert a.dtype == torch.float32 and torch.isfinite(a).all(), n
        ref_norm = float(g32[n].norm())
        ef = float((a - g32[n]).norm()) / ref_norm
        es = float((gs[n] - g32[n]).norm()) / ref_norm
        assert ef <= 1.5 * es + 1e-3, (n, ef, es)
        checked += 1
    assert checked == 2 * 13 + 13 + 2         # conv weights, BN weight and bias, fc weight and bias


# ------------------------------------------------------------------------------------------ 4. the gate
def test_fp16_autocast_keeps_stock_path():
    """Under fp16 autocast the fused model launches no batch-norm kernel and computes exactly what the stock modules
    compute."""
    from oktopk_b200.ops import ext
    torch.backends.cudnn.deterministic = True
    a = _vgg_pair()
    b = copy.deepcopy(a)
    a.fuse, b.fuse = True, False
    x = torch.randn(16, 3, 32, 32, device="cuda").contiguous(memory_format=torch.channels_last)
    n0 = ext.LAUNCH_COUNT["total"]
    with torch.autocast("cuda", torch.float16):
        oa = a(x)
    assert ext.LAUNCH_COUNT["total"] == n0
    with torch.autocast("cuda", torch.float16):
        ob = b(x)
    assert oa.dtype == torch.float16 and torch.equal(oa, ob)
    for (n, ba), bb in zip(a.named_buffers(), b.buffers()):
        assert torch.equal(ba, bb), n


def test_fp32_without_autocast_takes_fp32_kernel():
    """fp32 activations with autocast off: the fused model's launches are today's (13 + 13, no standalone pool), and a
    layer's outputs are bitwise those of a direct fp32 launch of the kernels."""
    from oktopk_b200.ops import ext
    from oktopk_b200.ops.fused_bn import bias_bn_relu
    net = _vgg_pair()
    x = torch.randn(16, 3, 32, 32, device="cuda").contiguous(memory_format=torch.channels_last)
    n0 = {k: ext.LAUNCH_COUNT.get(k, 0) for k in ("bn_forward", "bn_backward", "maxpool2_fwd")}
    net(x).float().sum().backward()
    d = {k: ext.LAUNCH_COUNT.get(k, 0) - v for k, v in n0.items()}
    assert d == {"bn_forward": 13, "bn_backward": 13, "maxpool2_fwd": 0}, d

    C = ext.require()
    shape = (16, 128, 16, 16)
    N, Ch, H, W = shape
    x, cbias, dy = (t.float() for t in _inputs(shape, 23, True))
    bn_a, bn_b = _bn(Ch, 23), _bn(Ch, 23)
    y, dx, dg, db = _run_fused(x, bn_a, cbias, torch.nn.MaxPool2d(2, 2), dy)
    assert y.dtype == torch.float32
    M = N * H * W
    rows = C.bn_tile_rows(M, Ch)
    partial = torch.empty((M + rows - 1) // rows * 2 * Ch, device="cuda")
    stats, dgb = torch.empty(2 * Ch, device="cuda"), torch.empty(2 * Ch, device="cuda")
    y2 = torch.empty_like(y)
    arg = torch.empty(y2.numel(), dtype=torch.uint8, device="cuda")
    dx2 = torch.empty_like(x)
    s = torch.cuda.current_stream().cuda_stream
    C.bn_forward(x.data_ptr(), y2.data_ptr(), arg.data_ptr(), partial.data_ptr(), bn_b.weight.data_ptr(),
                 bn_b.bias.data_ptr(), cbias.data_ptr(), stats.data_ptr(), stats.data_ptr() + 4 * Ch,
                 bn_b.running_mean.data_ptr(), bn_b.running_var.data_ptr(), bn_b.num_batches_tracked.data_ptr(),
                 bn_b.momentum, bn_b.eps, 1, M, Ch, W, 999, 0, s, 0)
    C.bn_backward(x.data_ptr(), dy.data_ptr(), arg.data_ptr(), dx2.data_ptr(), partial.data_ptr(), bn_b.weight.data_ptr(),
                  bn_b.bias.data_ptr(), stats.data_ptr(), stats.data_ptr() + 4 * Ch, dgb.data_ptr(),
                  dgb.data_ptr() + 4 * Ch, 1, M, Ch, W, 999, 0, s, 0)
    assert torch.equal(y, y2) and torch.equal(dx, dx2)
    assert torch.equal(dg, dgb[:Ch]) and torch.equal(db, dgb[Ch:])
    assert torch.equal(bn_a.running_mean, bn_b.running_mean) and torch.equal(bn_a.running_var, bn_b.running_var)


# ------------------------------------------------------------------------------------------ 5. CUDA graphs
def test_trainer_bf16_cuda_graph_matches_eager():
    """Trainer(autocast="bf16", cuda_graph=True) on VGG-16 Ok-Topk: the graph-captured steps (autocast entered inside the
    capture) over the dense-to-sparse transition and 36 sparse steps give the parameters of the same steps run eagerly,
    bit for bit."""
    import oktopk_b200 as okt
    from oktopk_b200.ops import ext
    from oktopk_b200.train.trainer import Trainer
    torch.backends.cudnn.deterministic = True
    cfg = okt.preset("vgg16", density=0.001, warmup_iters=4)
    kw = dict(dnn="vgg16", dataset="cifar10", batch_size=16, lr=0.05, compressor="oktopk", density=0.001, cfg=cfg,
              autocast="bf16", seed=0)
    tg = Trainer(cuda_graph=True, **kw)
    te = Trainer(cuda_graph=False, **kw)
    assert tg.graphed is not None and te.graphed is None
    for a, b in zip(tg.net.parameters(), te.net.parameters()):
        assert torch.equal(a, b)
    g = torch.Generator("cuda").manual_seed(2)
    batches = [(torch.randn(16, 3, 32, 32, device="cuda", generator=g).contiguous(memory_format=torch.channels_last),
                torch.randint(0, 10, (16,), device="cuda", generator=g)) for _ in range(4)]
    n_bn = ext.LAUNCH_COUNT.get("bn_forward", 0)
    for it in range(4 + 36):
        batch = batches[it % len(batches)]
        tg.graphed.step(batch)
        te.optimizer.zero_grad()
        loss, _ = te._forward_loss(batch)
        loss.backward()
        te.update_model()
    torch.cuda.synchronize()
    assert tg.graphed.enabled, tg.graphed.why_disabled
    assert len(tg.graphed.graphs) >= 2
    assert ext.LAUNCH_COUNT.get("bn_forward", 0) > n_bn
    for (n, a), b in zip(tg.net.named_parameters(), te.net.parameters()):
        assert torch.isfinite(a).all(), n
        assert torch.equal(a, b), n
    for (n, a), b in zip(tg.net.named_buffers(), te.net.buffers()):
        assert torch.equal(a, b), n
    tg.close()
    te.close()
