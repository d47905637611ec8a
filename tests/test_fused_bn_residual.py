"""The residual form of the fused batch-norm kernels (csrc/bnrelu.cu, kRes): relu(bn(x) + r), the end of a ResNet block.
Against the stock modules in fp32, bit for bit the fp32 kernel on widened bf16 / fp16 input, a capped grid, the
fallbacks, a whole ResNet-20 fused against stock, and whole-step CUDA graphs of a fused ResNet-20."""
import copy

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# the BN inputs of ResNet-20 at 32 images (one per stage), a ResNet-50 stage-1 and stage-4 shape at 8 images
RESNET20_SHAPES = [(32, 16, 32, 32), (32, 32, 16, 16), (32, 64, 8, 8)]
SHAPES = RESNET20_SHAPES + [(8, 256, 56, 56), (8, 2048, 7, 7)]


def _bn(C, seed):
    torch.manual_seed(seed)
    bn = torch.nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        bn.weight.normal_(1.0, 0.3); bn.bias.normal_(0.0, 0.5)
        bn.running_mean.normal_(0.0, 0.1); bn.running_var.uniform_(0.5, 1.5)
    return bn


def _inputs(shape, seed, dtype=torch.float32):
    g = torch.Generator("cuda").manual_seed(seed)
    cl = torch.channels_last
    x = (torch.randn(shape, device="cuda", generator=g) * 1.7 + 0.3).to(dtype).contiguous(memory_format=cl)
    r = (torch.randn(shape, device="cuda", generator=g) * 0.8).to(dtype).contiguous(memory_format=cl)
    dy = torch.randn(shape, device="cuda", generator=g).to(dtype).contiguous(memory_format=cl)
    return x, r, dy


def _fused(x, r, bn, dy, fp16=False):
    from oktopk_b200.ops.fused_bn import bias_bn_relu
    xa = x.detach().clone().requires_grad_(True)
    ra = r.detach().clone().requires_grad_(True)
    y = bias_bn_relu(xa, bn, None, True, None, fp16=fp16, residual=ra)
    y.backward(dy)
    return y, xa.grad, ra.grad, bn.weight.grad, bn.bias.grad


def _counts():
    from oktopk_b200.ops import ext
    return {k: ext.LAUNCH_COUNT.get(k, 0) for k in ("bn_forward", "bn_backward")}


def _delta(n0):
    return {k: v - n0[k] for k, v in _counts().items()}


# ------------------------------------------------------------------------------------------ 1. fp32 against stock
@pytest.mark.parametrize("shape", SHAPES)
def test_residual_matches_stock_modules(shape):
    x, r, dy = _inputs(shape, sum(shape))
    bn_a, bn_b = _bn(shape[1], 3), _bn(shape[1], 3)
    n0 = _counts()
    y, dx, dr, dg, db = _fused(x, r, bn_a, dy)
    assert _delta(n0) == {"bn_forward": 1, "bn_backward": 1}
    assert y.is_contiguous(memory_format=torch.channels_last) and dr.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(dr, dy * (y > 0))                      # the residual's gradient is dy under the ReLU mask, exactly
    xb, rb = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
    yb = F.relu(bn_b(xb) + rb)
    yb.backward(dy)
    torch.testing.assert_close(y, yb, rtol=2e-4, atol=2e-5)
    # an element within rounding of zero may take the other side of the ReLU: allow a few
    for got, want in ((dx, xb.grad), (dr, rb.grad)):
        bad = int((~torch.isclose(got, want, rtol=2e-3, atol=2e-4)).sum())
        assert bad <= max(4, got.numel() // 20000), bad
    torch.testing.assert_close(dg, bn_b.weight.grad, rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(db, bn_b.bias.grad, rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(bn_a.running_mean, bn_b.running_mean, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(bn_a.running_var, bn_b.running_var, rtol=1e-4, atol=1e-5)
    assert int(bn_a.num_batches_tracked) == int(bn_b.num_batches_tracked) == 1


# ------------------------------------------------------------------------------------------ 2. bf16 / fp16
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", RESNET20_SHAPES + [(8, 256, 56, 56)])
def test_16bit_residual_is_fp32_kernel_on_widened_input(shape, dtype):
    fp16 = dtype == torch.float16
    x, r, dy = _inputs(shape, 11, dtype)
    bn16, bn32 = _bn(shape[1], 5), _bn(shape[1], 5)
    y, dx, dr, dg, db = _fused(x, r, bn16, dy, fp16=fp16)
    y32, dx32, dr32, dg32, db32 = _fused(x.float(), r.float(), bn32, dy.float())
    assert y.dtype == dx.dtype == dr.dtype == dtype and dg.dtype == torch.float32
    assert torch.equal(y, y32.to(dtype))
    assert torch.equal(dx, dx32.to(dtype))
    assert torch.equal(dr, dr32.to(dtype))
    assert torch.equal(dg, dg32) and torch.equal(db, db32)
    assert torch.equal(bn16.running_mean, bn32.running_mean) and torch.equal(bn16.running_var, bn32.running_var)


# ------------------------------------------------------------------------------------------ 3. capped grid
@pytest.mark.parametrize("shape", [(32, 16, 32, 32), (8, 256, 56, 56), (2, 1032, 3, 3)])
def test_residual_capped_grid_is_bitwise_the_same(shape, monkeypatch):
    """Five CTAs looping over the tiles give the bits of one tile per CTA.  (8, 256, 56, 56) has tiles too large to hold
    on chip (phase 3 reads the dres written in phase 1 back), (2, 1032, 3, 3) more channels than one column tile."""
    from oktopk_b200.ops import fused_bn
    x, r, dy = _inputs(shape, 7)
    bn_a, bn_b = _bn(shape[1], 9), _bn(shape[1], 9)
    ref = _fused(x, r, bn_a, dy)
    monkeypatch.setattr(fused_bn, "MAX_CTAS", 5)
    got = _fused(x, r, bn_b, dy)
    for a, b in zip(ref, got):
        assert torch.equal(a, b)
    assert torch.equal(bn_a.running_mean, bn_b.running_mean) and torch.equal(bn_a.running_var, bn_b.running_var)


# ------------------------------------------------------------------------------------------ 4. fallbacks
@pytest.mark.parametrize("case", ["nchw", "eval", "res_dtype", "res_shape", "cpu"])
def test_residual_fallbacks_run_the_stock_ops(case):
    from oktopk_b200.ops.fused_bn import bias_bn_relu
    shape = (4, 16, 8, 8)
    x, r, dy = _inputs(shape, 2)
    bn_a, bn_b = _bn(16, 4), _bn(16, 4)
    if case == "nchw":
        x, r, dy = x.contiguous(), r.contiguous(), dy.contiguous()
    elif case == "eval":
        bn_a.eval(); bn_b.eval()
    elif case == "res_dtype":
        r = r.double()
    elif case == "res_shape":
        r = r[:, :, :1, :1].contiguous()                       # broadcasts in the stock add
    elif case == "cpu":
        x, r, dy, bn_a, bn_b = x.cpu(), r.cpu(), dy.cpu(), bn_a.cpu(), bn_b.cpu()
    n0 = _counts()
    xa, ra = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
    y = bias_bn_relu(xa, bn_a, residual=ra)
    y.backward(dy.to(y.dtype))
    assert _delta(n0) == {"bn_forward": 0, "bn_backward": 0}
    xb, rb = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
    yb = F.relu(bn_b(xb) + rb)
    yb.backward(dy.to(yb.dtype))
    assert torch.equal(y, yb) and torch.equal(xa.grad, xb.grad) and torch.equal(ra.grad, rb.grad)


def test_residual_needs_relu_and_no_pool():
    from oktopk_b200.ops.fused_bn import bias_bn_relu, conv_bn_relu
    x, r, _ = _inputs((4, 16, 8, 8), 1)
    bn = _bn(16, 1)
    with pytest.raises(ValueError):
        bias_bn_relu(x, bn, relu=False, residual=r)
    with pytest.raises(ValueError):
        bias_bn_relu(x, bn, pool=torch.nn.MaxPool2d(2, 2), residual=r)
    conv = torch.nn.Conv2d(16, 16, 3, 1, 1, bias=False).cuda().to(memory_format=torch.channels_last)
    with pytest.raises(ValueError):
        conv_bn_relu(x, conv, bn, relu=False, residual=r)


# ------------------------------------------------------------------------------------------ 5. whole ResNets
def _fp32_convs():
    """Full-fp32 convolutions for fused-vs-stock comparisons (see test_gpu_kernels: with TF32 the two paths may call
    different cuDNN kernels whose differences back-propagation amplifies)."""
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.allow_tf32 = False


def test_resnet20_fused_trains_like_stock_through_oktopk():
    import oktopk_b200 as okt
    from oktopk_b200.models import create_net
    tf32 = torch.backends.cudnn.allow_tf32
    _fp32_convs()
    try:
        torch.manual_seed(0)
        a, _ = create_net(10, "resnet20", fuse_bn=True)
        b = copy.deepcopy(a)
        b.fuse = False
        assert a.fuse and not b.fuse
        a = a.cuda().to(memory_format=torch.channels_last)
        b = b.cuda().to(memory_format=torch.channels_last)
        cfg = okt.preset("vgg16", density=0.02, warmup_iters=2)
        opts = [okt.DistributedOptimizer(torch.optim.SGD(n.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4),
                                         named_parameters=n.named_parameters(), compression=okt.compressors["oktopk"],
                                         is_sparse=True, cfg=cfg) for n in (a, b)]
        g = torch.Generator("cuda").manual_seed(1)
        x = torch.randn(32, 3, 32, 32, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (32,), device="cuda", generator=g)
        losses = {0: [], 1: []}
        for it in range(5):
            for i, (net, opt) in enumerate(zip((a, b), opts)):
                n0 = _counts()
                opt.zero_grad()
                loss = F.cross_entropy(net(x), y)
                loss.backward()
                opt.step()
                losses[i].append(float(loss.detach()))
                assert _delta(n0) == ({"bn_forward": 19, "bn_backward": 19} if i == 0 else
                                      {"bn_forward": 0, "bn_backward": 0})
            if it == 0:                                     # one dense step: close everywhere
                sa, sb = a.state_dict(), b.state_dict()
                assert list(sa) == list(sb)
                for k in sa:
                    if sa[k].dtype.is_floating_point:
                        err = float((sa[k] - sb[k]).norm()) / (float(sb[k].norm()) + 1e-6)
                        assert err < 2e-2, "%s: relative L2 error %.3g after one step" % (k, err)
                    else:
                        assert torch.equal(sa[k], sb[k]), k
        assert losses[0][0] == pytest.approx(losses[1][0], rel=1e-4), losses
        assert losses[0] == pytest.approx(losses[1], rel=0.05, abs=0.05), losses
        pa = torch.cat([p.detach().flatten() for p in a.parameters()])
        pb = torch.cat([p.detach().flatten() for p in b.parameters()])
        assert torch.isfinite(pa).all()
        assert float((pa - pb).norm()) / float(pb.norm()) < 1e-2
        for o in opts:
            o.close()
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


# ------------------------------------------------------------------------------------------ 6. CUDA graphs
@pytest.mark.parametrize("autocast", [None, "bf16"])
def test_fused_resnet20_cuda_graph_matches_eager(autocast):
    """Trainer(model_kwargs={"fuse_bn": True}, cuda_graph=True) on ResNet-20 Ok-Topk: the graph-captured steps over the
    dense-to-sparse transition replay the eager steps bit for bit."""
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    torch.backends.cudnn.deterministic = True
    cfg = okt.preset("vgg16", density=0.02, warmup_iters=4)
    kw = dict(dnn="resnet20", dataset="cifar10", batch_size=32, lr=0.1, compressor="oktopk", density=0.02, cfg=cfg,
              autocast=autocast, seed=0, model_kwargs={"fuse_bn": True})
    tg = Trainer(cuda_graph=True, **kw)
    te = Trainer(cuda_graph=False, **kw)
    assert tg.graphed is not None and te.graphed is None and tg.net.fuse and te.net.fuse
    for a, b in zip(tg.net.parameters(), te.net.parameters()):
        assert torch.equal(a, b)
    g = torch.Generator("cuda").manual_seed(2)
    batches = [(torch.randn(32, 3, 32, 32, device="cuda", generator=g).contiguous(memory_format=torch.channels_last),
                torch.randint(0, 10, (32,), device="cuda", generator=g)) for _ in range(4)]
    n0 = _counts()
    for it in range(4 + 16):
        batch = batches[it % len(batches)]
        tg.graphed.step(batch)
        te.optimizer.zero_grad()
        loss, _ = te._forward_loss(batch)
        loss.backward()
        te.update_model()
    torch.cuda.synchronize()
    assert tg.graphed.enabled, tg.graphed.why_disabled
    assert len(tg.graphed.graphs) >= 2
    assert _delta(n0)["bn_forward"] > 0
    for (n, a), b in zip(tg.net.named_parameters(), te.net.parameters()):
        assert torch.isfinite(a).all(), n
        assert torch.equal(a, b), n
    for (n, a), b in zip(tg.net.named_buffers(), te.net.buffers()):
        assert torch.equal(a, b), n
    tg.close()
    te.close()
