"""GPU tests: every sm_90a kernel against a plain PyTorch fp32 reference / the oracle.
Single-GPU tests run the full peer-memory protocol with P=1 (all mailboxes local)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


def _C():
    from oktopk_b200.ops import ext
    return ext.require()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def test_extension_loaded():
    C = _C()
    assert C.state_bytes() > 0 and C.max_coop_grid(0) >= torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("n,k", [(1000, 10), (100003, 1000), (1 << 22, 4194), (1 << 22, 400000)])
def test_kth_abs_matches_topk(n, k):
    C = _C()
    torch.manual_seed(n + k)
    x = torch.randn(n, device="cuda") * torch.rand(n, device="cuda")
    st = C.dev_alloc_zero(C.state_bytes())
    out = torch.zeros(1, device="cuda")
    C.kth_abs(x.data_ptr(), n, k, st, out.data_ptr(), C.max_coop_grid(0), _stream())
    ref = torch.topk(x.abs(), k).values[-1]
    assert float(out) == float(ref)


def test_fused_sgd_matches_torch():
    C = _C()
    torch.manual_seed(0)
    n = 100003
    p = torch.randn(n, device="cuda"); g = torch.randn(n, device="cuda")
    pr = p.clone().requires_grad_(True)
    opt = torch.optim.SGD([pr], lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=True)
    mom = torch.zeros(n, device="cuda")
    lr = torch.tensor([0.1], device="cuda")
    for it in range(3):
        pr.grad = g.clone()
        opt.step()
        gg = g.clone()
        C.fused_sgd(p.data_ptr(), gg.data_ptr(), mom.data_ptr(), n, 0.9, 0.0, 1e-4, 1, int(it == 0), 1, _stream(),
                    lr.data_ptr())
        assert float(gg.abs().max()) == 0.0          # gradient bucket zeroed in the same pass
    torch.testing.assert_close(p, pr.detach(), rtol=1e-5, atol=1e-6)


def test_fused_bert_adam_matches_reference_math():
    C = _C()
    torch.manual_seed(0)
    n = 65537
    p = torch.randn(n, device="cuda"); m = torch.zeros(n, device="cuda"); v = torch.zeros(n, device="cuda")
    pr, mr, vr = p.clone(), m.clone(), v.clone()
    lr = torch.tensor([2e-4], device="cuda")
    for it in range(3):
        g = torch.randn(n, device="cuda")
        mr.mul_(0.9).add_(g, alpha=0.1)
        vr.mul_(0.999).addcmul_(g, g, value=0.001)
        upd = mr / (vr.sqrt() + 1e-6) + 0.01 * pr
        pr.add_(upd, alpha=-2e-4)
        C.fused_bert_adam(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, 0.9, 0.999, 1e-6, 0.01, 1, _stream(),
                          lr.data_ptr())
    torch.testing.assert_close(p, pr, rtol=1e-5, atol=1e-6)


def _run_engine_vs_oracle(name, n, iters, cfg, tol_count=0, rtol=0.0):
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.oracle import run_oracle
    from oktopk_b200.parallel.state import SparseState
    from oktopk_b200.parallel.world import World
    w = World()
    eng = CudaBucketEngine(n, cfg, w, name="t")
    states = [SparseState(n, 1)]
    for it in range(iters):
        g = torch.Generator().manual_seed(77 * it + 5)
        x = torch.randn(n, generator=g) * (1.0 + 0.2 * it)
        eng.grad.copy_(x.cuda())
        eng.reduce(name)
        torch.cuda.synchronize()
        ref = run_oracle(name, [x.clone()], states, cfg)[0]
        got = eng.grad.cpu()
        st = eng.stats()
        ne = (lambda a, b: a != b) if rtol == 0.0 else (lambda a, b: ~torch.isclose(a, b, rtol=rtol, atol=5e-7))
        bad = int(ne(got, ref).sum())
        assert bad <= tol_count, "%s it %d: %d mismatching elements (stats %s)" % (name, it, bad, st)
        rbad = int(ne(eng.residual.cpu(), states[0].residual).sum())
        assert rbad <= tol_count, "%s it %d: residual mismatch %d" % (name, it, rbad)
        if tol_count == 0:
            assert st["local_count"] == states[0].last_local_count, (it, st, states[0].last_local_count)
            if name in ("oktopk", "topkAopt"):       # schemes whose threshold is carried across iterations
                assert abs(st["local_thr"] - states[0].local_thr) <= 1e-12 + 1e-7 * abs(states[0].local_thr)
        assert st["overflow_send"] == 0 and st["overflow_gather"] == 0
    eng.close()


@pytest.mark.parametrize("n", [4096, 100003, 3_000_000])
@pytest.mark.parametrize("fused,pull", [(True, "tma"), (True, "ldg"), (False, "tma")])
def test_oktopk_single_gpu_matches_oracle(n, fused, pull):
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=0.01, local_recompute_interval=4, global_recompute_interval=4, repartition_interval=8,
                       fused=fused, pull_mode=pull, slot_factor=64, gather_factor=64)
    _run_engine_vs_oracle("oktopk", n, 10, cfg)


@pytest.mark.parametrize("mode", ["list", "scan"])
@pytest.mark.parametrize("density", [0.002, 0.05])
def test_oktopk_global_selection_paths(mode, density):
    """Candidate-list and region-scan global selection are interchangeable (same result as the oracle)."""
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=density, local_recompute_interval=4, global_recompute_interval=3, repartition_interval=8,
                       gselect_mode=mode, slot_factor=64, gather_factor=64)
    _run_engine_vs_oracle("oktopk", 1_000_003, 8, cfg)
    if density == 0.05:
        _run_engine_vs_oracle("topkSA", 300_001, 4, cfg)


def test_oktopk_lstm_and_bert_presets():
    import oktopk_b200 as okt
    for preset in ("lstm_an4", "bert_base"):
        cfg = okt.preset(preset, density=0.005, warmup_iters=0, local_recompute_interval=3, global_recompute_interval=5,
                         slot_factor=64, gather_factor=64)
        _run_engine_vs_oracle("oktopk", 500_000, 8, cfg)


@pytest.mark.parametrize("name", ["topkSA", "gaussiankSA", "topkAopt", "topkA"])
def test_other_schemes_single_gpu_match_oracle(name):
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=0.01, topkaopt_recompute_interval=3, slot_factor=64, gather_factor=64)
    _run_engine_vs_oracle(name, 200_000, 5, cfg)


def test_gaussiank_single_gpu_close_to_oracle():
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=0.01, slot_factor=64, gather_factor=64)
    # the device computes the moments in one pass (double accumulation) => threshold may differ in the
    # last bits from torch.std; allow a handful of borderline elements
    _run_engine_vs_oracle("gaussiank", 400_000, 4, cfg, tol_count=40)


def test_distributed_optimizer_cuda_single_gpu_trains():
    import oktopk_b200 as okt
    from oktopk_b200.models import create_net
    torch.manual_seed(0)
    net, _ = create_net(10, "resnet20")
    net = net.cuda()
    opt = okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4),
                                   named_parameters=net.named_parameters(), compression=okt.compressors["oktopk"],
                                   is_sparse=True, density=0.05)
    x = torch.randn(32, 3, 32, 32, device="cuda"); y = torch.randint(0, 10, (32,), device="cuda")
    losses = []
    for it in range(30):
        opt.zero_grad()
        loss = torch.nn.functional.cross_entropy(net(x), y)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0] * 0.7, losses
    sd = opt.state_dict()
    assert "oktopk" in sd and len(sd["oktopk"]["buckets"]) >= 1
    opt.load_state_dict(sd)
    opt.close()


def test_dense_path_matches_torch_sgd_on_gpu():
    import copy
    import oktopk_b200 as okt
    from oktopk_b200.models import create_net
    torch.manual_seed(0)
    net, _ = create_net(10, "resnet20")
    net = net.cuda()
    ref = copy.deepcopy(net)
    o_ref = torch.optim.SGD(ref.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4)
    o = okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4),
                                 named_parameters=net.named_parameters(), compression=okt.compressors["none"])
    torch.backends.cudnn.deterministic = True
    for it in range(3):
        x = torch.randn(8, 3, 32, 32, device="cuda"); y = torch.randint(0, 10, (8,), device="cuda")
        for m, oo in ((ref, o_ref), (net, o)):
            oo.zero_grad()
            torch.nn.functional.cross_entropy(m(x), y).backward()
            oo.step()
    for a, b in zip(net.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
    o.close()


# ======================================================================================================
# round 2: lossless exchange, overflow policy, conservation, new native schemes
# ======================================================================================================
def _scale(it):
    """Gradient-scale jumps (x10, x100): the carried thresholds become far too small, the stale-threshold
    iterations select a large part of the bucket."""
    return 1.0 if it < 3 else (10.0 if it < 6 else 100.0)


def _conservation_run(name, n, iters, cfg, exact_tol=0):
    """P=1: after every call  acc (= grad + residual before) == residual after + result, element-wise and exactly:
    whatever is not delivered stays in the residual."""
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.world import World
    eng = CudaBucketEngine(n, cfg, World(), name="t")
    res_prev = torch.zeros(n)
    hist = []
    for it in range(iters):
        g = torch.Generator().manual_seed(991 * it + 3)
        x = torch.randn(n, generator=g) * _scale(it)
        acc = (x.cuda() + res_prev.cuda()).cpu()
        eng.grad.copy_(x.cuda())
        eng.reduce(name)
        torch.cuda.synchronize()
        out, res, st = eng.grad.cpu(), eng.residual.cpu(), eng.stats()
        bad = int((acc != res + out).sum())
        assert bad <= exact_tol, "%s it %d: %d elements not conserved (stats %s)" % (name, it, bad, st)
        assert st["fault"] == 0
        hist.append(st)
        res_prev = res
    eng.close()
    return hist


def test_lossless_slots_never_drop_under_scale_jumps():
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=0.01, local_recompute_interval=8, global_recompute_interval=8, repartition_interval=8)
    hist = _conservation_run("oktopk", 400_003, 12, cfg)
    assert all(h["lossless"] for h in hist)
    assert all(h["overflow_send"] == 0 and h["overflow_gather"] == 0 and h["redo"] == 0 for h in hist), hist
    assert max(h["local_count"] for h in hist) > 10 * 4000          # the stale threshold really over-selected


def test_bounded_slots_redo_policy_is_lossless_and_conserved():
    """slot_factor=1: the send slot holds ~k entries; after a x10 gradient-scale jump the stale threshold selects most
    of the bucket.  The in-kernel policy raises the threshold and redoes the pack: nothing is dropped, nothing is lost."""
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=0.01, local_recompute_interval=8, global_recompute_interval=8, repartition_interval=8,
                       slot_factor=1.0, gather_factor=64.0)
    hist = _conservation_run("oktopk", 400_003, 12, cfg)
    assert not hist[0]["lossless"]
    assert all(h["overflow_send"] == 0 for h in hist), [h["overflow_send"] for h in hist]
    assert sum(h["redo"] for h in hist) > 0, "the overflow policy never ran"
    assert all(h["local_count"] <= h["cap"] for h in hist)


def test_bounded_gather_slot_overflow_is_conserved():
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=0.01, local_recompute_interval=8, global_recompute_interval=8, repartition_interval=8,
                       slot_factor=0.0, gather_factor=1.0)
    hist = _conservation_run("oktopk", 400_003, 10, cfg)
    assert sum(h["overflow_gather"] for h in hist) > 0            # entries were dropped from the gather slot ...
    # ... and _conservation_run has checked that every one of them is still in the residual


@pytest.mark.parametrize("name,tol", [("gaussiankSA", 0), ("topkDSA", 1)])
def test_classic_residual_schemes_keep_unsent_entries(name, tol):
    """TopkDSA / gaussiankSA zero the residual at the selection: with a too-small send slot the entries that found no
    room must stay in the residual (round-1 bug: they were zeroed before the capacity check).  TopkDSA's reference
    quirk (the k-th element itself is cleared but not sent) accounts for one element."""
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=0.05, slot_factor=0.05, compressor=name)
    hist = _conservation_run(name, 400_003, 4, cfg, exact_tol=tol)
    assert all(h["overflow_send"] > 0 for h in hist), [h["overflow_send"] for h in hist]


@pytest.mark.parametrize("slot_factor", [0.0, 64.0])
def test_oktopk_matches_oracle_in_both_slot_layouts(slot_factor):
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=0.01, local_recompute_interval=4, global_recompute_interval=4, repartition_interval=8,
                       slot_factor=slot_factor, gather_factor=slot_factor)
    _run_engine_vs_oracle("oktopk", 1_000_003, 10, cfg)


@pytest.mark.parametrize("name", ["topkA2", "gtopk"])
def test_native_reselect_and_tree_schemes_single_gpu(name):
    from oktopk_b200.config import OkTopkConfig
    _run_engine_vs_oracle(name, 300_001, 4, OkTopkConfig(density=0.01))


@pytest.mark.parametrize("name", ["topkA", "topkA2", "gtopk"])
def test_norm_clip_on_the_cuda_path(name):
    """VGG/allreducer.py:1372-1379: the incoming gradient is scaled to L2 norm sqrt(1/P)*norm_clip inside the kernel."""
    from oktopk_b200.config import OkTopkConfig
    # (the device computes the norm with double accumulation, torch with an fp32 reduction: the scale factor differs by
    #  ~1e-6 relative, hence the tolerances -- absolute for elements where gradient and residual nearly cancel)
    _run_engine_vs_oracle(name, 200_000, 3, OkTopkConfig(density=0.01, norm_clip=5.0), tol_count=40, rtol=1e-5)


def test_land_grads_kernel_copies_every_tensor():
    C = _C()
    torch.manual_seed(1)
    sizes = [1, 3, 64, 1000, 8192, 8193, 100_003, 2_359_296] + [17] * 120        # > LAND_MAX tensors: several launches
    srcs = [torch.randn(s, device="cuda") for s in sizes]
    offs, o = [], 0
    for s in sizes:
        offs.append(o)
        o += (s + 63) // 64 * 64
    bucket = torch.full((o,), -7.0, device="cuda")
    C.land_grads([t.data_ptr() for t in srcs], offs, sizes, bucket.data_ptr(), _stream())
    torch.cuda.synchronize()
    for t, off, s in zip(srcs, offs, sizes):
        assert torch.equal(bucket[off:off + s], t)
    touched = torch.zeros(o, dtype=torch.bool, device="cuda")
    for off, s in zip(offs, sizes):
        touched[off:off + s] = True
    assert bool((bucket[~touched] == -7.0).all())                   # gaps untouched


def test_gradient_landing_matches_accumulating_into_views():
    """The landing path (fresh autograd gradients + one multi-tensor copy per bucket) must train exactly like the
    round-1 path (autograd accumulating into bucket views), including a channels_last model."""
    import copy
    import oktopk_b200 as okt
    from oktopk_b200.models import create_net
    torch.manual_seed(0)
    torch.backends.cudnn.deterministic = True
    base, _ = create_net(10, "vgg16")
    base = base.cuda().to(memory_format=torch.channels_last)
    nets = [copy.deepcopy(base), copy.deepcopy(base)]
    opts = []
    for net, land in zip(nets, (True, False)):
        cfg = okt.preset("vgg16", density=0.01, warmup_iters=1, land_grads=land)
        opts.append(okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4),
                                             named_parameters=net.named_parameters(), compression=okt.compressors["oktopk"],
                                             is_sparse=True, cfg=cfg))
    assert opts[0]._land and not opts[1]._land
    for it in range(4):
        x = torch.randn(8, 3, 32, 32, device="cuda").contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (8,), device="cuda")
        for net, opt in zip(nets, opts):
            opt.zero_grad()
            torch.nn.functional.cross_entropy(net(x), y).backward()
            opt.step()
    torch.cuda.synchronize()
    for a, b in zip(nets[0].parameters(), nets[1].parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    for o in opts:
        o.close()


def test_trace_ring_records_every_call():
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.world import World
    eng = CudaBucketEngine(200_000, OkTopkConfig(density=0.01), World(), name="t")
    for it in range(5):
        eng.grad.normal_()
        eng.reduce("oktopk")
    torch.cuda.synchronize()
    tr = eng.trace()
    assert [r["epoch"] for r in tr] == [1, 2, 3, 4, 5]
    assert all(r["us_pack"] > 0 and r["local_count"] > 0 for r in tr), tr
    eng.close()


def test_fused_update_is_skipped_when_the_bucket_faulted():
    C = _C()
    n = 10_000
    p = torch.ones(n, device="cuda"); g = torch.ones(n, device="cuda"); mom = torch.zeros(n, device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    lr = torch.tensor([0.1], device="cuda")
    C.fused_sgd(p.data_ptr(), g.data_ptr(), mom.data_ptr(), n, 0.0, 0.0, 0.0, 0, 1, 0, _stream(), lr.data_ptr(), flag.data_ptr())
    torch.cuda.synchronize()
    assert float(p[0]) == pytest.approx(0.9)
    flag.fill_(1)
    C.fused_sgd(p.data_ptr(), g.data_ptr(), mom.data_ptr(), n, 0.0, 0.0, 0.0, 0, 0, 0, _stream(), lr.data_ptr(), flag.data_ptr())
    torch.cuda.synchronize()
    assert float(p[0]) == pytest.approx(0.9)          # partial gradient not applied


def test_overselect_cap_bounds_the_volume_and_matches_oracle():
    """overselect_cap=2: even after x10 / x100 gradient-scale jumps a stale threshold never ships more than 2k entries
    (the ladder keeps climbing), nothing is lost (conservation), and the choice of rung is the oracle's."""
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=0.01, local_recompute_interval=8, global_recompute_interval=8, repartition_interval=8,
                       overselect_cap=2.0)
    hist = _conservation_run("oktopk", 400_003, 12, cfg)
    assert all(h["local_count"] <= 2 * 4000 for h in hist), [h["local_count"] for h in hist]
    assert all(h["overflow_send"] == 0 and h["redo"] == 0 for h in hist)
    cfg2 = OkTopkConfig(density=0.01, local_recompute_interval=6, global_recompute_interval=6, repartition_interval=4,
                        overselect_cap=1.5, overselect_guard_loops=0)
    _run_engine_vs_oracle("oktopk", 300_001, 9, cfg2)


@pytest.mark.parametrize("shape", [(16, 64, 32, 32), (16, 128, 16, 16), (16, 512, 2, 2), (4, 96, 5, 7), (2, 1024, 3, 3)])
@pytest.mark.parametrize("relu", [True, False])
def test_fused_bias_bn_relu_matches_torch(shape, relu):
    """csrc/bnrelu.cu against conv-bias add -> nn.BatchNorm2d -> ReLU in plain fp32 torch: output, input gradient,
    gamma/beta gradients, running statistics; the reference's own bias gradient is rounding noise."""
    from oktopk_b200.ops.fused_bn import bias_bn_relu
    torch.manual_seed(sum(shape))
    N, C, H, W = shape
    x = (torch.randn(N, C, H, W, device="cuda") * 1.7 + 0.3).contiguous(memory_format=torch.channels_last)
    cb = torch.randn(C, device="cuda")
    dy = torch.randn(N, C, H, W, device="cuda").contiguous(memory_format=torch.channels_last)
    bn_a, bn_b = torch.nn.BatchNorm2d(C).cuda(), torch.nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        bn_a.weight.normal_(1.0, 0.3); bn_a.bias.normal_(0.0, 0.5)
        bn_b.load_state_dict(bn_a.state_dict())
    xa = x.clone().requires_grad_(True); xb = x.clone().requires_grad_(True)
    cba = cb.clone().requires_grad_(True); cbb = cb.clone().requires_grad_(True)
    for it in range(2):                                     # two steps: running statistics accumulate
        ya = bias_bn_relu(xa, bn_a, cba, relu)
        zb = bn_b(xb + cbb.view(1, -1, 1, 1))
        yb = torch.relu(zb) if relu else zb
        for t in (xa, xb, cba, cbb, bn_a.weight, bn_a.bias, bn_b.weight, bn_b.bias):
            t.grad = None
        ya.backward(dy); yb.backward(dy)
    assert ya.is_contiguous(memory_format=torch.channels_last)
    torch.testing.assert_close(ya, yb, rtol=2e-4, atol=2e-5)
    # an element whose pre-activation is within rounding of zero may take the other side of the ReLU: allow a few
    bad = int((~torch.isclose(xa.grad, xb.grad, rtol=2e-3, atol=2e-4)).sum())
    assert bad <= max(4, xa.numel() // 20000), bad
    torch.testing.assert_close(bn_a.weight.grad, bn_b.weight.grad, rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(bn_a.bias.grad, bn_b.bias.grad, rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(bn_a.running_mean, bn_b.running_mean, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(bn_a.running_var, bn_b.running_var, rtol=1e-4, atol=1e-5)
    assert int(bn_a.num_batches_tracked) == int(bn_b.num_batches_tracked) == 2
    assert cba.grad is None                                  # the loss does not depend on a bias in front of a batch-norm ...
    assert float(cbb.grad.abs().max()) <= 1e-3 * float(dy.abs().sum(dim=(0, 2, 3)).max())     # ... autograd returns noise


def test_vgg16_fused_path_trains_like_the_stock_modules():
    import copy
    from oktopk_b200.models import create_net
    torch.manual_seed(0)
    torch.backends.cudnn.deterministic = True
    # full-fp32 convolutions for this comparison: with TF32 the two paths call different cuDNN kernels (bias epilogue or
    # not) whose 10-bit-mantissa products differ at the 1e-3 level, which 13 layers of back-propagation amplify to
    # several per cent in the first layer's gradients -- that is cuDNN-vs-cuDNN noise, not what is being tested here
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        _vgg_fused_vs_stock(create_net, copy)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


def _vgg_fused_vs_stock(create_net, copy):
    base, _ = create_net(10, "vgg16")
    base = base.cuda().to(memory_format=torch.channels_last)
    a, b = copy.deepcopy(base), copy.deepcopy(base)
    a.fuse, b.fuse = True, False
    oa = torch.optim.SGD(a.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    ob = torch.optim.SGD(b.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    x = torch.randn(16, 3, 32, 32, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (16,), device="cuda")
    la, lb = [], []
    for it in range(3):
        for net, opt, ls in ((a, oa, la), (b, ob, lb)):
            opt.zero_grad(set_to_none=True)
            loss = torch.nn.functional.cross_entropy(net(x), y)
            loss.backward()
            opt.step()
            ls.append(float(loss.detach()))
        if it == 0:                                          # after ONE step the two paths must agree closely everywhere
            sa, sb = a.state_dict(), b.state_dict()
            assert list(sa.keys()) == list(sb.keys())
            for k in sa:
                if sa[k].dtype.is_floating_point:      # per-tensor relative L2 error (13 stacked batch-norms in fp32)
                    err = float((sa[k] - sb[k]).norm()) / (float(sb[k].norm()) + 1e-6)
                    assert err < 2e-2, "%s: relative L2 error %.3g after one step" % (k, err)
                else:
                    assert torch.equal(sa[k], sb[k]), k
    assert la[0] == pytest.approx(lb[0], rel=1e-3), (la, lb)      # same forward pass
    assert la[1] == pytest.approx(lb[1], rel=0.1, abs=0.1), (la, lb)   # and still close after one update
    # (beyond that two fp32 trajectories of a 14.7 M-parameter net at lr 0.05 / momentum 0.9 drift apart chaotically)
    assert all(torch.isfinite(torch.tensor(la + lb)))


@pytest.mark.parametrize("shape", [(16, 64, 32, 32), (16, 512, 2, 2), (3, 20, 6, 10)])
def test_maxpool_2x2_channels_last_matches_torch(shape):
    from oktopk_b200.ops.fused_bn import max_pool_2x2
    torch.manual_seed(1)
    pool = torch.nn.MaxPool2d(2, 2)
    x = torch.relu(torch.randn(*shape, device="cuda")).contiguous(memory_format=torch.channels_last)   # many ties at 0
    xa = x.clone().requires_grad_(True); xb = x.clone().requires_grad_(True)
    ya, yb = max_pool_2x2(xa, pool), pool(xb)
    dy = torch.randn_like(yb)
    ya.backward(dy); yb.backward(dy)
    assert torch.equal(ya, yb)
    assert torch.equal(xa.grad, xb.grad)                     # same arg-max rule for ties (first maximum in window order)


def test_threaded_prefetcher_delivers_the_loader_order_on_the_device():
    from oktopk_b200.train import data as D
    ds = D.build_dataset("mnist", None, train=True)
    loader, sampler = D.build_loader(ds, "mnist", 8, 0, 1, train=False)
    pf = D.Prefetcher(loader, torch.device("cuda", 0), threaded=True)
    assert pf.threaded
    ref = [b for _, b in zip(range(12), iter(loader))]
    for want in ref:
        got = pf.next(defer=True)
        pf.advance()
        torch.cuda.current_stream().synchronize()
        assert got[0].is_cuda and torch.equal(got[0].cpu(), want[0]) and torch.equal(got[1].cpu(), want[1])
    assert pf.h2d_bytes == sum(t.numel() * t.element_size() for b in ref for t in b)
    pf.close()
    pf2 = D.Prefetcher(loader, torch.device("cuda", 0), threaded=False)
    b = pf2.next()
    assert torch.equal(b[0].cpu(), ref[0][0])
