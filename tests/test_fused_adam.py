"""GPU tests: ``DistributedOptimizer`` wrapping ``torch.optim.Adam`` / ``AdamW`` with ``fused=True`` runs the flat-bucket
``fused_adam`` kernel.  Against torch's own Adam (within fp32 rounding), bitwise across the gradient paths and CUDA graphs,
through checkpoints in both directions, and only when torch's options ask for a fused kernel the project implements."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = dict(rtol=1e-5, atol=1e-6)


def _C():
    from oktopk_b200.ops import ext
    return ext.require()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _scalars(lr, b1, b2, wd, t):
    """What the optimizer pushes to the device before step t: computed in double as torch's non-capturable Adam does."""
    return torch.tensor([1 - lr * wd, (lr / (1 - b1 ** t)) * -1, (1 - b2 ** t) ** 0.5], dtype=torch.float32,
                        device="cuda")


def _maxdiff(a, b):
    return float((a.detach() - b.detach()).abs().max())


# ---------------------------------------------------------------------------------------------------- 1. the kernel
@pytest.mark.parametrize("impl", ["foreach", "fused"])
@pytest.mark.parametrize("wd", [0.0, 1e-2])
@pytest.mark.parametrize("decoupled", [False, True])
def test_fused_adam_kernel_matches_torch(decoupled, wd, impl):
    """Adam (L2) and AdamW, 20 steps of fresh (partly all-zero) gradients over 100 003 elements (a 3-element tail);
    zero_grad=1 leaves the gradient all-zero."""
    C = _C()
    n, lr, b1, b2, eps = 100003, 1e-3, 0.9, 0.999, 1e-8
    gen = torch.Generator(device="cuda").manual_seed(1)
    p = torch.randn(n, device="cuda", generator=gen)
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pr = p.clone().requires_grad_(True)
    cls = torch.optim.AdamW if decoupled else torch.optim.Adam
    ref = cls([pr], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, **{impl: True})
    keep = []
    for t in range(1, 21):
        g = torch.randn(n, device="cuda", generator=gen)
        if t % 2 == 0:
            g.view(-1)[: n // 4 * 4].view(-1, 8)[:, :4] = 0          # every other float4 line all-zero
        pr.grad = g.clone()
        ref.step()
        scal = _scalars(lr, b1, b2, wd, t)
        keep.append(scal)
        C.fused_adam(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, b1, b2, eps, wd, int(decoupled), 1,
                     _stream(), scal.data_ptr())
        assert float(g.abs().max()) == 0.0, t
    st = ref.state[pr]
    print("fused_adam kernel vs torch %s %s wd=%g: max |dp| %.3e" % ("AdamW" if decoupled else "Adam", impl, wd,
                                                                    _maxdiff(p, pr)))
    torch.testing.assert_close(p, pr.detach(), **TOL)
    torch.testing.assert_close(m, st["exp_avg"], **TOL)
    torch.testing.assert_close(v, st["exp_avg_sq"], **TOL)


def test_fused_adam_kernel_skips_on_fault_and_keeps_gradient_without_zero_grad():
    C = _C()
    n = 4099
    p, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    m, v = torch.rand(n, device="cuda"), torch.rand(n, device="cuda")
    p0, g0, m0, v0 = p.clone(), g.clone(), m.clone(), v.clone()
    scal = _scalars(1e-3, 0.9, 0.999, 1e-2, 3)
    fault = torch.ones(1, dtype=torch.int32, device="cuda")
    C.fused_adam(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, 0.9, 0.999, 1e-8, 1e-2, 1, 1, _stream(),
                 scal.data_ptr(), fault.data_ptr())
    torch.cuda.synchronize()
    for a, b in ((p, p0), (g, g0), (m, m0), (v, v0)):
        assert torch.equal(a, b)
    fault.zero_()
    C.fused_adam(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, 0.9, 0.999, 1e-8, 1e-2, 1, 0, _stream(),
                 scal.data_ptr(), fault.data_ptr())
    torch.cuda.synchronize()
    assert torch.equal(g, g0) and not torch.equal(p, p0)


# ---------------------------------------------------------------------------------------------------- helpers
def _vgg(seed=0):
    from oktopk_b200.models import create_net
    torch.manual_seed(seed)
    net, _ = create_net(10, "vgg16")
    return net.cuda().to(memory_format=torch.channels_last)


def _groups(net, wd=1e-2):
    decay = [p for p in net.parameters() if p.dim() > 1]
    no_decay = [p for p in net.parameters() if p.dim() <= 1]
    return [{"params": decay, "weight_decay": wd}, {"params": no_decay, "weight_decay": 0.0}]


def _batches(k, bs=8, seed=7):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [(torch.randn(bs, 3, 32, 32, device="cuda", generator=g).contiguous(memory_format=torch.channels_last),
             torch.randint(0, 10, (bs,), device="cuda", generator=g)) for _ in range(k)]


def _dense_wrapper(net, **kw):
    import oktopk_b200 as okt
    return okt.DistributedOptimizer(torch.optim.AdamW(_groups(net), lr=1e-3, fused=True, **kw),
                                    named_parameters=net.named_parameters(), compression=okt.compressors["none"],
                                    is_sparse=False)


def _wrapped_grads_step(net, opt, batch):
    """Backward + reduction on the wrapped net; returns copies of the reduced gradients the wrapper is about to apply."""
    opt.zero_grad()
    torch.nn.functional.cross_entropy(net(batch[0]), batch[1]).backward()
    opt.synchronize()
    return [p.grad.clone() for p in net.parameters()]


def _feed(net, grads):
    for p, g in zip(net.parameters(), grads):
        p.grad = g.clone()


def _count(name):
    from oktopk_b200.ops import ext
    return ext.LAUNCH_COUNT.get(name, 0)


# ---------------------------------------------------------------------------------------------------- 2. wrapper vs torch
def test_wrapped_adamw_matches_torch_fused_adamw_on_vgg16():
    """Two param groups (decay / no decay), 30 steps, the learning rate changed at step 15."""
    a = _vgg()
    b = copy.deepcopy(a)
    opt = _dense_wrapper(a)
    ref = torch.optim.AdamW(_groups(b), lr=1e-3, fused=True)
    assert opt._okt_adam
    n0 = _count("fused_adam")
    for it, batch in enumerate(_batches(30)):
        if it == 15:
            for g in opt.param_groups + ref.param_groups:
                g["lr"] = 3e-4
        _feed(b, _wrapped_grads_step(a, opt, batch))
        opt.step()
        ref.step()
    torch.cuda.synchronize()
    assert _count("fused_adam") - n0 == 30 * sum(len(bk.group_slices) for bk in opt._buckets)
    assert opt.counter == 30
    worst = max(_maxdiff(p, q) for p, q in zip(a.parameters(), b.parameters()))
    print("wrapped AdamW vs torch AdamW(fused=True), VGG-16, 30 steps: max |dp| %.3e" % worst)
    for (name, p), q in zip(a.named_parameters(), b.parameters()):
        torch.testing.assert_close(p, q, **TOL, msg=name)
        torch.testing.assert_close(opt.state[p]["exp_avg"], ref.state[q]["exp_avg"], **TOL, msg=name)
        torch.testing.assert_close(opt.state[p]["exp_avg_sq"], ref.state[q]["exp_avg_sq"], **TOL, msg=name)
    opt.close()


# ---------------------------------------------------------------------------------------------------- 3. gradient paths
def _okt_opts(kinds, warmup_iters):
    import oktopk_b200 as okt
    base = _vgg()
    nets, opts = [], []
    for kind in kinds:
        net = copy.deepcopy(base)
        cfg = okt.preset("vgg16", density=0.01, warmup_iters=warmup_iters, land_grads=kind != "views")
        opt = okt.DistributedOptimizer(torch.optim.AdamW(_groups(net), lr=1e-3, fused=True),
                                       named_parameters=net.named_parameters(), compression=okt.compressors["oktopk"],
                                       is_sparse=True, cfg=cfg)
        if kind == "land":
            opt._direct = False
        nets.append(net)
        opts.append(opt)
    return nets, opts


def test_adamw_reading_sources_is_bitwise_like_landing_and_like_views():
    """36 VGG-16 steps (2 dense, then sparse with two exact-threshold iterations): in-place gradient reads, the landing
    copy and accumulation into bucket views give identical parameters, moments and residuals."""
    torch.backends.cudnn.deterministic = True
    nets, opts = _okt_opts(("direct", "land", "views"), warmup_iters=2)
    assert all(o._okt_adam for o in opts)
    assert opts[0]._direct and not opts[1]._direct and opts[1]._land and not opts[2]._land
    for it, (x, y) in enumerate(_batches(36)):
        for k, (net, opt) in enumerate(zip(nets, opts)):
            land0 = _count("land_grads")
            opt.zero_grad()
            torch.nn.functional.cross_entropy(net(x), y).backward()
            opt.step()
            if k == 0:
                landed = _count("land_grads") - land0
                assert landed == (1 if it < 2 else 0), (it, landed)
                torch.cuda.synchronize()
                assert all(float(b.grad.abs().max()) == 0.0 for b in opt._buckets), it
    torch.cuda.synchronize()
    for other in (1, 2):
        for (name, a), b in zip(nets[0].named_parameters(), nets[other].parameters()):
            assert torch.equal(a, b), (other, name)
        for ba, bb in zip(opts[0]._buckets, opts[other]._buckets):
            for key in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(opts[0]._flat_state[ba.index][key], opts[other]._flat_state[bb.index][key]), key
            ra = opts[0]._allreducer._engines[ba.name].residual
            rb = opts[other]._allreducer._engines[bb.name].residual
            assert torch.equal(ra, rb), other
    for o in opts:
        o.close()


# ---------------------------------------------------------------------------------------------------- 4. CUDA graphs
class _Shim:
    """The part of Trainer that GraphedTrainStep drives."""

    def __init__(self, net, opt):
        self.net, self.optimizer = net, opt

    def _forward_loss(self, batch):
        x, y = batch
        return torch.nn.functional.cross_entropy(self.net(x), y), None

    def update_model(self):
        self.optimizer.step()


def test_graphed_adamw_steps_match_eager_steps_bitwise():
    """Whole-step CUDA graphs across the dense-to-sparse transition, the learning rate changed between replays: the
    graphs stay on and every replay uses the current learning rate and bias correction, bit for bit like eager steps."""
    from oktopk_b200.train.graph_step import GraphedTrainStep
    torch.backends.cudnn.deterministic = True
    nets, opts = _okt_opts(("direct", "direct"), warmup_iters=4)
    gs = GraphedTrainStep(_Shim(nets[0], opts[0]), warmup_eager=2)
    n_steps = 12
    for it, batch in enumerate(_batches(n_steps)):
        if it == 7:
            for o in opts:
                for g in o.param_groups:
                    g["lr"] *= 0.25
        gs.step(batch)
        opts[1].zero_grad()
        torch.nn.functional.cross_entropy(nets[1](batch[0]), batch[1]).backward()
        opts[1].step()
        torch.cuda.synchronize()
        assert all(float(b.grad.abs().max()) == 0.0 for b in opts[0]._buckets), it
    torch.cuda.synchronize()
    assert gs.enabled, gs.why_disabled
    assert len(gs.graphs) >= 2
    assert opts[0].counter == opts[1].counter == n_steps
    # the scalars of the last (replayed) step: t = 12 and the lowered learning rate
    for gi, g in enumerate(opts[0].param_groups):
        want = _scalars(g["lr"], *g["betas"], g["weight_decay"], n_steps)
        assert torch.equal(opts[0]._lr_dev[3 * gi:3 * gi + 3], want), gi
    for (name, a), b in zip(nets[0].named_parameters(), nets[1].parameters()):
        assert torch.equal(a, b), name
    for o in opts:
        o.close()


def test_graphed_bert_adam_checkpoints_the_steps_taken():
    """BertAdam under whole-step CUDA graphs: the checkpointed per-parameter step is the number of steps taken (a replay
    runs no Python), and the parameters match eager steps bit for bit."""
    import oktopk_b200 as okt
    from oktopk_b200.train.graph_step import GraphedTrainStep
    torch.backends.cudnn.deterministic = True
    base = _vgg()
    nets, opts = [], []
    for _ in range(2):
        net = copy.deepcopy(base)
        cfg = okt.preset("vgg16", density=0.01, warmup_iters=4)
        nets.append(net)
        opts.append(okt.BertAdam(_groups(net), lr=1e-3, warmup=0.1, t_total=100, compressor="oktopk", density=0.01,
                                 named_parameters=list(net.named_parameters()), cfg=cfg))
    gs = GraphedTrainStep(_Shim(nets[0], opts[0]), warmup_eager=2)
    n_steps = 8
    for batch in _batches(n_steps):
        gs.step(batch)
        opts[1].zero_grad()
        torch.nn.functional.cross_entropy(nets[1](batch[0]), batch[1]).backward()
        opts[1].step()
    torch.cuda.synchronize()
    assert gs.enabled, gs.why_disabled
    assert len(gs.graphs) >= 2
    for o in opts:
        sd = o.state_dict()
        assert o.counter == sd["counter"] == n_steps
        assert sd["state"] and all(st["step"] == n_steps for st in sd["state"].values())
    for (name, a), b in zip(nets[0].named_parameters(), nets[1].parameters()):
        assert torch.equal(a, b), name
    for o in opts:
        o.close()


# ---------------------------------------------------------------------------------------------------- 5. checkpoints
def test_wrapper_state_dict_loads_into_torch_adamw():
    a = _vgg()
    opt = _dense_wrapper(a)
    batches = _batches(10)
    for batch in batches[:5]:
        _wrapped_grads_step(a, opt, batch)
        opt.step()
    sd = copy.deepcopy(opt.state_dict())         # a checkpoint: torch's load keeps (aliases) same-device tensors
    st0 = next(iter(sd["state"].values()))
    assert st0["step"].dtype == torch.float32 and st0["step"].dim() == 0 and st0["step"].is_cuda
    assert float(st0["step"]) == 5.0
    b = _vgg(seed=1)
    b.load_state_dict(a.state_dict())
    ref = torch.optim.AdamW(_groups(b), lr=1e-3, fused=True)
    ref.load_state_dict(sd)
    for batch in batches[5:]:
        _feed(b, _wrapped_grads_step(a, opt, batch))
        opt.step()
        ref.step()
    torch.cuda.synchronize()
    for (name, p), q in zip(a.named_parameters(), b.parameters()):
        torch.testing.assert_close(p, q, **TOL, msg=name)
        assert float(ref.state[q]["step"]) == 10.0
    opt.close()


def test_torch_adamw_state_dict_loads_into_wrapper():
    b = _vgg()
    ref = torch.optim.AdamW(_groups(b), lr=1e-3, fused=True)
    batches = _batches(10)
    for x, y in batches[:5]:
        ref.zero_grad()
        torch.nn.functional.cross_entropy(b(x), y).backward()
        ref.step()
    a = copy.deepcopy(b)
    opt = _dense_wrapper(a)
    opt.load_state_dict(copy.deepcopy(ref.state_dict()))
    assert opt._okt_adam and opt.counter == 5
    flat = {k: [opt._flat_state[bk.index][k] for bk in opt._buckets] for k in ("exp_avg", "exp_avg_sq")}

    def aliased():
        for p in a.parameters():
            for k, bufs in flat.items():
                t = opt.state[p][k]
                assert any(t.untyped_storage().data_ptr() == f.untyped_storage().data_ptr() for f in bufs), k
                assert "step" not in opt.state[p]

    aliased()
    for (name, p), q in zip(a.named_parameters(), b.parameters()):
        if q in ref.state:
            torch.testing.assert_close(opt.state[p]["exp_avg"], ref.state[q]["exp_avg"], rtol=0, atol=0, msg=name)
    for batch in batches[5:]:
        _feed(b, _wrapped_grads_step(a, opt, batch))
        opt.step()
        ref.step()
    torch.cuda.synchronize()
    aliased()
    for (name, p), q in zip(a.named_parameters(), b.parameters()):
        torch.testing.assert_close(p, q, **TOL, msg=name)
    opt.close()


def test_unequal_step_counts_fall_back_to_torch_step():
    b = _vgg()
    ref = torch.optim.AdamW(_groups(b), lr=1e-3, fused=True)
    batches = _batches(6)
    for x, y in batches[:3]:
        ref.zero_grad()
        torch.nn.functional.cross_entropy(b(x), y).backward()
        ref.step()
    sd = ref.state_dict()
    first = next(iter(sd["state"]))
    sd["state"][first]["step"] = sd["state"][first]["step"] + 1
    ref.load_state_dict(sd)
    a = copy.deepcopy(b)
    opt = _dense_wrapper(a)
    with pytest.warns(UserWarning, match="unequal step counts"):
        opt.load_state_dict(copy.deepcopy(sd))
    assert not opt._okt_adam
    n0 = _count("fused_adam")
    for batch in batches[3:]:
        _feed(b, _wrapped_grads_step(a, opt, batch))
        opt.step()
        ref.step()
    torch.cuda.synchronize()
    assert _count("fused_adam") == n0
    for (name, p), q in zip(a.named_parameters(), b.parameters()):
        torch.testing.assert_close(p, q, **TOL, msg=name)
    opt.close()


# ---------------------------------------------------------------------------------------------------- 6. gating
def _mlp():
    torch.manual_seed(3)
    return torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 10)).cuda()


@pytest.mark.parametrize("case", ["fused_none", "amsgrad", "maximize", "tensor_lr"])
def test_gate_leaves_other_adam_options_on_torch_step(case):
    import oktopk_b200 as okt
    kw = {"fused_none": dict(fused=None), "amsgrad": dict(fused=True, amsgrad=True),
          "maximize": dict(fused=True, maximize=True), "tensor_lr": dict(fused=True)}[case]

    def lr():
        return torch.tensor(1e-3, device="cuda") if case == "tensor_lr" else 1e-3

    a = _mlp()
    b = copy.deepcopy(a)
    opt = okt.DistributedOptimizer(torch.optim.AdamW(a.parameters(), lr=lr(), **kw),
                                   named_parameters=a.named_parameters(), compression=okt.compressors["none"],
                                   is_sparse=False)
    ref = torch.optim.AdamW(b.parameters(), lr=lr(), **kw)
    assert not opt._okt_adam and not hasattr(opt, "counter")
    n0 = _count("fused_adam")
    gen = torch.Generator(device="cuda").manual_seed(5)
    for _ in range(4):
        x = torch.randn(16, 32, device="cuda", generator=gen)
        y = torch.randint(0, 10, (16,), device="cuda", generator=gen)
        opt.zero_grad()
        torch.nn.functional.cross_entropy(a(x), y).backward()
        opt.synchronize()
        _feed(b, [p.grad for p in a.parameters()])
        opt.step()
        ref.step()
    torch.cuda.synchronize()
    assert _count("fused_adam") == n0
    for p, q in zip(a.parameters(), b.parameters()):
        if case == "fused_none":                  # today's path: torch's own (foreach) step on the reduced gradients
            assert torch.equal(p, q)
        else:
            torch.testing.assert_close(p, q, **TOL)
    opt.close()
