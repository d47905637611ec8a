"""GPU tests of gradient clipping on the device (csrc/optim.cu grad_sumsq / clip_coef, the factor applied by the fused
updates): the norm against float64, the factor against torch's formula (non-finite gradients included), bitwise
repeatability, a factor of 1 as a no-op, the clipped updates against torch (clip_grad_norm_, then torch's update),
loss scaling, CUDA-graph capture, the launch count, and the AN4 and PTB trainers with ``fused_clip`` against the stock
clip.

Tolerances: the device norm is the fp32 rounding of an fp64 sum, torch's the fp32 norm of fp32 per-tensor norms.  The
two factors differ by a few fp32 ulps at most, so a clipped update differs from torch's by a few ulps of the gradient
term; over a handful of steps that stays within rtol 1e-5 / atol 1e-6 (the fused Adam tests' tolerance)."""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = dict(rtol=1e-5, atol=1e-6)


def _C():
    from oktopk_b200.ops import ext
    return ext.require()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _launches():
    from oktopk_b200.ops import ext
    return ext.LAUNCH_COUNT["total"]


def _device_norm(g, max_norm, segs=None, bounds=None):
    """(norm, coef) of ``g`` through grad_sumsq + clip_coef: one norm, or one per (offset, length) of ``segs`` with the
    per-segment bounds ``bounds``."""
    C = _C()
    chunk = C.SUMSQ_CHUNK
    offs, lens = zip(*segs) if segs else ([0], [g.numel()])
    blk = [0]
    for n in lens:
        blk.append(blk[-1] + max(1, -(-n // chunk)))
    partial = torch.full((blk[-1],), float("nan"), dtype=torch.float64, device="cuda")
    C.grad_sumsq(g.data_ptr(), list(offs), list(lens), partial.data_ptr(), _stream())
    if segs is None:
        norm, coef = torch.empty(1, device="cuda"), torch.empty(1, device="cuda")
        C.clip_coef(partial.data_ptr(), blk[-1], 0, 0, 0, 0, max_norm, norm.data_ptr(), coef.data_ptr(), _stream())
    else:
        ns = len(segs)
        norm, coef = torch.empty(ns, device="cuda"), torch.empty(ns, device="cuda")
        seg_blk = torch.tensor(blk, dtype=torch.int32, device="cuda")
        seg_scal = torch.arange(ns, dtype=torch.int32, device="cuda")
        scal = torch.tensor(bounds, dtype=torch.float32, device="cuda")
        C.clip_coef(partial.data_ptr(), blk[-1], seg_blk.data_ptr(), seg_scal.data_ptr(), ns, scal.data_ptr(), 0.0,
                    norm.data_ptr(), coef.data_ptr(), _stream())
    torch.cuda.synchronize()
    return norm, coef


def _wide(n, seed):
    """Gradients spread over many orders of magnitude (|g| from 1e-8 to 1e4)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, device="cuda", generator=gen) * torch.pow(
        10.0, torch.empty(n, device="cuda").uniform_(-8, 4, generator=gen))


# ------------------------------------------------------------------------------------------------ 1. the kernels
@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, 2 ** 20 + 3, 66_034_000])
def test_norm_against_float64_and_bitwise_repeatable(n):
    g = _wide(n, n % 1000)
    ref = math.sqrt(float((g.double() ** 2).sum()))
    norm, coef = _device_norm(g, 0.5)
    again = _device_norm(g, 0.5)
    assert torch.equal(norm, again[0]) and torch.equal(coef, again[1])
    got = float(norm)
    assert abs(got - ref) <= 2 ** -23 * ref, (n, got, ref)        # the fp32 rounding of the fp64 norm, within 1 ulp
    # the factor is torch's formula applied to that norm, bit for bit
    want = torch.clamp(0.5 / (norm + 1e-6), max=1.0)
    assert torch.equal(coef, want), (coef, want)


@pytest.mark.parametrize("case", ["below", "above", "zero", "inf", "nan"])
def test_factor_follows_clip_grad_norm(case):
    """The factor and norm clip_grad_norm_ gives: exactly 1 below the bound, 1 for an all-zero gradient, 0 for an
    infinite gradient (finite entries become 0, infinite ones NaN) and NaN for a NaN gradient."""
    n = 4099
    g = torch.randn(n, device="cuda")
    max_norm = {"below": 1e4, "zero": 1.0}.get(case, 1.0)
    if case == "zero":
        g.zero_()
    elif case == "inf":
        g[17] = float("inf")
    elif case == "nan":
        g[4000] = float("nan")
    p = torch.nn.Parameter(torch.zeros(n, device="cuda"))
    p.grad = g.clone()
    total = torch.nn.utils.clip_grad_norm_([p], max_norm)
    norm, coef = _device_norm(g, max_norm)
    scaled = g * coef                                            # the update kernels' multiply
    if case == "below" or case == "zero":
        assert float(coef) == 1.0
    if case == "inf":
        assert float(coef) == 0.0 and math.isinf(float(norm))
    if case == "nan":
        assert math.isnan(float(coef)) and math.isnan(float(norm))
    if case in ("inf", "nan"):
        assert torch.equal(torch.isnan(scaled), torch.isnan(p.grad))
        assert torch.equal(scaled.nan_to_num(7.0), p.grad.nan_to_num(7.0))
        assert torch.equal(norm[0].isnan(), total.isnan()) and torch.equal(norm[0].isinf(), total.isinf())
    else:
        torch.testing.assert_close(norm[0], total, rtol=2e-6, atol=0)   # torch sums in fp32
        torch.testing.assert_close(scaled, p.grad, rtol=2e-6, atol=0)


def test_per_segment_factors_follow_bertadam_rule():
    """max / (norm + 1e-6) where norm > max > 0, else 1; an infinite segment gets 0, a NaN one 1 (it is not clipped,
    as float(nan) > max is False)."""
    n = 5 * 1024
    g = torch.randn(n, device="cuda")
    segs = [(0, 1000), (1024, 1024), (2048, 3), (3072, 1024), (4096, 1024)]
    bounds = [1.0, 1e4, 1.0, 1.0, 1.0]
    g[3072] = float("inf")
    g[4096 + 5] = float("nan")
    norm, coef = _device_norm(g, 0.0, segs, bounds)
    for s, ((o, L), mx) in enumerate(zip(segs, bounds)):
        nrm = float(g[o:o + L].double().norm())
        if math.isfinite(nrm):
            assert abs(float(norm[s]) - nrm) <= 2 ** -23 * nrm
        want = mx / (float(norm[s]) + 1e-6) if float(norm[s]) > mx else 1.0      # BertAdam's host arithmetic
        assert float(coef[s]) == float(torch.tensor(want, dtype=torch.float32)), (s, float(coef[s]), want)
    assert float(coef[1]) == 1.0 and float(coef[3]) == 0.0 and float(coef[4]) == 1.0
    _, off = _device_norm(g, 0.0, segs, [1.0, 1e4, 1.0, 0.0, -1.0])
    assert float(off[3]) == 1.0 and float(off[4]) == 1.0         # a bound <= 0 turns the clip off


# ------------------------------------------------------------------------------------------------ helpers
def _vgg(seed=0):
    from oktopk_b200.models import create_net
    torch.manual_seed(seed)
    net, _ = create_net(10, "vgg16")
    return net.cuda().to(memory_format=torch.channels_last)


def _batches(k, bs=8, seed=7, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [((torch.randn(bs, 3, 32, 32, device="cuda", generator=g) * scale).contiguous(
        memory_format=torch.channels_last), torch.randint(0, 10, (bs,), device="cuda", generator=g)) for _ in range(k)]


def _cfg(sparse, warmup=2, **kw):
    import oktopk_b200 as okt
    return okt.preset("vgg16", density=0.01, warmup_iters=warmup, **kw) if sparse else None


def _sgd_opt(net, max_norm, sparse, cfg=None, **sgd):
    import oktopk_b200 as okt
    base = torch.optim.SGD(net.parameters(), **(sgd or dict(lr=0.05, momentum=0.9, weight_decay=1e-4)))
    return okt.DistributedOptimizer(base, named_parameters=net.named_parameters(),
                                    compression=okt.compressors["oktopk" if sparse else "none"], is_sparse=sparse,
                                    cfg=cfg if cfg is not None else _cfg(sparse), max_grad_norm=max_norm)


def _adam_opt(net, max_norm, sparse, decoupled):
    import oktopk_b200 as okt
    cls = torch.optim.AdamW if decoupled else torch.optim.Adam
    base = cls(net.parameters(), lr=1e-3, weight_decay=1e-2, fused=True)
    return okt.DistributedOptimizer(base, named_parameters=net.named_parameters(),
                                    compression=okt.compressors["oktopk" if sparse else "none"], is_sparse=sparse,
                                    cfg=_cfg(sparse), max_grad_norm=max_norm)


def _bert_opt(net, sparse, clip, max_norm=1.0):
    from oktopk_b200.optimizer import BertAdam
    decay = [p for p in net.parameters() if p.dim() > 1]
    rest = [p for p in net.parameters() if p.dim() <= 1]
    groups = [{"params": decay, "weight_decay": 0.01}, {"params": rest, "weight_decay": 0.0}]
    kw = dict(compressor="oktopk", density=0.01, cfg=_cfg(True)) if sparse else {}
    return BertAdam(groups, lr=1e-3, max_grad_norm=max_norm, named_parameters=net.named_parameters(),
                    clip_reduced=clip, **kw)


def _step(net, opt, batch, stock_clip=None):
    opt.zero_grad()
    torch.nn.functional.cross_entropy(net(batch[0]), batch[1]).backward()
    if stock_clip is not None:
        opt.synchronize()
        torch.nn.utils.clip_grad_norm_(net.parameters(), stock_clip)
    opt.step()


def _state(net, opt):
    out = [p.detach().clone() for p in net.parameters()]
    for p in net.parameters():
        out += [v.clone() for k, v in sorted(opt.state[p].items()) if torch.is_tensor(v) and v.dim() > 0]
    return out


# ------------------------------------------------------------------------------------------------ 2. factor 1
@pytest.mark.parametrize("kind", ["sgd", "adam", "bertadam"])
def test_factor_one_is_bitwise_no_clip(kind):
    """With the norm far below the bound, five steps (two dense, three Ok-Topk) equal an unclipped run bit for bit."""
    torch.backends.cudnn.deterministic = True
    base = _vgg()
    nets = [copy.deepcopy(base) for _ in range(2)]
    if kind == "sgd":
        opts = [_sgd_opt(nets[0], None, True), _sgd_opt(nets[1], 1e30, True)]
    elif kind == "adam":
        opts = [_adam_opt(nets[0], None, True, True), _adam_opt(nets[1], 1e30, True, True)]
    else:
        opts = [_bert_opt(nets[0], True, False), _bert_opt(nets[1], True, True, max_norm=1e30)]
    assert opts[0]._clip is None and opts[1]._clip is not None
    for batch in _batches(5):
        for net, opt in zip(nets, opts):
            _step(net, opt, batch)
    torch.cuda.synchronize()
    assert float(opts[1].grad_norm().max()) > 0
    for a, b in zip(_state(nets[0], opts[0]), _state(nets[1], opts[1])):
        assert torch.equal(a, b)
    for o in opts:
        o.close()


# ------------------------------------------------------------------------------------------------ 3. against torch
def _against_torch(net, opt, make_ref, keys, max_norm, batches):
    """Each step from the same state: the clipped fused step against torch (clip_grad_norm_ over the reduced gradient,
    then ``make_ref``'s torch optimizer) started from the parameters and state the step began with.  Comparing step by
    step keeps the arms on one trajectory: otherwise an ulp of difference can flip an Ok-Topk selection later on."""
    params = list(net.parameters())
    clipped = 0
    for batch in batches:
        p0 = [p.detach().clone() for p in params]
        s0 = [{k: opt.state[p][k].clone() for k in keys if k in opt.state.get(p, {})} for p in params]
        t0 = getattr(opt, "counter", 0)
        opt.zero_grad()
        torch.nn.functional.cross_entropy(net(batch[0]), batch[1]).backward()
        opt.synchronize()
        grads = [p.grad.detach().clone() for p in params]
        opt.step()
        refs = [torch.nn.Parameter(q.clone()) for q in p0]
        for r, g in zip(refs, grads):
            r.grad = g
        total = torch.nn.utils.clip_grad_norm_(refs, max_norm)
        clipped += int(float(total) > max_norm)
        ref = make_ref(refs)
        for r, st in zip(refs, s0):
            if st:
                ref.state[r] = dict({k: v.clone() for k, v in st.items()},
                                    **({"step": torch.tensor(float(t0), device="cuda")} if "exp_avg" in st else {}))
        ref.step()
        torch.cuda.synchronize()
        for p, r in zip(params, refs):
            torch.testing.assert_close(p.detach(), r.detach(), **TOL)
            for k in keys:
                torch.testing.assert_close(opt.state[p][k], ref.state[r][k], **TOL)
    assert clipped == len(batches)


@pytest.mark.parametrize("ahead", [False, True])
def test_sgd_clip_matches_torch(ahead):
    """Six VGG-16 steps (two dense, four Ok-Topk), the gradient norm above the bound, with the early SGD update on and
    off: the fused clip against clip_grad_norm_ then torch.optim.SGD."""
    from oktopk_b200.ops import ext
    torch.backends.cudnn.deterministic = True
    net = _vgg()
    hyper = dict(lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
    opt = _sgd_opt(net, 0.5, True, cfg=_cfg(True, sgd_ahead=ahead), **hyper)
    a0 = ext.LAUNCH_COUNT.get("sgd_ahead", 0)
    _against_torch(net, opt, lambda ps: torch.optim.SGD(ps, foreach=False, **hyper), ("momentum_buffer",), 0.5,
                   _batches(6))
    assert (ext.LAUNCH_COUNT.get("sgd_ahead", 0) > a0) is ahead
    opt.close()


@pytest.mark.parametrize("decoupled", [False, True])
def test_adam_clip_matches_torch(decoupled):
    torch.backends.cudnn.deterministic = True
    net = _vgg()
    opt = _adam_opt(net, 0.5, True, decoupled)
    assert opt._okt_adam and opt._clip is not None
    cls = torch.optim.AdamW if decoupled else torch.optim.Adam
    _against_torch(net, opt, lambda ps: cls(ps, lr=1e-3, weight_decay=1e-2, fused=True), ("exp_avg", "exp_avg_sq"),
                   0.5, _batches(6))
    opt.close()


@pytest.mark.parametrize("sparse", [False, True])
def test_bertadam_per_parameter_clip_matches_torch(sparse):
    """BertAdam(clip_reduced=True) on the device, each step from the same state, against the per-parameter clip in torch
    (float(norm) per parameter, scaled where norm > max_grad_norm) followed by BertAdam's update in torch ops; a bound
    that clips many parameters."""
    torch.backends.cudnn.deterministic = True
    net = _vgg()
    opt = _bert_opt(net, sparse, True, max_norm=0.05)
    assert opt._clip is not None
    params = list(net.parameters())
    group = {p: g for g in opt.param_groups for p in g["params"]}
    clipped = 0
    for batch in _batches(5):
        p0 = [p.detach().clone() for p in params]
        s0 = [(opt.state[p]["next_m"].clone(), opt.state[p]["next_v"].clone()) if "next_m" in opt.state.get(p, {})
              else (torch.zeros_like(p), torch.zeros_like(p)) for p in params]
        opt.zero_grad()
        torch.nn.functional.cross_entropy(net(batch[0]), batch[1]).backward()
        opt.synchronize()
        grads = [p.grad.detach().clone() for p in params]
        lr = opt._scheduled_lr(opt.param_groups[0], opt.counter)
        opt.step()
        torch.cuda.synchronize()
        for p, q, (m, v), g in zip(params, p0, s0, grads):
            h = group[p]
            nrm = float(g.norm())
            if nrm > h["max_grad_norm"]:
                g = g * (h["max_grad_norm"] / (nrm + 1e-6))
                clipped += 1
            m = m * h["b1"] + g * (1 - h["b1"])
            v = v * h["b2"] + g * g * (1 - h["b2"])
            u = m / (v.sqrt() + h["e"])
            if h["weight_decay"] > 0:
                u = u + h["weight_decay"] * q
            torch.testing.assert_close(p.detach(), q - lr * u, **TOL)
            torch.testing.assert_close(opt.state[p]["next_m"], m, **TOL)
            torch.testing.assert_close(opt.state[p]["next_v"], v, **TOL)
    assert clipped >= 5 * 10
    norms = opt.grad_norm()
    assert norms.numel() == len(params)
    opt.close()


# ------------------------------------------------------------------------------------------------ 4. loss scaling
def test_skipped_step_leaves_everything_and_clears_the_gradient():
    import oktopk_b200 as okt
    torch.backends.cudnn.deterministic = True
    net = _vgg()
    opt = okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9),
                                   named_parameters=net.named_parameters(), compression=okt.compressors["oktopk"],
                                   is_sparse=True, cfg=_cfg(True), loss_scale=okt.LossScale(init_scale=2.0 ** 10),
                                   max_grad_norm=0.5)
    batches = _batches(4)
    for batch in batches[:3]:
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            loss = torch.nn.functional.cross_entropy(net(batch[0]), batch[1])
        opt.scale_loss(loss).backward()
        opt.step()
    torch.cuda.synchronize()
    before = _state(net, opt)
    skipped0 = opt.loss_scale_state()["skipped_steps"]
    opt.zero_grad()
    with torch.autocast("cuda", dtype=torch.float16):
        loss = torch.nn.functional.cross_entropy(net(batches[3][0]), batches[3][1]) * float("inf")
    opt.scale_loss(loss).backward()
    opt.step()
    torch.cuda.synchronize()
    assert opt.loss_scale_state()["skipped_steps"] == skipped0 + 1
    for a, b in zip(before, _state(net, opt)):
        assert torch.equal(a, b)
    assert all(float(b.grad.abs().max()) == 0.0 for b in opt._buckets)
    opt.close()


# ------------------------------------------------------------------------------------------------ 5. graphs
def _mlp(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(256, 512), torch.nn.GELU(), torch.nn.Linear(512, 512), torch.nn.GELU(),
                               torch.nn.Linear(512, 10)).cuda()


def _mlp_batches(k):
    g = torch.Generator(device="cuda").manual_seed(5)
    return [(torch.randn(64, 256, device="cuda", generator=g) * 3, torch.randint(0, 10, (64,), device="cuda",
                                                                                   generator=g)) for _ in range(k)]


def _graphed_against_eager(make_opt, lrs):
    nets = [_mlp(), _mlp()]
    opts = [make_opt(n) for n in nets]
    batches = _mlp_batches(3 + len(lrs))

    def step(net, opt, x, y):
        opt.zero_grad()
        torch.nn.functional.cross_entropy(net(x), y).backward()
        opt.step()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for x, y in batches[:3]:
            for n, o in zip(nets, opts):
                step(n, o, x, y)
    torch.cuda.current_stream().wait_stream(s)
    sx, sy = batches[0][0].clone(), batches[0][1].clone()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        step(nets[1], opts[1], sx, sy)
    for i, (lr, (x, y)) in enumerate(zip(lrs, batches[3:])):
        for o in opts:
            for grp in o.param_groups:
                grp["lr"] = lr
        step(nets[0], opts[0], x, y)
        opts[1].refresh_lr()
        sx.copy_(x)
        sy.copy_(y)
        g.replay()
    torch.cuda.synchronize()
    for a, b in zip(_state(nets[0], opts[0]), _state(nets[1], opts[1])):
        assert torch.equal(a, b)
    for o in opts:
        o.close()


def test_graphed_sgd_step_with_clip_replays_like_eager():
    import oktopk_b200 as okt

    def make(net):
        return okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4),
                                        named_parameters=net.named_parameters(), compression=okt.compressors["none"],
                                        max_grad_norm=0.5)
    _graphed_against_eager(make, [0.1 * (0.8 ** i) for i in range(10)])


def test_graphed_bertadam_clip_reduced_step_captures_and_matches_eager():
    from oktopk_b200.optimizer import BertAdam

    def make(net):
        return BertAdam(net.parameters(), lr=1e-3, max_grad_norm=0.05, named_parameters=net.named_parameters(),
                        clip_reduced=True)
    _graphed_against_eager(make, [1e-3 * (0.8 ** i) for i in range(10)])


# ------------------------------------------------------------------------------------------------ 6. launch count
@pytest.mark.parametrize("buckets", [1, 2])
def test_two_launches_more_per_step(buckets):
    """grad_sumsq once per bucket and clip_coef once: two launches more than an unclipped one-bucket step."""
    import oktopk_b200 as okt
    counts = []
    for clip in (None, 0.5):
        net = _mlp()
        cfg = okt.preset("vgg16", density=0.01, bucket_elems=(1 << 30) if buckets == 1 else 200_000)
        opt = okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9),
                                       named_parameters=net.named_parameters(), compression=okt.compressors["none"],
                                       cfg=cfg, max_grad_norm=clip)
        assert len(opt._buckets) == buckets
        x, y = _mlp_batches(1)[0]
        for _ in range(2):
            opt.zero_grad()
            torch.nn.functional.cross_entropy(net(x), y).backward()
            opt.synchronize()
            n0 = _launches()
            opt.step()
            n1 = _launches()
        counts.append(n1 - n0)
        opt.close()
    assert counts[1] - counts[0] == buckets + 1


# ------------------------------------------------------------------------------------------------ 7. trainers
def _an4_trainer(fused_clip, autocast=None):
    """Dense reduction: under Ok-Topk at density 0.001 an ulp of difference flips selections within a few steps."""
    import bench
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    kw = {"fuse_lstm": True, "fuse_ctc": True, "fuse_bn": True}
    if autocast:
        kw["fuse_lstm_autocast"] = True
    return Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, density=0.001,
                   cfg=okt.preset(preset, density=0.001, warmup_iters=5), t_total=100000, warmup=0.1, seed=0,
                   cuda_graph=True, an4_pad_multiple=32, autocast=autocast, model_kwargs=kw, compressor="none",
                   compression=False, fused_clip=fused_clip)


def _an4_batches(n, bs=2):
    from oktopk_b200.train.data import SyntheticAN4, an4_collate
    ds = SyntheticAN4(n=n * bs, seed=3)
    return [tuple(t.cuda() for t in an4_collate([ds[i * bs + j] for j in range(bs)])) for i in range(n)]


def test_an4_graphed_padded_fused_clip_follows_stock_clip():
    """Ten graphed steps at m = 32 with fuse_lstm, fuse_ctc and fuse_bn.  The two clips' factors differ by the rounding
    of the norm (torch sums in fp32), and this training carries that difference forward fast once the clip is active;
    so the losses must agree within 1e-4 or within four times the drift of a stock run whose bound moves by 1e-6 (the
    size of that rounding), whichever is larger."""
    pool = _an4_batches(4)
    losses = {}
    for arm in ("stock", "fused", "control"):
        tr = _an4_trainer(arm == "fused")
        if arm == "control":
            tr.clip_norm *= 1 + 1e-6
        assert tr.graphed is not None and tr.graphed.enabled, tr.graphed.why_disabled
        assert (tr.optimizer._clip is not None) is (arm == "fused")
        seq = []
        for it in range(10):
            seq.append(tr.step(pool[it % len(pool)]).clone())
        assert len(tr.graphed.graphs) > 0
        losses[arm] = [float(x) for x in seq]
        tr.close()
    print("AN4 graphed m=32 losses:", losses)
    for a, b, c in zip(losses["stock"], losses["fused"], losses["control"]):
        assert abs(a - b) <= max(1e-4 * abs(a), 4 * abs(a - c)), losses


def test_ptb_bf16_fused_clip_follows_stock_clip():
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    losses = {}
    for fused in (False, True):
        cfg = okt.preset("lstm_an4", density=0.02, warmup_iters=2)
        tr = Trainer(dnn="lstm", dataset="ptb", batch_size=20, lr=22, compressor="oktopk", density=0.02, cfg=cfg,
                     seed=0, autocast="bf16", model_kwargs={"fuse_lstm": True, "fuse_xent": True}, fused_clip=fused)
        tr.net.dropout.p = 0.0
        tr.net.lstm.dropout = 0.0
        assert (tr.optimizer._clip is not None) is fused
        seq = []
        for _ in range(10):
            tr.train_step()
            seq.append(float(tr.last_loss()))
        if fused:
            assert float(tr.optimizer.grad_norm()) > 0.25           # the clip was active
        losses[fused] = seq
        tr.close()
    print("PTB bf16 losses, stock clip %s\n fused clip %s" % (losses[False], losses[True]))
    for a, b in zip(losses[False], losses[True]):
        assert abs(a - b) <= 1e-4 * abs(a), losses
