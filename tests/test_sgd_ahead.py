"""Early SGD update (csrc/optim.cu sgd_ahead_kernel / fused_sgd_tail_kernel): the zero-gradient update applied during
backward over the early-pack segments' ranges, then the tail after the call, must leave parameters, momentum and the
gradient bucket bit for bit where one fused_sgd pass leaves them."""
import random

import pytest
import torch


# ---------------------------------------------------------------------------------------------------------- ranges (CPU)
@pytest.mark.parametrize("seed", range(30))
def test_ahead_and_rest_cover_every_vector_once_per_group(seed):
    """The segments' ranges (the ahead pass) plus ``rest()`` (the tail's dense part), each clipped to a param group's
    slice, cover each whole float4 vector of the slice exactly once; the slice's scalar tail is left to the tail kernel."""
    from oktopk_b200.optimizer import _clip_ranges
    from oktopk_b200.parallel.early_pack import PackPlanner
    rng = random.Random(seed)
    sizes = [rng.choice([1, 3, 5, 10, 64, 301, 4097, 20000]) for _ in range(rng.randrange(1, 30))]
    offs, o = [], 0
    for s in sizes:
        offs.append(o)
        o += (s + 3) // 4 * 4
    n = o - rng.randrange(4) if o > offs[-1] + 4 else o
    cuts = sorted(rng.sample(range(1, len(offs)), min(rng.randrange(3), len(offs) - 1)))
    bounds = [0] + [offs[c] for c in cuts] + [n]
    slices = list(zip(bounds, bounds[1:]))                         # param-group slices start at parameter offsets
    pl = PackPlanner(offs, n, min_elems=rng.choice([1, 50, 4096, 30000]), max_ranges=rng.choice([2, 4, 32]))
    order = list(range(len(sizes)))
    rng.shuffle(order)
    for i in order[:len(order) - rng.randrange(len(order) + 1) // 3]:
        pl.ready(i)
    ahead = [r for seg in pl.segments for r in seg]
    rest = pl.rest()
    for s, e in slices:
        a, d = _clip_ranges(ahead, s, e), _clip_ranges(rest, s, e)
        assert len(a) <= pl.max_ranges and len(d) <= pl.max_ranges
        cover = [0] * (e - s)
        for lo, hi in a + d:
            assert lo % 4 == 0 and hi % 4 == 0 and 0 <= lo < hi <= 4 * ((e - s) // 4)
            for x in range(lo, hi):
                cover[x] += 1
        for x in range(4 * ((e - s) // 4), e - s):
            cover[x] += 1
        assert all(c == 1 for c in cover)


# ---------------------------------------------------------------------------------------------------------- kernels (GPU)
def _sparse_grad(n, gen):
    """A call-written bucket: mostly +0, some normal values, signed zeros and subnormals."""
    g = torch.zeros(n, device="cuda")
    idx = torch.randperm(n, generator=gen, device="cuda")[: max(n // 50, 8)]
    vals = torch.randn(idx.numel(), generator=gen, device="cuda")
    kinds = torch.randint(0, 4, (idx.numel(),), generator=gen, device="cuda")
    vals = torch.where(kinds == 1, torch.full_like(vals, -0.0), vals)
    vals = torch.where(kinds == 2, vals.sign() * 1e-40, vals)          # subnormal
    g[idx] = vals
    return g


def _ranges(n, gen_py):
    """Ahead ranges and their complement over the whole vectors of an n-element slice, at multiples of 4."""
    top = 4 * (n // 4)
    cuts = sorted({0, top, *(4 * gen_py.randrange(top // 4 + 1) for _ in range(6))})
    spans = list(zip(cuts, cuts[1:]))
    ahead = [r for k, r in enumerate(spans) if k % 2 == 0 and r[0] < r[1]]
    dense = [r for k, r in enumerate(spans) if k % 2 == 1 and r[0] < r[1]]
    return ahead, dense


def _bits(t):
    return t.view(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("momentum,dampening,nesterov", [(0.0, 0.0, 0), (0.9, 0.0, 0), (0.9, 0.1, 0), (0.9, 0.0, 1)])
@pytest.mark.parametrize("wd", [0.0, 5e-4])
@pytest.mark.parametrize("n", [4096 * 3 + 4, 100_003])
def test_ahead_then_tail_matches_fused_sgd(momentum, dampening, nesterov, wd, n):
    from oktopk_b200.ops import ext
    C = ext.require()
    gen = torch.Generator(device="cuda").manual_seed(n + int(momentum * 10) + nesterov)
    rng = random.Random(n)
    s = torch.cuda.current_stream().cuda_stream
    lr = torch.tensor([0.05], device="cuda")
    p0 = torch.randn(n, generator=gen, device="cuda")
    p0[:7] = torch.tensor([0.0, -0.0, 1e-40, -1e-40, 0.0, -0.0, 3.0])    # signed zeros and subnormals in p too
    m0 = torch.randn(n, generator=gen, device="cuda")
    m0[:4] = torch.tensor([0.0, -0.0, -0.0, 0.0])
    g0 = _sparse_grad(n, gen)
    ahead, dense = _ranges(n, rng)
    for zero_grad in (1, 0):
        pa, ma, ga = p0.clone(), m0.clone(), g0.clone()
        C.fused_sgd(pa.data_ptr(), ga.data_ptr(), ma.data_ptr(), n, momentum, dampening, wd, nesterov, 0, zero_grad,
                    s, lr.data_ptr())
        pb, mb, gb = p0.clone(), m0.clone(), g0.clone()
        sp, sm = torch.full_like(p0, float("nan")), torch.full_like(m0, float("nan"))
        C.sgd_ahead(pb.data_ptr(), mb.data_ptr(), sp.data_ptr(), sm.data_ptr(), n, ahead, momentum, dampening, wd,
                    nesterov, 7, s, lr.data_ptr())
        C.fused_sgd_tail(pb.data_ptr(), gb.data_ptr(), mb.data_ptr(), sp.data_ptr(), sm.data_ptr(), n, ahead, dense,
                         momentum, dampening, wd, nesterov, 0, zero_grad, s, lr.data_ptr())
        torch.cuda.synchronize()
        assert torch.equal(_bits(pa), _bits(pb))
        if momentum != 0.0:
            assert torch.equal(_bits(ma), _bits(mb))
        assert torch.equal(_bits(ga), _bits(gb))


@pytest.mark.gpu
@pytest.mark.parametrize("flag", ["fault", "skip"])
def test_tail_restores_the_stash_when_the_step_is_not_applied(flag):
    """A timed-out cross-GPU wait (the fault word, written here as the host's fault mirror writes it) or a loss-scaling
    skip: p and m are bitwise what they were before the ahead pass; the gradient is what fused_sgd leaves."""
    from oktopk_b200.ops import ext
    C = ext.require()
    n = 50_001
    gen = torch.Generator(device="cuda").manual_seed(7)
    s = torch.cuda.current_stream().cuda_stream
    lr = torch.tensor([0.05], device="cuda")
    word = torch.ones(1, dtype=torch.int32, device="cuda")
    p0, m0, g0 = torch.randn(n, generator=gen, device="cuda"), torch.randn(n, generator=gen, device="cuda"), \
        _sparse_grad(n, gen)
    ahead, dense = _ranges(n, random.Random(3))
    pa, ma, ga = p0.clone(), m0.clone(), g0.clone()
    ptrs = dict(fault_ptr=word.data_ptr()) if flag == "fault" else dict(skip_ptr=word.data_ptr())
    C.fused_sgd(pa.data_ptr(), ga.data_ptr(), ma.data_ptr(), n, 0.9, 0.0, 5e-4, 0, 0, 1, s, lr.data_ptr(), **ptrs)
    pb, mb, gb = p0.clone(), m0.clone(), g0.clone()
    sp, sm = torch.empty_like(p0), torch.empty_like(m0)
    C.sgd_ahead(pb.data_ptr(), mb.data_ptr(), sp.data_ptr(), sm.data_ptr(), n, ahead, 0.9, 0.0, 5e-4, 0, 32, s,
                lr.data_ptr())
    C.fused_sgd_tail(pb.data_ptr(), gb.data_ptr(), mb.data_ptr(), sp.data_ptr(), sm.data_ptr(), n, ahead, dense, 0.9,
                     0.0, 5e-4, 0, 0, 1, s, lr.data_ptr(), **ptrs)
    torch.cuda.synchronize()
    assert torch.equal(_bits(pb), _bits(p0)) and torch.equal(_bits(mb), _bits(m0))
    assert torch.equal(_bits(pa), _bits(pb)) and torch.equal(_bits(ma), _bits(mb)) and torch.equal(_bits(ga), _bits(gb))


# ---------------------------------------------------------------------------------------------------------- trainer (GPU)
@pytest.mark.gpu
def test_vgg_trainer_with_and_without_sgd_ahead_agree():
    """40 sparse VGG-16 steps after a short dense warm-up, in whole-step CUDA graphs: parameters, momentum buffers and
    residuals are bit for bit the same with the early SGD update on and off."""
    import bench
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, _ = bench.MODELS["vgg16"]
    trs, calls = [], []
    for on in (False, True):
        torch.manual_seed(0)
        cfg = okt.preset("vgg16", density=0.001, warmup_iters=3, sgd_ahead=on)
        tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001,
                     compression=True, cfg=cfg, seq_len=128, t_total=100000, warmup=0.1, cuda_graph=True)
        if on:
            inner = tr.optimizer._sgd_ahead
            tr.optimizer._sgd_ahead = lambda *a: (calls.append(1), inner(*a))
        trs.append(tr)
    pool = [tuple(t.to(trs[0].device) for t in bench.make_batch("vgg16", i, 0, bs, 128)) for i in range(4)]
    for it in range(3 + 40):
        for tr in trs:
            tr.step(pool[it % 4])
    torch.cuda.synchronize()
    assert calls, "the early SGD update never ran"
    a, b = (tr.optimizer for tr in trs)
    for pa, pb in zip(trs[0].net.parameters(), trs[1].net.parameters()):
        assert torch.equal(_bits(pa.detach()), _bits(pb.detach()))
    for ba, bb in zip(a._buckets, b._buckets):
        assert torch.equal(_bits(a._flat_state[ba.index]["momentum_buffer"]),
                           _bits(b._flat_state[bb.index]["momentum_buffer"]))
        assert torch.equal(_bits(a._allreducer._engines[ba.name].residual),
                           _bits(b._allreducer._engines[bb.name].residual))
        assert torch.equal(_bits(ba.grad), _bits(bb.grad))
    for tr in trs:
        tr.close()
