"""Early pack (parallel/early_pack.py): a threshold-reuse Ok-Topk call whose bucket was partly packed during backward by
segment launches must compute exactly what the single launch computes."""
import copy
import random

import pytest
import torch


# ---------------------------------------------------------------------------------------------------------- planner (CPU)
def _layout(sizes, rng):
    offs, o = [], 0
    for s in sizes:
        offs.append(o)
        o += (s + 3) // 4 * 4 + 4 * rng.randrange(3)          # padding gaps of 0 - 8 elements
    return offs, o - rng.randrange(4)                         # a bucket length that need not be a multiple of 4


@pytest.mark.parametrize("seed", range(40))
def test_planner_packs_every_element_exactly_once(seed):
    from oktopk_b200.parallel.early_pack import PackPlanner
    rng = random.Random(seed)
    sizes = [rng.choice([1, 3, 5, 10, 64, 301, 4097, 20000]) for _ in range(rng.randrange(1, 30))]
    offs, n = _layout(sizes, rng)
    n = max(n, offs[-1] + 1)
    pl = PackPlanner(offs, n, min_elems=rng.choice([1, 50, 4096, 30000]), max_ranges=rng.choice([2, 4, 32]))
    for _ in range(2):                                        # a second call after reset() plans afresh
        order = list(range(len(sizes)))
        rng.shuffle(order)
        arrived = order[:len(order) - rng.randrange(len(order) + 1) // 3]   # some parameters get no gradient
        segs = [r for r in (pl.ready(i) for i in arrived) if r is not None]
        assert all(pl.ready(i) is None for i in arrived)      # a second hook of the same parameter packs nothing
        assert segs == pl.segments
        ranges = [r for seg in segs for r in seg]
        assert len(ranges) <= pl.max_ranges - 1
        rest = pl.rest()
        assert len(rest) <= pl.max_ranges
        cover = [0] * (4 * (n // 4))
        for lo, hi in ranges + rest:
            assert lo % 4 == 0 and hi % 4 == 0 and lo < hi
            for e in range(lo, hi):
                cover[e] += 1
        assert all(c == 1 for c in cover)
        for seg in segs:                                      # a segment covers only parameters that had arrived
            assert sum(hi - lo for lo, hi in seg) >= pl.min_elems
            assert seg == sorted(seg) and all(a[1] < b[0] for a, b in zip(seg, seg[1:]))
            for lo, hi in seg:
                for i, o in enumerate(offs):
                    if lo <= o < hi:
                        assert i in arrived
        assert rest == sorted(rest) and all(a[1] < b[0] for a, b in zip(rest, rest[1:]))
        pl.reset()


def test_planner_rejects_unaligned_offsets():
    from oktopk_b200.parallel.early_pack import PackPlanner
    with pytest.raises(ValueError):
        PackPlanner([0, 6], 16, 1, 4)


# ---------------------------------------------------------------------------------------------------------- engine (GPU)
def _engine_layout(sizes):
    offs, o = [], 0
    for s in sizes:
        offs.append(o)
        o += (s + 63) // 64 * 64
    return offs, o


@pytest.mark.gpu
@pytest.mark.parametrize("plan", ["one", "many", "unaligned", "scattered"])
def test_segments_then_call_match_the_single_launch(plan):
    """1 .. many segments of 1 .. many ranges, with a tile boundary (4096 elements) and a partial last vector inside one, then
    the call over what they left: bucket, residual, thresholds and counts are those of one launch, bit for bit, over
    threshold-reuse iterations and the exact-threshold ones in between (which take no segments)."""
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.early_pack import PackPlanner
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.world import World
    sizes = [1_000_003, 300, 10, 64, 4097, 2_359_296, 7, 5, 123_457]
    has_grad = [True, False, True, True, True, True, True, True, True]
    offs, n = _engine_layout(sizes)
    cfg = OkTopkConfig(density=0.01, local_recompute_interval=4, global_recompute_interval=4, repartition_interval=8)
    w = World()
    ea, eb = CudaBucketEngine(n, cfg, w, name="single"), CudaBucketEngine(n, cfg, w, name="segments")
    arrive = {"one": [5, 6, 7, 8], "many": [8, 7, 6, 5, 4, 3, 2, 0], "unaligned": [4, 0, 2, 3, 8, 6],
              "scattered": [5, 0, 8, 3, 2]}[plan]
    min_elems = {"one": 2_000_000, "many": 1, "unaligned": 3000, "scattered": 3_400_000}[plan]
    pl = PackPlanner(offs, n, min_elems, eb.C.PACK_RANGE_MAX)
    segments_run = 0
    for it in range(10):
        gen = torch.Generator(device="cuda").manual_seed(2000 + it)
        grads = [torch.randn(s, device="cuda", generator=gen) * (1.0 + 0.3 * it) if h else None
                 for s, h in zip(sizes, has_grad)]

        def table(lo=0, hi=n):
            keep = [(g, o) for g, o in zip(grads, offs) if g is not None and lo <= o < hi]
            return [g.data_ptr() for g, _ in keep], [o for _, o in keep], [g.numel() for g, _ in keep]

        ea.reduce("oktopk", srcs=table())
        pl.reset()
        early = eb.packs_early("oktopk")
        assert early == (it % 4 != 0)
        if early:
            for i in arrive:
                seg = pl.ready(i)
                if seg is not None:
                    keep = [t for lo, hi in seg for t in zip(*table(lo, hi))]
                    eb.pack_segment("oktopk", seg, tuple(list(c) for c in zip(*keep)))
                    segments_run += 1
        eb.reduce("oktopk", srcs=table(), pack_ranges=pl.rest() if pl.segments else None)
        torch.cuda.synchronize()
        assert torch.equal(ea.grad, eb.grad), it
        assert torch.equal(ea.residual, eb.residual), it
        sa, sb = ea.stats(), eb.stats()
        for k in ("local_thr", "local_thr_used", "global_thr", "local_count", "global_count", "recv_total",
                  "gather_total", "overflow_send", "overflow_gather", "redo"):
            if k in sa:
                assert sa[k] == sb[k], (it, k, sa[k], sb[k])
        ea.grad.zero_()
        eb.grad.zero_()
    assert segments_run >= {"one": 7, "many": 14, "unaligned": 7, "scattered": 7}[plan]
    ea.close()
    eb.close()


@pytest.mark.gpu
def test_vgg_optimizer_with_and_without_early_pack_agree():
    """VGG-16 through DistributedOptimizer, eager and in whole-step CUDA graphs: the hooks' segments (one per
    threshold-reuse step: 4 eager, 1 captured) change nothing in the parameters or the residual."""
    import oktopk_b200 as okt
    from oktopk_b200.models import create_net
    torch.manual_seed(0)
    base, _ = create_net(10, "vgg16")
    base = base.cuda().to(memory_format=torch.channels_last)
    nets, opts = [], []
    for on in (False, True):
        net = copy.deepcopy(base)
        cfg = okt.preset("vgg16", density=0.001, warmup_iters=0, local_recompute_interval=4,
                         global_recompute_interval=4, early_pack=on)
        opts.append(okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4),
                                             named_parameters=net.named_parameters(),
                                             compression=okt.compressors["oktopk"], is_sparse=True, cfg=cfg))
        nets.append(net)
    segs = []
    inner = opts[1]._allreducer.pack_segment
    opts[1]._allreducer.pack_segment = lambda *a, **k: (segs.append(a[1]), inner(*a, **k))
    x = torch.randn(16, 3, 32, 32, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (16,), device="cuda")
    graphs = [None, None]
    for it in range(12):
        for a in range(2):
            if it < 6:
                opts[a].zero_grad()
                torch.nn.functional.cross_entropy(nets[a](x), y).backward()
                opts[a].step()
            else:                                               # one graph of a threshold-reuse step, replayed
                if graphs[a] is None:
                    s = torch.cuda.Stream()
                    s.wait_stream(torch.cuda.current_stream())
                    graphs[a] = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graphs[a]):
                        opts[a].zero_grad()
                        torch.nn.functional.cross_entropy(nets[a](x), y).backward()
                        opts[a].step()
                graphs[a].replay()
        torch.cuda.synchronize()
        for pa, pb in zip(nets[0].parameters(), nets[1].parameters()):
            assert torch.equal(pa, pb), it
        ra = opts[0]._allreducer._engines[opts[0]._buckets[0].name].residual
        rb = opts[1]._allreducer._engines[opts[1]._buckets[0].name].residual
        assert torch.equal(ra, rb), it
    assert len(segs) == 5 and not opts[0]._allreducer.packs_early(opts[0]._buckets[0].name)
    for o in opts:
        o.close()
