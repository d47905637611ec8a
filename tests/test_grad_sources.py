"""GPU tests: the Ok-Topk reduction reading the gradient straight from autograd's tensors (a gradient-source table)
instead of from a bucket the gradients were first copied into.  Results must be bitwise those of the landing path."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu


def _layout(sizes):
    offs, o = [], 0
    for s in sizes:
        offs.append(o)
        o += (s + 63) // 64 * 64
    return offs, o


@pytest.mark.parametrize("slot_factor", [0.0, 64.0])
def test_oktopk_run_reads_gradient_sources_like_the_bucket(slot_factor):
    """Padding gaps, a parameter without a gradient, a 10-element tail (and 1- and 3-element ones), small and large
    tensors: the source-table call and the bucket-resident call agree exactly on result, residual, thresholds and counts,
    over exact-threshold and threshold-reuse iterations."""
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.world import World
    sizes = [1_000_003, 300, 10, 64, 4097, 2_359_296, 7, 5]
    has_grad = [True, False, True, True, True, True, True, True]
    offs, n = _layout(sizes)
    cfg = OkTopkConfig(density=0.01, local_recompute_interval=4, global_recompute_interval=4, repartition_interval=8,
                       slot_factor=slot_factor, gather_factor=slot_factor)
    w = World()
    ea, eb = CudaBucketEngine(n, cfg, w, name="bucket"), CudaBucketEngine(n, cfg, w, name="sources")
    for it in range(10):
        gen = torch.Generator(device="cuda").manual_seed(1000 + it)
        grads = [torch.randn(s, device="cuda", generator=gen) * (1.0 + 0.3 * it) if h else None
                 for s, h in zip(sizes, has_grad)]
        keep = [None if g is None else g.clone() for g in grads]
        ea.grad.zero_()
        for g, o in zip(grads, offs):
            if g is not None:
                ea.grad[o:o + g.numel()].copy_(g)
        ea.reduce("oktopk")
        assert eb.reads_sources("oktopk")
        assert float(eb.grad.abs().max()) == 0.0
        srcs = ([g.data_ptr() for g in grads if g is not None], [o for g, o in zip(grads, offs) if g is not None],
                [g.numel() for g in grads if g is not None])
        eb.reduce("oktopk", srcs=srcs)
        torch.cuda.synchronize()
        assert torch.equal(ea.grad, eb.grad), it
        assert torch.equal(ea.residual, eb.residual), it
        sa, sb = ea.stats(), eb.stats()
        for k in ("local_thr", "local_thr_used", "global_thr", "local_count", "global_count", "recv_total",
                  "gather_total", "overflow_send", "overflow_gather", "redo"):
            if k in sa:
                assert sa[k] == sb[k], (it, k, sa[k], sb[k])
        assert sa["local_count"] > 0 and sa["global_count"] > 0
        for g, k in zip(grads, keep):                       # the sources are only read
            assert g is None or torch.equal(g, k)
        eb.grad.zero_()                                     # what the fused update does to the few written entries
    ea.close()
    eb.close()


def _vgg_opts(kinds, warmup_iters, seed=0):
    import oktopk_b200 as okt
    from oktopk_b200.models import create_net
    torch.manual_seed(seed)
    base, _ = create_net(10, "vgg16")
    base = base.cuda().to(memory_format=torch.channels_last)
    nets, opts = [], []
    for kind in kinds:
        net = copy.deepcopy(base)
        cfg = okt.preset("vgg16", density=0.01, warmup_iters=warmup_iters, land_grads=kind != "views")
        opt = okt.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4),
                                       named_parameters=net.named_parameters(), compression=okt.compressors["oktopk"],
                                       is_sparse=True, cfg=cfg)
        if kind == "land":
            opt._direct = False                              # the landing copy + bucket-resident reduction
        nets.append(net)
        opts.append(opt)
    return nets, opts


def _batches(k):
    g = torch.Generator(device="cuda").manual_seed(7)
    return [(torch.randn(8, 3, 32, 32, device="cuda", generator=g).contiguous(memory_format=torch.channels_last),
             torch.randint(0, 10, (8,), device="cuda", generator=g)) for _ in range(k)]


def test_reading_sources_trains_bitwise_like_landing_and_like_accumulating_into_views():
    """VGG-16 over 36 steps (2 dense, then sparse steps 0..33: two exact-threshold iterations at 0 and 32): reading
    autograd's gradients in place, landing them with one copy, and accumulating into bucket views give identical bits."""
    from oktopk_b200.ops import ext
    torch.backends.cudnn.deterministic = True
    nets, opts = _vgg_opts(("direct", "land", "views"), warmup_iters=2)
    assert opts[0]._direct and not opts[1]._direct and opts[1]._land and not opts[2]._land
    for it, (x, y) in enumerate(_batches(36)):
        for k, (net, opt) in enumerate(zip(nets, opts)):
            land0 = ext.LAUNCH_COUNT.get("land_grads", 0)
            opt.zero_grad()
            torch.nn.functional.cross_entropy(net(x), y).backward()
            opt.step()
            if k == 0:
                landed = ext.LAUNCH_COUNT.get("land_grads", 0) - land0
                assert landed == (1 if it < 2 else 0), (it, landed)
                torch.cuda.synchronize()
                assert float(opt._buckets[0].grad.abs().max()) == 0.0, it     # the update left the bucket all-zero
    torch.cuda.synchronize()
    for other in (1, 2):
        for (name, a), b in zip(nets[0].named_parameters(), nets[other].parameters()):
            assert torch.equal(a, b), (other, name)
        ra = opts[0]._allreducer._engines[opts[0]._buckets[0].name].residual
        rb = opts[other]._allreducer._engines[opts[other]._buckets[0].name].residual
        assert torch.equal(ra, rb), other
    for o in opts:
        o.close()


class _Shim:
    """The part of Trainer that GraphedTrainStep drives."""

    def __init__(self, net, opt):
        self.net, self.optimizer = net, opt

    def _forward_loss(self, batch):
        x, y = batch
        return torch.nn.functional.cross_entropy(self.net(x), y), None

    def update_model(self):
        self.optimizer.step()


def test_graphed_steps_read_sources_across_the_dense_to_sparse_transition():
    """Whole-step CUDA graphs: the dense warm-up graph lands the gradients, the sparse graphs do not, the bucket is
    all-zero after every step, and the parameters match eager steps through the landing path exactly."""
    from oktopk_b200.ops import ext
    from oktopk_b200.train.graph_step import GraphedTrainStep
    torch.backends.cudnn.deterministic = True
    nets, opts = _vgg_opts(("direct", "land"), warmup_iters=4)
    gs = GraphedTrainStep(_Shim(nets[0], opts[0]), warmup_eager=2)
    landed = []
    for it, batch in enumerate(_batches(12)):
        land0 = ext.LAUNCH_COUNT.get("land_grads", 0)                # (capture counts the launches a graph records)
        gs.step(batch)
        landed.append(ext.LAUNCH_COUNT.get("land_grads", 0) - land0)
        torch.cuda.synchronize()
        assert float(opts[0]._buckets[0].grad.abs().max()) == 0.0, it
        opts[1].zero_grad()
        torch.nn.functional.cross_entropy(nets[1](batch[0]), batch[1]).backward()
        opts[1].step()
    torch.cuda.synchronize()
    assert gs.enabled, gs.why_disabled
    assert len(gs.graphs) >= 2
    assert landed[:3] == [1, 1, 1] and not any(landed[4:]), landed     # eager, eager, dense capture; sparse steps: none
    for (name, a), b in zip(nets[0].named_parameters(), nets[1].parameters()):
        assert torch.equal(a, b), name
    for o in opts:
        o.close()
