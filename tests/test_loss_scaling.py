"""Dynamic loss scaling (``LossScale``): gradients are unscaled before they reach a residual, a threshold or a momentum; a
bucket with a non-finite value on any rank is skipped on every rank, leaving its sparse state bitwise unchanged; a step
with a skipped bucket updates nothing and backs the scale off as ``torch.amp.GradScaler`` does.

CPU: the oracle's rules, the torch.distributed path (gloo) and the torch update path.  GPU: the ``unscale_check`` kernel,
every native scheme at P = 1, the fused Adam against torch's, and VGG-16 under fp16 autocast with whole-step CUDA graphs.
"""
import copy
import os
import struct
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from mp_util import run_distributed  # noqa: E402

gpu = pytest.mark.gpu


def _grad(it, rank, n):
    g = torch.Generator().manual_seed(1000 * it + rank)
    return torch.randn(n, generator=g) * torch.linspace(0.2, 2.0, n)


# ================================================================================================ CPU: oracle
def test_oracle_poisoned_bucket_keeps_its_state_while_clean_buckets_proceed():
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.oracle import inv_scale_of, run_oracle, run_oracle_scaled
    from oktopk_b200.parallel.state import SparseState
    P, n, scale = 2, 4000, 1024.0
    inv = inv_scale_of(scale)
    cfg = OkTopkConfig(density=0.02, local_recompute_interval=1, global_recompute_interval=1, repartition_interval=1)
    states = {b: [SparseState(n, P) for _ in range(P)] for b in ("clean", "poisoned")}
    ref = [SparseState(n, P) for _ in range(P)]
    for it in range(3):
        for b, sts in states.items():
            grads = [_grad(it, r, n) * scale for r in range(P)]
            if b == "poisoned" and it == 2:
                grads[1][17] = float("nan")
                before = [(st.residual.clone(), st.local_thr, st.global_thr, list(st.region_offsets)) for st in sts]
            out, skipped = run_oracle_scaled("oktopk", grads, sts, cfg, inv)
            assert skipped == (b == "poisoned" and it == 2)
            if skipped:
                for st, (res, lt, gt, off) in zip(sts, before):
                    assert torch.equal(st.residual, res) and st.local_thr == lt and st.global_thr == gt
                    assert st.region_offsets == off
            elif b == "clean":
                # scaling by a power of two and unscaling is exact: the same as reducing the unscaled gradients
                want = run_oracle("oktopk", [_grad(it, r, n) for r in range(P)], ref, cfg)
                for o, w in zip(out, want):
                    assert torch.equal(o, w)
    assert states["poisoned"][0].counter == 3          # iteration counters advance on a skipped call


def _gradscaler_sequence(verdicts, init, growth, backoff, interval):
    p = torch.nn.Parameter(torch.ones(3))
    opt = torch.optim.SGD([p], lr=0.0)
    scaler = torch.amp.GradScaler("cpu", init_scale=init, growth_factor=growth, backoff_factor=backoff,
                                  growth_interval=interval)
    out = []
    for bad in verdicts:
        opt.zero_grad()
        scaler.scale((p * (float("inf") if bad else 1.0)).sum()).backward()
        scaler.step(opt)
        scaler.update()
        out.append((float(scaler.get_scale()), int(scaler._growth_tracker)))
    return out


def test_scale_sequence_matches_gradscaler():
    from oktopk_b200.config import LossScale
    from oktopk_b200.parallel.oracle import update_scale
    verdicts = [False] * 7 + [True] + [False] * 3 + [True, True] + [False] * 12
    for ls in (LossScale(init_scale=2.0 ** 10, growth_interval=3), LossScale(init_scale=3.0, growth_factor=1.5,
                                                                            backoff_factor=0.25, growth_interval=2),
               LossScale(init_scale=2.0 ** 127, growth_interval=1)):          # growth to inf is refused
        want = _gradscaler_sequence(verdicts, ls.init_scale, ls.growth_factor, ls.backoff_factor, ls.growth_interval)
        scale, tracker, got = ls.init_scale, 0, []
        for bad in verdicts:
            scale, tracker = update_scale(scale, tracker, bad, ls)
            got.append((scale, tracker))
        assert got == want


def test_loss_scale_parse_and_momentum_correction_conflict():
    from oktopk_b200.config import LossScale
    from oktopk_b200.optimizer import DistributedOptimizer
    assert LossScale.parse(None) is None
    assert LossScale.parse("dynamic") == LossScale()
    assert LossScale.parse("128") == LossScale(init_scale=128.0, growth_factor=1.0, backoff_factor=1.0)
    with pytest.raises(ValueError):
        LossScale(backoff_factor=2.0)
    m = torch.nn.Linear(4, 2)
    opt = DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9),
                               named_parameters=m.named_parameters(), loss_scale=LossScale())
    with pytest.raises(ValueError):
        opt.momentum_correction = True
    plain = DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters())
    plain.momentum_correction = True
    assert plain.loss_scale_state() is None


# ================================================================================================ CPU: gloo
def _model(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.Tanh(), torch.nn.Linear(32, 4))


def _batch(it, rank):
    g = torch.Generator().manual_seed(31 * it + rank)
    return torch.randn(8, 16, generator=g), torch.randint(0, 4, (8,), generator=g)


def _train_step(model, opt, it, rank, poison=False):
    x, y = _batch(it, rank)
    loss = torch.nn.functional.cross_entropy(model(x), y)
    if poison:
        loss = loss * float("inf")
    opt.scale_loss(loss).backward()
    opt.step()
    opt.zero_grad()


def _skip_worker(rank, P, name):
    from oktopk_b200.config import LossScale, OkTopkConfig
    from oktopk_b200.optimizer import DistributedOptimizer
    cfg = OkTopkConfig(compressor=name, density=0.05, local_recompute_interval=1, global_recompute_interval=1,
                       repartition_interval=1, backend="dist")
    model = _model()

    def make(m):
        return DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9),
                                    named_parameters=m.named_parameters(), compression=name, is_sparse=True, cfg=cfg,
                                    loss_scale=LossScale(init_scale=2.0 ** 12))
    opt = make(model)
    for it in range(3):
        _train_step(model, opt, it, rank)
    before = [p.detach().clone() for p in model.parameters()]
    sd = copy.deepcopy(opt.state_dict())
    scale0 = opt.loss_scale_state()
    _train_step(model, opt, 3, rank, poison=(rank == P - 1))
    after_skip = [p.detach().clone() for p in model.parameters()]
    scale1 = opt.loss_scale_state()
    _train_step(model, opt, 4, rank)
    after_next = [p.detach().clone() for p in model.parameters()]
    # the same clean step, run from the state before the skip
    model2 = _model()
    with torch.no_grad():
        for p, q in zip(model2.parameters(), before):
            p.copy_(q)
    opt2 = make(model2)
    opt2.load_state_dict(sd)
    _train_step(model2, opt2, 4, rank)
    replay = [p.detach().clone() for p in model2.parameters()]
    return before, after_skip, after_next, replay, scale0, scale1


@pytest.mark.parametrize("P", [2, 4])
@pytest.mark.parametrize("name", ["oktopk", "gtopk"])
def test_gloo_inf_on_one_rank_skips_on_every_rank(name, P):
    got = run_distributed(_skip_worker, P, (name,), backend="gloo", timeout=240)
    for r in range(P):
        before, after_skip, after_next, replay, scale0, scale1 = got[r]
        for a, b in zip(before, after_skip):
            assert torch.equal(a, b), "rank %d: a skipped step changed a parameter" % r
        for a, b in zip(after_skip, got[0][1]):
            assert torch.equal(a, b), "rank %d diverged from rank 0" % r
        assert scale1["scale"] == scale0["scale"] / 2 and scale1["skipped_steps"] == scale0["skipped_steps"] + 1
        assert scale1["growth_tracker"] == 0
        for a, b in zip(after_next, replay):          # one bucket: the skip was a complete no-op
            assert torch.equal(a, b), "rank %d: the step after a skip differs from the same step without it" % r


# ================================================================================================ CPU: torch update path
def test_sgd_cpu_path_matches_torch_sgd_with_gradscaler():
    from oktopk_b200.config import LossScale
    from oktopk_b200.optimizer import DistributedOptimizer
    ls = LossScale(init_scale=2.0 ** 8, growth_interval=5)
    m1, m2 = _model(), _model()
    opt = DistributedOptimizer(torch.optim.SGD(m1.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-3),
                               named_parameters=m1.named_parameters(), loss_scale=ls)
    ref = torch.optim.SGD(m2.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-3)
    scaler = torch.amp.GradScaler("cpu", init_scale=ls.init_scale, growth_interval=ls.growth_interval)
    poison = {6, 17}
    for it in range(30):
        _train_step(m1, opt, it, 0, poison=it in poison)
        x, y = _batch(it, 0)
        loss = torch.nn.functional.cross_entropy(m2(x), y)
        if it in poison:
            loss = loss * float("inf")
        scaler.scale(loss).backward()
        scaler.step(ref)
        scaler.update()
        ref.zero_grad()
        st = opt.loss_scale_state()
        assert (st["scale"], st["growth_tracker"]) == (float(scaler.get_scale()), int(scaler._growth_tracker)), it
    assert opt.loss_scale_state()["skipped_steps"] == 2
    for a, b in zip(m1.parameters(), m2.parameters()):
        torch.testing.assert_close(a, b)


def test_state_dict_round_trip_resumes_like_an_uninterrupted_run():
    from oktopk_b200.config import LossScale, OkTopkConfig
    from oktopk_b200.optimizer import DistributedOptimizer
    cfg = OkTopkConfig(compressor="oktopk", density=0.1, backend="dist")

    def make(m):
        return DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9),
                                    named_parameters=m.named_parameters(), compression="oktopk", is_sparse=True,
                                    cfg=cfg, loss_scale=LossScale(init_scale=2.0 ** 6, growth_interval=2))
    m1 = _model()
    o1 = make(m1)
    for it in range(8):
        _train_step(m1, o1, it, 0, poison=it == 2)
    m2 = _model()
    o2 = make(m2)
    for it in range(4):
        _train_step(m2, o2, it, 0, poison=it == 2)
    sd, params = copy.deepcopy(o2.state_dict()), [p.detach().clone() for p in m2.parameters()]
    assert sd["loss_scale"]["skipped_steps"] == 1
    m3 = _model(seed=1)
    with torch.no_grad():
        for p, q in zip(m3.parameters(), params):
            p.copy_(q)
    o3 = make(m3)
    o3.load_state_dict(sd)
    for it in range(4, 8):
        _train_step(m3, o3, it, 0)
    assert o3.loss_scale_state() == o1.loss_scale_state()
    for a, b in zip(m1.parameters(), m3.parameters()):
        assert torch.equal(a, b)
    # a checkpoint without scale state starts from init_scale
    sd.pop("loss_scale")
    o3.load_state_dict(sd)
    assert o3.loss_scale_state() == {"scale": 2.0 ** 6, "growth_tracker": 0, "skipped_steps": 0}


# ================================================================================================ GPU
def _ls_state(buf):
    raw = bytes(buf.cpu().numpy())
    scale, inv, tracker, found, skipped, adam_step = struct.unpack("<ffiiqq", raw)
    return scale, inv, found


@gpu
@pytest.mark.parametrize("n", [4096, 100003, 1_000_001])
def test_unscale_check_output_and_flag(n):
    from oktopk_b200.config import LossScale, OkTopkConfig
    from oktopk_b200.optimizer import _ScaleState
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.world import World
    eng = CudaBucketEngine(n, OkTopkConfig(density=0.01), World(), name="t")
    ls = _ScaleState(LossScale(init_scale=3.0 * 2 ** 9), torch.device("cuda"))
    inv = ls.state()["scale"]
    inv_f = torch.tensor(1.0 / inv, dtype=torch.float64).float().cuda()
    gen = torch.Generator(device="cuda").manual_seed(3)
    # the direct path's source table: three tensors at offsets that are multiples of 4, lengths that need not be
    lens = [n // 3 - (n // 3) % 4, 5, n - (n // 3 - (n // 3) % 4) - 5 - 3]

    def run(values, table):
        ls.reset()
        if table:
            srcs = [values[sum(lens[:i]):sum(lens[:i + 1])].clone() for i in range(3)]
            eng.unscale_check(ls.ptr, srcs=([s.data_ptr() for s in srcs], [0, lens[0], lens[0] + lens[1]], lens))
            torch.cuda.synchronize()
            out = torch.cat(srcs)
        else:
            eng.grad.copy_(values)
            eng.unscale_check(ls.ptr)
            torch.cuda.synchronize()
            out = eng.grad.clone()
        return out, ls.state()["found_inf"]

    base = torch.randn(n, device="cuda", generator=gen) * 1e4
    for table in (False, True):
        m = sum(lens) if table else n
        x = base[:m].clone()
        out, found = run(x, table)
        assert found == 0 and torch.equal(out, x * inv_f), "output is not bitwise g * inv_scale"
        y = x.clone()
        y[::7] = torch.finfo(torch.float32).max
        assert run(y, table)[1] == 0, "FLT_MAX is finite"
        tail = m - 1 - (m % 4 == 0) * 2                    # the non-multiple-of-4 tail (or just before the end)
        # first and last element, the global tail, the scalar tail of the 5-element middle segment, a middle CTA
        for pos in (0, m - 1, tail, lens[0] + 4, m // 2 + 1):
            for bad in (float("inf"), float("-inf"), float("nan")):
                z = x.clone()
                z[pos] = bad
                assert run(z, table)[1] == 1, (table, pos, bad)
    eng.close()


def _scheme_cfg(name):
    from oktopk_b200.config import OkTopkConfig
    kw = dict(compressor=name, density=0.01, local_recompute_interval=2, global_recompute_interval=2,
              repartition_interval=2, topkaopt_recompute_interval=2, slot_factor=64, gather_factor=64)
    if name == "warmup":
        kw.update(compressor="oktopk", warmup_iters=100)
    return OkTopkConfig(**kw)


@gpu
@pytest.mark.parametrize("name", ["oktopk", "oktopk-direct", "topkA", "topkA2", "gaussiank", "gtopk", "topkDSA",
                                  "warmup"])
def test_every_native_scheme_skips_a_poisoned_call(name):
    from oktopk_b200.config import LossScale
    from oktopk_b200.optimizer import _ScaleState
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.oracle import run_oracle_scaled
    from oktopk_b200.parallel.state import SparseState
    from oktopk_b200.parallel.world import World
    direct = name == "oktopk-direct"
    scheme = {"oktopk-direct": "oktopk", "warmup": "oktopk"}.get(name, name)
    cfg = _scheme_cfg("oktopk" if direct else name)
    n = 200_003
    eng = CudaBucketEngine(n, cfg, World(), name="t")
    ls = _ScaleState(LossScale(init_scale=2.0 ** 10), torch.device("cuda"))
    inv = ls.state()["scale"] and (1.0 / ls.state()["scale"])
    states = [SparseState(n, 1)]
    for it in range(4):
        x = torch.randn(n, generator=torch.Generator().manual_seed(it)) * (1 + it)
        xs = x * 2.0 ** 10
        if it == 2:
            xs[n // 2] = float("inf")
        ls.reset()
        before = (eng.residual.clone(), {k: v for k, v in eng.stats().items() if k in ("local_thr", "global_thr",
                                                                                       "edges", "epoch")})
        if direct:
            src = xs.cuda()
            srcs = ([src.data_ptr()], [0], [n])
            eng.unscale_check(ls.ptr, srcs=srcs)
            eng.reduce(scheme, srcs=srcs, skip=eng.verdict_ptr)
        else:
            eng.grad.copy_(xs.cuda())
            eng.unscale_check(ls.ptr)
            eng.reduce(scheme, skip=eng.verdict_ptr)
        torch.cuda.synchronize()
        ref, skipped = run_oracle_scaled(scheme, [xs.clone()], states, cfg, inv)
        assert bool(ls.state()["found_inf"]) == skipped == (it == 2)
        if skipped:
            assert torch.equal(eng.residual, before[0]), "a skipped call changed the residual"
            st = eng.stats()
            assert {k: st[k] for k in before[1]} == before[1], "a skipped call changed thresholds / edges / epoch"
            if direct:
                assert float(eng.grad.abs().max()) == 0.0, "the direct-path bucket must stay all-zero"
            else:
                eng.grad.zero_()
            continue
        assert torch.equal(eng.grad.cpu(), ref[0]), "%s it %d differs from the oracle" % (name, it)
        if states[0].residual is not None:
            assert torch.equal(eng.residual.cpu(), states[0].residual)
        if direct:
            eng.grad.zero_()                      # what the fused update does after every step
    eng.close()


@gpu
def test_fused_adamw_with_dynamic_scaling_matches_torch_gradscaler():
    from oktopk_b200.config import LossScale, OkTopkConfig
    from oktopk_b200.optimizer import DistributedOptimizer
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 10)).cuda()
    ref_net = copy.deepcopy(net)
    ls = LossScale(init_scale=2.0 ** 12, growth_interval=20)
    opt = DistributedOptimizer(torch.optim.AdamW(net.parameters(), lr=1e-3, weight_decay=1e-2, fused=True),
                               named_parameters=net.named_parameters(), compression="none",
                               cfg=OkTopkConfig(compressor="none", sparse=False), loss_scale=ls)
    ref = torch.optim.AdamW(ref_net.parameters(), lr=1e-3, weight_decay=1e-2, fused=True)
    scaler = torch.amp.GradScaler("cuda", init_scale=ls.init_scale, growth_interval=ls.growth_interval)
    poison = {3, 30}
    for it in range(50):
        # each step starts from the same parameters and moments: under fp16 autocast a last-bit difference would
        # otherwise be amplified step after step by the fp16 rounding of the activations
        with torch.no_grad():
            for p, q in zip(net.parameters(), ref_net.parameters()):
                q.copy_(p)
                if q in ref.state:
                    ref.state[q]["exp_avg"].copy_(opt.state[p]["exp_avg"])
                    ref.state[q]["exp_avg_sq"].copy_(opt.state[p]["exp_avg_sq"])
        g = torch.Generator(device="cuda").manual_seed(it)
        x, y = torch.randn(32, 64, device="cuda", generator=g), torch.randint(0, 10, (32,), device="cuda", generator=g)
        for model, which in ((net, 0), (ref_net, 1)):
            with torch.autocast("cuda", dtype=torch.float16):
                loss = torch.nn.functional.cross_entropy(model(x), y)
            if it in poison:
                loss = loss * float("inf")
            if which == 0:
                opt.scale_loss(loss).backward()
                opt.step()
                opt.zero_grad()
            else:
                scaler.scale(loss).backward()
                scaler.step(ref)
                scaler.update()
                ref.zero_grad()
    st = opt.loss_scale_state()
    assert st["scale"] == float(scaler.get_scale()) and st["growth_tracker"] == int(scaler._growth_tracker)
    assert st["skipped_steps"] == 2
    sd = opt.state_dict()
    for i, (p, q) in enumerate(zip(net.parameters(), ref_net.parameters())):
        torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)
        rs = ref.state[q]
        torch.testing.assert_close(opt.state[p]["exp_avg"], rs["exp_avg"], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(opt.state[p]["exp_avg_sq"], rs["exp_avg_sq"], rtol=1e-5, atol=1e-6)
        assert float(sd["state"][i]["step"]) == float(rs["step"]) == 48.0


@gpu
def test_vgg16_fp16_graphed_overflow_skips_until_the_first_applied_step():
    """VGG-16 (the bench workload: Ok-Topk 0.001, SGD), fp16 autocast, LossScale(2^40): the fp16 backward overflows.
    Every overflowing replay leaves parameters, momentum and residual bitwise unchanged and halves the scale; graphed and
    eager runs agree, and the replay loop adds no host synchronisation."""
    from oktopk_b200.config import LossScale, preset
    from oktopk_b200.train.trainer import Trainer, preset_for

    def make(graph):
        return Trainer(dnn="vgg16", dataset="cifar10", batch_size=16, lr=0.01, density=0.001, cuda_graph=graph, seed=0,
                       cfg=preset(preset_for("vgg16"), density=0.001, warmup_iters=0), autocast="fp16",
                       loss_scale=LossScale(init_scale=2.0 ** 40))

    def eager(tr, batch):
        tr.optimizer.zero_grad()
        loss, _ = tr._forward_loss(batch)
        tr.backward(loss)
        tr.update_model()

    runs = {}
    for graph in (False, True):
        tr = make(graph)
        tr.net.train()
        opt = tr.optimizer
        assert len(opt._buckets) == 1
        batch = tuple(t.cuda() for t in next(iter(tr.loader)))
        eng = opt._allreducer._engines[opt._buckets[0].name]
        hist, applied = [], 0
        for i in range(48):
            snap = ([p.detach().clone() for p in tr.net.parameters()],
                    [t.clone() for fs in opt._flat_state.values() for t in fs.values()], eng.residual.clone())
            scale_before = opt.loss_scale_state()["scale"]
            if graph and i >= 4:                  # replays only: the first graphed step captured every flavour
                torch.cuda.set_sync_debug_mode("error")
            try:
                tr.graphed.step(batch) if graph else eager(tr, batch)
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
