"""The fused softmax + CTC loss (``csrc/ctc.cu``, ``ops/fused_ctc.py``) on the GPU: loss and logits' gradient against
``F.ctc_loss`` in float64 on the CPU, no worse than the stock fp32 op on the GPU; the edge cases of the kernels' header
(zero_infinity, frames past Tn, a bad label, Ln = 0, Tn = 0); the loss scale and an fp16 overflow; determinism; no host
synchronisation and CUDA-graph replay; launch counts; the whole DeepSpeech model; and Trainer steps against stock."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oktopk_b200.models import create_net
from oktopk_b200.ops import ext
from oktopk_b200.ops.fused_ctc import ctc_loss

pytestmark = pytest.mark.gpu

C = 29


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _launches():
    return ext.LAUNCH_COUNT.get("ctc_forward", 0), ext.LAUNCH_COUNT.get("ctc_backward", 0)


def _stock(x, targets, tn, ln, reduction="sum"):
    return F.ctc_loss(F.log_softmax(x, -1).float(), targets.long(), tn.long(), ln.long(), blank=0,
                      reduction=reduction, zero_infinity=True)


def _need(labels):
    """Frames the labels need: one each, plus a blank between equal neighbours."""
    return len(labels) + sum(1 for a, b in zip(labels, labels[1:]) if a == b)


def _batch(N, T, seed, infeasible=False):
    """Logits [T, N, C] and a batch with mixed Tn (the first utterance full length), Ln from 0 up to feasibility, runs
    of repeated labels, and with `infeasible` one utterance that cannot be aligned."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, N, C, generator=g) * 2
    tn = [T] + [int(torch.randint(1, T + 1, (1,), generator=g)) for _ in range(N - 1)]
    tgts, lns = [], []
    for n in range(N):
        cap = tn[n]
        L = int(torch.randint(0, cap + 1, (1,), generator=g)) if n else min(cap, 33)
        lab = torch.randint(1, C, (L,), generator=g).tolist()
        if L >= 4:
            lab[1] = lab[2] = lab[3] = lab[0]                  # a run of repeats
        while lab and _need(lab) > cap:
            lab.pop()
        if infeasible and n == N - 1:                        # cap repeats need 2 cap - 1 > cap frames
            lab = [7] * cap if cap >= 2 else [3, 4]
        tgts += lab
        lns.append(len(lab))
    return x, torch.tensor(tgts, dtype=torch.int64), torch.tensor(tn, dtype=torch.int32), torch.tensor(lns, dtype=torch.int32)


def _fused(x, targets, tn, ln, g=1.0):
    xi = x.detach().clone().requires_grad_(True)
    loss = ctc_loss(xi, targets, tn, ln)
    (dx,) = torch.autograd.grad(loss, xi, torch.tensor(g, device=loss.device))
    return loss.detach(), dx


def _ctc64(x, targets, tn, ln):
    """F.ctc_loss in float64 on the CPU, on log_softmax of the widened logits (no .float() in between)."""
    return F.ctc_loss(F.log_softmax(x.double().cpu(), -1), targets.cpu().long(), tn.cpu().long(), ln.cpu().long(),
                      blank=0, reduction="sum", zero_infinity=True)


def _ref(x, targets, tn, ln):
    xi = x.detach().double().cpu().requires_grad_(True)
    loss = _ctc64(xi, targets, tn, ln)
    (dx,) = torch.autograd.grad(loss, xi)
    return loss.detach(), dx


def _stock_gpu(x, targets, tn, ln):
    xi = x.detach().float().cuda().requires_grad_(True)
    loss = _stock(xi, targets.cuda(), tn.cuda(), ln.cuda())
    (dx,) = torch.autograd.grad(loss, xi)
    return loss.detach(), dx


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("N,T", [(1, 1), (2, 2), (2, 48), (5, 48), (1, 198), (2, 198), (5, 198), (2, 400), (5, 400)])
def test_loss_and_gradient_against_float64(N, T, dtype):
    x, targets, tn, ln = _batch(N, T, seed=N * 1000 + T, infeasible=T >= 2 and N >= 2)
    x = x.to(dtype)                                           # the reference sees the same (widened) values
    n0 = _launches()
    lf, df = _fused(x.cuda(), targets.cuda(), tn, ln)
    n1 = _launches()
    assert (n1[0] - n0[0], n1[1] - n0[1]) == (2, 1)
    assert df.dtype == dtype
    lr, dr = _ref(x, targets, tn, ln)
    ls, ds = _stock_gpu(x, targets, tn, ln)
    el, es_l = abs(lf.double().cpu() - lr).item(), abs(ls.double().cpu() - lr).item()
    assert el <= 2 * es_l + 1e-5 * max(1.0, abs(lr.item())), (el, es_l, lr.item())
    ef = (df.cpu().double() - dr).abs()
    es = (ds.cpu().double() - dr).abs().max().item()
    rnd = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}[dtype]
    tol = rnd * dr.abs() + 2 * es + 1e-5
    assert bool((ef <= tol).all()), (ef.max().item(), es)
    for n in range(N):                                        # frames past Tn: exactly 0
        assert torch.all(df[int(tn[n]):, n] == 0)


def test_zero_infinity_leaves_the_others_unchanged():
    x, targets, tn, ln = _batch(4, 60, seed=11)
    bad_t = torch.cat([targets, torch.tensor([6, 6, 6, 6])])   # 4 repeats need 7 frames; the extra utterance has 5
    bad_tn = torch.cat([tn, torch.tensor([5], dtype=torch.int32)])
    bad_ln = torch.cat([ln, torch.tensor([4], dtype=torch.int32)])
    xb = torch.cat([x, torch.randn(60, 1, C)], dim=1)
    l4, d4 = _fused(x.cuda(), targets.cuda(), tn, ln)
    l5, d5 = _fused(xb.cuda(), bad_t.cuda(), bad_tn, bad_ln)
    assert torch.all(d5[:, 4] == 0)
    assert torch.equal(d5[:, :4], d4)
    assert l5.item() == pytest.approx(l4.item(), rel=1e-6)
    per = _stock(xb.double(), bad_t, bad_tn, bad_ln, reduction="none")
    assert per[4].item() == 0 and torch.isfinite(l5)


def test_frames_past_tn_are_never_read():
    g = torch.Generator().manual_seed(12)
    x = torch.randn(80, 3, C, generator=g)
    tn = torch.tensor([80, 50, 70], dtype=torch.int32)
    ln = torch.tensor([10, 12, 8], dtype=torch.int32)
    targets = torch.randint(1, C, (30,), generator=g)
    l0, d0 = _fused(x.cuda(), targets.cuda(), tn, ln)
    xp = x.clone()
    xp[50:, 1] = float("nan")
    xp[60:, 1, 3] = float("inf")
    l1, d1 = _fused(xp.cuda(), targets.cuda(), tn, ln)
    assert torch.equal(l0, l1) and torch.equal(d0, d1)
    assert torch.all(d1[50:, 1] == 0) and torch.isfinite(d1).all()
    assert torch.all(d1[70:, 2] == 0) and d1[:50, 1].abs().max() > 0


def test_label_out_of_range_is_nan_for_that_utterance():
    x, targets, tn, ln = _batch(3, 40, seed=13)
    ln = torch.tensor([3, 4, 2], dtype=torch.int32)
    targets = torch.tensor([1, 2, 3, 4, C, 5, 6, 7, 8])         # the second utterance holds C
    tn = torch.tensor([40, 30, 20], dtype=torch.int32)
    loss, dx = _fused(x.cuda(), targets.cuda(), tn, ln)
    assert torch.isnan(loss)
    assert torch.isnan(dx[:30, 1]).all() and torch.all(dx[30:, 1] == 0)
    assert torch.isfinite(dx[:, 0]).all() and torch.isfinite(dx[:, 2]).all()
    ref = _fused(x[:, [0, 2]].contiguous().cuda(), torch.tensor([1, 2, 3, 7, 8]).cuda(), torch.tensor([40, 20], dtype=torch.int32),
                 torch.tensor([3, 2], dtype=torch.int32))[1]
    assert torch.equal(dx[:, 0], ref[:, 0]) and torch.equal(dx[:, 2], ref[:, 1])


def test_empty_targets_and_zero_length_inputs():
    g = torch.Generator().manual_seed(14)
    x = torch.randn(30, 4, C, generator=g)
    targets = torch.tensor([4, 9], dtype=torch.int64)
    tn = torch.tensor([30, 0, 0, 17], dtype=torch.int32)
    ln = torch.tensor([0, 0, 2, 0], dtype=torch.int32)            # Ln = 0 twice, Tn = 0 with and without labels
    lf, df = _fused(x.cuda(), targets.cuda(), tn, ln)
    lr, dr = _ref(x, targets, tn, ln)
    assert lf.item() == pytest.approx(lr.item(), rel=1e-5)
    assert (df.cpu().double() - dr).abs().max().item() < 1e-5
    assert torch.all(df[:, 1] == 0) and torch.all(df[:, 2] == 0) and torch.all(df[17:, 3] == 0)
    lf0, df0 = _fused(x.cuda(), targets[:0].cuda(), tn, torch.zeros(4, dtype=torch.int32))   # no targets at all
    lr0, dr0 = _ref(x, targets[:0], tn, torch.zeros(4, dtype=torch.int32))
    assert lf0.item() == pytest.approx(lr0.item(), rel=1e-5) and (df0.cpu().double() - dr0).abs().max() < 1e-5


def test_loss_scale_and_fp16_overflow():
    x, targets, tn, ln = _batch(2, 100, seed=15)
    _, d1 = _fused(x.cuda(), targets.cuda(), tn, ln)
    _, d2 = _fused(x.cuda(), targets.cuda(), tn, ln, g=1024.0)
    assert torch.equal(d2, d1 * 1024)
    _, dh = _fused(x.half().cuda(), targets.cuda(), tn, ln, g=2.0 ** 17)
    assert torch.isinf(dh).any()
    assert not torch.isnan(dh).any()


def test_deterministic():
    x, targets, tn, ln = _batch(5, 198, seed=16)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        outs = [_fused(x.cuda(), targets.cuda(), tn.cuda(), ln.cuda()) for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(old)
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_no_host_synchronisation():
    x, targets, tn, ln = _batch(2, 198, seed=17)
    xs = x.cuda().requires_grad_(True)
    ts, tns, lns = targets.cuda(), tn.cuda(), ln.cuda()
    torch.cuda.synchronize()
    old = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = ctc_loss(xs, ts, tns, lns)
        (dx,) = torch.autograd.grad(loss, xs)
    finally:
        torch.cuda.set_sync_debug_mode(old)
    assert torch.isfinite(dx).all()


def test_graph_replay_on_new_logits_and_lengths():
    x, targets, tn, ln = _batch(2, 198, seed=17)
    xs = x.cuda().requires_grad_(True)
    ts, tns, lns = targets.cuda(), tn.cuda(), ln.cuda()

    def run():
        loss = ctc_loss(xs, ts, tns, lns)
        (dx,) = torch.autograd.grad(loss, xs)
        return loss, dx

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss_s, dx_s = run()
    # new logits and lengths (the same total of targets), copied into the static inputs
    x2 = _batch(2, 198, seed=18)[0]
    tn2 = torch.tensor([150, 198], dtype=torch.int32)
    k = int(ln.sum()) // 2
    ln2 = torch.tensor([int(ln.sum()) - k, k], dtype=torch.int32)
    with torch.no_grad():
        xs.copy_(x2)
    tns.copy_(tn2)
    lns.copy_(ln2)
    graph.replay()
    le, de = _fused(x2.cuda(), targets.cuda(), tn2, ln2)
    assert torch.equal(loss_s, le) and torch.equal(dx_s, de)


def _an4_loss(out, targets, out_lens, tsizes, kind):
    if kind == "fused":
        return ctc_loss(out.transpose(0, 1), targets, out_lens, tsizes) / out.size(0)
    if kind == "ref":
        return _ctc64(out.transpose(0, 1), targets, out_lens, tsizes) / out.size(0)
    return _stock(out.transpose(0, 1), targets, out_lens, tsizes) / out.size(0)


@pytest.mark.parametrize("fuse_lstm", [False, True])
def test_whole_model_against_float64(fuse_lstm):
    torch.manual_seed(0)
    net, _ = create_net(29, "lstman4")
    ref = copy.deepcopy(net).double()
    stock = net.cuda()
    fused = copy.deepcopy(stock)
    fused.fuse_ctc = True
    stock.fuse_lstm = fused.fuse_lstm = fuse_lstm
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 1, 161, 400, generator=g)
    lens = torch.tensor([400, 290], dtype=torch.int32)
    tsizes = torch.tensor([20, 14])
    targets = torch.randint(1, 29, (int(tsizes.sum()),), generator=g)
    res = {}
    for name, m, dev, dt in (("ref", ref, "cpu", torch.float64), ("stock", stock, "cuda", torch.float32),
                             ("fused", fused, "cuda", torch.float32)):
        m.train()
        n0 = _launches()
        out, out_lens = m(x.to(dev, dt), lens)
        loss = _an4_loss(out, targets.to(dev), out_lens, tsizes.to(dev), name)
        loss.backward()
        assert (_launches() != n0) == (name == "fused"), name
        res[name] = [loss.detach().cpu().double()] + [p.grad.detach().cpu().double() for p in m.parameters()]
    assert torch.isfinite(res["fused"][0])
    names = ["ctc"] + [n for n, _ in net.named_parameters()]
    for i, name in enumerate(names):
        r = res["ref"][i]
        es = (res["stock"][i] - r).abs().max().item()
        ef = (res["fused"][i] - r).abs().max().item()
        floor = 1e-5 * max(1.0, r.abs().max().item())
        assert ef <= 2 * es + floor, (name, ef, es, floor)


@pytest.mark.parametrize("precision", ["fp32", "bf16", "fp16"])
def test_trainer_steps_follow_stock(precision):
    """Five steps on the bench's AN4 batches with the fused LSTM on in both arms, stock loss against fused loss (fp16
    with dynamic loss scaling)."""
    import bench
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    autocast = None if precision == "fp32" else precision
    losses = {}
    for fuse in (False, True):
        cfg = okt.preset(preset, density=0.001, warmup_iters=2)
        tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                     t_total=100000, warmup=0.1, seed=0, autocast=autocast,
                     loss_scale=okt.LossScale() if precision == "fp16" else None,
                     model_kwargs={"fuse_lstm": True, "fuse_lstm_autocast": autocast is not None, "fuse_ctc": fuse})
        assert tr.net.fuse_ctc is fuse
        seq = []
        n0 = _launches()
        for i in range(5):
            batch = tuple(t.to(tr.device) for t in bench.make_batch("lstman4", i, 0, bs, 128))
            tr.net.train()
            tr.optimizer.zero_grad()
            loss, _ = tr._forward_loss(batch)
            tr.backward(loss)
            tr.update_model()
            seq.append(float(loss))
        n1 = _launches()
        assert (n1[0] - n0[0], n1[1] - n0[1]) == ((10, 5) if fuse else (0, 0))
        assert all(torch.isfinite(p).all() for p in tr.net.parameters())
        assert all(torch.isfinite(torch.tensor(seq)))
        tr.close()
        losses[fuse] = seq
    rel = 2e-2 if precision == "fp32" else 5e-2
    for a, b in zip(losses[False], losses[True]):
        assert b == pytest.approx(a, rel=rel), losses


@pytest.mark.parametrize("case", ["fp64", "wide_c", "many_targets", "padded_targets"])
def test_fallbacks_on_the_gpu_are_the_stock_expression(case):
    g = torch.Generator().manual_seed(19)
    T, N = 12, 3
    x = torch.randn(T, N, C, generator=g)
    tn = torch.tensor([12, 9, 5], dtype=torch.int32)
    ln = torch.tensor([4, 3, 2], dtype=torch.int32)
    t = torch.randint(1, C, (9,), generator=g)
    if case == "fp64":
        x = x.double()
    elif case == "wide_c":
        x = torch.randn(T, N, 200, generator=g)
    elif case == "many_targets":                              # 2048 targets, though each utterance's are feasible
        ln = torch.tensor([4, 3, 2041], dtype=torch.int32)
        tn = torch.tensor([12, 9, 12], dtype=torch.int32)
        t = torch.randint(1, C, (2048,), generator=g)
    else:
        t = torch.randint(1, C, (N, 4), generator=g)
    x, t = x.cuda(), t.cuda()
    outs = []
    for fused in (True, False):
        xi = x.clone().requires_grad_(True)
        n0 = _launches()
        loss = ctc_loss(xi, t, tn, ln) if fused else _stock(xi, t, tn, ln)
        loss.backward()
        assert _launches() == n0
        outs.append((loss.detach(), xi.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
