"""The fused softmax cross-entropy (csrc/xent.cu, ops/fused_xent.py): loss and gradient against a float64 reference in
fp32, bf16 and fp16 over aligned and misaligned rows and labelled fractions 1, ~0.11 and 0; loss scales including an
fp16 overflow; non-finite logits, out-of-range targets and NaN in ignored rows; determinism and CUDA-graph replay; the
launch counts; the fallbacks; and BERT pre-training under autocast, recompute, loss scaling and whole-step graphs."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

IGN = -1                                              # BERT's ignore_index
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


# ------------------------------------------------------------------------------------------ helpers
def _inputs(R, V, frac_ignored, dtype, seed):
    """Logits with per-row offsets (so the max matters), targets with ~frac_ignored rows ignored (row 0 is labelled
    unless every row is ignored)."""
    g = torch.Generator("cuda").manual_seed(seed)
    x = (torch.randn(R, V, device="cuda", generator=g) * 3 + torch.randn(R, 1, device="cuda", generator=g) * 20)
    t = torch.randint(0, V, (R,), device="cuda", generator=g)
    if frac_ignored >= 1:
        t.fill_(IGN)
    elif frac_ignored > 0:
        ign = torch.rand(R, device="cuda", generator=g) < frac_ignored
        ign[0] = False
        t[ign] = IGN
    return x.to(dtype), t


def _fused(x, t, g=1.0):
    from oktopk_b200.ops.fused_xent import softmax_cross_entropy
    xi = x.detach().clone().requires_grad_(True)
    loss = softmax_cross_entropy(xi, t, ignore_index=IGN)
    loss.backward(torch.tensor(g, device="cuda"))
    return loss.detach(), xi.grad


def _reference(x, t, g=1.0):
    """float64 loss and gradient of the widened logits; ignored rows are never read (their gradient is 0)."""
    xd = x.double()
    lab = t != IGN
    n = int(lab.sum())
    lse = torch.logsumexp(xd, 1)
    tc = t.clamp(0, x.size(1) - 1)
    rowloss = lse - xd.gather(1, tc[:, None])[:, 0]
    loss = rowloss[lab].sum() / n if n else torch.tensor(float("nan"), dtype=torch.float64, device=x.device)
    grad = torch.softmax(xd, 1)
    grad[torch.arange(len(t), device=x.device), tc] -= 1
    grad = torch.where(lab[:, None], grad * (g / max(n, 1)), torch.zeros_like(grad))
    return loss, grad


def _ulps(a, b):
    """Element-wise distance in units in the last place between two tensors of one 16-bit type (inf counts as a value)."""
    def key(v):
        i = v.view(torch.int16).int()
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return (key(a) - key(b)).abs()


def _check_grad(got, want64, dtype, g, n, t):
    """fp32: within 2e-5 of each element (the rounding of the saved fp32 log-sum-exp, ~|lse| 2^-24, dominates), and of
    g / n at the target, where p - 1 cancels.  16-bit: within 1 ulp of the float64 gradient rounded to the dtype."""
    if dtype == torch.float32:
        tol = 2e-5 * want64.abs()
        rows = torch.nonzero(t != IGN)[:, 0]
        tol[rows, t[rows]] = 2e-5 * abs(g) / n
        assert bool(((got.double() - want64).abs() <= tol).all()), float(((got.double() - want64).abs() - tol).max())
    else:
        assert int(_ulps(got, want64.to(dtype)).max()) <= 1


def _counts():
    from oktopk_b200.ops import ext
    return {k: ext.LAUNCH_COUNT.get(k, 0) for k in ("xent_forward", "xent_backward")}


def _delta(n0):
    return {k: v - n0[k] for k, v in _counts().items()}


# ------------------------------------------------------------------------------------------ 1. float64 reference
SHAPES = [(1, 1), (1, 2), (7, 10), (300, 10000), (1024, 30522), (64, 50257)]


@pytest.mark.parametrize("frac", [0.0, 0.89, 1.0])
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_matches_float64_reference(dtype, shape, frac):
    R, V = shape
    x, t = _inputs(R, V, frac, dtype, seed=R + V)
    g = 0.75
    n0 = _counts()
    loss, grad = _fused(x, t, g)
    assert _delta(n0) == {"xent_forward": 2, "xent_backward": 1}
    want_loss, want_grad = _reference(x, t, g)
    n = int((t != IGN).sum())
    assert loss.dtype == torch.float32 and loss.dim() == 0 and grad.dtype == dtype
    if n == 0:
        assert torch.isnan(loss) and torch.count_nonzero(grad) == 0
        return
    assert abs(float(loss) - float(want_loss)) <= 1e-5 * max(1.0, abs(float(want_loss))), (float(loss), float(want_loss))
    _check_grad(grad, want_grad, dtype, g, n, t)
    assert torch.count_nonzero(grad[t == IGN]) == 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_matches_stock_cross_entropy(dtype):
    """Against F.cross_entropy with autocast's dtype handling (fp32 math, the gradient narrowed to the logits' type)."""
    x, t = _inputs(1024, 30522, 0.89, dtype, seed=1)
    loss, grad = _fused(x, t)
    xs = x.clone().requires_grad_(True)
    ref = F.cross_entropy(xs.float(), t, ignore_index=IGN)
    ref.backward()
    torch.testing.assert_close(loss, ref, rtol=1e-5, atol=0)
    if dtype == torch.float32:
        torch.testing.assert_close(grad, xs.grad, rtol=1e-4, atol=1e-9)
    else:
        assert int(_ulps(grad, xs.grad).max()) <= 1


def test_misaligned_and_non_contiguous_logits():
    """Logits that start off a 16-byte boundary or are a transposed view are copied once and give the same results."""
    x, t = _inputs(33, 1001, 0.5, torch.bfloat16, seed=2)
    want = _fused(x, t, 2.0)
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device="cuda")
    off = buf[1:].view(33, 1001)
    off.copy_(x)
    assert off.data_ptr() % 16 != 0
    for v in (off, x.t().contiguous().t()):
        got = _fused(v, t, 2.0)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


# ------------------------------------------------------------------------------------------ 2. edge cases
def test_fp16_loss_scale_overflows_to_inf():
    """g = 65536 on one labelled row: the dominant non-target logit's gradient p · 65536 rounds past 65504 to inf."""
    x = torch.full((4, 37), -3.0, device="cuda")
    x[1, 5] = 12.0
    t = torch.tensor([IGN, 9, IGN, IGN], device="cuda")
    xh = x.half()
    loss, grad = _fused(xh, t, 65536.0)
    _, want = _reference(xh, t, 65536.0)
    assert torch.isinf(grad[1, 5]) and grad[1, 5] > 0
    assert torch.equal(torch.isinf(grad), torch.isinf(want.half()))
    assert int(_ulps(grad, want.half()).max()) <= 1
    assert torch.isfinite(loss)


@pytest.mark.parametrize("dtype", DTYPES)
def test_non_finite_logits_in_labelled_rows(dtype):
    x, t = _inputs(8, 333, 0.0, dtype, seed=3)
    x[2, 7] = float("nan")
    x[3, 100] = float("inf")
    x[4, 11] = float("-inf")                          # isolated -inf: contributes exp = 0
    x[4, 200] = float("-inf")
    t[4] = 5
    loss, grad = _fused(x, t)
    assert torch.isnan(loss)
    assert torch.isnan(grad[2]).all() and torch.isnan(grad[3]).all()
    ok = torch.tensor([0, 1, 4, 5, 6, 7], device="cuda")
    assert torch.isfinite(grad[ok]).all()
    assert float(grad[4, 11]) == 0.0 and float(grad[4, 200]) == 0.0
    # the finite rows match the reference over the same n
    _, want = _reference(x[ok], t[ok], 6 / 8)
    _check_grad(grad[ok], want, dtype, 6 / 8, 6, t[ok])
    # -inf alone: a finite loss matching float64
    x2, t2 = _inputs(4, 333, 0.0, dtype, seed=4)
    x2[:, ::7] = float("-inf")
    t2[:] = 1
    l2, g2 = _fused(x2, t2)
    wl, wg = _reference(x2, t2)
    assert torch.isfinite(l2) and abs(float(l2) - float(wl)) <= 1e-5 * max(1.0, abs(float(wl)))
    assert torch.count_nonzero(g2[:, ::7]) == 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_out_of_range_target_gives_nan_without_trapping(dtype):
    """Fused path only: torch's own kernel device-asserts on these targets."""
    x, t = _inputs(6, 129, 0.0, dtype, seed=5)
    t[1], t[4] = 129, -5
    t[5] = IGN
    loss, grad = _fused(x, t)
    torch.cuda.synchronize()
    assert torch.isnan(loss)
    assert torch.isnan(grad[1]).all() and torch.isnan(grad[4]).all()
    assert torch.count_nonzero(grad[5]) == 0
    ok = torch.tensor([0, 2, 3], device="cuda")
    _, want = _reference(x[ok], t[ok], 3 / 5)          # n counts the bad rows: 5 rows are not ignored
    _check_grad(grad[ok], want, dtype, 3 / 5, 3, t[ok])


@pytest.mark.parametrize("dtype", DTYPES)
def test_nan_in_ignored_row_gives_zero_gradient(dtype):
    """Deliberately unlike stock, whose log_softmax backward turns such a row into NaN: an ignored row is never read."""
    x, t = _inputs(5, 1000, 0.0, dtype, seed=6)
    t[2] = IGN
    x[2, :] = float("nan")
    x[2, 3] = float("inf")
    loss, grad = _fused(x, t)
    keep = t != IGN
    want_loss, want = _reference(x[keep], t[keep])
    assert abs(float(loss) - float(want_loss)) <= 1e-5 * max(1.0, abs(float(want_loss)))
    assert torch.count_nonzero(grad[2]) == 0 and torch.isfinite(grad).all()
    _check_grad(grad[keep], want, dtype, 1.0, 4, t[keep])


# ------------------------------------------------------------------------------------------ 3. determinism, graphs
@pytest.mark.parametrize("dtype", DTYPES)
def test_bitwise_deterministic(dtype):
    x, t = _inputs(1024, 30522, 0.89, dtype, seed=7)
    a, b = _fused(x, t), _fused(x, t)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_cuda_graph_replays_bitwise_equal_to_eager(dtype):
    from oktopk_b200.ops.fused_xent import softmax_cross_entropy
    x, t = _inputs(1024, 30522, 0.89, dtype, seed=8)
    xs = x.clone().requires_grad_(True)
    scale = torch.tensor(3.0, device="cuda")

    def step():
        loss = softmax_cross_entropy(xs, t, ignore_index=IGN)
        (gx,) = torch.autograd.grad(loss * scale, xs)
        return loss, gx

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gl, gg = step()
    for seed, sc in ((9, 3.0), (10, 0.5)):            # new inputs and a new scale, written in place
        x2, t2 = _inputs(1024, 30522, 0.89, dtype, seed=seed)
        with torch.no_grad():
            xs.copy_(x2)
        t.copy_(t2)
        scale.fill_(sc)
        graph.replay()
        torch.cuda.synchronize()
        el, eg = _fused(x2, t2, sc)
        assert torch.equal(gl, el) and torch.equal(gg, eg)


# ------------------------------------------------------------------------------------------ 4. fallbacks
@pytest.mark.parametrize("case", ["cpu", "3d", "fp64", "no_rows"])
def test_fallbacks_run_stock_cross_entropy(case):
    from oktopk_b200.ops.fused_xent import softmax_cross_entropy
    x, t = _inputs(16, 50, 0.5, torch.float32, seed=11)
    if case == "cpu":
        x, t = x.cpu(), t.cpu()
    elif case == "3d":
        x, t = x.view(4, 4, 50).transpose(1, 2), t.view(4, 4)
    elif case == "fp64":
        x = x.double()
    elif case == "no_rows":
        x, t = x[:0], t[:0]
    n0 = _counts()
    outs = []
    for fused in (True, False):
        xi = x.clone().requires_grad_(True)
        loss = softmax_cross_entropy(xi, t, ignore_index=IGN) if fused else F.cross_entropy(xi, t, ignore_index=IGN)
        loss.backward()
        outs.append((loss.detach(), xi.grad))
    assert _delta(n0) == {"xent_forward": 0, "xent_backward": 0}
    (la, ga), (lb, gb) = outs
    assert torch.equal(la, lb) or (la.isnan() and lb.isnan())
    assert torch.equal(ga, gb)


# ------------------------------------------------------------------------------------------ 5. BERT
def _bert(**kw):
    from oktopk_b200.models.bert import BertConfig, BertForPreTraining
    torch.manual_seed(0)
    cfg = BertConfig(num_hidden_layers=4, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    return BertForPreTraining(cfg, depth=4, **kw).cuda()


def _batch(seed=1):
    from oktopk_b200.models.bert import synthetic_batch
    return synthetic_batch(8, 128, device="cuda", generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_bert_pretraining_fused_matches_stock_under_autocast(dtype):
    a = _bert()
    b = copy.deepcopy(a)
    a.fuse_xent = True
    batch = _batch()
    res = []
    for net in (a, b):
        n0 = _counts()
        with torch.autocast("cuda", dtype):
            loss = net(*batch)
        loss.backward()
        res.append((float(loss.detach()), [p.grad for p in net.parameters()], _delta(n0)))
    (la, ga, na), (lb, gb, nb) = res
    assert na == {"xent_forward": 2, "xent_backward": 1} and nb == {"xent_forward": 0, "xent_backward": 0}
    # stock cross_entropy under autocast differs from fp32 cross_entropy on the same 16-bit logits by ~1e-4 relative;
    # the fused loss is the latter
    assert la == pytest.approx(lb, rel=1e-3)
    for (n, _), u, v in zip(a.named_parameters(), ga, gb):
        err = float((u.float() - v.float()).norm()) / (float(v.float().norm()) + 1e-12)
        assert err < 2e-2, (n, err)


def test_bert_recompute_with_fused_loss():
    a = _bert(fuse_xent=True, fuse_ln=True)
    b = copy.deepcopy(a)
    b.recompute = True
    batch = _batch(2)
    for net in (a, b):
        net.train()
        net(*batch).backward()
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        torch.testing.assert_close(pa.grad, pb.grad, rtol=1e-3, atol=1e-5, msg=n)


def _trainer(cuda_graph, fuse_ln, **kw):
    import oktopk_b200 as okt
    from oktopk_b200.models.bert import BertConfig
    from oktopk_b200.train.trainer import Trainer
    cfg = BertConfig(num_hidden_layers=2, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    return Trainer(dnn="bert_base", dataset="wikipedia", batch_size=8, lr=1e-4, compressor="oktopk", density=0.001,
                   cfg=okt.preset("bert_base", density=0.001, warmup_iters=2), seed=0, seq_len=128,
                   cuda_graph=cuda_graph, model_kwargs={"config": cfg, "depth": 2, "fuse_ln": fuse_ln,
                                                        "fuse_xent": True}, **kw)


def _bert_batches(n):
    return [_batch(40 + i) for i in range(n)]


@pytest.mark.parametrize("fuse_ln", [False, True])
def test_graphed_trainer_matches_eager(fuse_ln):
    tg, te = _trainer(True, fuse_ln), _trainer(False, fuse_ln)
    assert tg.graphed is not None and tg.net.fuse_xent and tg.net.fuse_ln == fuse_ln
    batches = _bert_batches(3)
    lg, le = [], []
    n0 = _counts()
    for it in range(8):
        b = batches[it % len(batches)]
        lg.append(float(tg.graphed.step(b)))
        te.optimizer.zero_grad()
        loss, _ = te._forward_loss(b)
        loss.backward()
        te.update_model()
        le.append(float(loss.detach()))
    torch.cuda.synchronize()
    assert tg.graphed.enabled and len(tg.graphed.graphs) >= 1, tg.graphed.why_disabled
    assert _delta(n0)["xent_forward"] >= 2 * 8
    assert lg == pytest.approx(le, rel=1e-3, abs=1e-3), (lg, le)
    pa = torch.cat([p.detach().flatten() for p in tg.net.parameters()])
    pb = torch.cat([p.detach().flatten() for p in te.net.parameters()])
    assert float((pa - pb).norm()) / float(pb.norm()) < 1e-3
    tg.close()
    te.close()


def test_graphed_fp16_loss_scaled_trainer_runs():
    from oktopk_b200.config import LossScale
    tr = _trainer(True, True, autocast="fp16", loss_scale=LossScale())
    batches = _bert_batches(3)
    losses = [float(tr.graphed.step(batches[i % 3])) for i in range(10)]
    torch.cuda.synchronize()
    assert tr.graphed.enabled and len(tr.graphed.graphs) >= 1, tr.graphed.why_disabled
    assert np.isfinite(losses).all(), losses
    assert all(torch.isfinite(p).all() for p in tr.net.parameters())
    tr.close()
