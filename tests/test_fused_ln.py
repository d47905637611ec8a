"""The fused dropout + residual add + LayerNorm kernels (csrc/layernorm.cu, ops/fused_ln.py): the Philox mask against a
numpy Philox4x32-10, fp32 against a float64 reference on off-centre and constant rows, 16-bit ``a`` bit for bit the fp32
kernel on ``a.float()``, mask statistics and determinism, stock parity, the fallbacks, activation recomputation and
whole-step CUDA graphs of a fused BERT."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

EPS = 1e-12                                           # BERT's layer_norm_eps


# ------------------------------------------------------------------------------------------ numpy Philox4x32-10
def philox4x32_10(ctr, key):
    """``ctr``: [n, 4] uint32 counters, ``key``: (k0, k1).  Returns [n, 4] uint32 words (Random123's round order)."""
    c = [ctr[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    m0, m1, mask = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0xFFFFFFFF)
    for r in range(10):
        if r > 0:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & mask, (k1 + np.uint64(0xBB67AE85)) & mask
        p0, p1 = m0 * c[0], m1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & mask]
    return np.stack(c, 1).astype(np.uint32)


def test_philox_reference_known_answers():
    z = philox4x32_10(np.zeros((1, 4), np.uint32), (0, 0))
    assert [int(v) for v in z[0]] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    o = philox4x32_10(np.full((1, 4), 0xFFFFFFFF, np.uint32), (0xFFFFFFFF, 0xFFFFFFFF))
    assert [int(v) for v in o[0]] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


def seed_of(s):
    """The seed the fused op draws as its first CUDA random call after ``torch.cuda.manual_seed(s)``."""
    torch.cuda.manual_seed(s)
    return int(torch.empty(1, dtype=torch.int64, device="cuda").random_().item())


def keep_mask(seed, R, H, p):
    from oktopk_b200.ops.fused_ln import keep_threshold
    n = R * H
    q = np.arange(n // 4, dtype=np.uint64)
    ctr = np.zeros((n // 4, 4), np.uint32)
    ctr[:, 0] = (q & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    ctr[:, 1] = (q >> np.uint64(32)).astype(np.uint32)
    u = seed & ((1 << 64) - 1)
    words = philox4x32_10(ctr, (u & 0xFFFFFFFF, u >> 32)).reshape(-1)
    return torch.from_numpy(words.astype(np.int64) < keep_threshold(p)).view(R, H).cuda()


# ------------------------------------------------------------------------------------------ helpers
def _ln(H, seed=0):
    torch.manual_seed(seed)
    ln = torch.nn.LayerNorm(H, eps=EPS).cuda()
    with torch.no_grad():
        ln.weight.normal_(1.0, 0.3)
        ln.bias.normal_(0.0, 0.5)
    return ln


def _inputs(R, H, seed, adtype=torch.float32, centre=0.0):
    g = torch.Generator("cuda").manual_seed(seed)
    x = torch.randn(R, H, device="cuda", generator=g) * 0.7 + centre
    a = (torch.randn(R, H, device="cuda", generator=g) * 0.9).to(adtype)
    dy = torch.randn(R, H, device="cuda", generator=g)
    return x, a, dy


def _fused(x, a, ln, dy, p, cuda_seed=None):
    from oktopk_b200.ops.fused_ln import residual_dropout_layer_norm
    if cuda_seed is not None:
        torch.cuda.manual_seed(cuda_seed)
    ln.zero_grad(set_to_none=True)
    xa = x.detach().clone().requires_grad_(True)
    aa = a.detach().clone().requires_grad_(True)
    y = residual_dropout_layer_norm(xa, aa, ln, p)
    y.backward(dy)
    return y.detach(), xa.grad, aa.grad, ln.weight.grad.clone(), ln.bias.grad.clone()


def _counts():
    from oktopk_b200.ops import ext
    return {k: ext.LAUNCH_COUNT.get(k, 0) for k in ("ln_forward", "ln_backward")}


def _delta(n0):
    return {k: v - n0[k] for k, v in _counts().items()}


def _close(got, want, tol):
    """max |got - want| within tol of the reference's largest magnitude (at least 1)."""
    err = float((got.double() - want).abs().max())
    assert err <= tol * max(1.0, float(want.abs().max())), err


# ------------------------------------------------------------------------------------------ 1. fp32 against float64
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("H", [128, 768, 1024])
@pytest.mark.parametrize("R", [1, 1024, 4096])
def test_fp32_matches_float64_reference(R, H, p):
    """Off-centre rows (mean 40, std ~1): a one-pass E[z^2] - E[z]^2 variance would lose most of its digits."""
    x, a, dy = _inputs(R, H, R + H, centre=40.0)
    ln = _ln(H, 1)
    s = 1000 + R + H
    n0 = _counts()
    y, dx, da, dg, db = _fused(x, a, ln, dy, p, cuda_seed=s)
    assert _delta(n0) == {"ln_forward": 1, "ln_backward": 2}
    keep = keep_mask(seed_of(s), R, H, p) if p > 0 else torch.ones(R, H, dtype=torch.bool, device="cuda")
    scale = 1.0 / (1.0 - p)
    assert torch.equal(da, dx * keep * scale)
    xd, ad = x.double().requires_grad_(True), a.double().requires_grad_(True)
    gd, bd = ln.weight.detach().double().requires_grad_(True), ln.bias.detach().double().requires_grad_(True)
    yd = F.layer_norm(xd + ad * keep * scale, (H,), gd, bd, EPS)
    yd.backward(dy.double())
    _close(y, yd.detach(), 2e-5)
    _close(dx, xd.grad, 2e-4)
    _close(da, ad.grad, 2e-4)
    _close(dg, gd.grad, 5e-4)
    _close(db, bd.grad, 5e-4)


def test_constant_row_is_kept_finite_by_eps():
    """var = 0 on a constant row: only eps keeps rstd finite (1e6 at eps 1e-12), y is beta there."""
    R, H = 8, 768
    x, a, dy = _inputs(R, H, 3)
    x[3] = 2.5
    a[3] = 0.0
    ln = _ln(H, 2)
    y, dx, da, dg, db = _fused(x, a, ln, dy, 0.0)
    for t in (y, dx, da, dg, db):
        assert torch.isfinite(t).all()
    torch.testing.assert_close(y[3], ln.bias.detach(), rtol=0, atol=1e-6)
    xd, ad = x.double().requires_grad_(True), a.double().requires_grad_(True)
    yd = F.layer_norm(xd + ad, (H,), ln.weight.detach().double(), ln.bias.detach().double(), EPS)
    yd.backward(dy.double())
    _close(dx, xd.grad, 2e-4)
    _close(y, yd.detach(), 2e-5)


# ------------------------------------------------------------------------------------------ 2. bf16 / fp16 a
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("R,H", [(1, 128), (1024, 768), (4096, 1024), (300, 384)])
def test_16bit_a_is_fp32_kernel_on_widened_a(R, H, dtype, p):
    x, a, dy = _inputs(R, H, 7 + H, dtype, centre=3.0)
    ln16, ln32 = _ln(H, 4), _ln(H, 4)
    y, dx, da, dg, db = _fused(x, a, ln16, dy, p, cuda_seed=77)
    y32, dx32, da32, dg32, db32 = _fused(x, a.float(), ln32, dy, p, cuda_seed=77)
    assert y.dtype == dx.dtype == dg.dtype == torch.float32 and da.dtype == dtype
    assert torch.equal(y, y32) and torch.equal(dx, dx32)
    assert torch.equal(dg, dg32) and torch.equal(db, db32)
    assert torch.equal(da, da32.to(dtype))


@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_non_finite_a_propagates_to_its_row(dtype, bad):
    R, H = 16, 768
    x, a, dy = _inputs(R, H, 5, dtype)
    a[5, 100] = bad
    y, *_ = _fused(x, a, _ln(H), dy, 0.1)
    assert torch.isnan(y[5]).all()
    assert torch.isfinite(torch.cat([y[:5], y[6:]])).all()


# ------------------------------------------------------------------------------------------ 3. statistics, determinism
def test_kept_fraction_and_fresh_masks():
    R, H, p = 1024, 768, 0.1                           # 786,432 elements
    x, a, dy = _inputs(R, H, 9)
    ln = _ln(H)
    _, dx1, da1, _, _ = _fused(x, a, ln, dy, p)
    _, dx2, da2, _, _ = _fused(x, a, ln, dy, p)
    assert (dx1 != 0).all() and (dx2 != 0).all()
    k1, k2 = da1 != 0, da2 != 0
    n = R * H
    sigma = (p * (1 - p) / n) ** 0.5
    for k in (k1, k2):
        assert abs(float(k.float().mean()) - (1 - p)) < 6 * sigma
    assert not torch.equal(k1, k2)                     # two calls draw two seeds
    assert float((k1 != k2).float().mean()) > 0.1      # independent masks differ in ~18% of the elements


def test_same_seed_is_bitwise_reproducible():
    x, a, dy = _inputs(4096, 1024, 13, torch.bfloat16)
    ln = _ln(1024)
    r1 = _fused(x, a, ln, dy, 0.1, cuda_seed=21)
    r2 = _fused(x, a, ln, dy, 0.1, cuda_seed=21)
    for u, v in zip(r1, r2):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------ 4. stock parity
def test_p0_matches_stock_layer_norm():
    x, a, dy = _inputs(2048, 768, 17)
    ln = _ln(768)
    y, dx, da, dg, db = _fused(x, a, ln, dy, 0.0)
    xs, as_ = x.clone().requires_grad_(True), a.clone().requires_grad_(True)
    ln.zero_grad(set_to_none=True)
    ys = F.layer_norm(xs + as_, (768,), ln.weight, ln.bias, EPS)
    ys.backward(dy)
    torch.testing.assert_close(y, ys, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(dx, xs.grad, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(da, as_.grad, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(dg, ln.weight.grad, rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(db, ln.bias.grad, rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_bert_layer_fused_matches_stock_under_autocast(dtype):
    from oktopk_b200.models.bert import BertConfig, BertLayer
    torch.manual_seed(0)
    cfg = BertConfig(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    a = BertLayer(cfg).cuda()
    b = copy.deepcopy(a)
    a.fuse_ln = True
    x = torch.randn(8, 128, 768, device="cuda")
    dy = torch.randn(8, 128, 768, device="cuda")
    outs = []
    for layer in (a, b):
        xi = x.clone().requires_grad_(True)
        n0 = _counts()
        with torch.autocast("cuda", dtype):
            y = layer(xi, None)
        y.backward(dy.to(y.dtype))
        outs.append((y.detach(), xi.grad, [q.grad for q in layer.parameters()], _delta(n0)))
    (ya, dxa, ga, na), (yb, dxb, gb, nb) = outs
    assert na == {"ln_forward": 2, "ln_backward": 4} and nb == {"ln_forward": 0, "ln_backward": 0}
    assert ya.dtype == yb.dtype == torch.float32
    tol = 3e-2 if dtype == torch.bfloat16 else 5e-3
    torch.testing.assert_close(ya, yb, rtol=tol, atol=tol)
    torch.testing.assert_close(dxa, dxb, rtol=tol, atol=tol)
    for (n, _), u, v in zip(a.named_parameters(), ga, gb):
        err = float((u.float() - v.float()).norm()) / (float(v.float().norm()) + 1e-6)
        assert err < 2 * tol, (n, err)


# ------------------------------------------------------------------------------------------ 5. fallbacks
@pytest.mark.parametrize("case", ["cpu", "h96", "h1152", "h_mismatch", "x_bf16", "a_fp64", "shape", "no_affine",
                                  "params_bf16"])
def test_fallbacks_run_the_stock_ops(case):
    from oktopk_b200.ops.fused_ln import residual_dropout_layer_norm
    R, H, p = 64, 768, 0.1
    x, a, dy = _inputs(R, H, 31)
    ln = _ln(H)
    autocast = None
    if case == "cpu":
        x, a, dy, ln = x.cpu(), a.cpu(), dy.cpu(), ln.cpu()
    elif case in ("h96", "h1152"):
        H = int(case[1:])
        x, a, dy = _inputs(R, H, 32)
        ln = _ln(H)
    elif case == "h_mismatch":                          # normalises over the last two dimensions
        x, a, dy = x.view(8, 8, H), a.view(8, 8, H), dy.view(8, 8, H)
        ln = torch.nn.LayerNorm((8, H), eps=EPS).cuda()
    elif case == "x_bf16":
        x = x.bfloat16()
    elif case == "a_fp64":
        x, a, dy, ln = x.double(), a.double(), dy.double(), ln.double()
    elif case == "shape":
        a = a[:1]                                       # broadcasts in the stock add
    elif case == "no_affine":
        ln = torch.nn.LayerNorm(H, eps=EPS, elementwise_affine=False).cuda()
    elif case == "params_bf16":                         # under autocast the stock layer_norm runs in fp32
        ln = ln.bfloat16()
        a = a.bfloat16()
        autocast = torch.bfloat16
    results = []
    n0 = _counts()
    for fused in (True, False):
        torch.manual_seed(3)
        xi, ai = x.clone().requires_grad_(True), a.clone().requires_grad_(True)
        with torch.autocast("cuda", autocast or torch.bfloat16, enabled=autocast is not None):
            y = residual_dropout_layer_norm(xi, ai, ln, p) if fused else ln(xi + F.dropout(ai, p, True))
        y.backward(dy.to(y.dtype).expand_as(y))
        results.append((y.detach(), xi.grad, ai.grad))
    assert _delta(n0) == {"ln_forward": 0, "ln_backward": 0}
    for u, v in zip(*results):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------ 6. recompute
def test_recompute_regenerates_the_same_masks():
    from oktopk_b200.models.bert import BertConfig, BertForPreTraining, synthetic_batch
    torch.manual_seed(0)
    cfg = BertConfig(num_hidden_layers=4)
    a = BertForPreTraining(cfg, depth=4, fuse_ln=True).cuda()
    b = copy.deepcopy(a)
    b.recompute = True
    batch = synthetic_batch(4, 128, device="cuda", generator=torch.Generator().manual_seed(1))
    counts = []
    for net in (a, b):
        net.train()
        n0 = _counts()
        torch.manual_seed(5)
        net(*batch).backward()
        counts.append(_delta(n0))
    # 4 layers x 2 sites forward; with recompute the two middle stages' layers run forward again in the backward pass
    assert counts == [{"ln_forward": 8, "ln_backward": 16}, {"ln_forward": 12, "ln_backward": 16}]
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        torch.testing.assert_close(pa.grad, pb.grad, rtol=1e-3, atol=1e-5, msg=n)


# ------------------------------------------------------------------------------------------ 7. CUDA graphs
def _trainer(cuda_graph, dropout, lr):
    import oktopk_b200 as okt
    from oktopk_b200.models.bert import BertConfig
    from oktopk_b200.train.trainer import Trainer
    cfg = BertConfig(num_hidden_layers=2, hidden_dropout_prob=dropout, attention_probs_dropout_prob=dropout)
    return Trainer(dnn="bert_base", dataset="wikipedia", batch_size=8, lr=lr, compressor="oktopk", density=0.001,
                   cfg=okt.preset("bert_base", density=0.001, warmup_iters=2), seed=0, seq_len=128,
                   cuda_graph=cuda_graph, model_kwargs={"config": cfg, "depth": 2, "fuse_ln": True})


def _bert_batches(n):
    from oktopk_b200.models.bert import synthetic_batch
    return [synthetic_batch(8, 128, device="cuda", generator=torch.Generator().manual_seed(40 + i)) for i in range(n)]


def test_graph_replays_draw_fresh_masks():
    """lr 0 keeps the parameters fixed: replays of one captured step on one batch differ only by their dropout masks."""
    tr = _trainer(True, 0.1, 0.0)
    assert tr.graphed is not None and tr.net.fuse_ln
    batch = _bert_batches(1)[0]
    n0 = _counts()
    losses = [float(tr.graphed.step(batch)) for _ in range(8)]
    torch.cuda.synchronize()
    assert tr.graphed.enabled and len(tr.graphed.graphs) >= 1, tr.graphed.why_disabled
    # 2 layers x 2 sites per step: the 3 eager warm-up steps and every capture launch them (replays are not counted)
    steps = 3 + len(tr.graphed.graphs)
    assert _delta(n0) == {"ln_forward": 4 * steps, "ln_backward": 8 * steps}
    assert all(np.isfinite(losses))
    assert losses[-1] != losses[-2], losses
    tr.close()


def test_graph_matches_eager_without_dropout():
    tg, te = _trainer(True, 0.0, 1e-4), _trainer(False, 0.0, 1e-4)
    for u, v in zip(tg.net.parameters(), te.net.parameters()):
        assert torch.equal(u, v)
    batches = _bert_batches(3)
    lg, le = [], []
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
    assert lg == pytest.approx(le, rel=1e-3, abs=1e-3), (lg, le)
    pa = torch.cat([p.detach().flatten() for p in tg.net.parameters()])
    pb = torch.cat([p.detach().flatten() for p in te.net.parameters()])
    assert float((pa - pb).norm()) / float(pb.norm()) < 1e-3
    tg.close()
    te.close()
