"""The fused embedding sum + LayerNorm + dropout kernels (csrc/embedding.cu, ops/fused_emb.py): y and every gradient
against a float64 reference on constant and off-centre rows and four id patterns, untouched table rows exactly 0, the
Philox mask against a numpy Philox4x32-10, mask statistics and bitwise determinism, stock parity, autocast, the
fallbacks, out-of-range ids, and whole-step CUDA graphs of a fused BERT."""
import copy
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_fused_ln import keep_mask, seed_of  # noqa: E402  (numpy Philox4x32-10 mask, the op's seed)

pytestmark = pytest.mark.gpu

EPS = 1e-12
VOCAB = 30522
LAUNCHES = ("emb_forward", "emb_backward")


def _emb(H, vocab=VOCAB, max_pos=512, types=2, seed=0):
    from oktopk_b200.models.bert import BertConfig, BertEmbeddings
    torch.manual_seed(seed)
    cfg = BertConfig(vocab_size=vocab, hidden_size=H, max_position_embeddings=max_pos, type_vocab_size=types)
    emb = BertEmbeddings(cfg).cuda()
    with torch.no_grad():
        for e in (emb.word_embeddings, emb.position_embeddings, emb.token_type_embeddings):
            e.weight.normal_(0.0, 0.5)
        emb.LayerNorm.weight.normal_(1.0, 0.3)
        emb.LayerNorm.bias.normal_(0.0, 0.5)
    return emb


def _ids(pattern, B, S, vocab=VOCAB, seed=0):
    g = torch.Generator().manual_seed(seed)
    R = B * S
    if pattern == "same":
        ids = torch.full((R,), 4242)
    elif pattern == "distinct":
        ids = torch.randperm(vocab, generator=g)[:R]
    elif pattern == "ends":                                # only the first and the last row of the table
        ids = torch.where(torch.rand(R, generator=g) < 0.5, 0, vocab - 1)
    else:                                                  # heavy duplicates: 7 ids, one of them most of the tokens
        ids = torch.tensor([100, 103, 0, 7, vocab - 523, 512, 1234 % vocab])[
            torch.randint(0, 7, (R,), generator=g) * (torch.rand(R, generator=g) < 0.5)]
    tt = torch.randint(0, 2, (R,), generator=g)
    return ids.view(B, S).cuda(), tt.view(B, S).cuda()


def _counts():
    from oktopk_b200.ops import ext
    return {k: ext.LAUNCH_COUNT.get(k, 0) for k in LAUNCHES}


def _delta(n0):
    return {k: v - n0[k] for k, v in _counts().items()}


def _fused(emb, ids, tt, dy, p, cuda_seed=None):
    from oktopk_b200.ops.fused_emb import embedding_layer_norm
    if cuda_seed is not None:
        torch.cuda.manual_seed(cuda_seed)
    emb.zero_grad(set_to_none=True)
    y = embedding_layer_norm(ids, tt, emb, p)
    y.backward(dy)
    return [y.detach()] + [q.grad.clone() for q in _params(emb)]


def _params(emb):
    return [emb.word_embeddings.weight, emb.position_embeddings.weight, emb.token_type_embeddings.weight,
            emb.LayerNorm.weight, emb.LayerNorm.bias]


def _reference(emb, ids, tt, dy, keep, scale):
    """float64 y and gradients from the fp32 stock-order sum; out-of-range ids and types contribute 0."""
    W, P, T = (q.detach() for q in _params(emb)[:3])
    gam, bet = emb.LayerNorm.weight.detach().double(), emb.LayerNorm.bias.detach().double()
    B, S = ids.shape
    H = W.size(1)
    i, t = ids.reshape(-1), tt.reshape(-1)
    iok, tok = (i >= 0) & (i < W.size(0)), (t >= 0) & (t < T.size(0))
    wi, ti = torch.where(iok, i, 0), torch.where(tok, t, 0)
    s = torch.arange(S, device=ids.device).repeat(B)
    e = (W[wi] * iok[:, None] + P[s]) + T[ti] * tok[:, None]           # fp32, the stock order
    ed = e.double().requires_grad_(True)
    gd, bd = gam.clone().requires_grad_(True), bet.clone().requires_grad_(True)
    yd = F.layer_norm(ed, (H,), gd, bd, EPS) * keep.view(-1, H).double() * scale
    yd.backward(dy.reshape(-1, H).double())
    de = ed.grad
    dw = torch.zeros(W.shape, dtype=torch.float64, device=W.device).index_add_(0, wi[iok], de[iok])
    dp = torch.zeros(P.shape, dtype=torch.float64, device=W.device).index_add_(0, s, de)
    dt = torch.zeros(T.shape, dtype=torch.float64, device=W.device).index_add_(0, ti[tok], de[tok])
    return [yd.detach().view(B, S, H), dw, dp, dt, gd.grad, bd.grad]


def _close_rows(got, want, tol):
    """Every row (a vector: the whole of it) within tol of its largest reference magnitude (at least 1)."""
    g, w = got.double().reshape(-1, got.size(-1)), want.reshape(-1, want.size(-1))
    err = (g - w).abs().amax(1)
    lim = tol * w.abs().amax(1).clamp_min(1.0)
    assert bool((err <= lim).all()), float((err / lim).max())


TOL = (2e-5, 5e-4, 5e-4, 5e-4, 5e-4, 5e-4)                # y, dword, dpos, dtype, dgamma, dbeta


# ------------------------------------------------------------------------------------------ 1. against float64
@pytest.mark.parametrize("pattern", ["same", "distinct", "ends", "dups"])
@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("S", [1, 128, 512])
@pytest.mark.parametrize("H", [768, 1024])
def test_matches_float64_reference(H, S, B, pattern):
    """Token (0, 0) sums three constant rows (variance 0: only eps keeps rstd finite); type 0 is off-centre (+40)."""
    emb = _emb(H, seed=H + S)
    ids, tt = _ids(pattern, B, S, seed=S + B)
    tt[0, 0] = 1
    with torch.no_grad():
        emb.word_embeddings.weight[ids[0, 0]] = 2.5
        emb.position_embeddings.weight[0] = 0.5
        emb.token_type_embeddings.weight[1] = 0.25
        emb.token_type_embeddings.weight[0] += 40.0
    dy = torch.randn(B, S, H, device="cuda", generator=torch.Generator("cuda").manual_seed(5))
    p, s = 0.1, 100 + H + S + B
    n0 = _counts()
    got = _fused(emb, ids, tt, dy, p, cuda_seed=s)
    assert _delta(n0) == {"emb_forward": 1, "emb_backward": 3}
    keep = keep_mask(seed_of(s), B * S, H, p)
    want = _reference(emb, ids, tt, dy, keep, 1.0 / (1.0 - p))
    assert torch.equal(got[0][0, 0], emb.LayerNorm.bias.detach() * keep[0] * (1.0 / (1.0 - p)))   # y = beta there
    for u, v, tol in zip(got, want, TOL):
        assert torch.isfinite(u).all()
        _close_rows(u, v, tol)
    # rows no token touches are exactly 0
    used = torch.zeros(VOCAB, dtype=torch.bool, device="cuda")
    used[ids.reshape(-1)] = True
    assert bool((got[1][~used] == 0).all())
    assert bool((got[2][S:] == 0).all())


# ------------------------------------------------------------------------------------------ 2. mask, statistics
def test_mask_matches_numpy_philox():
    H, B, S, p = 768, 4, 128, 0.1
    emb = _emb(H)
    ids, tt = _ids("distinct", B, S)
    dy = torch.randn(B, S, H, device="cuda")
    y0 = _fused(emb, ids, tt, dy, 0.0)[0]
    yp = _fused(emb, ids, tt, dy, p, cuda_seed=11)[0]
    keep = keep_mask(seed_of(11), B * S, H, p).view(B, S, H)
    assert torch.equal(yp, y0 * keep * (1.0 / (1.0 - p)))


def test_keep_rate_fresh_masks_and_bitwise_determinism():
    H, B, S, p = 768, 8, 128, 0.1                         # 786,432 elements
    emb = _emb(H)
    ids, tt = _ids("dups", B, S)
    dy = torch.randn(B, S, H, device="cuda")
    y1 = _fused(emb, ids, tt, dy, p)[0]
    y2 = _fused(emb, ids, tt, dy, p)[0]
    n = y1.numel()
    sigma = (p * (1 - p) / n) ** 0.5
    for y in (y1, y2):
        assert abs(float((y != 0).float().mean()) - (1 - p)) < 6 * sigma
    assert float(((y1 != 0) != (y2 != 0)).float().mean()) > 0.1
    r1 = _fused(emb, ids, tt, dy, p, cuda_seed=21)
    r2 = _fused(emb, ids, tt, dy, p, cuda_seed=21)
    for u, v in zip(r1, r2):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------ 3. stock parity
@pytest.mark.parametrize("B,S,H", [(8, 128, 768), (2, 512, 1024)])
def test_p0_matches_stock(B, S, H):
    emb = _emb(H)
    ids, tt = _ids("dups", B, S)
    dy = torch.randn(B, S, H, device="cuda")
    got = _fused(emb, ids, tt, dy, 0.0)
    emb.zero_grad(set_to_none=True)
    emb.eval()
    y = emb(ids, tt)
    y.backward(dy)
    want = [y.detach()] + [q.grad for q in _params(emb)]
    tols = (1e-5, 1e-4, 1e-4, 1e-4, 1e-4, 1e-4)
    for u, v, tol in zip(got, want, tols):
        err = float((u - v).abs().max())
        assert err <= tol * max(1.0, float(v.abs().max())), err


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_autocast_runs_the_fp32_op(dtype):
    B, S, H = 8, 128, 768
    emb = _emb(H)
    ids, tt = _ids("dups", B, S)
    dy = torch.randn(B, S, H, device="cuda")
    ref = _fused(emb, ids, tt, dy, 0.1, cuda_seed=3)
    with torch.autocast("cuda", dtype):
        got = _fused(emb, ids, tt, dy, 0.1, cuda_seed=3)
        emb.eval()
        stock = emb(ids, tt)
        emb.train()
    assert got[0].dtype == stock.dtype == torch.float32
    for u, v in zip(got, ref):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------ 4. fallbacks
@pytest.mark.parametrize("case", ["cpu", "h96", "h1152", "bf16", "sparse", "padding_idx", "max_norm",
                                  "scale_grad_by_freq", "tokens_4608"])
def test_fallbacks_run_the_stock_ops(case):
    from oktopk_b200.ops.fused_emb import embedding_layer_norm
    B, S, H, p = 4, 64, 768, 0.1
    emb = _emb(H, vocab=1000)
    ids, tt = _ids("dups", B, S, vocab=1000)
    if case == "cpu":
        emb, ids, tt = emb.cpu(), ids.cpu(), tt.cpu()
    elif case in ("h96", "h1152"):
        emb = _emb(int(case[1:]), vocab=1000)
    elif case == "bf16":
        emb = emb.bfloat16()
    elif case == "sparse":
        emb.word_embeddings.sparse = True
    elif case == "padding_idx":
        emb.word_embeddings.padding_idx = 0
    elif case == "max_norm":
        emb.word_embeddings.max_norm = 1.0
    elif case == "scale_grad_by_freq":
        emb.token_type_embeddings.scale_grad_by_freq = True
    elif case == "tokens_4608":
        ids, tt = _ids("dups", 9, 512, vocab=1000)
    results = []
    n0 = _counts()
    for fused in (True, False):
        e = copy.deepcopy(emb)                           # max_norm renormalises the table in place
        torch.manual_seed(3)
        y = embedding_layer_norm(ids, tt, e, p) if fused else e.train()(ids, tt)
        y.float().sum().backward()
        grads = [q.grad.to_dense() if q.grad.is_sparse else q.grad for q in _params(e)]
        results.append([y.detach()] + grads)
    assert _delta(n0) == {"emb_forward": 0, "emb_backward": 0}
    assert torch.equal(results[0][0], results[1][0])
    # stock embedding_dense_backward adds duplicate rows with atomics: its gradients differ run to run in the last bits
    for u, v in zip(results[0][1:], results[1][1:]):
        torch.testing.assert_close(u, v, rtol=1e-5, atol=1e-4)


# ------------------------------------------------------------------------------------------ 5. out-of-range ids
def test_out_of_range_ids_are_counted_and_contribute_zero():
    B, S, H, V = 4, 128, 768, 1000
    emb = _emb(H, vocab=V)
    ids, tt = _ids("distinct", B, S, vocab=V)
    bad_ids = {(0, 3): -1, (1, 5): V, (2, 7): V + 5, (3, 127): -(2 ** 40)}
    bad_tt = {(0, 3): 2, (1, 9): -3}
    for (b, s), v in bad_ids.items():
        ids[b, s] = v
    for (b, s), v in bad_tt.items():
        tt[b, s] = v
    dy = torch.randn(B, S, H, device="cuda")
    emb.id_overflow.zero_()
    got = _fused(emb, ids, tt, dy, 0.0)
    torch.cuda.synchronize()
    assert int(emb.id_overflow) == len(bad_ids) + len(bad_tt)
    want = _reference(emb, ids, tt, dy, torch.ones(B * S, H, dtype=torch.bool, device="cuda"), 1.0)
    for u, v, tol in zip(got, want, TOL):
        assert torch.isfinite(u).all()
        _close_rows(u, v, tol)
    # a good token's y does not depend on the other tokens' ids
    ok_ids, ok_tt = ids.clamp(0, V - 1), tt.clamp(0, 1)
    y_ok = _fused(emb, ok_ids, ok_tt, dy, 0.0)[0]
    good = torch.ones(B, S, dtype=torch.bool, device="cuda")
    for b, s in list(bad_ids) + list(bad_tt):
        good[b, s] = False
    assert torch.equal(got[0][good], y_ok[good])
    assert int(emb.id_overflow) == len(bad_ids) + len(bad_tt)


# ------------------------------------------------------------------------------------------ 6. CUDA graphs
def _trainer(cuda_graph, dropout, lr, fuse_emb=True):
    import oktopk_b200 as okt
    from oktopk_b200.models.bert import BertConfig
    from oktopk_b200.train.trainer import Trainer
    cfg = BertConfig(num_hidden_layers=2, hidden_dropout_prob=dropout, attention_probs_dropout_prob=dropout)
    return Trainer(dnn="bert_base", dataset="wikipedia", batch_size=8, lr=lr, compressor="oktopk", density=0.001,
                   cfg=okt.preset("bert_base", density=0.001, warmup_iters=2), seed=0, seq_len=128,
                   cuda_graph=cuda_graph, model_kwargs={"config": cfg, "depth": 2, "fuse_emb": fuse_emb})


def _bert_batches(n):
    from oktopk_b200.models.bert import synthetic_batch
    return [synthetic_batch(8, 128, device="cuda", generator=torch.Generator().manual_seed(40 + i)) for i in range(n)]


def test_graph_replays_draw_fresh_masks():
    """lr 0 keeps the parameters fixed: replays of one captured step on one batch differ only by their dropout masks."""
    tr = _trainer(True, 0.1, 0.0)
    assert tr.graphed is not None and tr.net.fuse_emb
    batch = _bert_batches(1)[0]
    n0 = _counts()
    losses = [float(tr.graphed.step(batch)) for _ in range(8)]
    torch.cuda.synchronize()
    assert tr.graphed.enabled and len(tr.graphed.graphs) >= 1, tr.graphed.why_disabled
    assert _delta(n0)["emb_forward"] >= 1
    assert all(np.isfinite(losses))
    assert losses[-1] != losses[-2], losses
    tr.close()


def test_graph_fused_matches_eager_stock_without_dropout():
    tg, te = _trainer(True, 0.0, 1e-4), _trainer(False, 0.0, 1e-4, fuse_emb=False)
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
    assert int(tg.net.stages[0].embeddings.id_overflow) == 0
    tg.close()
    te.close()
