"""The fixed-capacity gather of BERT's labelled masked-LM rows (csrc/mlm_gather.cu, ops/mlm_gather.py) on the GPU: the
select, gather and scatter kernels bit for bit against the torch implementation in fp32, bf16 and fp16, for R from 1 to
32768 and H in {768, 1024, 100} (100 takes the scalar path), with overflow and its accumulation; the scatter writing
every row; launch counts and CUDA-graph capture; BERT pre-training with the sparse head against the stock head in fp32,
under bf16 / fp16 autocast, with and without the fused loss, with recompute and with fp16 dynamic loss scaling; and a
whole-step graph replayed over batches whose labelled-row counts differ, against eager steps."""
import copy

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

IGN = -1
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
ROWS = [1, 7, 100, 1024, 1025, 4099, 32768]


def _counts():
    from oktopk_b200.ops import ext
    return {k: ext.LAUNCH_COUNT.get(k, 0) for k in ("mlm_select", "mlm_gather", "mlm_scatter")}


def _delta(n0):
    return {k: v - n0[k] for k, v in _counts().items()}


def _labels(R, frac, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    t = torch.randint(0, 30522, (R,), device="cuda", generator=g)
    t[torch.rand(R, device="cuda", generator=g) >= frac] = IGN
    return t


def _torch_path(x, labels, M, dy, overflow):
    """The torch implementation on CPU copies: (xg, tgt, rows, slot, count, dx)."""
    from oktopk_b200.ops import mlm_gather
    rows, tgt, slot, count = mlm_gather.select_labelled(labels.cpu(), M, IGN, overflow)
    xc = x.detach().cpu().requires_grad_(True)
    xg, _ = mlm_gather.gather_labelled(xc, labels.cpu(), M, IGN)
    xg.backward(dy.cpu())
    return xg.detach(), tgt, rows, slot, count, xc.grad


def _check(R, H, dtype, frac, seed):
    from oktopk_b200.ops import mlm_gather
    labels = _labels(R, frac, seed)
    M = mlm_gather.capacity_rows(R, 0.25)
    g = torch.Generator("cuda").manual_seed(seed + 1)
    x = torch.randn(R, H, device="cuda", generator=g).to(dtype).requires_grad_(True)
    dy = torch.randn(M, H, device="cuda", generator=g).to(dtype)
    ov = torch.full((1,), 11, dtype=torch.int64, device="cuda")
    n0 = _counts()
    rows, tgt, slot, count = mlm_gather.select_labelled(labels, M, IGN, ov)
    xg, tgt2 = mlm_gather.gather_labelled(x, labels, M, IGN, ov)
    xg.backward(dy)
    assert _delta(n0) == {"mlm_select": 2, "mlm_gather": 1, "mlm_scatter": 1}
    ov_cpu = torch.full((1,), 11, dtype=torch.int64)
    ref_xg, ref_tgt, ref_rows, ref_slot, ref_count, ref_dx = _torch_path(x, labels, M, dy, ov_cpu)
    mlm_gather.select_labelled(labels.cpu(), M, IGN, ov_cpu)            # the second call, as above
    assert torch.equal(rows.cpu(), ref_rows) and torch.equal(slot.cpu(), ref_slot)
    assert torch.equal(tgt.cpu(), ref_tgt) and torch.equal(tgt2.cpu(), ref_tgt)
    assert int(count) == int(ref_count) == int((labels != IGN).sum())
    assert int(ov) == int(ov_cpu) == 11 + 2 * max(int(ref_count) - M, 0)
    assert xg.dtype == dtype and x.grad.dtype == dtype
    assert torch.equal(_bits(xg.cpu()), _bits(ref_xg)) and torch.equal(_bits(x.grad.cpu()), _bits(ref_dx))
    return int(ref_count), M


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


@pytest.mark.parametrize("H", [768, 1024, 100])
@pytest.mark.parametrize("R", ROWS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_kernels_match_the_torch_path_bitwise(dtype, R, H):
    n, M = _check(R, H, dtype, 0.15, seed=R + H)
    if R >= 1024:
        assert 0 < n <= M


@pytest.mark.parametrize("R", [1, 100, 1025, 32768])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H", [768, 100])
def test_overflow_is_dropped_and_accumulated(dtype, R, H):
    n, M = _check(R, H, dtype, 0.6 if R > 1 else 1.0, seed=3 * R + H)
    assert n > M or R == 1


def test_no_labels_and_all_labels():
    from oktopk_b200.ops import mlm_gather
    for fill in ("none", "all"):
        R, H = 2048, 768
        labels = torch.full((R,), IGN, device="cuda") if fill == "none" else torch.arange(R, device="cuda")
        x = torch.randn(R, H, device="cuda", requires_grad=True)
        ov = torch.zeros(1, dtype=torch.int64, device="cuda")
        xg, tgt = mlm_gather.gather_labelled(x, labels, 512, IGN, ov)
        xg.backward(torch.ones_like(xg))
        if fill == "none":
            assert int(xg.abs().max()) == 0 and bool((tgt == IGN).all()) and int(x.grad.abs().max()) == 0
            assert int(ov) == 0
        else:
            assert torch.equal(xg, x[:512]) and torch.equal(tgt, labels[:512]) and int(ov) == R - 512
            assert bool((x.grad[:512] == 1).all()) and int(x.grad[512:].abs().max()) == 0


@pytest.mark.parametrize("H", [768, 100])
@pytest.mark.parametrize("dtype", DTYPES)
def test_scatter_writes_every_row(dtype, H):
    """Into a NaN-filled gradient: after one scatter no row is left unwritten."""
    from oktopk_b200.ops import ext, mlm_gather
    C = ext.require()
    R = 5000
    labels = _labels(R, 0.15, 9)
    M = mlm_gather.capacity_rows(R, 0.25)
    _, _, slot, _ = mlm_gather.select_labelled(labels, M, IGN)
    dout = torch.randn(M, H, device="cuda").to(dtype)
    dx = torch.full((R, H), float("nan"), device="cuda").to(dtype)
    C.mlm_scatter(dout.data_ptr(), slot.data_ptr(), dx.data_ptr(), R, H, ext.DTYPE_CODE[dtype],
                  torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert not bool(dx.isnan().any())
    s = slot.long()
    assert torch.equal(dx[s >= 0], dout[s[s >= 0]]) and int(dx[s < 0].abs().max()) == 0


def test_misaligned_rows_take_the_scalar_path():
    from oktopk_b200.ops import mlm_gather
    R, H = 300, 768
    base = torch.randn(R * H + 1, device="cuda")
    x = base[1:].view(R, H)                                            # 4 bytes off a 16-byte boundary
    labels = _labels(R, 0.3, 4)
    xg, tgt = mlm_gather.gather_labelled(x, labels, 96, IGN)
    ref, _ = mlm_gather.gather_labelled(x.cpu(), labels.cpu(), 96, IGN)
    assert torch.equal(xg.cpu(), ref)


def test_cuda_graph_replay_follows_new_labels():
    from oktopk_b200.ops import mlm_gather
    R, H, M = 1024, 768, 256
    x = torch.randn(R, H, device="cuda", requires_grad=True)
    labels = _labels(R, 0.1, 1)
    ov = torch.zeros(1, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        xg, _ = mlm_gather.gather_labelled(x, labels, M, IGN, ov)
        (gx,) = torch.autograd.grad(xg.sum(), x)
    torch.cuda.current_stream().wait_stream(s)
    del xg, gx                                           # drop the warm-up's autograd graph before the capture
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        xg, tgt = mlm_gather.gather_labelled(x, labels, M, IGN, ov)
        (gx,) = torch.autograd.grad((xg * xg).sum(), x)
    for seed, frac in ((2, 0.05), (3, 0.2), (4, 0.4)):
        labels.copy_(_labels(R, frac, seed))
        ov.zero_()
        g.replay()
        torch.cuda.synchronize()
        ref_xg, ref_tgt = mlm_gather.gather_labelled(x.detach().cpu(), labels.cpu(), M, IGN)
        n = int((labels != IGN).sum())
        assert torch.equal(xg.cpu(), ref_xg) and torch.equal(tgt.cpu(), ref_tgt)
        assert int(ov) == max(n - M, 0)
        kept = torch.zeros(R, dtype=torch.bool)
        kept[(labels != IGN).nonzero()[:M, 0].cpu()] = True
        assert torch.equal(gx.cpu()[kept], 2 * x.detach().cpu()[kept]) and int(gx.cpu()[~kept].abs().max()) == 0


# ------------------------------------------------------------------------------------------ BERT
def _bert(**kw):
    from oktopk_b200.models.bert import BertConfig, BertForPreTraining
    torch.manual_seed(0)
    cfg = BertConfig(num_hidden_layers=4, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    return BertForPreTraining(cfg, depth=4, **kw).cuda()


def _batch(seed=1, mask_prob=0.15):
    from oktopk_b200.models.bert import synthetic_batch
    return synthetic_batch(8, 128, device="cuda", generator=torch.Generator().manual_seed(seed), mask_prob=mask_prob)


def _grad_err(u, v):
    return float((u.float() - v.float()).norm()) / (float(v.float().norm()) + 1e-12)


@pytest.mark.parametrize("fuse_xent", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_bert_sparse_head_matches_stock(dtype, fuse_xent):
    b = _bert(fuse_xent=fuse_xent)
    a = copy.deepcopy(b)
    a.sparse_mlm = True
    batch = _batch()
    res = []
    for net in (a, b):
        net.train()
        n0 = _counts()
        with torch.autocast("cuda", dtype, enabled=dtype != torch.float32):
            loss = net(*batch)
        loss.backward()
        res.append((loss.detach().double(), [p.grad for p in net.parameters()], _delta(n0)))
    (la, ga, na), (lb, gb, nb) = res
    assert na == {"mlm_select": 1, "mlm_gather": 1, "mlm_scatter": 1} and nb == {k: 0 for k in nb}
    assert int(a.stages[-1].heads.mlm_overflow) == 0
    names = [n for n, _ in a.named_parameters()]
    if dtype == torch.float32:
        assert float(la) == pytest.approx(float(lb), rel=1e-5)
        for n, u, v in zip(names, ga, gb):
            torch.testing.assert_close(u, v, rtol=1e-3, atol=1e-5, msg=n)
    else:                                                # test_fused_xent's autocast tolerances
        assert float(la) == pytest.approx(float(lb), rel=1e-3)
        for n, u, v in zip(names, ga, gb):
            assert _grad_err(u, v) < 2e-2, (n, _grad_err(u, v))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_sequence_gradient_is_bitwise_zero_on_unlabelled_rows(dtype):
    net = _bert(sparse_mlm=True, fuse_xent=True)
    heads = net.stages[-1].heads
    _, _, _, labels, nxt = _batch(3)
    seq = torch.randn(8, 128, 768, device="cuda", requires_grad=True)
    pooled = torch.randn(8, 768, device="cuda")
    with torch.autocast("cuda", dtype, enabled=dtype != torch.float32):
        scores, nsp, tgt = heads(seq, pooled, labels)
        loss = net.criterion(scores, nsp, tgt, nxt)
    assert scores.shape == (256, 30522) and tgt.shape == (256,)
    loss.backward()
    g = seq.grad.reshape(-1, 768)
    off = labels.reshape(-1) == IGN
    assert int((g[off] != 0).sum()) == 0 and bool((g[~off] != 0).any(1).all())


def test_bert_sparse_head_with_recompute():
    b = _bert(fuse_xent=True, fuse_ln=True)
    a = copy.deepcopy(b)
    a.sparse_mlm = True
    a.recompute = True
    batch = _batch(2)
    losses = []
    for net in (a, b):
        net.train()
        loss = net(*batch)
        loss.backward()
        losses.append(float(loss.detach()))
    assert losses[0] == pytest.approx(losses[1], rel=1e-5)
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        torch.testing.assert_close(pa.grad, pb.grad, rtol=1e-3, atol=1e-5, msg=n)


def _trainer(cuda_graph, sparse, **kw):
    import oktopk_b200 as okt
    from oktopk_b200.models.bert import BertConfig
    from oktopk_b200.train.trainer import Trainer
    cfg = BertConfig(num_hidden_layers=2, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    return Trainer(dnn="bert_base", dataset="wikipedia", batch_size=8, lr=1e-4, compressor="oktopk", density=0.001,
                   cfg=okt.preset("bert_base", density=0.001, warmup_iters=2), seed=0, seq_len=128,
                   cuda_graph=cuda_graph, model_kwargs={"config": cfg, "depth": 2, "fuse_ln": True, "fuse_xent": True,
                                                        "sparse_mlm": sparse}, **kw)


def _varied_batches():
    """Labelled-row counts from ~40 to ~200 of 1024 (every one under the capacity of 256)."""
    return [_batch(40 + i, p) for i, p in enumerate((0.05, 0.15, 0.25, 0.1))]


def test_graphed_trainer_over_varied_label_counts_matches_eager():
    tg, te = _trainer(True, True), _trainer(False, True)
    assert tg.graphed is not None and tg.net.sparse_mlm and te.net.sparse_mlm
    batches = _varied_batches()
    counts = [int((b[3] != IGN).sum()) for b in batches]
    assert len(set(counts)) == len(counts) and max(counts) < 256, counts
    lg, le = [], []
    n0 = _counts()
    for it in range(10):
        b = batches[it % len(batches)]
        lg.append(float(tg.graphed.step(b)))
        te.optimizer.zero_grad()
        loss, _ = te._forward_loss(b)
        loss.backward()
        te.update_model()
        le.append(float(loss.detach()))
    torch.cuda.synchronize()
    assert tg.graphed.enabled and len(tg.graphed.graphs) >= 1, tg.graphed.why_disabled
    assert _delta(n0)["mlm_select"] >= 10
    assert lg == pytest.approx(le, rel=1e-3, abs=1e-3), (lg, le)
    pa = torch.cat([p.detach().flatten() for p in tg.net.parameters()])
    pb = torch.cat([p.detach().flatten() for p in te.net.parameters()])
    assert float((pa - pb).norm()) / float(pb.norm()) < 1e-3
    tg.flush_losses()                                    # reads the overflow counter: nothing was dropped
    assert int(tg.net.stages[-1].heads.mlm_overflow) == 0
    tg.close()
    te.close()


def test_graphed_trainer_raises_on_overflow():
    tr = _trainer(True, True)
    tr.net.mlm_capacity = 0.0625                         # 64 rows of 1024
    batches = _varied_batches()
    for it in range(6):
        tr.graphed.step(batches[it % len(batches)])
    with pytest.raises(RuntimeError, match="--mlm-capacity"):
        tr.flush_losses()
    tr.close()


def test_fp16_dynamic_loss_scaling_sparse_matches_stock():
    from oktopk_b200.config import LossScale
    ta = _trainer(False, True, autocast="fp16", loss_scale=LossScale())
    tb = _trainer(False, False, autocast="fp16", loss_scale=LossScale())
    batches = _varied_batches()
    la, lb = [], []
    for it in range(8):
        for tr, out in ((ta, la), (tb, lb)):
            b = batches[it % len(batches)]
            tr.optimizer.zero_grad()
            loss, _ = tr._forward_loss(b)
            tr.backward(loss)
            tr.update_model()
            out.append(float(loss.detach()))
    torch.cuda.synchronize()
    assert np.isfinite(la).all() and np.isfinite(lb).all(), (la, lb)
    assert la[0] == pytest.approx(lb[0], rel=1e-3)
    assert la == pytest.approx(lb, rel=2e-2), (la, lb)
    assert all(torch.isfinite(p).all() for p in ta.net.parameters())
    ta.close()
    tb.close()
