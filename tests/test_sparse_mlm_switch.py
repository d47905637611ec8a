"""BERT's sparse masked-LM head on the CPU: the semantics of ``ops/mlm_gather.py`` (slots, padding, overflow, gradient)
through its torch implementation, ``create_net(..., "bert_base", sparse_mlm=True)`` against the stock network (loss,
gradients, inference outputs, ``state_dict`` keys), the run-time switches, the ``--sparse-mlm`` / ``--mlm-capacity``
flags, the Trainer's overflow error and the default capacity against the repository's masking."""
import copy

import pytest
import torch

from oktopk_b200.models import bert_synthetic_batch, create_net
from oktopk_b200.models.bert import BertConfig
from oktopk_b200.models.bert_heads import BertForMaskedLM
from oktopk_b200.ops import mlm_gather
from oktopk_b200.train import cli


def _reference(labels, M, ignore=-1):
    """Loop form of the contract: (rows, tgt, slot, count)."""
    rows, tgt, slot, n = [-1] * M, [ignore] * M, [], 0
    for r, lab in enumerate(labels.tolist()):
        if lab == ignore:
            slot.append(-1)
            continue
        if n < M:
            rows[n], tgt[n] = r, lab
            slot.append(n)
        else:
            slot.append(-1)
        n += 1
    return rows, tgt, slot, n


def _patterns():
    R, M = 64, 16
    full = torch.arange(R) + 5
    ign = torch.full((R,), -1)
    out = {"none": ign.clone(), "all": full.clone()}
    for name, k in (("exactly_M", M), ("M_plus_1", M + 1)):
        t = ign.clone()
        idx = torch.randperm(R, generator=torch.Generator().manual_seed(k))[:k]
        t[idx] = full[idx]
        out[name] = t
    t = ign.clone()
    t[R - 16::3] = full[R - 16::3]                      # labels only in the last of four 16-token sequences
    out["last_sequence"] = t
    return out, M


@pytest.mark.parametrize("name", ["none", "all", "exactly_M", "M_plus_1", "last_sequence"])
def test_select_and_gather_follow_the_contract(name):
    pats, M = _patterns()
    labels = pats[name]
    R = labels.numel()
    rows_ref, tgt_ref, slot_ref, n_ref = _reference(labels, M)
    ov = torch.full((1,), 3, dtype=torch.int64)
    rows, tgt, slot, count = mlm_gather.select_labelled(labels, M, -1, ov)
    assert rows.dtype == torch.int32 and slot.dtype == torch.int32 and tgt.dtype == torch.int64
    assert rows.tolist() == rows_ref and tgt.tolist() == tgt_ref and slot.tolist() == slot_ref
    assert int(count) == n_ref and int(ov) == 3 + max(n_ref - M, 0)

    x = torch.randn(R, 12, generator=torch.Generator().manual_seed(1), requires_grad=True)
    xg, t = mlm_gather.gather_labelled(x, labels, M, -1)
    assert xg.shape == (M, 12) and t.tolist() == tgt_ref and not t.requires_grad
    for s, r in enumerate(rows_ref):
        assert torch.equal(xg[s], x[r] if r >= 0 else torch.zeros(12)), s
    dy = torch.randn(M, 12, generator=torch.Generator().manual_seed(2))
    xg.backward(dy)
    for r, s in enumerate(slot_ref):
        assert torch.equal(x.grad[r], dy[s] if s >= 0 else torch.zeros(12)), r    # exactly 0: unlabelled or dropped


def test_capacity_rows():
    assert mlm_gather.capacity_rows(8 * 128, 0.25) == 256
    assert mlm_gather.capacity_rows(1, 0.25) == 8
    assert mlm_gather.capacity_rows(1000, 1.0) == 1000 and mlm_gather.capacity_rows(1001, 1.0) == 1008
    for bad in (0.0, -0.1, 1.5):
        with pytest.raises(ValueError):
            mlm_gather.capacity_rows(64, bad)


def _pair(**kw):
    torch.manual_seed(0)
    a, _ = create_net(2, "bert_base", num_hidden_layers=2, depth=2, sparse_mlm=True, **kw)
    torch.manual_seed(0)
    b, _ = create_net(2, "bert_base", num_hidden_layers=2, depth=2)
    return a, b


def test_sparse_mlm_matches_the_stock_network():
    a, b = _pair()
    assert a.sparse_mlm is True and b.sparse_mlm is False and a.mlm_capacity == 0.25
    assert list(a.state_dict()) == list(b.state_dict())
    ids, seg, mask, labels, nxt = bert_synthetic_batch(4, 32, generator=torch.Generator().manual_seed(3))
    a.eval(); b.eval()
    with torch.no_grad():                               # inference (no labels) is the stock forward pass
        for oa, ob in zip(a(ids, seg, mask), b(ids, seg, mask)):
            assert oa.shape == ob.shape and torch.equal(oa, ob)
    a.train(); b.train()
    torch.manual_seed(7)
    la = a(ids, seg, mask, labels, nxt)
    la.backward()
    torch.manual_seed(7)
    lb = b(ids, seg, mask, labels, nxt)
    lb.backward()
    torch.testing.assert_close(la, lb, rtol=1e-5, atol=0)
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        torch.testing.assert_close(pa.grad, pb.grad, rtol=1e-4, atol=1e-6, msg=n)
    assert int(a.stages[-1].heads.mlm_overflow) == 0


def test_sequence_gradient_is_zero_on_unlabelled_rows():
    a, b = _pair()
    heads_a, heads_b = a.stages[-1].heads, b.stages[-1].heads
    _, _, _, labels, nxt = bert_synthetic_batch(4, 32, generator=torch.Generator().manual_seed(5))
    seq = torch.randn(4, 32, 768, generator=torch.Generator().manual_seed(6))
    pooled = torch.randn(4, 768, generator=torch.Generator().manual_seed(7))
    grads = []
    for h in (heads_a, heads_b):
        s = seq.clone().requires_grad_(True)
        scores, nsp, tgt = h(s, pooled, labels)
        a.criterion(scores, nsp, tgt, nxt).backward()
        grads.append(s.grad.reshape(-1, 768))
    off = labels.reshape(-1) == -1
    assert torch.equal(grads[0][off], torch.zeros_like(grads[0][off]))
    assert torch.equal(grads[1][off], torch.zeros_like(grads[1][off]))
    torch.testing.assert_close(grads[0], grads[1], rtol=1e-4, atol=1e-7)


def test_overflowing_rows_leave_the_loss_and_are_counted():
    a, b = _pair(mlm_capacity=0.0625)                   # 8 of 128 rows
    ids, seg, mask, labels, nxt = bert_synthetic_batch(4, 32, generator=torch.Generator().manual_seed(3))
    n = int((labels != -1).sum())
    assert n > 8
    kept = labels.clone().reshape(-1)
    kept[(kept != -1).nonzero()[8:, 0]] = -1            # stock with only the first 8 labelled rows
    a.eval(); b.eval()
    la = a(ids, seg, mask, labels, nxt)
    lb = b(ids, seg, mask, kept.view_as(labels), nxt)
    torch.testing.assert_close(la, lb, rtol=1e-5, atol=0)
    assert int(a.stages[-1].heads.mlm_overflow) == n - 8
    a(ids, seg, mask, labels, nxt)
    assert int(a.stages[-1].heads.mlm_overflow) == 2 * (n - 8)


def test_sparse_mlm_is_a_run_time_switch():
    a, b = _pair()
    a.sparse_mlm = False
    assert a.sparse_mlm is False and a.stages[-1].heads.sparse_mlm is False
    a.sparse_mlm = True
    a.mlm_capacity = 0.5
    assert a.stages[-1].heads.mlm_capacity == 0.5
    with pytest.raises(ValueError):
        a.mlm_capacity = 0.0
    assert a.fuse_xent is False and a.fuse_ln is False
    a.fuse_xent = a.fuse_ln = True
    assert a.sparse_mlm is True
    assert list(a.state_dict()) == list(b.state_dict())
    assert not any("mlm" in k for k in a.state_dict())
    # fuse_xent on the CPU is stock cross_entropy: the sparse head feeds it (M, V) scores
    ids, seg, mask, labels, nxt = bert_synthetic_batch(2, 32, generator=torch.Generator().manual_seed(8))
    a.eval(); b.eval()
    torch.testing.assert_close(a(ids, seg, mask, labels, nxt), b(ids, seg, mask, labels, nxt), rtol=1e-5, atol=0)


def test_masked_lm_model_switch():
    cfg = BertConfig(num_hidden_layers=1)
    torch.manual_seed(0)
    a = BertForMaskedLM(cfg, sparse_mlm=True, mlm_capacity=0.5)
    b = copy.deepcopy(a)
    b.sparse_mlm = False
    assert a.sparse_mlm and a.mlm_capacity == 0.5 and not b.sparse_mlm
    assert list(a.state_dict()) == list(b.state_dict())
    ids, seg, mask, labels, _ = bert_synthetic_batch(2, 16, generator=torch.Generator().manual_seed(4))
    a.eval(); b.eval()
    assert torch.equal(a(ids, seg, mask), b(ids, seg, mask))
    la, lb = a(ids, seg, mask, labels), b(ids, seg, mask, labels)
    la.backward(); lb.backward()
    torch.testing.assert_close(la, lb, rtol=1e-5, atol=0)
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        if pb.grad is None:
            assert pa.grad is None, n
        else:
            torch.testing.assert_close(pa.grad, pb.grad, rtol=1e-4, atol=1e-6, msg=n)


def test_cli_sparse_mlm_flags():
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "bert_base", "--sparse-mlm"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("bert_base", {"sparse_mlm": True})
    args = p.parse_args(["--module", "models.bert12.depth=4", "--sparse-mlm", "--mlm-capacity", "0.5", "--fused-xent"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("bert_base", {"num_hidden_layers": 12, "depth": 4, "fuse_xent": True,
                                                  "sparse_mlm": True, "mlm_capacity": 0.5})
    for bad in (["--dnn", "vgg16", "--sparse-mlm"], ["--dnn", "lstman4", "--sparse-mlm", "--mlm-capacity", "0.5"],
                ["--dnn", "bert_base", "--mlm-capacity", "0.5"],
                ["--dnn", "bert_base", "--sparse-mlm", "--mlm-capacity", "0"],
                ["--dnn", "bert_base", "--sparse-mlm", "--mlm-capacity", "1.5"]):
        with pytest.raises(SystemExit):
            cli.main(bad)


def test_trainer_raises_on_overflow():
    from oktopk_b200.train.trainer import Trainer
    cfg = BertConfig(num_hidden_layers=2, hidden_size=64, num_attention_heads=2, intermediate_size=128, vocab_size=512)
    tr = Trainer(dnn="bert_base", dataset="wikipedia", batch_size=2, lr=1e-4, compression=False, seq_len=32,
                 device=torch.device("cpu"),
                 model_kwargs={"config": cfg, "depth": 2, "sparse_mlm": True, "mlm_capacity": 0.125})
    try:
        assert tr.net.sparse_mlm and tr._mlm_heads == [tr.net.stages[-1].heads]
        tr.check_mlm_overflow()                          # nothing dropped yet
        tr.net.stages[-1].heads.mlm_overflow.fill_(5)
        with pytest.raises(RuntimeError, match=r"left 5 labelled rows.*--mlm-capacity"):
            tr.flush_losses()
        tr.net.sparse_mlm = False                        # the counter is only read while the switch is on
        tr.flush_losses()
    finally:
        tr.close()


def test_default_capacity_covers_the_synthetic_batches():
    R = 8 * 128
    M = mlm_gather.capacity_rows(R, 0.25)
    worst = 0
    for seed in range(200):
        labels = bert_synthetic_batch(8, 128, generator=torch.Generator().manual_seed(seed))[3]
        worst = max(worst, int((labels != -1).sum()))
    # Bernoulli(0.15) over at most 1024 tokens: mean <= 154, standard deviation <= 11.5; 256 is 8.9 deviations out
    assert worst < M, (worst, M)


def test_default_capacity_covers_capped_masking(tmp_path):
    from oktopk_b200.train.bert_data import BERTDatasetPartitioned, PretrainingDataCreator, synthetic_corpus
    from oktopk_b200.utils.tokenization import BertTokenizer
    tok = BertTokenizer.synthetic(3000)
    (tmp_path / "corpus.txt").write_text("\n".join(synthetic_corpus(n_docs=20, sents=12, words=14)))
    pc = PretrainingDataCreator.from_corpus(str(tmp_path / "corpus.txt"), tok, max_seq_length=128, dupe_factor=1, seed=1)
    pc.save_partitions(str(tmp_path / "parts"), 2)
    ds = BERTDatasetPartitioned(tok, str(tmp_path / "parts"), max_seq_length=128, max_predictions_per_seq=20)
    # at most 20 labels per 128 tokens is at most 15.6 % of any batch's rows, under the default 25 %
    per_seq = [int((ds[i][3] != -1).sum()) for i in range(len(ds))]
    assert max(per_seq) <= 20 and max(per_seq) > 0
    for b in range(0, len(ds) - 8, 8):
        assert sum(per_seq[b:b + 8]) <= mlm_gather.capacity_rows(8 * 128, 0.25)
