"""BERT's fused embedding switch on the CPU: ``create_net(..., "bert_base", fuse_emb=True)`` is the stock network
wherever the fused kernels do not run (outputs, loss, every gradient, ``state_dict`` keys), ``net.fuse_emb`` is a
run-time switch, and the ``--fused-emb`` flag."""
import pytest
import torch

from oktopk_b200.models import bert_synthetic_batch, create_net
from oktopk_b200.models.bert import BertConfig, BertEmbeddings
from oktopk_b200.train import cli


def _pair():
    torch.manual_seed(0)
    a, _ = create_net(2, "bert_base", num_hidden_layers=2, depth=2, fuse_emb=True)
    torch.manual_seed(0)
    b, _ = create_net(2, "bert_base", num_hidden_layers=2, depth=2)
    return a, b


def test_fuse_emb_on_cpu_is_the_stock_network():
    a, b = _pair()
    assert a.fuse_emb is True and b.fuse_emb is False
    assert list(a.state_dict()) == list(b.state_dict())
    assert [n for n, _ in a.named_buffers()] == [n for n, _ in b.named_buffers()]
    for (k, va), vb in zip(a.state_dict().items(), b.state_dict().values()):
        assert torch.equal(va, vb), k
    ids, seg, mask, labels, nxt = bert_synthetic_batch(2, 32, generator=torch.Generator().manual_seed(3))
    a.eval(); b.eval()
    with torch.no_grad():
        for oa, ob in zip(a(ids, seg, mask), b(ids, seg, mask)):
            assert torch.equal(oa, ob)
    a.train(); b.train()
    torch.manual_seed(7)
    la = a(ids, seg, mask, labels, nxt)
    la.backward()
    torch.manual_seed(7)
    lb = b(ids, seg, mask, labels, nxt)
    lb.backward()
    assert torch.equal(la, lb)
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        assert torch.equal(pa.grad, pb.grad), n


def test_fused_emb_op_on_cpu_is_the_stock_expression():
    from oktopk_b200.ops.fused_emb import embedding_layer_norm
    torch.manual_seed(1)
    emb = BertEmbeddings(BertConfig(vocab_size=50, hidden_size=128, max_position_embeddings=16, type_vocab_size=2))
    ids = torch.randint(0, 50, (3, 9))
    tt = torch.randint(0, 2, (3, 9))
    emb.train()
    torch.manual_seed(2)
    y = embedding_layer_norm(ids, tt, emb, 0.1)
    y.sum().backward()
    g = [p.grad.clone() for p in emb.parameters()]
    emb.zero_grad(set_to_none=True)
    torch.manual_seed(2)
    r = emb(ids, tt)
    r.sum().backward()
    assert torch.equal(y, r)
    for u, p in zip(g, emb.parameters()):
        assert torch.equal(u, p.grad)


def test_fuse_emb_is_a_run_time_switch():
    a, _ = _pair()
    mods = [m for m in a.modules() if isinstance(m, BertEmbeddings)]
    assert len(mods) == 1 and mods[0].fuse_emb
    a.fuse_emb = False
    assert a.fuse_emb is False and not mods[0].fuse_emb
    a.fuse_emb = True
    assert a.fuse_emb is True and mods[0].fuse_emb
    assert not any("fuse_emb" in k or "id_overflow" in k for k in a.state_dict())


def test_glue_models_take_the_switch():
    from oktopk_b200.models.bert_heads import BertModel
    cfg = BertConfig(num_hidden_layers=1, hidden_size=128, num_attention_heads=2, intermediate_size=256)
    torch.manual_seed(0)
    m = BertModel(cfg)
    ids = torch.randint(0, cfg.vocab_size, (2, 8))
    m.eval()
    with torch.no_grad():
        ref = m(ids)
        m.embeddings.fuse_emb = True
        got = m(ids)
    assert all(torch.equal(u, v) for u, v in zip(got, ref))


def test_cli_fused_emb_flag():
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "bert_base", "--fused-emb"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("bert_base", {"fuse_emb": True})
    args = p.parse_args(["--module", "models.bert12.depth=4", "--fused-emb", "--fused-ln"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("bert_base", {"num_hidden_layers": 12, "depth": 4, "fuse_ln": True,
                                                  "fuse_emb": True})
    assert cli.model_args(p.parse_args(["--dnn", "bert"])) == ("bert", {})
    for bad in (["--dnn", "vgg16", "--fused-emb"], ["--dnn", "lstm", "--fused-emb"]):
        with pytest.raises(SystemExit):
            cli.main(bad)
