"""BERT's fused LayerNorm switch on the CPU: ``create_net(..., "bert_base", fuse_ln=True)`` is the stock network wherever
the fused kernels do not run (outputs, parameters, ``state_dict`` keys), ``net.fuse_ln`` is a run-time switch, and the
``--fused-ln`` flag."""
import pytest
import torch

from oktopk_b200.models import bert_synthetic_batch, create_net
from oktopk_b200.models.bert import BertLayer
from oktopk_b200.train import cli


def _pair():
    torch.manual_seed(0)
    a, _ = create_net(2, "bert_base", num_hidden_layers=2, depth=2, fuse_ln=True)
    torch.manual_seed(0)
    b, _ = create_net(2, "bert_base", num_hidden_layers=2, depth=2)
    return a, b


def test_fuse_ln_on_cpu_is_the_stock_network():
    a, b = _pair()
    assert a.fuse_ln is True and b.fuse_ln is False
    assert list(a.state_dict()) == list(b.state_dict())
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


def test_fuse_ln_is_a_run_time_switch():
    a, _ = _pair()
    layers = [m for m in a.modules() if isinstance(m, BertLayer)]
    assert len(layers) == 2 and all(m.fuse_ln for m in layers)
    a.fuse_ln = False
    assert a.fuse_ln is False and not any(m.fuse_ln for m in layers)
    layers[0].fuse_ln = True
    assert a.fuse_ln is False                      # only when every layer is fused
    a.fuse_ln = True
    assert a.fuse_ln is True
    assert "fuse_ln" not in a.state_dict()


def test_cli_fused_ln_flag():
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "bert_base", "--fused-ln"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("bert_base", {"fuse_ln": True})
    args = p.parse_args(["--module", "models.bert12.depth=4", "--fused-ln", "--recompute_step"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("bert_base", {"num_hidden_layers": 12, "depth": 4, "recompute": True,
                                                  "fuse_ln": True})
    assert cli.model_args(p.parse_args(["--dnn", "bert"])) == ("bert", {})
    for bad in (["--dnn", "vgg16", "--fused-ln"], ["--dnn", "resnet20", "--fused-ln"]):
        with pytest.raises(SystemExit):
            cli.main(bad)
