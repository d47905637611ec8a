"""BERT's fused masked-LM loss switch on the CPU: ``create_net(..., "bert_base", fuse_xent=True)`` is the stock network
wherever the fused kernels do not run (outputs, loss, gradients, ``state_dict`` keys), ``net.fuse_xent`` is a run-time
switch, every fallback of ``softmax_cross_entropy`` calls stock ``F.cross_entropy``, and the ``--fused-xent`` flag."""
from unittest import mock

import pytest
import torch
import torch.nn.functional as F

from oktopk_b200.models import bert_synthetic_batch, create_net
from oktopk_b200.models.bert import BertConfig
from oktopk_b200.models.bert_heads import BertForMaskedLM
from oktopk_b200.ops import ext, fused_xent
from oktopk_b200.train import cli


def _pair():
    torch.manual_seed(0)
    a, _ = create_net(2, "bert_base", num_hidden_layers=2, depth=2, fuse_xent=True)
    torch.manual_seed(0)
    b, _ = create_net(2, "bert_base", num_hidden_layers=2, depth=2)
    return a, b


def test_fuse_xent_on_cpu_is_the_stock_network():
    a, b = _pair()
    assert a.fuse_xent is True and b.fuse_xent is False
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


def test_fuse_xent_is_a_run_time_switch():
    a, _ = _pair()
    assert a.criterion.fuse_xent is True
    a.fuse_xent = False
    assert a.fuse_xent is False and a.criterion.fuse_xent is False
    a.fuse_xent = True
    assert a.fuse_xent is True and a.fuse_ln is False       # independent of fuse_ln
    a.fuse_ln = True
    assert a.fuse_xent is True and a.fuse_ln is True
    assert not any("fuse" in k for k in a.state_dict())
    assert sum(1 for _ in a.buffers()) == sum(1 for _ in _pair()[1].buffers())


def test_masked_lm_head_switch_on_cpu():
    cfg = BertConfig(num_hidden_layers=1)
    torch.manual_seed(0)
    a = BertForMaskedLM(cfg, fuse_xent=True)
    torch.manual_seed(0)
    b = BertForMaskedLM(cfg)
    assert a.fuse_xent and not b.fuse_xent and list(a.state_dict()) == list(b.state_dict())
    ids, seg, mask, labels, _ = bert_synthetic_batch(2, 16, generator=torch.Generator().manual_seed(4))
    a.eval(); b.eval()
    la, lb = a(ids, seg, mask, labels), b(ids, seg, mask, labels)
    la.backward(); lb.backward()
    assert torch.equal(la, lb)
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        assert (pa.grad is None and pb.grad is None) or torch.equal(pa.grad, pb.grad), n   # the NSP head has none
    a.fuse_xent = False
    assert not a.fuse_xent


def _case(name):
    g = torch.Generator().manual_seed(5)
    x, t = torch.randn(6, 11, generator=g), torch.randint(0, 11, (6,), generator=g)
    t[1] = -1
    if name == "3d":
        x, t = x.view(2, 3, 11).transpose(1, 2), t.view(2, 3)      # [N, C, d] with per-position targets
    elif name == "fp64":
        x = x.double()
    elif name == "no_rows":
        x, t = x[:0], t[:0]
    elif name == "int32_target":
        t = t.int()
    elif name == "target_shape":
        t = t.view(6, 1)
    return x, t


@pytest.mark.parametrize("case", ["cpu", "no_extension", "3d", "fp64", "no_rows", "int32_target", "target_shape"])
def test_fallbacks_call_stock_cross_entropy(case):
    x, t = _case(case)
    if case in ("int32_target", "target_shape"):     # stock refuses these targets, and so does the fallback
        with pytest.raises(Exception):
            F.cross_entropy(x, t, ignore_index=-1)
        with mock.patch.object(fused_xent.F, "cross_entropy", wraps=F.cross_entropy) as ce, pytest.raises(Exception):
            fused_xent.softmax_cross_entropy(x, t, ignore_index=-1)
        assert ce.call_count == 1
        return
    outs = []
    for fused in (True, False):
        xi = x.clone().requires_grad_(True)
        if fused:
            with mock.patch.object(fused_xent.F, "cross_entropy", wraps=F.cross_entropy) as ce, \
                    mock.patch.object(ext, "available", return_value=case != "no_extension"):
                loss = fused_xent.softmax_cross_entropy(xi, t, ignore_index=-1)
            assert ce.call_count == 1 and ce.call_args.kwargs == {"ignore_index": -1}
        else:
            loss = F.cross_entropy(xi, t, ignore_index=-1)
        loss.backward()
        outs.append((loss.detach(), xi.grad))
    (la, ga), (lb, gb) = outs
    assert torch.equal(la, lb) or (la.isnan() and lb.isnan())
    assert torch.equal(ga, gb)


def test_cli_fused_xent_flag():
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "bert_base", "--fused-xent"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("bert_base", {"fuse_xent": True})
    args = p.parse_args(["--module", "models.bert12.depth=4", "--fused-xent", "--fused-ln"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("bert_base", {"num_hidden_layers": 12, "depth": 4, "fuse_ln": True,
                                                  "fuse_xent": True})
    for bad in (["--dnn", "vgg16", "--fused-xent"], ["--dnn", "resnet20", "--fused-xent"]):
        with pytest.raises(SystemExit):
            cli.main(bad)
