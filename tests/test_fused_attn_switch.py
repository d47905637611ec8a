"""BERT's fused self-attention switch on the CPU: ``create_net(..., "bert_base", fuse_attn=True)`` is the stock network
wherever the fused kernels do not run (outputs, loss, every gradient, ``state_dict`` keys), ``net.fuse_attn`` is a
run-time switch, and the ``--fused-attn`` flag."""
import pytest
import torch

from oktopk_b200.models import bert_synthetic_batch, create_net
from oktopk_b200.models.bert import BertSelfAttention
from oktopk_b200.train import cli


def _pair():
    torch.manual_seed(0)
    a, _ = create_net(2, "bert_base", num_hidden_layers=2, depth=2, fuse_attn=True)
    torch.manual_seed(0)
    b, _ = create_net(2, "bert_base", num_hidden_layers=2, depth=2)
    return a, b


def test_fuse_attn_on_cpu_is_the_stock_network():
    a, b = _pair()
    assert a.fuse_attn is True and b.fuse_attn is False
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


def test_fused_attn_op_on_cpu_is_the_stock_expression():
    import torch.nn.functional as F
    from oktopk_b200.ops.fused_attn import self_attention
    torch.manual_seed(1)
    B, S, H = 2, 9, 3
    qkv = torch.randn(B, S, 3 * H * 64, requires_grad=True)
    mask = torch.zeros(B, 1, 1, S)
    mask[1, ..., 5:] = -10000.0
    torch.manual_seed(2)
    o = self_attention(qkv, H, mask, 0.1)
    o.sum().backward()
    g, qkv.grad = qkv.grad, None
    torch.manual_seed(2)
    q, k, v = qkv.view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    r = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=0.1).transpose(1, 2).reshape(B, S, H * 64)
    r.sum().backward()
    assert torch.equal(o, r) and torch.equal(g, qkv.grad)


def test_fuse_attn_is_a_run_time_switch():
    a, _ = _pair()
    mods = [m for m in a.modules() if isinstance(m, BertSelfAttention)]
    assert len(mods) == 2 and all(m.fuse_attn for m in mods)
    a.fuse_attn = False
    assert a.fuse_attn is False and not any(m.fuse_attn for m in mods)
    mods[0].fuse_attn = True
    assert a.fuse_attn is False                      # only when every layer is fused
    a.fuse_attn = True
    assert a.fuse_attn is True
    assert not any("fuse_attn" in k for k in a.state_dict())


def test_cli_fused_attn_flag():
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "bert_base", "--fused-attn"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("bert_base", {"fuse_attn": True})
    args = p.parse_args(["--module", "models.bert12.depth=4", "--fused-attn", "--fused-ln", "--recompute_step"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("bert_base", {"num_hidden_layers": 12, "depth": 4, "recompute": True,
                                                  "fuse_ln": True, "fuse_attn": True})
    assert cli.model_args(p.parse_args(["--dnn", "bert"])) == ("bert", {})
    for bad in (["--dnn", "vgg16", "--fused-attn"], ["--dnn", "lstman4", "--fused-attn"]):
        with pytest.raises(SystemExit):
            cli.main(bad)
