"""The ResNets' fused batch-norm switch on the CPU: ``create_net(..., fuse_bn=True)`` keeps the stock network (outputs,
parameters, ``state_dict`` keys) wherever the fused kernels do not run, and the ``--fused-bn`` flag."""
import pytest
import torch

from oktopk_b200.models import FUSED_BN_RESNETS, create_net
from oktopk_b200.train import cli


@pytest.mark.parametrize("dnn,shape", [("resnet20", (2, 3, 32, 32)), ("resnet32", (2, 3, 32, 32))])
def test_fuse_bn_on_cpu_is_the_stock_network(dnn, shape):
    torch.manual_seed(0)
    a, _ = create_net(10, dnn, fuse_bn=True)
    torch.manual_seed(0)
    b, _ = create_net(10, dnn)
    assert a.fuse is True and b.fuse is False and a.fuse_fp16 is False
    assert list(a.state_dict()) == list(b.state_dict())
    assert sum(p.numel() for p in a.parameters()) == sum(p.numel() for p in b.parameters())
    for (ka, va), vb in zip(a.state_dict().items(), b.state_dict().values()):
        assert torch.equal(va, vb), ka
    x = torch.randn(shape)
    a.train(); b.train()
    torch.testing.assert_close(a(x), b(x), rtol=0, atol=0)
    for ba, bb in zip(a.buffers(), b.buffers()):
        assert torch.equal(ba, bb)


def test_fuse_bn_is_a_run_time_switch_and_carries_fuse_fp16():
    net, _ = create_net(10, "resnet56", fuse_bn=True, fuse_fp16=True)
    assert net.fuse and net.fuse_fp16
    net.fuse = False
    assert not net.fuse
    assert create_net(10, "resnet110")[0].fuse is False
    assert set(FUSED_BN_RESNETS) == {"resnet20", "resnet32", "resnet44", "resnet56", "resnet110"}


def test_cli_fused_bn_flag():
    p = cli.build_parser()
    args = p.parse_args(["--dnn", "resnet20", "--fused-bn"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("resnet20", {"fuse_bn": True})
    args = p.parse_args(["--dnn", "resnet56", "--fp16", "--fused-bn", "--fused-bn-fp16"])
    cli.check_switch_args(p, args)
    assert cli.model_args(args) == ("resnet56", {"fuse_fp16": True, "fuse_bn": True})
    assert cli.model_args(p.parse_args(["--dnn", "resnet20"])) == ("resnet20", {})
    for bad in (["--dnn", "vgg16", "--fused-bn"], ["--dnn", "preresnet110", "--fused-bn"],
                ["--dnn", "resnet50", "--fused-bn"], ["--dnn", "densenet100", "--fused-bn"],
                ["--dnn", "resnet20", "--fp16", "--fused-bn-fp16"]):
        with pytest.raises(SystemExit):
            cli.main(bad)
