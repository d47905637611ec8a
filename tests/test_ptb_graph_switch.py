"""Whole-step CUDA graphs for the PTB language model, on the CPU: a CPU trainer has no graph step, which PTB
configurations get graphs and the reasons of those that do not, and the ``--cuda-graph --dnn lstm`` wiring."""
import pytest
import torch

from oktopk_b200.models import create_net
from oktopk_b200.train import cli
from oktopk_b200.train.graph_step import ptb_graph_error


def _ptb_trainer(**kw):
    from oktopk_b200.train.trainer import Trainer
    return Trainer(dnn="lstm", dataset="ptb", batch_size=2, lr=22.0, compressor="none", compression=False, seed=0,
                   device=torch.device("cpu"), cuda_graph=True, **kw)


def test_cpu_trainer_has_no_graph_step():
    tr = _ptb_trainer(model_kwargs={"fuse_lstm": True, "fuse_lstm_fp32": True})
    assert tr.graphed is None
    tr.close()


@pytest.mark.parametrize("kw,autocast,why", [
    ({"fuse_lstm": True}, torch.bfloat16, None),
    ({"fuse_lstm": True, "fuse_xent": True}, torch.float16, None),
    ({"fuse_lstm": True, "fuse_lstm_fp32": True}, None, None),
    ({"fuse_lstm": True, "fuse_lstm_fp32": True, "fuse_xent": True}, None, None),
    ({}, None, None),                                          # the stock cuDNN layer in fp32
    ({"fuse_lstm": True}, None, None),                         # fuse_lstm alone in fp32 is the stock layer
    ({"fuse_lstm_fp32": True}, None, None),                    # so is fuse_lstm_fp32 alone
    ({}, torch.bfloat16, "stock nn.LSTM under bfloat16 autocast"),
    ({"fuse_xent": True}, torch.float16, "stock nn.LSTM under float16 autocast"),
    ({"fuse_lstm_fp32": True}, torch.bfloat16, "stock nn.LSTM under bfloat16 autocast"),
])
def test_which_configurations_get_graphs(kw, autocast, why):
    net, _ = create_net(10000, "lstm", **kw)
    got = ptb_graph_error(net, autocast)
    if why is None:
        assert got is None
    else:
        assert why in got and "fuse_lstm" in got


def test_cli_wiring():
    parser = cli.build_parser()
    args = parser.parse_args(["--dnn", "lstm", "--cuda-graph", "--bf16", "--fused-lstm-lm", "--fused-xent"])
    cli.check_switch_args(parser, args)
    assert args.cuda_graph and args.dnn == "lstm"
    assert cli.model_args(args)[1]["fuse_lstm"] is True
    args = parser.parse_args(["--dnn", "lstm", "--cuda-graph", "--fused-lstm-lm-fp32"])
    cli.check_switch_args(parser, args)
    assert cli.model_args(args)[1]["fuse_lstm_fp32"] is True
    assert not parser.parse_args(["--dnn", "lstm"]).cuda_graph
    help_text = " ".join(parser.format_help().split())
    assert "PTB --dnn lstm" in help_text and "--fused-lstm-lm-fp32" in help_text
