"""Which model takes which opt-in switch, on the CPU: every switch flag (with the flags and precision it needs) against
every ``--dnn``, and every ``create_net`` switch keyword against the models that take it and one that does not.  The
model sets are written out here rather than read from ``models/switches.py``, so this is the specification."""
from unittest import mock

import pytest

from oktopk_b200.models import DNNS, BertConfig, create_net
from oktopk_b200.train import cli

VGG = {"vgg11", "vgg13", "vgg16", "vgg19"}
CIFAR_RESNETS = {"resnet20", "resnet32", "resnet44", "resnet56", "resnet110"}
BERT = {"bert", "bert_base"}

# (argv with its prerequisites, the models that accept it, the create_net keywords it gives)
FLAGS = [
    (["--fp16", "--fused-bn-fp16"], VGG, {"fuse_fp16": True}),
    (["--fp16", "--fused-bn", "--fused-bn-fp16"], CIFAR_RESNETS, {"fuse_bn": True, "fuse_fp16": True}),
    (["--fused-bn"], CIFAR_RESNETS | {"lstman4"}, {"fuse_bn": True}),
    (["--fused-ln"], BERT, {"fuse_ln": True}),
    (["--fused-xent"], BERT | {"lstm"}, {"fuse_xent": True}),
    (["--sparse-mlm"], BERT, {"sparse_mlm": True}),
    (["--sparse-mlm", "--mlm-capacity", "0.5"], BERT, {"sparse_mlm": True, "mlm_capacity": 0.5}),
    (["--fused-attn"], BERT, {"fuse_attn": True}),
    (["--fused-emb"], BERT, {"fuse_emb": True}),
    (["--fused-lstm"], {"lstman4"}, {"fuse_lstm": True}),
    (["--bf16", "--fused-lstm-lm"], {"lstm"}, {"fuse_lstm": True}),
    (["--fp16", "--fused-lstm-lm"], {"lstm"}, {"fuse_lstm": True}),
    (["--fused-lstm-lm-fp32"], {"lstm"}, {"fuse_lstm": True, "fuse_lstm_fp32": True}),
    (["--bf16", "--fused-lstm", "--fused-lstm-autocast"], {"lstman4"}, {"fuse_lstm": True, "fuse_lstm_autocast": True}),
    (["--fused-ctc"], {"lstman4"}, {"fuse_ctc": True}),
    (["--an4-pad-multiple", "8"], {"lstman4"}, {}),
    (["--bidirectional"], {"lstman4"}, {"bidirectional": True}),
    (["--fused-lstm", "--bidirectional", "--fused-lstm-bidirectional"], {"lstman4"},
     {"fuse_lstm": True, "bidirectional": True, "fuse_lstm_bidirectional": True}),
]

# create_net keyword -> the models that take it
TAKES = {
    "fuse_fp16": VGG | CIFAR_RESNETS,
    "fuse_bn": CIFAR_RESNETS | {"lstman4"},
    "fuse_ln": BERT,
    "fuse_xent": BERT | {"lstm"},
    "sparse_mlm": BERT,
    "mlm_capacity": BERT,
    "fuse_attn": BERT,
    "fuse_emb": BERT,
    "fuse_lstm": {"lstman4", "lstm"},
    "fuse_lstm_fp32": {"lstm"},
    "fuse_lstm_autocast": {"lstman4"},
    "fuse_ctc": {"lstman4"},
    "bidirectional": {"lstman4"},
    "fuse_lstm_bidirectional": {"lstman4"},
}


def _check(argv):
    """``model_args`` of ``argv`` if ``check_switch_args`` accepts it, else the error message."""
    p = cli.build_parser()
    args = p.parse_args(argv)
    with mock.patch.object(p, "error", side_effect=SystemExit) as err:
        try:
            cli.check_switch_args(p, args)
        except SystemExit:
            return err.call_args[0][0]
    return cli.model_args(args)


@pytest.mark.parametrize("argv,models,kwargs", FLAGS, ids=[" ".join(f[0]) for f in FLAGS])
def test_flag_accepted_exactly_on_its_models(argv, models, kwargs):
    for dnn in DNNS:
        got = _check(["--dnn", dnn] + argv)
        if dnn in models:
            assert got == (dnn, kwargs), (dnn, got)
        else:
            assert isinstance(got, str), (dnn, got)


def test_flags_checked_against_the_module_model():
    assert _check(["--module", "models.bert12.depth=4", "--fused-ln"]) == (
        "bert_base", {"num_hidden_layers": 12, "depth": 4, "fuse_ln": True})
    assert "not bert_base" in _check(["--module", "models.bert12.depth=4", "--fused-bn"])
    assert "not bert_base" in _check(["--module", "models.bert12.depth=4", "--fp16", "--fused-bn-fp16"])


def _small(dnn):
    """Construction arguments that keep the model small."""
    if dnn in BERT:
        return {"config": BertConfig(vocab_size=64, hidden_size=32, num_hidden_layers=2, num_attention_heads=2,
                                     intermediate_size=64, max_position_embeddings=16), "depth": 2}
    if dnn == "lstm":
        return {"vocab_size": 64}
    if dnn == "lstman4":
        return {"hidden_size": 16, "hidden_layers": 2}
    return {}


@pytest.mark.parametrize("keyword", sorted(TAKES))
def test_create_net_switch_only_on_its_models(keyword):
    value = 0.5 if keyword == "mlm_capacity" else True
    for dnn in sorted(TAKES[keyword]):
        create_net(10, dnn, **{keyword: value}, **_small(dnn))
    other = next(d for d in DNNS if d not in TAKES[keyword])
    with pytest.raises(ValueError, match=keyword):
        create_net(10, other, **{keyword: value}, **_small(other))
