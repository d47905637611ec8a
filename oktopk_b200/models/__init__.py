"""Model factory: ``create_net(num_classes, dnn, **kw)`` (``VGG/dl_trainer.py:81-102``) over fresh
implementations of the reference's architectures, plus synthetic-batch generators of the dataset shapes."""
from __future__ import annotations

import torch

from .vgg import VGG, vgg16, vgg19                                    # noqa: F401
from .deepspeech import DeepSpeech, lstman4, PTBLSTM, AN4_LABELS      # noqa: F401
from .bert import (BertConfig, BertForPreTraining, bert_base, build_stages, synthetic_batch as bert_synthetic_batch,  # noqa: F401
                   StartingStage, IntermediateStage, EndingStage, PretrainingCriterion)
from . import zoo
from .switches import FUSED_BN_RESNETS, SWITCH_MODELS                 # noqa: F401

DNNS = ["vgg16", "vgg19", "vgg11", "vgg13", "resnet20", "resnet32", "resnet44", "resnet56", "resnet110",
        "preresnet110", "resnext29", "densenet100", "caffe_cifar", "alexnet", "resnet18", "resnet34", "resnet50",
        "resnet101", "resnet152", "mnistnet", "lstman4", "lstm", "bert_base", "bert"]


def create_net(num_classes: int, dnn: str = "resnet20", **kwargs):
    """Returns ``(net, ext)`` like the reference (``ext`` carries e.g. the AN4 label set).  The opt-in switches, such as
    ``fuse_bn=True``, and the models that take each are listed in ``switches.py``; a switch the model does not take
    raises ``ValueError``."""
    ext = None
    d = dnn.lower()
    switches = {k: kwargs.pop(k) for k in list(kwargs) if k in SWITCH_MODELS}
    for k in switches:
        if d not in SWITCH_MODELS[k]:
            raise ValueError("%s applies to %s, not %s" % (k, ", ".join(SWITCH_MODELS[k]), dnn))
    if d.startswith("vgg"):
        net = VGG(d, num_classes, **switches)
    elif d in ("resnet20", "resnet32", "resnet44", "resnet56", "resnet110"):
        net = zoo.CifarResNet(int(d[6:]), num_classes, **switches)
    elif d.startswith("preresnet"):
        net = zoo.PreResNet(int(d[9:]), num_classes)
    elif d == "resnext29":
        net = zoo.CifarResNeXt(8, 29, num_classes)
    elif d == "densenet100":
        net = zoo.DenseNet(100, 12, 0.5, num_classes)
    elif d == "caffe_cifar":
        net = zoo.CifarCaffeNet(num_classes)
    elif d == "alexnet":
        net = zoo.AlexNet(num_classes)
    elif d in ("resnet18", "resnet34", "resnet50", "resnet101", "resnet152"):
        net = zoo.imagenet_resnet(d, num_classes)
    elif d == "mnistnet":
        net = zoo.MnistNet()
    elif d == "lstman4":
        net = lstman4(**kwargs, **switches)
        ext = {"labels": AN4_LABELS}
    elif d == "lstm":
        net = PTBLSTM(vocab_size=kwargs.get("vocab_size", 10000), batch_size=kwargs.get("batch_size", 20), **switches)
    elif d in ("bert", "bert_base"):
        cfg = kwargs.get("config")
        if isinstance(cfg, str):
            cfg = BertConfig.from_json_file(cfg)
        cfg = cfg or BertConfig.bert_base()
        if kwargs.get("num_hidden_layers"):
            import dataclasses
            cfg = dataclasses.replace(cfg, num_hidden_layers=int(kwargs["num_hidden_layers"]))
        net = BertForPreTraining(cfg, kwargs.get("depth", 4), recompute=bool(kwargs.get("recompute", False)),
                                 **switches)
    else:
        raise ValueError("unknown dnn %r (have %s)" % (dnn, DNNS))
    return net, ext
