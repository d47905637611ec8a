"""Model factory: ``create_net(num_classes, dnn, **kw)`` (``VGG/dl_trainer.py:81-102``) over fresh
implementations of the reference's architectures, plus synthetic-batch generators of the dataset shapes."""
from __future__ import annotations

import torch

from .vgg import VGG, vgg16, vgg19                                    # noqa: F401
from .deepspeech import DeepSpeech, lstman4, PTBLSTM, AN4_LABELS      # noqa: F401
from .bert import (BertConfig, BertForPreTraining, bert_base, build_stages, synthetic_batch as bert_synthetic_batch,  # noqa: F401
                   StartingStage, IntermediateStage, EndingStage, PretrainingCriterion)
from . import zoo

DNNS = ["vgg16", "vgg19", "vgg11", "vgg13", "resnet20", "resnet32", "resnet44", "resnet56", "resnet110",
        "preresnet110", "resnext29", "densenet100", "caffe_cifar", "alexnet", "resnet18", "resnet34", "resnet50",
        "resnet101", "resnet152", "mnistnet", "lstman4", "lstm", "bert_base", "bert"]


# the ResNets whose batch-norms take the fused kernels with ``fuse_bn=True`` (VGG fuses by default; the ImageNet
# ResNets keep the stock modules, see ROADMAP)
FUSED_BN_RESNETS = ("resnet20", "resnet32", "resnet44", "resnet56", "resnet110")


def create_net(num_classes: int, dnn: str = "resnet20", **kwargs):
    """Returns ``(net, ext)`` like the reference (``ext`` carries e.g. the AN4 label set).  For the ResNets of
    ``FUSED_BN_RESNETS``, ``fuse_bn=True`` turns on ``net.fuse`` (and ``fuse_fp16=True`` ``net.fuse_fp16``); for BERT,
    ``fuse_ln=True`` turns on ``net.fuse_ln``, ``fuse_xent=True`` ``net.fuse_xent`` and ``sparse_mlm=True``
    ``net.sparse_mlm`` (``mlm_capacity=F`` sets ``net.mlm_capacity``), ``fuse_attn=True`` ``net.fuse_attn`` and
    ``fuse_emb=True`` ``net.fuse_emb``; for
    ``lstman4``,
    ``fuse_lstm=True`` turns on ``net.fuse_lstm``, ``fuse_lstm_autocast=True`` ``net.fuse_lstm_autocast`` and
    ``fuse_lstm_bidirectional=True`` ``net.fuse_lstm_bidirectional`` (with ``bidirectional=True``), ``fuse_ctc=True``
    ``net.fuse_ctc`` and ``fuse_bn=True`` ``net.fuse_bn``; for ``lstm`` (PTB),
    ``fuse_lstm=True`` turns on ``net.fuse_lstm``, ``fuse_lstm_fp32=True`` ``net.fuse_lstm_fp32`` and ``fuse_xent=True``
    ``net.fuse_xent``."""
    ext = None
    d = dnn.lower()
    if d.startswith("vgg"):
        net = VGG(d, num_classes, fuse_fp16=bool(kwargs.get("fuse_fp16", False)))
    elif d in ("resnet20", "resnet32", "resnet44", "resnet56", "resnet110"):
        net = zoo.CifarResNet(int(d[6:]), num_classes)
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
        kw = dict(kwargs)
        fuse_lstm = bool(kw.pop("fuse_lstm", False))
        fuse_ctc = bool(kw.pop("fuse_ctc", False))
        net = lstman4(**kw)
        net.fuse_lstm = fuse_lstm
        net.fuse_ctc = fuse_ctc
        ext = {"labels": AN4_LABELS}
    elif d == "lstm":
        net = PTBLSTM(vocab_size=kwargs.get("vocab_size", 10000), batch_size=kwargs.get("batch_size", 20),
                      fuse_lstm=bool(kwargs.get("fuse_lstm", False)), fuse_xent=bool(kwargs.get("fuse_xent", False)),
                      fuse_lstm_fp32=bool(kwargs.get("fuse_lstm_fp32", False)))
    elif d in ("bert", "bert_base"):
        cfg = kwargs.get("config")
        if isinstance(cfg, str):
            cfg = BertConfig.from_json_file(cfg)
        cfg = cfg or BertConfig.bert_base()
        if kwargs.get("num_hidden_layers"):
            import dataclasses
            cfg = dataclasses.replace(cfg, num_hidden_layers=int(kwargs["num_hidden_layers"]))
        net = BertForPreTraining(cfg, kwargs.get("depth", 4), recompute=bool(kwargs.get("recompute", False)),
                                 fuse_ln=bool(kwargs.get("fuse_ln", False)),
                                 fuse_xent=bool(kwargs.get("fuse_xent", False)),
                                 sparse_mlm=bool(kwargs.get("sparse_mlm", False)),
                                 mlm_capacity=float(kwargs.get("mlm_capacity", 0.25)),
                                 fuse_attn=bool(kwargs.get("fuse_attn", False)),
                                 fuse_emb=bool(kwargs.get("fuse_emb", False)))
    else:
        raise ValueError("unknown dnn %r (have %s)" % (dnn, DNNS))
    if d in FUSED_BN_RESNETS:
        net.fuse = bool(kwargs.get("fuse_bn", False))
        net.fuse_fp16 = bool(kwargs.get("fuse_fp16", False))
    return net, ext
