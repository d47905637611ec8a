"""The rest of the reference's model zoo, selectable through ``--dnn`` (``VGG/dl_trainer.py:59-102``,
``VGG/models/__init__.py:16-26``): CIFAR ResNet-20/32/44/56/110 (He et al. option-A shortcuts),
pre-activation ResNets, ResNeXt-29, DenseNet-BC-100, a Caffe-style CIFAR-quick net, AlexNet (with
LRN), ImageNet ResNet-18/34/50/101/152 and the MNIST net.  Fresh compact implementations."""
from __future__ import annotations

import math
from typing import List, Sequence, Type

import torch
import torch.nn as nn
import torch.nn.functional as F


# ---------------------------------------------------------------------------- CIFAR ResNet (6n+2)
class _BasicA(nn.Module):
    """3x3-3x3 block with parameter-free (stride + zero-pad) shortcut."""

    def __init__(self, cin: int, cout: int, stride: int):
        super().__init__()
        self.c1 = nn.Conv2d(cin, cout, 3, stride, 1, bias=False)
        self.b1 = nn.BatchNorm2d(cout)
        self.c2 = nn.Conv2d(cout, cout, 3, 1, 1, bias=False)
        self.b2 = nn.BatchNorm2d(cout)
        self.stride, self.pad = stride, cout - cin

    def forward(self, x):
        y = self.b2(self.c2(F.relu(self.b1(self.c1(x)), inplace=True)))
        if self.stride != 1 or self.pad:
            x = x[:, :, ::self.stride, ::self.stride]
            x = F.pad(x, (0, 0, 0, 0, self.pad // 2, self.pad - self.pad // 2))
        return F.relu(x + y, inplace=True)

    def forward_fused(self, x, fp16: bool = False):
        """``forward`` through the fused batch-norm kernels, the residual add and ReLU folded into the second one."""
        from ..ops.fused_bn import conv_bn_relu
        y = conv_bn_relu(x, self.c1, self.b1, fp16=fp16)
        if self.stride != 1 or self.pad:
            x = x[:, :, ::self.stride, ::self.stride]
            x = F.pad(x, (0, 0, 0, 0, self.pad // 2, self.pad - self.pad // 2))
        return conv_bn_relu(y, self.c2, self.b2, fp16=fp16, residual=x)


class CifarResNet(nn.Module):
    """``net.fuse`` (default off; ``create_net(..., fuse_bn=True)``) runs every conv -> BN [+ shortcut] -> ReLU through
    the fused batch-norm kernels in training on the GPU, ``net.fuse_fp16`` adds fp16 activations to that path (as for
    VGG).  The option-A shortcut (stride slice + channel zero-pad) stays stock torch ops."""

    def __init__(self, depth: int = 20, num_classes: int = 10, fuse_bn: bool = False, fuse_fp16: bool = False):
        super().__init__()
        self.fuse, self.fuse_fp16 = bool(fuse_bn), bool(fuse_fp16)
        assert (depth - 2) % 6 == 0
        n = (depth - 2) // 6
        self.stem = nn.Sequential(nn.Conv2d(3, 16, 3, 1, 1, bias=False), nn.BatchNorm2d(16), nn.ReLU(inplace=True))
        blocks, cin = [], 16
        for width, stride in ((16, 1), (32, 2), (64, 2)):
            for i in range(n):
                blocks.append(_BasicA(cin, width, stride if i == 0 else 1))
                cin = width
        self.blocks = nn.Sequential(*blocks)
        self.fc = nn.Linear(64, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight)

    def forward(self, x):
        if self.fuse and x.is_cuda and self.training:
            from ..ops.fused_bn import conv_bn_relu
            x = conv_bn_relu(x, self.stem[0], self.stem[1], fp16=self.fuse_fp16)
            for b in self.blocks:
                x = b.forward_fused(x, self.fuse_fp16)
            return self.fc(torch.flatten(F.adaptive_avg_pool2d(x, 1), 1))
        x = self.blocks(self.stem(x))
        return self.fc(torch.flatten(F.adaptive_avg_pool2d(x, 1), 1))


# ---------------------------------------------------------------------------- pre-activation ResNet
class _PreAct(nn.Module):
    def __init__(self, cin: int, cout: int, stride: int):
        super().__init__()
        self.b1 = nn.BatchNorm2d(cin)
        self.c1 = nn.Conv2d(cin, cout, 3, stride, 1, bias=False)
        self.b2 = nn.BatchNorm2d(cout)
        self.c2 = nn.Conv2d(cout, cout, 3, 1, 1, bias=False)
        self.short = None if (stride == 1 and cin == cout) else nn.Conv2d(cin, cout, 1, stride, bias=False)

    def forward(self, x):
        o = F.relu(self.b1(x), inplace=True)
        s = x if self.short is None else self.short(o)
        o = self.c2(F.relu(self.b2(self.c1(o)), inplace=True))
        return o + s


class PreResNet(nn.Module):
    def __init__(self, depth: int = 110, num_classes: int = 10):
        super().__init__()
        n = (depth - 2) // 6
        self.stem = nn.Conv2d(3, 16, 3, 1, 1, bias=False)
        blocks, cin = [], 16
        for width, stride in ((16, 1), (32, 2), (64, 2)):
            for i in range(n):
                blocks.append(_PreAct(cin, width, stride if i == 0 else 1))
                cin = width
        self.blocks = nn.Sequential(*blocks)
        self.bn = nn.BatchNorm2d(64)
        self.fc = nn.Linear(64, num_classes)

    def forward(self, x):
        x = F.relu(self.bn(self.blocks(self.stem(x))), inplace=True)
        return self.fc(torch.flatten(F.adaptive_avg_pool2d(x, 1), 1))


# ---------------------------------------------------------------------------- ResNeXt-29
class _XBlock(nn.Module):
    def __init__(self, cin: int, cout: int, stride: int, cardinality: int, base_width: int, widen: int):
        super().__init__()
        d = cardinality * int(base_width * (cout / (widen * 64.0)))
        self.reduce = nn.Conv2d(cin, d, 1, bias=False)
        self.bn_r = nn.BatchNorm2d(d)
        self.conv = nn.Conv2d(d, d, 3, stride, 1, groups=cardinality, bias=False)
        self.bn = nn.BatchNorm2d(d)
        self.expand = nn.Conv2d(d, cout, 1, bias=False)
        self.bn_e = nn.BatchNorm2d(cout)
        self.short = None
        if cin != cout or stride != 1:
            self.short = nn.Sequential(nn.Conv2d(cin, cout, 1, stride, bias=False), nn.BatchNorm2d(cout))

    def forward(self, x):
        o = F.relu(self.bn_r(self.reduce(x)), inplace=True)
        o = F.relu(self.bn(self.conv(o)), inplace=True)
        o = self.bn_e(self.expand(o))
        s = x if self.short is None else self.short(x)
        return F.relu(o + s, inplace=True)


class CifarResNeXt(nn.Module):
    def __init__(self, cardinality: int = 8, depth: int = 29, num_classes: int = 10, base_width: int = 64, widen: int = 4):
        super().__init__()
        n = (depth - 2) // 9
        stages = [64, 64 * widen, 128 * widen, 256 * widen]
        self.stem = nn.Sequential(nn.Conv2d(3, 64, 3, 1, 1, bias=False), nn.BatchNorm2d(64), nn.ReLU(inplace=True))
        blocks, cin = [], stages[0]
        for width, stride in zip(stages[1:], (1, 2, 2)):
            for i in range(n):
                blocks.append(_XBlock(cin, width, stride if i == 0 else 1, cardinality, base_width, widen))
                cin = width
        self.blocks = nn.Sequential(*blocks)
        self.fc = nn.Linear(stages[3], num_classes)

    def forward(self, x):
        x = self.blocks(self.stem(x))
        return self.fc(torch.flatten(F.adaptive_avg_pool2d(x, 1), 1))


# ---------------------------------------------------------------------------- DenseNet-BC
class _DenseLayer(nn.Module):
    def __init__(self, cin: int, growth: int):
        super().__init__()
        self.b1 = nn.BatchNorm2d(cin)
        self.c1 = nn.Conv2d(cin, 4 * growth, 1, bias=False)
        self.b2 = nn.BatchNorm2d(4 * growth)
        self.c2 = nn.Conv2d(4 * growth, growth, 3, padding=1, bias=False)

    def forward(self, x):
        o = self.c1(F.relu(self.b1(x), inplace=True))
        o = self.c2(F.relu(self.b2(o), inplace=True))
        return torch.cat([x, o], 1)


class DenseNet(nn.Module):
    def __init__(self, depth: int = 100, growth: int = 12, reduction: float = 0.5, num_classes: int = 10):
        super().__init__()
        n = (depth - 4) // 6
        c = 2 * growth
        layers: List[nn.Module] = [nn.Conv2d(3, c, 3, padding=1, bias=False)]
        for stage in range(3):
            for _ in range(n):
                layers.append(_DenseLayer(c, growth))
                c += growth
            if stage < 2:
                co = int(math.floor(c * reduction))
                layers += [nn.BatchNorm2d(c), nn.ReLU(inplace=True), nn.Conv2d(c, co, 1, bias=False), nn.AvgPool2d(2)]
                c = co
        self.features = nn.Sequential(*layers)
        self.bn = nn.BatchNorm2d(c)
        self.fc = nn.Linear(c, num_classes)

    def forward(self, x):
        x = F.relu(self.bn(self.features(x)), inplace=True)
        return self.fc(torch.flatten(F.adaptive_avg_pool2d(x, 1), 1))


# ---------------------------------------------------------------------------- small nets
class CifarCaffeNet(nn.Module):
    """CIFAR10-quick style 3-conv network (``VGG/models/caffe_cifar.py``)."""

    def __init__(self, num_classes: int = 10):
        super().__init__()
        self.features = nn.Sequential(
            nn.Conv2d(3, 32, 3, padding=1), nn.MaxPool2d(2), nn.ReLU(inplace=True), nn.BatchNorm2d(32),
            nn.Conv2d(32, 64, 3, padding=1), nn.ReLU(inplace=True), nn.AvgPool2d(2), nn.BatchNorm2d(64),
            nn.Conv2d(64, 128, 3, padding=1), nn.ReLU(inplace=True), nn.AvgPool2d(2), nn.BatchNorm2d(128))
        self.classifier = nn.Sequential(nn.Linear(128 * 4 * 4, 512), nn.ReLU(inplace=True), nn.Linear(512, num_classes))

    def forward(self, x):
        return self.classifier(torch.flatten(self.features(x), 1))


class AlexNet(nn.Module):
    """Single-tower AlexNet with local response normalisation (``VGG/models/alexnet.py``)."""

    def __init__(self, num_classes: int = 1000):
        super().__init__()
        self.features = nn.Sequential(
            nn.Conv2d(3, 96, 11, 4, 2), nn.ReLU(inplace=True), nn.LocalResponseNorm(5, 1e-4, 0.75, 2), nn.MaxPool2d(3, 2),
            nn.Conv2d(96, 256, 5, padding=2, groups=2), nn.ReLU(inplace=True), nn.LocalResponseNorm(5, 1e-4, 0.75, 2),
            nn.MaxPool2d(3, 2),
            nn.Conv2d(256, 384, 3, padding=1), nn.ReLU(inplace=True),
            nn.Conv2d(384, 384, 3, padding=1, groups=2), nn.ReLU(inplace=True),
            nn.Conv2d(384, 256, 3, padding=1, groups=2), nn.ReLU(inplace=True), nn.MaxPool2d(3, 2))
        self.classifier = nn.Sequential(nn.Linear(256 * 6 * 6, 4096), nn.ReLU(inplace=True), nn.Dropout(),
                                        nn.Linear(4096, 4096), nn.ReLU(inplace=True), nn.Dropout(),
                                        nn.Linear(4096, num_classes))

    def forward(self, x):
        return self.classifier(torch.flatten(self.features(x), 1))


class MnistNet(nn.Module):
    """``VGG/dl_trainer.py:59-76``."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(1, 10, kernel_size=5)
        self.conv2 = nn.Conv2d(10, 20, kernel_size=5)
        self.drop = nn.Dropout2d()
        self.fc1 = nn.Linear(320, 50)
        self.fc2 = nn.Linear(50, 10)

    def forward(self, x):
        x = F.relu(F.max_pool2d(self.conv1(x), 2))
        x = F.relu(F.max_pool2d(self.drop(self.conv2(x)), 2))
        x = F.dropout(F.relu(self.fc1(x.reshape(-1, 320))), training=self.training)
        return self.fc2(x)


# ---------------------------------------------------------------------------- ImageNet ResNet
class _Basic(nn.Module):
    expansion = 1

    def __init__(self, cin, planes, stride=1, down=None):
        super().__init__()
        self.c1 = nn.Conv2d(cin, planes, 3, stride, 1, bias=False)
        self.b1 = nn.BatchNorm2d(planes)
        self.c2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.b2 = nn.BatchNorm2d(planes)
        self.down = down

    def forward(self, x):
        o = self.b2(self.c2(F.relu(self.b1(self.c1(x)), inplace=True)))
        return F.relu(o + (x if self.down is None else self.down(x)), inplace=True)


class _Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, cin, planes, stride=1, down=None):
        super().__init__()
        self.c1 = nn.Conv2d(cin, planes, 1, bias=False)
        self.b1 = nn.BatchNorm2d(planes)
        self.c2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
        self.b2 = nn.BatchNorm2d(planes)
        self.c3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.b3 = nn.BatchNorm2d(planes * 4)
        self.down = down

    def forward(self, x):
        o = F.relu(self.b1(self.c1(x)), inplace=True)
        o = F.relu(self.b2(self.c2(o)), inplace=True)
        o = self.b3(self.c3(o))
        return F.relu(o + (x if self.down is None else self.down(x)), inplace=True)


class ImageNetResNet(nn.Module):
    def __init__(self, block: Type[nn.Module], layers: Sequence[int], num_classes: int = 1000):
        super().__init__()
        self.cin = 64
        self.stem = nn.Sequential(nn.Conv2d(3, 64, 7, 2, 3, bias=False), nn.BatchNorm2d(64), nn.ReLU(inplace=True),
                                  nn.MaxPool2d(3, 2, 1))
        self.stages = nn.Sequential(*[self._stage(block, 64 * 2 ** i, n, 1 if i == 0 else 2) for i, n in enumerate(layers)])
        self.fc = nn.Linear(512 * block.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")

    def _stage(self, block, planes, n, stride):
        down = None
        if stride != 1 or self.cin != planes * block.expansion:
            down = nn.Sequential(nn.Conv2d(self.cin, planes * block.expansion, 1, stride, bias=False),
                                 nn.BatchNorm2d(planes * block.expansion))
        blocks = [block(self.cin, planes, stride, down)]
        self.cin = planes * block.expansion
        blocks += [block(self.cin, planes) for _ in range(1, n)]
        return nn.Sequential(*blocks)

    def forward(self, x):
        x = self.stages(self.stem(x))
        return self.fc(torch.flatten(F.adaptive_avg_pool2d(x, 1), 1))


_IMAGENET = {"resnet18": (_Basic, (2, 2, 2, 2)), "resnet34": (_Basic, (3, 4, 6, 3)), "resnet50": (_Bottleneck, (3, 4, 6, 3)),
             "resnet101": (_Bottleneck, (3, 4, 23, 3)), "resnet152": (_Bottleneck, (3, 8, 36, 3))}


def imagenet_resnet(name: str, num_classes: int = 1000) -> ImageNetResNet:
    block, layers = _IMAGENET[name]
    return ImageNetResNet(block, layers, num_classes)
