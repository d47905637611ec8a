"""CIFAR-style VGG-11/13/16/19 with BatchNorm (the reference's flagship CNN).

Architecture parity with ``VGG/models/vgg.py:6-38``: 3x3 conv + BN + ReLU stacks, five 2x2 max-pools,
a 1x1 average pool and ``Linear(512, num_classes)``.  VGG-16 = 14,728,266 parameters in 54 tensors.

``net.fuse`` (default on, ``OKTOPK_FUSED_BN=0`` turns it off) runs the Conv -> BN -> ReLU [-> pool] blocks through the
fused batch-norm kernels in fp32 and bf16.  ``net.fuse_fp16`` (``VGG(..., fuse_fp16=True)``, default off) adds fp16
activations and fp16 autocast to that path; without it fp16 keeps the stock modules.
"""
from __future__ import annotations

import torch
import torch.nn as nn

_PLANS = {
    "vgg11": (1, 1, 2, 2, 2),
    "vgg13": (2, 2, 2, 2, 2),
    "vgg16": (2, 2, 3, 3, 3),
    "vgg19": (2, 2, 4, 4, 4),
}
_WIDTHS = (64, 128, 256, 512, 512)


class VGG(nn.Module):
    def __init__(self, name: str = "vgg16", num_classes: int = 10, in_channels: int = 3, fuse_fp16: bool = False):
        super().__init__()
        plan = _PLANS[name.lower()]
        layers, c = [], in_channels
        for reps, width in zip(plan, _WIDTHS):
            for _ in range(reps):
                layers += [nn.Conv2d(c, width, kernel_size=3, padding=1), nn.BatchNorm2d(width), nn.ReLU(inplace=True)]
                c = width
            layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
        layers.append(nn.AvgPool2d(kernel_size=1, stride=1))
        self.features = nn.Sequential(*layers)
        self.fc = nn.Linear(512, num_classes)
        import os
        self.fuse = os.environ.get("OKTOPK_FUSED_BN", "1") == "1"
        self.fuse_fp16 = bool(fuse_fp16)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        # Conv -> BN -> ReLU runs go through the fused sm_90a batch-norm kernels when the activations are channels_last
        # fp32 or bf16 (fp16 too with fuse_fp16) on the GPU in training mode (ops/fused_bn.py); everywhere else this is
        # exactly self.features(x)
        if self.fuse and x.is_cuda and self.training:
            from ..ops.fused_bn import run_fused_sequential
            x = run_fused_sequential(self.features, x, fp16=self.fuse_fp16)
        else:
            x = self.features(x)
        return self.fc(torch.flatten(x, 1))


def vgg16(num_classes: int = 10) -> VGG:
    return VGG("vgg16", num_classes)


def vgg19(num_classes: int = 10) -> VGG:
    return VGG("vgg19", num_classes)
