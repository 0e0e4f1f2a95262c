"""ResNet-18/34 for the larger-bucket / overlap-stress configuration (BASELINE.json config 4:
"ResNet-18 on synthetic 3×224×224, DDP 8×H100").  Own implementation of the standard
architecture (He et al. 2015); parameter names follow the common torchvision layout
(``conv1``, ``bn1``, ``layer{1..4}.{i}.conv{1,2}``, ``downsample.{0,1}``, ``fc``) so the bucket
plan matches torch DDP's (62 tensors, 46,758,048 B → 3 buckets).
"""
from __future__ import annotations

from typing import List, Optional, Type

import torch
import torch.nn as nn


def _conv3x3(cin, cout, stride=1):
    return nn.Conv2d(cin, cout, 3, stride, 1, bias=False)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, cin: int, cout: int, stride: int = 1, downsample: Optional[nn.Module] = None):
        super().__init__()
        self.conv1 = _conv3x3(cin, cout, stride)
        self.bn1 = nn.BatchNorm2d(cout)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = _conv3x3(cout, cout)
        self.bn2 = nn.BatchNorm2d(cout)
        self.downsample = downsample

    def forward(self, x):
        idt = x if self.downsample is None else self.downsample(x)
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        return self.relu(out + idt)


class ResNet(nn.Module):
    def __init__(self, block: Type[BasicBlock], layers: List[int], num_classes: int = 1000, in_channels: int = 3):
        super().__init__()
        self.inplanes = 64
        self.conv1 = nn.Conv2d(in_channels, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], 2)
        self.layer3 = self._make_layer(block, 256, layers[2], 2)
        self.layer4 = self._make_layer(block, 512, layers[3], 2)
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(512 * block.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    def _make_layer(self, block, planes, blocks, stride=1):
        down = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            down = nn.Sequential(nn.Conv2d(self.inplanes, planes * block.expansion, 1, stride, bias=False),
                                 nn.BatchNorm2d(planes * block.expansion))
        layers = [block(self.inplanes, planes, stride, down)]
        self.inplanes = planes * block.expansion
        layers += [block(self.inplanes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def forward(self, x):
        x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(torch.flatten(self.avgpool(x), 1))


def resnet18(num_classes: int = 1000, **kw) -> ResNet:
    return ResNet(BasicBlock, [2, 2, 2, 2], num_classes, **kw)


def resnet34(num_classes: int = 1000, **kw) -> ResNet:
    return ResNet(BasicBlock, [3, 4, 6, 3], num_classes, **kw)
