"""ResNet-18/34/50/101/152 ([DRIVER] BASELINE.json configs 1-3; not present in the
reference, whose only model is the LSTM — SURVEY.md §0 item 6).

``state_dict`` keys follow the familiar torchvision naming (``conv1.weight``,
``layer1.0.bn1.running_mean`` …) so ``hvd.broadcast_parameters(model.state_dict())`` moves
parameters **and** BN buffers (SURVEY.md §7.3).  ResNet-50 here has 25 557 032 parameters
in 161 tensors, matching the survey's count.

H100-first layout: activations are NHWC (``channels_last``) bf16, so every 1x1 convolution
is a plain ``[N*H*W, Cin] x [Cin, Cout]`` GEMM for the wgmma kernel and BN/ReLU/residual
are fused row-wise epilogues/prologues (``ops.functional.conv_bn_act``).  Each
conv+BN(+ReLU)(+residual) is ONE functional call so the fused kernels can replace it as a
unit; the PyTorch composition is the fallback and the numerics oracle.
"""
from __future__ import annotations

from typing import List, Type, Union

from torch import nn

from ..ops import functional as F2


def _conv(cin, cout, k, stride=1, padding=0):
    return nn.Conv2d(cin, cout, k, stride=stride, padding=padding, bias=False)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = _conv(inplanes, planes, 3, stride, 1)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = _conv(planes, planes, 3, 1, 1)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        identity = x
        out = F2.conv_bn_act(x, self.conv1, self.bn1, relu=True)
        if self.downsample is not None:
            identity = F2.conv_bn_act(x, self.downsample[0], self.downsample[1], relu=False)
        return F2.conv_bn_act(out, self.conv2, self.bn2, relu=True, residual=identity)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = _conv(inplanes, planes, 1)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = _conv(planes, planes, 3, stride, 1)      # stride on the 3x3 (v1.5)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = _conv(planes, planes * 4, 1)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        return F2.bottleneck(x, self)


class ResNet(nn.Module):
    def __init__(self, block: Type[Union[BasicBlock, Bottleneck]], layers: List[int],
                 num_classes: int = 1000, zero_init_residual: bool = False,
                 small_input: bool = False):
        super().__init__()
        self.inplanes = 64
        self.small_input = small_input
        if small_input:   # 32x32 synthetic plumbing config: 3x3 stem, no max-pool
            self.conv1 = _conv(3, 64, 3, 1, 1)
        else:
            self.conv1 = _conv(3, 64, 7, 2, 3)
        self.bn1 = nn.BatchNorm2d(64)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], stride=2)
        self.layer3 = self._make_layer(block, 256, layers[2], stride=2)
        self.layer4 = self._make_layer(block, 512, layers[3], stride=2)
        self.fc = nn.Linear(512 * block.expansion, num_classes)

        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        if zero_init_residual:
            for m in self.modules():
                if isinstance(m, Bottleneck):
                    nn.init.constant_(m.bn3.weight, 0)
                elif isinstance(m, BasicBlock):
                    nn.init.constant_(m.bn2.weight, 0)

    def _make_layer(self, block, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(
                _conv(self.inplanes, planes * block.expansion, 1, stride),
                nn.BatchNorm2d(planes * block.expansion))
        layers = [block(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes))
        return nn.Sequential(*layers)

    def forward(self, x):
        x = F2.conv_bn_act(x, self.conv1, self.bn1, relu=True)
        if not self.small_input:
            x = F2.max_pool_3x3_s2(x)
        x = self.layer1(x)
        x = self.layer2(x)
        x = self.layer3(x)
        x = self.layer4(x)
        x = F2.global_avg_pool(x)
        return F2.linear(x, self.fc.weight, self.fc.bias)


def resnet18(**kw):
    return ResNet(BasicBlock, [2, 2, 2, 2], **kw)


def resnet34(**kw):
    return ResNet(BasicBlock, [3, 4, 6, 3], **kw)


def resnet50(**kw):
    return ResNet(Bottleneck, [3, 4, 6, 3], **kw)


def resnet101(**kw):
    return ResNet(Bottleneck, [3, 4, 23, 3], **kw)


def resnet152(**kw):
    return ResNet(Bottleneck, [3, 8, 36, 3], **kw)
