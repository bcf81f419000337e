"""ORACLE / TEST INFRASTRUCTURE ONLY — never imported by the product path.

Stand-in for the un-vendored dependency `timm==0.5.4`
(team_code_transfuser/requirements.txt:104), restating from its
published definition the single model the hot path constructs:
`timm.create_model('regnety_032', ...)` (call sites transfuser.py:380,442).

Parity note: timm's source is not in the container — this restatement follows
timm 0.5.4's `regnet.py` module/attribute names (stem.conv / stem.bn,
s1..s4.b{k}.{conv1,conv2,se,conv3,downsample}, feature_info, num_features, head)
and is cross-checked structurally (per-stage widths / depths / groups / SE sizes
and total parameter count) against torchvision's `regnet_y_3_2gf` in
tests/test_oracle.py.  "parity unpinned" against historical timm checkpoints.
"""
import math

import torch
from torch import nn


class BatchNormAct2d(nn.BatchNorm2d):
    """timm 0.5.4 `BatchNormAct2d`: BatchNorm2d with the activation inside
    (the reference relies on this: transfuser.py:386 'The Relu is part of the batch norm')."""

    def __init__(self, num_features, apply_act=True):
        super().__init__(num_features, eps=1e-5, momentum=0.1)
        self.act = nn.ReLU(inplace=True) if apply_act else nn.Identity()

    def forward(self, x):
        return self.act(super().forward(x))


class ConvBnAct(nn.Module):
    def __init__(self, cin, cout, kernel_size=1, stride=1, groups=1, apply_act=True):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, kernel_size, stride=stride, padding=kernel_size // 2,
                              groups=groups, bias=False)
        self.bn = BatchNormAct2d(cout, apply_act=apply_act)

    def forward(self, x):
        return self.bn(self.conv(x))


class SEModule(nn.Module):
    def __init__(self, channels, rd_channels):
        super().__init__()
        self.fc1 = nn.Conv2d(channels, rd_channels, kernel_size=1, bias=True)
        self.bn = nn.Identity()
        self.act = nn.ReLU(inplace=True)
        self.fc2 = nn.Conv2d(rd_channels, channels, kernel_size=1, bias=True)
        self.gate = nn.Sigmoid()

    def forward(self, x):
        x_se = x.mean((2, 3), keepdim=True)
        x_se = self.fc2(self.act(self.bn(self.fc1(x_se))))
        return x * self.gate(x_se)


class Bottleneck(nn.Module):
    """RegNet Y block: 1x1 -> grouped 3x3 (stride) -> SE -> 1x1 (no act) -> +shortcut -> ReLU."""

    def __init__(self, in_chs, out_chs, stride, group_width, se_ratio):
        super().__init__()
        bottleneck_chs = out_chs  # bottle_ratio = 1
        groups = bottleneck_chs // group_width
        self.conv1 = ConvBnAct(in_chs, bottleneck_chs, 1)
        self.conv2 = ConvBnAct(bottleneck_chs, bottleneck_chs, 3, stride=stride, groups=groups)
        self.se = SEModule(bottleneck_chs, rd_channels=int(round(in_chs * se_ratio)))
        self.conv3 = ConvBnAct(bottleneck_chs, out_chs, 1, apply_act=False)
        self.act3 = nn.ReLU(inplace=True)
        if in_chs != out_chs or stride != 1:
            self.downsample = ConvBnAct(in_chs, out_chs, 1, stride=stride, apply_act=False)
        else:
            self.downsample = None

    def zero_init_last_bn(self):
        nn.init.zeros_(self.conv3.bn.weight)

    def forward(self, x):
        shortcut = x
        x = self.conv1(x)
        x = self.conv2(x)
        x = self.se(x)
        x = self.conv3(x)
        if self.downsample is not None:
            shortcut = self.downsample(shortcut)
        x += shortcut
        x = self.act3(x)
        return x


class RegStage(nn.Module):
    def __init__(self, in_chs, out_chs, stride, depth, group_width, se_ratio):
        super().__init__()
        for i in range(depth):
            self.add_module('b{}'.format(i + 1),
                            Bottleneck(in_chs if i == 0 else out_chs, out_chs,
                                       stride if i == 0 else 1, group_width, se_ratio))

    def forward(self, x):
        for block in self.children():
            x = block(x)
        return x


class ClassifierHead(nn.Module):
    def __init__(self, in_chs, num_classes):
        super().__init__()
        self.global_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(in_chs, num_classes)

    def forward(self, x):
        return self.fc(self.global_pool(x).flatten(1))


REGNETY_032 = dict(stem_width=32, widths=(72, 216, 576, 1512), depths=(2, 5, 13, 1),
                   group_w=24, se_ratio=0.25)


class RegNet(nn.Module):
    def __init__(self, cfg, in_chans=3, num_classes=1000):
        super().__init__()
        self.num_classes = num_classes
        self.stem = ConvBnAct(in_chans, cfg['stem_width'], 3, stride=2)
        self.feature_info = [dict(num_chs=cfg['stem_width'], reduction=2, module='stem')]
        prev, red = cfg['stem_width'], 2
        for i, (w, d) in enumerate(zip(cfg['widths'], cfg['depths'])):
            name = 's{}'.format(i + 1)
            self.add_module(name, RegStage(prev, w, 2, d, cfg['group_w'], cfg['se_ratio']))
            prev, red = w, red * 2
            self.feature_info.append(dict(num_chs=w, reduction=red, module=name))
        self.num_features = prev
        self.head = ClassifierHead(prev, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                fan_out = m.kernel_size[0] * m.kernel_size[1] * m.out_channels // m.groups
                m.weight.data.normal_(0, math.sqrt(2.0 / fan_out))
                if m.bias is not None:
                    m.bias.data.zero_()
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
            elif isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, mean=0.0, std=0.01)
                nn.init.zeros_(m.bias)
        for m in self.modules():
            if hasattr(m, 'zero_init_last_bn'):
                m.zero_init_last_bn()

    def forward_features(self, x):
        # timm 0.5.4: every child but the last (the head), in registration order.
        for block in list(self.children())[:-1]:
            x = block(x)
        return x

    def forward(self, x):
        for block in self.children():
            x = block(x)
        return x


def create_model(model_name, pretrained=False, in_chans=3, **kwargs):
    # pretrained=True (transfuser.py:380) would download ImageNet weights; there is
    # no network here, so random init is used (documented in DESIGN.md).
    if model_name != 'regnety_032':
        raise RuntimeError('oracle timm shim only restates regnety_032, got %r' % (model_name,))
    return RegNet(REGNETY_032, in_chans=in_chans)
