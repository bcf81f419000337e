"""ORACLE / TEST INFRASTRUCTURE ONLY — never imported by the product path.

timm 0.5.4's BasicBlock ResNets `resnet18` / `resnet34` (the reference's default trunks, model.py:545), restated from timm's
published `resnet.py`: conv1 / bn1 / act1 / maxpool, layer1..4 of BasicBlocks with 1x1 downsample convs, global average pool +
flatten, fc; `in_chans`, `feature_info`, `num_features`, timm's initialisation (kaiming fan-out convs, zero last BatchNorm
scale of every block). timm and torchvision name these parameters alike; tests/test_resnet_trunks.py checks the names, shapes
and counts against torchvision's resnet18 / resnet34.

`with_resnets(timm_module)` lets the verbatim reference build them through the regnety_032 shim in oracle/shims/timm
(oracle/make_golden_resnet.py)."""
import contextlib

from torch import nn


class SelectAdaptivePool2d(nn.Module):
    """timm's global pool with pool_type='avg', flatten=True."""

    def forward(self, x):
        return x.mean((2, 3), keepdim=True).flatten(1)


class BasicBlock(nn.Module):
    """timm 0.5.4 ResNet BasicBlock (expansion 1): conv1 (3x3, stride) -> bn1 -> act1 -> conv2 (3x3) -> bn2 -> +shortcut -> act2."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.act1 = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.act2 = nn.ReLU(inplace=True)
        self.downsample = downsample

    def zero_init_last_bn(self):
        nn.init.zeros_(self.bn2.weight)

    def forward(self, x):
        shortcut = x
        x = self.act1(self.bn1(self.conv1(x)))
        x = self.bn2(self.conv2(x))
        if self.downsample is not None:
            shortcut = self.downsample(shortcut)
        x += shortcut
        return self.act2(x)


class ResNet(nn.Module):
    """timm 0.5.4 `ResNet` with BasicBlocks, the default stem (7x7 / 2 conv, 3x3 / 2 max-pool) and 1x1 downsample convs."""

    def __init__(self, layers, in_chans=3, num_classes=1000):
        super().__init__()
        self.num_classes = num_classes
        self.conv1 = nn.Conv2d(in_chans, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.act1 = nn.ReLU(inplace=True)
        self.feature_info = [dict(num_chs=64, reduction=2, module='act1')]
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        inplanes, red = 64, 4
        for i, (planes, depth) in enumerate(zip((64, 128, 256, 512), layers)):
            stride = 1 if i == 0 else 2
            blocks = []
            for b in range(depth):
                ds = None
                if b == 0 and (stride != 1 or inplanes != planes):
                    ds = nn.Sequential(nn.Conv2d(inplanes, planes, 1, stride=stride, bias=False), nn.BatchNorm2d(planes))
                blocks.append(BasicBlock(inplanes, planes, stride if b == 0 else 1, ds))
                inplanes = planes
            name = 'layer{}'.format(i + 1)
            self.add_module(name, nn.Sequential(*blocks))
            self.feature_info.append(dict(num_chs=planes, reduction=red, module=name))
            red *= 2
        self.num_features = 512
        self.global_pool = SelectAdaptivePool2d()
        self.fc = nn.Linear(self.num_features, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        for m in self.modules():
            if hasattr(m, 'zero_init_last_bn'):
                m.zero_init_last_bn()

    def forward_features(self, x):
        x = self.maxpool(self.act1(self.bn1(self.conv1(x))))
        return self.layer4(self.layer3(self.layer2(self.layer1(x))))

    def forward(self, x):
        return self.fc(self.global_pool(self.forward_features(x)))


RESNET_LAYERS = {'resnet18': (2, 2, 2, 2), 'resnet34': (3, 4, 6, 3)}


def create_model(model_name, pretrained=False, in_chans=3, **kwargs):
    """timm.create_model for resnet18 / resnet34 (random init: pretrained weights would need a download)."""
    if model_name not in RESNET_LAYERS:
        raise RuntimeError('oracle.timm_resnet restates resnet18 and resnet34 only, got %r' % (model_name,))
    return ResNet(RESNET_LAYERS[model_name], in_chans=in_chans)


@contextlib.contextmanager
def with_resnets(timm_module):
    """Inside the block, timm_module.create_model builds resnet18 / resnet34 here and every other name as before."""
    base = timm_module.create_model

    def create(model_name, pretrained=False, in_chans=3, **kwargs):
        if model_name in RESNET_LAYERS:
            return create_model(model_name, pretrained, in_chans, **kwargs)
        return base(model_name, pretrained=pretrained, in_chans=in_chans, **kwargs)
    timm_module.create_model = create
    try:
        yield
    finally:
        timm_module.create_model = base
