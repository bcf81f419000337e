"""ORACLE / TEST INFRASTRUCTURE ONLY — never imported by the product path.

The CPU oracle (oracle/torch_oracle.py) with the reference's default ResNet trunks (image resnet34, LiDAR resnet18; model.py:545)
in place of RegNetY-032: TransfuserBackbone.forward (transfuser.py:120-211, the ResNet branch of its stem: conv1 -> bn1 -> act1
-> maxpool, transfuser.py:136-143) and LateFusionBackbone.forward (late_fusion.py:72-111), restated with torch_oracle's own
contraction helpers, so its BF16_OPERANDS mode applies to them too. Pinned to the verbatim reference by
tests/golden/reference_resnet.npz (oracle/make_golden_resnet.py)."""
import contextlib

import torch
import torch.nn.functional as F

from oracle import torch_oracle as O

DEPTHS = {'resnet18': (2, 2, 2, 2), 'resnet34': (3, 4, 6, 3)}


def _basic_block(P, pre, x, train, stride):
    """timm 0.5.4 BasicBlock: conv1 (3x3, stride) -> bn1 -> ReLU -> conv2 -> bn2 -> + shortcut (downsample.0 / .1) -> ReLU."""
    y = O._bn(P, pre + 'bn1.', O._conv2d(x, P[pre + 'conv1.weight'], stride=stride, padding=1), train, True)
    y = O._bn(P, pre + 'bn2.', O._conv2d(y, P[pre + 'conv2.weight'], padding=1), train, False)
    if pre + 'downsample.0.weight' in P:
        x = O._bn(P, pre + 'downsample.1.', O._conv2d(x, P[pre + 'downsample.0.weight'], stride=stride), train, False)
    return F.relu(y + x)


def stem(P, pre, x, train):
    """conv1 (7x7 / 2) -> bn1 -> ReLU -> 3x3 / 2 max-pool."""
    return F.max_pool2d(O._bn(P, pre + 'bn1.', O._conv2d(x, P[pre + 'conv1.weight'], stride=2, padding=3), train, True), 3, 2, 1)


def stage(P, pre, arch, s, x, train):
    """layer{s+1} (s = 0..3): stride 1 for layer1, 2 for the others."""
    for i in range(DEPTHS[arch][s]):
        x = _basic_block(P, '%slayer%d.%d.' % (pre, s + 1, i), x, train, 2 if (i == 0 and s > 0) else 1)
    return x


def _conv1x1_or_skip(P, name, x):
    """change_channel_conv_* / reduce_channels_conv_*: parameterless nn.Sequential()s in the reference when the trunk already ends
    at perception_output_features (transfuser.py:92-97, late_fusion.py:45-52)."""
    return O._conv2d(x, P[name + '.weight'], P[name + '.bias']) if name + '.weight' in P else x


def _top_down(P, pre, l):
    up = lambda t: F.interpolate(t, scale_factor=2, mode='bilinear', align_corners=False)
    p5 = F.relu(O._conv2d(l, P[pre + 'c5_conv.weight'], P[pre + 'c5_conv.bias']))
    p4 = F.relu(O._conv2d(up(p5), P[pre + 'up_conv5.weight'], P[pre + 'up_conv5.bias']))
    p3 = F.relu(O._conv2d(up(p4), P[pre + 'up_conv4.weight'], P[pre + 'up_conv4.bias']))
    p2 = F.relu(O._conv2d(up(p3), P[pre + 'up_conv3.weight'], P[pre + 'up_conv3.bias']))
    return p2, p3, p4, p5


def _normalize(image):
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    return ((image / 255.0) - mean) / std


def backbone(P, image, lidar, trunks, cfg=O.Cfg, train=True, drop=None, pre='_model.', taps=None):
    """TransfuserBackbone.forward with ResNet trunks (image, LiDAR). `taps` (dict) collects the per-stage activations."""
    drop = drop or (lambda t, p: t)
    ie, le = pre + 'image_encoder.features.', pre + 'lidar_encoder._model.'
    x, l = stem(P, ie, _normalize(image), train), stem(P, le, lidar, train)
    for s in range(4):
        x, l = stage(P, ie, trunks[0], s, x, train), stage(P, le, trunks[1], s, l, train)
        xe = F.adaptive_avg_pool2d(x, (cfg.img_vert_anchors, cfg.img_horz_anchors))
        lemb = F.adaptive_avg_pool2d(l, (cfg.lidar_vert_anchors, cfg.lidar_horz_anchors))
        xo, lo = O._gpt(P, '%stransformer%d.' % (pre, s + 1), xe, lemb, cfg, train, drop)
        x = x + F.interpolate(xo, size=x.shape[2:], mode='bilinear', align_corners=False)
        l = l + F.interpolate(lo, size=l.shape[2:], mode='bilinear', align_corners=False)
        if taps is not None:
            taps['img_s%d' % (s + 1)], taps['lid_s%d' % (s + 1)] = x, l
    x = _conv1x1_or_skip(P, pre + 'change_channel_conv_image', x)
    l = _conv1x1_or_skip(P, pre + 'change_channel_conv_lidar', l)
    return _top_down(P, pre, l), x, x.mean((2, 3)) + l.mean((2, 3))


def backbone_late_fusion(P, image, lidar, trunks, cfg=O.Cfg, train=True, pre='_model.'):
    """LateFusionBackbone.forward with ResNet trunks: independent trunks, pooled sum, top-down on the LiDAR grid."""
    ie, le = pre + 'image_encoder.features.', pre + 'lidar_encoder._model.'
    x, l = stem(P, ie, _normalize(image), train), stem(P, le, lidar, train)
    for s in range(4):
        x, l = stage(P, ie, trunks[0], s, x, train), stage(P, le, trunks[1], s, l, train)
    x = _conv1x1_or_skip(P, pre + 'reduce_channels_conv_image', x)
    l = _conv1x1_or_skip(P, pre + 'reduce_channels_conv_lidar', l)
    return _top_down(P, pre, l), x, x.mean((2, 3)) + l.mean((2, 3))


@contextlib.contextmanager
def _backbone_of(trunks):
    """torch_oracle.forward with the backbone above in place of its RegNet one (same heads, decoders, GRU and losses)."""
    base = O._run_backbone

    def run(P, batch, cfg, train, drop, taps, backbone_name):
        lidar = torch.cat((batch['lidar'], batch['target_point_image']), dim=1)
        if backbone_name == 'late_fusion':
            return backbone_late_fusion(P, batch['rgb'], lidar, trunks, cfg, train)
        if backbone_name == 'transFuser':
            return backbone(P, batch['rgb'], lidar, trunks, cfg, train, drop, taps=taps)
        raise RuntimeError('%s cannot be built with ResNet trunks (the reference fails too)' % (backbone_name,))
    O._run_backbone = run
    try:
        yield
    finally:
        O._run_backbone = base


def forward(P, batch, trunks=('resnet34', 'resnet18'), cfg=O.Cfg, train=True, drop=None, taps=None, backbone_name='transFuser'):
    """LidarCenterNet.forward (model.py:733-805) with ResNet trunks: dict of the 11 losses."""
    if not all(t in DEPTHS for t in trunks):
        raise RuntimeError('resnet_oracle restates resnet18 / resnet34 trunks only, got %r' % (trunks,))
    with _backbone_of(tuple(trunks)):
        return O.forward(P, batch, cfg, train, drop, taps, backbone_name)
