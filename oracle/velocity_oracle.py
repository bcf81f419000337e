"""ORACLE / TEST INFRASTRUCTURE ONLY — never imported by the product path.

The CPU oracle (oracle/torch_oracle.py) with the ego-speed input, use_velocity=True, for the four backbones: a Linear(1, C)
embedding of the speed [B, 1] added
  - to every token of each GPT before the embedding dropout (transFuser, latentTF: transfuser.py:352-355, latentTF.py:288-292);
  - to the fused vector (late_fusion.py:107-109);
  - to the LiDAR and the image map of each scale, after that scale's residual adds (geometric_fusion.py:142-271).
Restated with torch_oracle's own helpers, so its BF16_OPERANDS mode applies here too. forward / forward_ego are torch_oracle's,
with the backbone below in their place (as oracle/resnet_oracle.py does). Pinned to the verbatim reference by
tests/golden/reference_velocity.npz (oracle/make_golden_velocity.py)."""
import contextlib
import math

import torch
import torch.nn.functional as F

from oracle import torch_oracle as O


def vel_emb(P, name, velocity):
    """vel_emb(v) = Linear(1, C) of the ego speed [B, 1] -> [B, C]."""
    return F.linear(velocity, P[name + '.weight'], P[name + '.bias'])


def _gpt(P, pre, img, lid, cfg, train, drop, velocity):
    """torch_oracle._gpt with vel_emb(velocity) added to every token (transfuser.py:352-355)."""
    bz, C = img.shape[0], img.shape[1]
    ih, iw, lh, lw = img.shape[2], img.shape[3], lid.shape[2], lid.shape[3]
    tok = torch.cat((img.permute(0, 2, 3, 1).reshape(bz, -1, C), lid.permute(0, 2, 3, 1).reshape(bz, -1, C)), dim=1)
    x = drop(P[pre + 'pos_emb'] + tok + vel_emb(P, pre + 'vel_emb', velocity).unsqueeze(1), cfg.embd_pdrop)
    T, nh = x.shape[1], cfg.n_head
    for i in range(cfg.n_layer):
        b = '%sblocks.%d.' % (pre, i)
        h = F.layer_norm(x, (C,), P[b + 'ln1.weight'], P[b + 'ln1.bias'])
        k = O._linear(h, P[b + 'attn.key.weight'], P[b + 'attn.key.bias']).view(bz, T, nh, C // nh).transpose(1, 2)
        q = O._linear(h, P[b + 'attn.query.weight'], P[b + 'attn.query.bias']).view(bz, T, nh, C // nh).transpose(1, 2)
        v = O._linear(h, P[b + 'attn.value.weight'], P[b + 'attn.value.bias']).view(bz, T, nh, C // nh).transpose(1, 2)
        if O.BF16_OPERANDS[0]:
            q, k, v = O._q(q), O._q(k), O._q(v)
            sc = (q @ k.transpose(-2, -1))
            e = ((sc - sc.amax(-1, keepdim=True)) * (1.0 / math.sqrt(C // nh))).exp()
            y = ((O._q(e) @ v) / e.sum(-1, keepdim=True)).transpose(1, 2).reshape(bz, T, C)
        else:
            att = drop(F.softmax((q @ k.transpose(-2, -1)) * (1.0 / math.sqrt(C // nh)), dim=-1), cfg.attn_pdrop)
            y = (att @ v).transpose(1, 2).reshape(bz, T, C)
        x = x + drop(O._linear(y, P[b + 'attn.proj.weight'], P[b + 'attn.proj.bias']), cfg.resid_pdrop)
        h = F.layer_norm(x, (C,), P[b + 'ln2.weight'], P[b + 'ln2.bias'])
        h = F.relu(O._linear(h, P[b + 'mlp.0.weight'], P[b + 'mlp.0.bias']))
        x = x + drop(O._linear(h, P[b + 'mlp.2.weight'], P[b + 'mlp.2.bias']), cfg.resid_pdrop)
    x = F.layer_norm(x, (C,), P[pre + 'ln_f.weight'], P[pre + 'ln_f.bias'])
    n_img = ih * iw
    return x[:, :n_img, :].contiguous().view(bz, -1, ih, iw), x[:, n_img:, :].contiguous().view(bz, -1, lh, lw)


def _image_prep(image):
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    return ((image / 255.0) - mean) / std


def _top_down(P, pre, l):
    up = lambda t: F.interpolate(t, scale_factor=2, mode='bilinear', align_corners=False)
    p5 = F.relu(O._conv2d(l, P[pre + 'c5_conv.weight'], P[pre + 'c5_conv.bias']))
    p4 = F.relu(O._conv2d(up(p5), P[pre + 'up_conv5.weight'], P[pre + 'up_conv5.bias']))
    p3 = F.relu(O._conv2d(up(p4), P[pre + 'up_conv4.weight'], P[pre + 'up_conv4.bias']))
    p2 = F.relu(O._conv2d(up(p3), P[pre + 'up_conv3.weight'], P[pre + 'up_conv3.bias']))
    return p2, p3, p4, p5


def backbone(P, image, lidar, velocity, cfg=O.Cfg, train=True, drop=None, pre='_model.', lidar_bn='stem.bn.'):
    """TransfuserBackbone.forward (transfuser.py:120-211) with use_velocity."""
    drop = drop or (lambda t, p: t)
    ie, le = pre + 'image_encoder.features.', pre + 'lidar_encoder._model.'
    x = O._bn(P, ie + 'stem.bn.', O._conv2d(_image_prep(image), P[ie + 'stem.conv.weight'], None, stride=2, padding=1), train, True)
    l = O._bn(P, le + lidar_bn, O._conv2d(lidar, P[le + 'conv1.weight'], None, stride=2, padding=1), train, True)
    for s in range(4):
        x = O._stage(P, '%ss%d.' % (ie, s + 1), x, train, O.REGNET_DEPTHS[s])
        l = O._stage(P, '%ss%d.' % (le, s + 1), l, train, O.REGNET_DEPTHS[s])
        xe = F.adaptive_avg_pool2d(x, (cfg.img_vert_anchors, cfg.img_horz_anchors))
        lemb = F.adaptive_avg_pool2d(l, (cfg.lidar_vert_anchors, cfg.lidar_horz_anchors))
        xo, lo = _gpt(P, '%stransformer%d.' % (pre, s + 1), xe, lemb, cfg, train, drop, velocity)
        x = x + F.interpolate(xo, size=x.shape[2:], mode='bilinear', align_corners=False)
        l = l + F.interpolate(lo, size=l.shape[2:], mode='bilinear', align_corners=False)
    x = O._conv2d(x, P[pre + 'change_channel_conv_image.weight'], P[pre + 'change_channel_conv_image.bias'])
    l = O._conv2d(l, P[pre + 'change_channel_conv_lidar.weight'], P[pre + 'change_channel_conv_lidar.bias'])
    return _top_down(P, pre, l), x, x.mean((2, 3)) + l.mean((2, 3))


def backbone_latent_tf(P, image, lidar, velocity, cfg=O.Cfg, train=True, drop=None, pre='_model.'):
    """latentTFBackbone.forward (latentTF.py:118-217) with use_velocity: the positional grid in place of the LiDAR histogram."""
    H, W = lidar.shape[2], lidar.shape[3]
    rows = torch.linspace(-1, 1, cfg.lidar_resolution_width).view(1, 1, H, 1).expand(lidar.shape[0], 1, H, W)
    cols = torch.linspace(-1, 1, cfg.lidar_resolution_height).view(1, 1, 1, W).expand(lidar.shape[0], 1, H, W)
    lidar = torch.cat((rows.to(lidar.dtype), cols.to(lidar.dtype), lidar[:, 2:]), dim=1)
    return backbone(P, image, lidar, velocity, cfg, train, drop, pre, lidar_bn='bn1.')


def backbone_late_fusion(P, image, lidar, velocity, cfg=O.Cfg, train=True, pre='_model.'):
    """LateFusionBackbone.forward (late_fusion.py:72-111) with use_velocity: the embedding is added to the fused vector only."""
    feats, grid, fused = O.backbone_late_fusion(P, image, lidar, cfg, train, pre)
    return feats, grid, fused + vel_emb(P, pre + 'vel_emb', velocity)


def backbone_geometric_fusion(P, image, lidar, bev_points, img_points, velocity, cfg=O.Cfg, train=True, pre='_model.'):
    """GeometricFusionBackbone.forward (geometric_fusion.py:98-296) with use_velocity: torch_oracle's restatement, with
    vel_emb_i(velocity) added to both full-resolution maps of scale i after that scale's residual adds, in the reference's order."""
    ie, le = pre + 'image_encoder.features.', pre + 'lidar_encoder._model.'
    x = O._bn(P, ie + 'stem.bn.', O._conv2d(_image_prep(image), P[ie + 'stem.conv.weight'], None, stride=2, padding=1), train, True)
    l = O._bn(P, le + 'bn1.', O._conv2d(lidar, P[le + 'conv1.weight'], None, stride=2, padding=1), train, True)
    c1 = lambda t, n: O._conv2d(t, P[pre + n + '.weight'], P[pre + n + '.bias'])
    prev_lidar_embd = None
    for s in range(4):
        i = s + 1
        x = O._stage(P, '%ss%d.' % (ie, i), x, train, O.REGNET_DEPTHS[s])
        l = O._stage(P, '%ss%d.' % (le, i), l, train, O.REGNET_DEPTHS[s])
        xe = F.adaptive_avg_pool2d(c1(x, 'image_conv%d' % i), (cfg.img_vert_anchors, cfg.img_horz_anchors))
        lemb = F.adaptive_avg_pool2d(c1(l, 'lidar_conv%d' % i), (cfg.lidar_vert_anchors, cfg.lidar_horz_anchors))
        bev_enc = O._proj3(P, '%simage_projection%d.' % (pre, i), O._gather_sum(xe, bev_points))
        img_enc = O._proj3(P, '%slidar_projection%d.' % (pre, i), O._gather_sum(prev_lidar_embd if i == 4 else lemb, img_points))
        if i < 4:
            sf = 2 ** (3 - s)
            bev_enc = F.interpolate(bev_enc, scale_factor=sf, mode='bilinear', align_corners=False)
            img_enc = F.interpolate(img_enc, scale_factor=sf, mode='bilinear', align_corners=False)
        e = vel_emb(P, '%svel_emb%d' % (pre, i), velocity)[:, :, None, None]
        l = l + c1(bev_enc, 'lidar_deconv%d' % i) + e
        x = x + c1(img_enc, 'image_deconv%d' % i) + e
        prev_lidar_embd = lemb
    x = c1(x, 'change_channel_conv_image')
    l = c1(l, 'change_channel_conv_lidar')
    return _top_down(P, pre, l), x, x.mean((2, 3)) + l.mean((2, 3))


def run_backbone(P, batch, cfg, train, drop, taps, backbone_name):
    """torch_oracle._run_backbone with use_velocity: reads batch['ego_vel'] [B, 1]. (`taps` is not collected.)"""
    lidar = torch.cat((batch['lidar'], batch['target_point_image']), dim=1)
    v = batch['ego_vel']
    if backbone_name == 'late_fusion':
        return backbone_late_fusion(P, batch['rgb'], lidar, v, cfg, train)
    if backbone_name == 'geometric_fusion':
        return backbone_geometric_fusion(P, batch['rgb'], lidar, batch['bev_points'], batch['cam_points'], v, cfg, train)
    if backbone_name == 'latentTF':
        return backbone_latent_tf(P, batch['rgb'], lidar, v, cfg, train, drop)
    return backbone(P, batch['rgb'], lidar, v, cfg, train, drop)


@contextlib.contextmanager
def _with_velocity():
    base = O._run_backbone
    O._run_backbone = run_backbone
    try:
        yield
    finally:
        O._run_backbone = base


def forward(P, batch, cfg=O.Cfg, train=True, drop=None, backbone_name='transFuser'):
    """LidarCenterNet.forward (model.py:733-805) with use_velocity: dict of the 11 losses."""
    with _with_velocity():
        return O.forward(P, batch, cfg, train, drop, None, backbone_name)


def forward_ego(P, batch, cfg=O.Cfg, backbone_name='transFuser'):
    """LidarCenterNet.forward_ego (model.py:685-731) in eval mode with use_velocity."""
    with _with_velocity():
        return O.forward_ego(P, batch, cfg, backbone_name)
