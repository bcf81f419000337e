"""ORACLE / TEST INFRASTRUCTURE ONLY — never imported by the product path (only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs may use it, and only as the checker / the CPU arm).

CPU restatement, in stock fp32 PyTorch functional ops, of the reference's training hot path:
  LidarCenterNet.forward            team_code_transfuser/model.py:733-805
  TransfuserBackbone.forward        transfuser.py:120-211   (GPT 333-366, Block 545-549, SelfAttention 510-527)
  SegDecoder / DepthDecoder         transfuser.py:239-246, 273-281
  forward_gru                       model.py:611-646
  LidarCenterNetHead.forward_single / get_targets / loss   model.py:127-147, 285-374, 149-248
  timm 0.5.4 RegNetY-032 blocks and mmdet 2.25 losses: restated from their published definitions (sources are not in the
  container; see oracle/shims/* — "parity unpinned" against the historical third-party packages).
It is a *functional* restatement over a flat {reference state_dict name: tensor} mapping, so that it cannot share code
(or bugs) with either the reference's nn.Module classes or the CUDA product.  It is pinned against the reference itself:
tests/test_oracle.py runs the verbatim reference (oracle/ref_import.py) and this file on the same weights/inputs in the
build container, and tests/golden/model_golden.npz holds reference outputs that this file must reproduce anywhere.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

REGNET_DEPTHS = (2, 5, 13, 1)
REGNET_WIDTHS = (72, 216, 576, 1512)
GROUP_W = 24


class Cfg:
    """The subset of GlobalConfig (config.py) the hot path reads, with train.py's overrides (n_layer 4, train.py:56)."""
    n_layer = 4
    n_head = 4
    img_vert_anchors, img_horz_anchors = 5, 22
    lidar_vert_anchors, lidar_horz_anchors = 8, 8
    embd_pdrop = attn_pdrop = resid_pdrop = 0.1
    bev_resolution_height = bev_resolution_width = 160
    lidar_resolution_height = lidar_resolution_width = 256
    num_dir_bins = 12
    pred_len = 4
    lidar_pos_x = 1.3
    ls_seg, ls_depth = 1.0, 10.0
    deconv_scale_factor_1, deconv_scale_factor_2 = 8, 4
    multitask = True


# ---- optional bf16-OPERAND mode (BASELINE config 2 is quoted in bf16): the same fp32 restatement, but every contraction the
# product runs on the tensor cores in its bf16 mode takes its two operands rounded to bf16 (round-to-nearest-even), accumulates in
# fp32 and keeps everything else (BatchNorm, softmax statistics, residuals, losses) in fp32 — the rounding POINTS of
# transfuser_b200's bf16 mode restated on the CPU, so its activations can be compared layer by layer at a tight tolerance instead of
# against the fp32 evaluation (which any bf16-operand implementation misses by 20-40 % at the deep stages of the batch-2 test point).
# Forward only: the rounding of gradients in the product's backward is not restated.
BF16_OPERANDS = [False]


def _q(t):
    return t.bfloat16().float()


def _tc_gemm(M, N, K):
    """Shapes transfuser_b200.gemm.tc_ok sends to the tensor-core GEMM (TMA: 16-byte aligned rows); the rest stays exact fp32."""
    return M >= 32 and N >= 16 and K >= 16 and K % 8 == 0 and N % 8 == 0


def _tc_conv(x, w, stride, groups):
    Cout, Cin, k = w.shape[0], w.shape[1] * groups, w.shape[2]
    if k == 1:
        Ho, Wo = (x.shape[2] - 1) // stride + 1, (x.shape[3] - 1) // stride + 1
        return groups == 1 and _tc_gemm(x.shape[0] * Ho * Wo, Cout, Cin)
    if Cin % 8 != 0:
        return False                                   # the two 3-channel stems
    if groups > 1:
        return Cin // groups == 24 and Cout // groups == 24
    nb = 16 if Cout <= 16 else 32 if Cout <= 32 else 64 if Cout <= 64 else 128
    return not (Cin <= 32 and nb > 64)


def _conv2d(x, w, b=None, stride=1, padding=0, groups=1):
    if BF16_OPERANDS[0] and _tc_conv(x, w, stride, groups):
        x, w = _q(x), _q(w)
    return F.conv2d(x, w, b, stride=stride, padding=padding, groups=groups)


def _linear(x, w, b=None):
    if BF16_OPERANDS[0] and _tc_gemm(x.numel() // x.shape[-1], w.shape[0], w.shape[1]):
        x, w = _q(x), _q(w)
    return F.linear(x, w, b)


def _bn(P, pre, x, train, act):
    y = F.batch_norm(x, P[pre + 'running_mean'], P[pre + 'running_var'], P[pre + 'weight'], P[pre + 'bias'],
                     training=train, momentum=0.1, eps=1e-5)
    return F.relu(y) if act else y


def _cba(P, pre, x, train, stride=1, groups=1, act=True, k=1):
    y = _conv2d(x, P[pre + 'conv.weight'], None, stride=stride, padding=k // 2, groups=groups)
    return _bn(P, pre + 'bn.', y, train, act)


def _bottleneck(P, pre, x, train, stride, has_ds):
    width = P[pre + 'conv1.conv.weight'].shape[0]
    y = _cba(P, pre + 'conv1.', x, train)
    y = _cba(P, pre + 'conv2.', y, train, stride=stride, groups=width // GROUP_W, k=3)
    s = y.mean((2, 3), keepdim=True)
    s = F.relu(_conv2d(s, P[pre + 'se.fc1.weight'], P[pre + 'se.fc1.bias']))
    s = torch.sigmoid(_conv2d(s, P[pre + 'se.fc2.weight'], P[pre + 'se.fc2.bias']))
    y = y * s
    y = _cba(P, pre + 'conv3.', y, train, act=False)
    sc = _cba(P, pre + 'downsample.', x, train, stride=stride, act=False) if has_ds else x
    return F.relu(y + sc)


def _stage(P, pre, x, train, depth):
    for i in range(depth):
        x = _bottleneck(P, '%sb%d.' % (pre, i + 1), x, train, 2 if i == 0 else 1, i == 0)
    return x


def _gpt(P, pre, img, lid, cfg, train, drop):
    bz, C = img.shape[0], img.shape[1]
    ih, iw, lh, lw = img.shape[2], img.shape[3], lid.shape[2], lid.shape[3]
    tok = torch.cat((img.permute(0, 2, 3, 1).reshape(bz, -1, C), lid.permute(0, 2, 3, 1).reshape(bz, -1, C)), dim=1)
    x = drop(P[pre + 'pos_emb'] + tok, cfg.embd_pdrop)
    T, nh = x.shape[1], cfg.n_head
    for i in range(cfg.n_layer):
        b = '%sblocks.%d.' % (pre, i)
        h = F.layer_norm(x, (C,), P[b + 'ln1.weight'], P[b + 'ln1.bias'])
        k = _linear(h, P[b + 'attn.key.weight'], P[b + 'attn.key.bias']).view(bz, T, nh, C // nh).transpose(1, 2)
        q = _linear(h, P[b + 'attn.query.weight'], P[b + 'attn.query.bias']).view(bz, T, nh, C // nh).transpose(1, 2)
        v = _linear(h, P[b + 'attn.value.weight'], P[b + 'attn.value.bias']).view(bz, T, nh, C // nh).transpose(1, 2)
        if BF16_OPERANDS[0]:
            # csrc/attn_tc.cu: q, k, v rounded to bf16, fp32 scores, the UNNORMALISED exp(s - max) rounded to bf16 as the operand of
            # the second product, row sum of the unrounded values applied afterwards (dropout is off in parity runs)
            q, k, v = _q(q), _q(k), _q(v)
            sc = (q @ k.transpose(-2, -1))
            e = ((sc - sc.amax(-1, keepdim=True)) * (1.0 / math.sqrt(C // nh))).exp()
            y = ((_q(e) @ v) / e.sum(-1, keepdim=True)).transpose(1, 2).reshape(bz, T, C)
        else:
            att = drop(F.softmax((q @ k.transpose(-2, -1)) * (1.0 / math.sqrt(C // nh)), dim=-1), cfg.attn_pdrop)
            y = (att @ v).transpose(1, 2).reshape(bz, T, C)
        x = x + drop(_linear(y, P[b + 'attn.proj.weight'], P[b + 'attn.proj.bias']), cfg.resid_pdrop)
        h = F.layer_norm(x, (C,), P[b + 'ln2.weight'], P[b + 'ln2.bias'])
        h = F.relu(_linear(h, P[b + 'mlp.0.weight'], P[b + 'mlp.0.bias']))
        x = x + drop(_linear(h, P[b + 'mlp.2.weight'], P[b + 'mlp.2.bias']), cfg.resid_pdrop)
    x = F.layer_norm(x, (C,), P[pre + 'ln_f.weight'], P[pre + 'ln_f.bias'])
    n_img = ih * iw
    # token-major buffers re-interpreted as NCHW without permuting back (transfuser.py:363-364)
    return x[:, :n_img, :].contiguous().view(bz, -1, ih, iw), x[:, n_img:, :].contiguous().view(bz, -1, lh, lw)


def backbone(P, image, lidar, cfg=Cfg, train=True, drop=None, pre='_model.', taps=None, lidar_bn='stem.bn.'):
    """TransfuserBackbone.forward (transfuser.py:120-211). `taps` (dict) collects per-stage activations."""
    drop = drop or (lambda t, p: t)
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    x = ((image / 255.0) - mean) / std
    ie, le = pre + 'image_encoder.features.', pre + 'lidar_encoder._model.'
    x = _bn(P, ie + 'stem.bn.', _conv2d(x, P[ie + 'stem.conv.weight'], None, stride=2, padding=1), train, True)
    l = _bn(P, le + lidar_bn, _conv2d(lidar, P[le + 'conv1.weight'], None, stride=2, padding=1), train, True)
    for s in range(4):
        x = _stage(P, '%ss%d.' % (ie, s + 1), x, train, REGNET_DEPTHS[s])
        l = _stage(P, '%ss%d.' % (le, s + 1), l, train, REGNET_DEPTHS[s])
        xe = F.adaptive_avg_pool2d(x, (cfg.img_vert_anchors, cfg.img_horz_anchors))
        lemb = F.adaptive_avg_pool2d(l, (cfg.lidar_vert_anchors, cfg.lidar_horz_anchors))
        xo, lo = _gpt(P, '%stransformer%d.' % (pre, s + 1), xe, lemb, cfg, train, drop)
        x = x + F.interpolate(xo, size=x.shape[2:], mode='bilinear', align_corners=False)
        l = l + F.interpolate(lo, size=l.shape[2:], mode='bilinear', align_corners=False)
        if taps is not None:
            taps['img_s%d' % (s + 1)], taps['lid_s%d' % (s + 1)] = x, l
    x = _conv2d(x, P[pre + 'change_channel_conv_image.weight'], P[pre + 'change_channel_conv_image.bias'])
    l = _conv2d(l, P[pre + 'change_channel_conv_lidar.weight'], P[pre + 'change_channel_conv_lidar.bias'])
    fused = x.mean((2, 3)) + l.mean((2, 3))
    up = lambda t: F.interpolate(t, scale_factor=2, mode='bilinear', align_corners=False)
    p5 = F.relu(_conv2d(l, P[pre + 'c5_conv.weight'], P[pre + 'c5_conv.bias']))
    p4 = F.relu(_conv2d(up(p5), P[pre + 'up_conv5.weight'], P[pre + 'up_conv5.bias']))
    p3 = F.relu(_conv2d(up(p4), P[pre + 'up_conv4.weight'], P[pre + 'up_conv4.bias']))
    p2 = F.relu(_conv2d(up(p3), P[pre + 'up_conv3.weight'], P[pre + 'up_conv3.bias']))
    return (p2, p3, p4, p5), x, fused


def backbone_latent_tf(P, image, lidar, cfg=Cfg, train=True, drop=None, pre='_model.'):
    """latentTFBackbone.forward (latentTF.py:118-217): the TransFuser architecture with the two LiDAR histogram channels replaced
    by a fixed positional grid in [-1, 1] (channel 0 varies top-down, channel 1 left-right, latentTF.py:132-137); the target
    point channel is kept. Its LidarEncoder deletes the whole stem, so the stem BN is keyed `bn1` (latentTF.py:195-196)."""
    H, W = lidar.shape[2], lidar.shape[3]
    rows = torch.linspace(-1, 1, cfg.lidar_resolution_width).view(1, 1, H, 1).expand(lidar.shape[0], 1, H, W)
    cols = torch.linspace(-1, 1, cfg.lidar_resolution_height).view(1, 1, 1, W).expand(lidar.shape[0], 1, H, W)
    lidar = torch.cat((rows.to(lidar.dtype), cols.to(lidar.dtype), lidar[:, 2:]), dim=1)
    return backbone(P, image, lidar, cfg, train, drop, pre, lidar_bn='bn1.')


def backbone_late_fusion(P, image, lidar, cfg=Cfg, train=True, pre='_model.'):
    """LateFusionBackbone.forward (late_fusion.py:72-111): independent trunks, 1x1 reduce, pooled sum, top-down on the LiDAR grid."""
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    x = ((image / 255.0) - mean) / std
    ie, le = pre + 'image_encoder.features.', pre + 'lidar_encoder._model.'
    x = _bn(P, ie + 'stem.bn.', _conv2d(x, P[ie + 'stem.conv.weight'], None, stride=2, padding=1), train, True)
    l = _bn(P, le + 'stem.bn.', _conv2d(lidar, P[le + 'stem.conv.weight'], None, stride=2, padding=1), train, True)
    for s in range(4):
        x = _stage(P, '%ss%d.' % (ie, s + 1), x, train, REGNET_DEPTHS[s])
        l = _stage(P, '%ss%d.' % (le, s + 1), l, train, REGNET_DEPTHS[s])
    x = _conv2d(x, P[pre + 'reduce_channels_conv_image.weight'], P[pre + 'reduce_channels_conv_image.bias'])
    l = _conv2d(l, P[pre + 'reduce_channels_conv_lidar.weight'], P[pre + 'reduce_channels_conv_lidar.bias'])
    fused = x.mean((2, 3)) + l.mean((2, 3))
    up = lambda t: F.interpolate(t, scale_factor=2, mode='bilinear', align_corners=False)
    p5 = F.relu(_conv2d(l, P[pre + 'c5_conv.weight'], P[pre + 'c5_conv.bias']))
    p4 = F.relu(_conv2d(up(p5), P[pre + 'up_conv5.weight'], P[pre + 'up_conv5.bias']))
    p3 = F.relu(_conv2d(up(p4), P[pre + 'up_conv4.weight'], P[pre + 'up_conv4.bias']))
    p2 = F.relu(_conv2d(up(p3), P[pre + 'up_conv3.weight'], P[pre + 'up_conv3.bias']))
    return (p2, p3, p4, p5), x, fused


def _gather_sum(emb, pts):
    """Sum of the 5 correspondences per cell (geometric_fusion.py:145-148): emb [B,C,h,w], pts [B,H,W,5,2] int64 (x, y) -> [B,C,H,W].
    The reference indexes B x B and takes the diagonal; per-sample advanced indexing is the same selection."""
    B, C = emb.shape[:2]
    H, W = pts.shape[1], pts.shape[2]
    e = emb.permute(0, 2, 3, 1)
    bi = torch.arange(B).view(B, 1)
    g = e[bi, pts[..., 1].reshape(B, -1), pts[..., 0].reshape(B, -1)]          # [B, H*W*5, C]
    return g.view(B, H, W, 5, C).sum(3).permute(0, 3, 1, 2)


def _proj3(P, pre, x):
    """image/lidar_projection{i}: 3 x (Linear + ReLU) over the channel dim (geometric_fusion.py:66-74)."""
    x = x.permute(0, 2, 3, 1)
    for j in (0, 2, 4):
        x = F.relu(_linear(x, P['%s%d.weight' % (pre, j)], P['%s%d.bias' % (pre, j)]))
    return x.permute(0, 3, 1, 2)


def backbone_geometric_fusion(P, image, lidar, bev_points, img_points, cfg=Cfg, train=True, pre='_model.'):
    """GeometricFusionBackbone.forward (geometric_fusion.py:98-296), n_scale 4, use_velocity False. Per scale: 1x1 embed to
    n_embd, pool to the anchor grids, gather-sum 5 projected correspondences from the other modality, 3-layer MLP,
    bilinear x(8,4,2,1), 1x1 back to the trunk width, residual add. Scale 4's image branch gathers from the scale-3
    LiDAR embedding (geometric_fusion.py:277, reproduced)."""
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    x = ((image / 255.0) - mean) / std
    ie, le = pre + 'image_encoder.features.', pre + 'lidar_encoder._model.'
    x = _bn(P, ie + 'stem.bn.', _conv2d(x, P[ie + 'stem.conv.weight'], None, stride=2, padding=1), train, True)
    l = _bn(P, le + 'bn1.', _conv2d(lidar, P[le + 'conv1.weight'], None, stride=2, padding=1), train, True)
    c1 = lambda t, n: _conv2d(t, P[pre + n + '.weight'], P[pre + n + '.bias'])
    prev_lidar_embd = None
    for s in range(4):
        i = s + 1
        x = _stage(P, '%ss%d.' % (ie, i), x, train, REGNET_DEPTHS[s])
        l = _stage(P, '%ss%d.' % (le, i), l, train, REGNET_DEPTHS[s])
        xe = F.adaptive_avg_pool2d(c1(x, 'image_conv%d' % i), (cfg.img_vert_anchors, cfg.img_horz_anchors))
        lemb = F.adaptive_avg_pool2d(c1(l, 'lidar_conv%d' % i), (cfg.lidar_vert_anchors, cfg.lidar_horz_anchors))
        bev_enc = _proj3(P, '%simage_projection%d.' % (pre, i), _gather_sum(xe, bev_points))
        img_enc = _proj3(P, '%slidar_projection%d.' % (pre, i), _gather_sum(prev_lidar_embd if i == 4 else lemb, img_points))
        if i < 4:
            sf = 2 ** (3 - s)
            bev_enc = F.interpolate(bev_enc, scale_factor=sf, mode='bilinear', align_corners=False)
            img_enc = F.interpolate(img_enc, scale_factor=sf, mode='bilinear', align_corners=False)
        l = l + c1(bev_enc, 'lidar_deconv%d' % i)
        x = x + c1(img_enc, 'image_deconv%d' % i)
        prev_lidar_embd = lemb
    x = c1(x, 'change_channel_conv_image')
    l = c1(l, 'change_channel_conv_lidar')
    fused = x.mean((2, 3)) + l.mean((2, 3))
    up = lambda t: F.interpolate(t, scale_factor=2, mode='bilinear', align_corners=False)
    p5 = F.relu(c1(l, 'c5_conv'))
    p4 = F.relu(c1(up(p5), 'up_conv5'))
    p3 = F.relu(c1(up(p4), 'up_conv4'))
    p2 = F.relu(c1(up(p3), 'up_conv3'))
    return (p2, p3, p4, p5), x, fused


def synthetic_correspondences(B, seed=0, cfg=Cfg):
    """Seeded int64 LiDAR<->camera correspondence indices of data.py:632-673's shape: bev_points [B,8,8,5,2] index the
    5x22 image anchor grid (x<22, y<5), cam_points [B,5,22,5,2] index the 8x8 BEV anchor grid."""
    g = torch.Generator().manual_seed(7000 + seed)
    ri = lambda hi, *s: torch.randint(0, hi, s, generator=g)
    lh, lw, ih, iw = cfg.lidar_vert_anchors, cfg.lidar_horz_anchors, cfg.img_vert_anchors, cfg.img_horz_anchors
    bev = torch.stack((ri(iw, B, lh, lw, 5), ri(ih, B, lh, lw, 5)), -1)
    cam = torch.stack((ri(lw, B, ih, iw, 5), ri(lh, B, ih, iw, 5)), -1)
    return bev, cam


def _decoder(P, pre, x, cfg):
    c = lambda t, n, act=True: (F.relu if act else (lambda z: z))(_conv2d(t, P['%s%s.weight' % (pre, n)], P['%s%s.bias' % (pre, n)], padding=1))
    x = c(c(x, 'deconv1.0'), 'deconv1.2')
    x = F.interpolate(x, scale_factor=cfg.deconv_scale_factor_1, mode='bilinear', align_corners=False)
    x = c(c(x, 'deconv2.0'), 'deconv2.2')
    x = F.interpolate(x, scale_factor=cfg.deconv_scale_factor_2, mode='bilinear', align_corners=False)
    return c(c(x, 'deconv3.0'), 'deconv3.2', act=False)


def gru_waypoints(P, fused, target_point, cfg):
    z = fused
    for i in (0, 2, 4):
        z = F.relu(_linear(z, P['join.%d.weight' % i], P['join.%d.bias' % i]))
    x = torch.zeros(z.shape[0], 2)
    tp = target_point.clone()
    tp[:, 1] *= -1
    out = []
    for _ in range(cfg.pred_len):
        gi = _linear(torch.cat([x, tp], dim=1), P['decoder.weight_ih'], P['decoder.bias_ih'])
        gh = _linear(z, P['decoder.weight_hh'], P['decoder.bias_hh'])
        i_r, i_z, i_n = gi.chunk(3, 1)
        h_r, h_z, h_n = gh.chunk(3, 1)
        r, u = torch.sigmoid(i_r + h_r), torch.sigmoid(i_z + h_z)
        n = torch.tanh(i_n + r * h_n)
        z = (1 - u) * n + u * z
        x = _linear(z, P['output.weight'], P['output.bias'])[:, :2] + x
        out.append(x)
    wp = torch.stack(out, dim=1)
    return torch.cat((wp[:, :, :1] - cfg.lidar_pos_x, wp[:, :, 1:]), dim=2)


def _gaussian_radius(h, w, mo=0.1):
    r1 = ((h + w) - math.sqrt((h + w) ** 2 - 4 * (w * h * (1 - mo) / (1 + mo)))) / 2
    r2 = (2 * (h + w) - math.sqrt((2 * (h + w)) ** 2 - 16 * ((1 - mo) * w * h))) / 8
    a3, b3, c3 = 4 * mo, -2 * mo * (h + w), (mo - 1) * w * h
    r3 = (b3 + math.sqrt(b3 ** 2 - 4 * a3 * c3)) / (2 * a3)
    return min(r1, r2, r3)


def centernet_targets(label, cfg, H=64, W=64):
    """get_targets (model.py:285-374). Returns dict of target maps and avg_factor."""
    B = label.shape[0]
    ratio = float(W / cfg.lidar_resolution_width)
    ratio_h = float(H / cfg.lidar_resolution_height)
    heat = torch.zeros(B, 1, H, W)
    t = {k: torch.zeros(B, c, H, W) for k, c in (('wh', 2), ('offset', 2), ('yaw_res', 1), ('velocity', 1), ('weight', 2))}
    yaw_cls = torch.zeros(B, H, W, dtype=torch.long)
    brake = torch.zeros(B, H, W, dtype=torch.long)
    apc = 2 * np.pi / float(cfg.num_dir_bins)
    for b in range(B):
        for j in range(label.shape[1]):
            box = label[b, j]
            if float(box.sum()) == 0.:
                continue
            ct = box[:2] * ratio
            x, y = int(ct[0]), int(ct[1])
            bh, bw = box[3] * ratio_h, box[2] * ratio
            r = max(2, int(_gaussian_radius(float(bh), float(bw))))
            sig = (2 * r + 1) / 6
            g = torch.arange(-r, r + 1, dtype=torch.float32)
            k = (-(g.view(1, -1) ** 2 + g.view(-1, 1) ** 2) / (2 * sig * sig)).exp()
            k[k < torch.finfo(torch.float32).eps * k.max()] = 0
            le, ri, to, bo = min(x, r), min(W - x, r + 1), min(y, r), min(H - y, r + 1)
            region = heat[b, 0, y - to:y + bo, x - le:x + ri]
            heat[b, 0, y - to:y + bo, x - le:x + ri] = torch.maximum(region, k[r - to:r + bo, r - le:r + ri])
            t['wh'][b, 0, y, x], t['wh'][b, 1, y, x] = bw, bh
            ang = box[4] % (2 * np.pi)
            sh = (ang + apc / 2) % (2 * np.pi)
            cls = torch.div(sh, apc, rounding_mode='trunc')
            yaw_cls[b, y, x] = cls.long()
            t['yaw_res'][b, 0, y, x] = sh - (cls * apc + apc / 2)
            t['velocity'][b, 0, y, x] = box[5]
            brake[b, y, x] = box[6].long()
            t['offset'][b, 0, y, x], t['offset'][b, 1, y, x] = ct[0] - x, ct[1] - y
            t['weight'][b, :, y, x] = 1
    t.update(heat=heat, yaw_cls=yaw_cls, brake=brake)
    return t, max(1, int(heat.eq(1).sum()))


def centernet_losses(preds, label, cfg):
    """LidarCenterNetHead.loss (model.py:149-248) with mmdet's weighted-loss reduction (sum / avg_factor)."""
    heat, wh, off, ycls, yres, vel, brk = preds
    t, avg = centernet_targets(label, cfg, heat.shape[2], heat.shape[3])
    eps = 1e-12
    pos = t['heat'].eq(1)
    focal = (-(heat + eps).log() * (1 - heat).pow(2) * pos - (1 - heat + eps).log() * heat.pow(2) * (1 - t['heat']).pow(4))
    w2, w1 = t['weight'], t['weight'][:, :1]
    out = {'loss_center_heatmap': focal.sum() / avg,
           'loss_wh': 0.1 * ((wh - t['wh']).abs() * w2).sum() / (avg * 2),
           'loss_offset': ((off - t['offset']).abs() * w2).sum() / (avg * 2)}
    # CE maps are (B,H,W); the weight is (B,1,H,W): the product broadcasts to (B,B,H,W) (model.py:220-224, 235-239)
    out['loss_yaw_class'] = (F.cross_entropy(ycls, t['yaw_cls'], reduction='none') * w1).sum() / avg
    d = (yres - t['yaw_res']).abs()
    out['loss_yaw_res'] = (torch.where(d < 1.0, 0.5 * d * d, d - 0.5) * w1).sum() / avg
    out['loss_velocity'] = ((vel - t['velocity']).abs() * w1).sum() / avg
    out['loss_brake'] = (F.cross_entropy(brk, t['brake'], reduction='none') * w1).sum() / avg
    return out


HEAD_NAMES = ('heatmap_head', 'wh_head', 'offset_head', 'yaw_class_head', 'yaw_res_head', 'velocity_head', 'brake_head')


def _run_backbone(P, batch, cfg, train, drop, taps, backbone_name):
    lidar = torch.cat((batch['lidar'], batch['target_point_image']), dim=1)
    if backbone_name == 'late_fusion':
        return backbone_late_fusion(P, batch['rgb'], lidar, cfg, train)
    if backbone_name == 'geometric_fusion':
        return backbone_geometric_fusion(P, batch['rgb'], lidar, batch['bev_points'], batch['cam_points'], cfg, train)
    if backbone_name == 'latentTF':
        return backbone_latent_tf(P, batch['rgb'], lidar, cfg, train, drop)
    return backbone(P, batch['rgb'], lidar, cfg, train, drop, taps=taps)


def _conv_pair(P, name, x):
    return _conv2d(F.relu(_conv2d(x, P[name + '.0.weight'], P[name + '.0.bias'], padding=1)), P[name + '.2.weight'], P[name + '.2.bias'])


def head_preds(P, feat):
    """LidarCenterNetHead.forward_single (model.py:101-125): seven conv3x3+ReLU+conv1x1 branches, sigmoid on the heatmap."""
    preds = [_conv_pair(P, 'head.' + n, feat) for n in HEAD_NAMES]
    preds[0] = preds[0].sigmoid()
    return preds


def forward(P, batch, cfg=Cfg, train=True, drop=None, taps=None, backbone_name='transFuser'):
    """LidarCenterNet.forward (model.py:733-805): dict of the 11 losses. `P` maps reference state_dict names to tensors."""
    feats, img_grid, fused = _run_backbone(P, batch, cfg, train, drop, taps, backbone_name)
    loss = {}
    wp = gru_waypoints(P, fused, batch['target_point'], cfg)
    pb = F.interpolate(_conv_pair(P, 'pred_bev', feats[0]), (cfg.bev_resolution_height, cfg.bev_resolution_width), mode='bilinear', align_corners=True)
    loss['loss_wp'] = (wp - batch['ego_waypoint']).abs().mean()
    loss['loss_bev'] = F.cross_entropy(pb, batch['bev'], weight=torch.tensor([1., 1., 3.]))
    loss.update(centernet_losses(head_preds(P, feats[0]), batch['label'], cfg))
    if cfg.multitask:
        seg = _decoder(P, 'seg_decoder.', img_grid, cfg)
        depth = torch.sigmoid(_decoder(P, 'depth_decoder.', img_grid, cfg)).squeeze(1)
        loss['loss_depth'] = cfg.ls_depth * F.l1_loss(depth, batch['depth'])
        loss['loss_semantic'] = cfg.ls_seg * F.cross_entropy(seg, batch['semantic'])
    if taps is not None:
        taps.update(p2=feats[0], img_grid=img_grid, fused=fused, pred_wp=wp)
    return loss


# ------------------------------------------------------------------ inference: CenterNet decode + forward_ego
def decode_heatmap(preds, num_dir_bins=12, k=100, kernel=3, ratio=4.0, stable=False):
    """LidarCenterNetHead.decode_heatmap (model.py:436-497) with mmdet 2.25.0's get_local_maximum / get_topk_from_heatmap /
    transpose_and_gather_feat folded in. preds: the 7 NCHW maps of head_preds (heatmap already a probability).
    Returns boxes [B,k,8] = (x, y, w, h in LiDAR-BEV pixels, yaw, velocity, brake class, score) sorted by score, labels [B,k].
    torch.topk leaves the order of equal scores unspecified; `stable=True` fixes it (equal scores by ascending cell index,
    the CUDA kernel's rule) and is otherwise the same computation."""
    heat, wh, off, yaw_cls, yaw_res, vel, brake = preds
    B, _, H, W = heat.shape
    peak = F.max_pool2d(heat, kernel, stride=1, padding=(kernel - 1) // 2) == heat
    kept = (heat * peak.float()).view(B, -1)
    if stable:
        score, flat = torch.sort(kept, dim=1, descending=True, stable=True)
        score, flat = score[:, :k], flat[:, :k]
    else:
        score, flat = torch.topk(kept, k)
    labels, cell = flat // (H * W), flat % (H * W)
    ys, xs = (cell // W).float(), (cell % W).float()
    at = lambda t: t.permute(0, 2, 3, 1).reshape(B, H * W, t.shape[1]).gather(1, cell.unsqueeze(2).expand(-1, -1, t.shape[1]))
    wh, off = at(wh), at(off)
    yaw = at(yaw_cls).argmax(-1).float() * (2 * np.pi / float(num_dir_bins)) + at(yaw_res).squeeze(2)   # class2angle, model.py:269-283
    yaw = torch.where(yaw > np.pi, yaw - 2 * np.pi, yaw)
    geom = torch.stack([xs + off[..., 0], ys + off[..., 1], wh[..., 0], wh[..., 1]], dim=2) * ratio
    rest = torch.stack([yaw, at(vel)[..., 0], at(brake).argmax(-1).float(), score], dim=2)
    return torch.cat((geom, rest), dim=2), labels


def bbox_local_metric(bbox, pixels_per_meter=8.0, bounding_box_divisor=2.0, lidar_pos=(1.3, 0.0, 2.5)):
    """LidarCenterNet.get_bbox_local_metric (model.py:810-844): one decoded row -> (6x3 array: 4 corners, centre, velocity
    tip in the ego frame, metres; brake; confidence). The BEV-pixel -> LiDAR map is the inverse of utils.py:29-37's T = 8*[[0,-1,16],[-1,0,32]]."""
    x, y, w, h, yaw, speed, brake, confidence = bbox
    w = w / bounding_box_divisor / pixels_per_meter
    h = h / bounding_box_divisor / pixels_per_meter
    T = np.array([[0, -1, 16], [-1, 0, 32], [0, 0, 1]], dtype=np.float32)
    T[:2, :] *= 8
    c = np.linalg.inv(T) @ np.array([x, y, 1.0]) + np.array(lidar_pos)
    c[1] = -c[1]
    pts = np.array([[-h, -w, 1], [-h, w, 1], [h, w, 1], [h, -w, 1], [0, 0, 1], [0, h * speed * 0.5, 1]])
    R = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
    return pts @ R.T + np.array([c[0], c[1], 0]), brake, confidence


def forward_ego(P, batch, cfg=Cfg, backbone_name='transFuser', bb_confidence_threshold=0.3):
    """LidarCenterNet.forward_ego (model.py:685-731) in eval mode: (pred_wp, list of 6x3 boxes of sample 0 above threshold)."""
    feats, _, fused = _run_backbone(P, batch, cfg, False, None, None, backbone_name)
    wp = gru_waypoints(P, fused, batch['target_point'], cfg)
    boxes, _ = decode_heatmap(head_preds(P, feats[0]), cfg.num_dir_bins)
    b0 = boxes[0]
    b0 = b0[b0[:, -1] > bb_confidence_threshold]
    return wp, [bbox_local_metric(r) for r in b0.detach().cpu().numpy()], boxes


# ------------------------------------------------------------------ deterministic synthetic data / weights
def synthetic_batch(B, seed=0, n_boxes=None):
    """Seeded synthetic batch of SURVEY.md §8(d)'s shape (CPU tensors, reference dtypes)."""
    g = torch.Generator().manual_seed(1000 + seed)
    r = lambda *s: torch.rand(*s, generator=g)
    batch = dict(
        rgb=torch.randint(0, 256, (B, 3, 160, 704), generator=g).float(),
        lidar=(torch.randint(0, 6, (B, 2, 256, 256), generator=g).float() / 5) * (r(B, 2, 256, 256) < 0.1),
        target_point_image=(r(B, 1, 256, 256) < 0.002).float(),
        target_point=r(B, 2) * 20 - 10,
        ego_vel=r(B, 1) * 8,
        ego_waypoint=torch.randn(B, 4, 2, generator=g) * 3,
        bev=torch.randint(0, 3, (B, 160, 160), generator=g),
        semantic=torch.randint(0, 7, (B, 160, 704), generator=g),
        depth=r(B, 160, 704),
    )
    label = torch.zeros(B, 20, 7)
    for b in range(B):
        k = int(torch.randint(0, 21, (1,), generator=g)) if n_boxes is None else n_boxes
        if k:
            label[b, :k, 0:2] = r(k, 2) * 253 + 1
            label[b, :k, 2:4] = r(k, 2) * 32 + 8
            label[b, :k, 4] = r(k) * 2 * math.pi - math.pi
            label[b, :k, 5] = r(k) * 8
            label[b, :k, 6] = (r(k) < 0.5).float()
    batch['label'] = label
    return batch


def deterministic_state(named_shapes, seed=0):
    """Machine-independent parameter values keyed by name (CPU generator): scaled normal weights, positive BN scales /
    variances, so that every layer (including zero-initialised ones in the reference) carries signal in parity tests."""
    import zlib
    out = {}
    for name, shape in named_shapes:
        g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(name.encode()))
        leaf = name.rsplit('.', 1)[-1]
        if leaf == 'num_batches_tracked':
            out[name] = torch.zeros((), dtype=torch.long)
        elif leaf == 'running_var':
            out[name] = torch.rand(shape, generator=g) * 0.5 + 0.75
        elif leaf == 'running_mean':
            out[name] = torch.randn(shape, generator=g) * 0.1
        elif len(shape) <= 1 and leaf == 'weight':       # norm scales
            out[name] = torch.rand(shape, generator=g) * 0.5 + 0.75
        elif len(shape) <= 1:                             # biases
            out[name] = torch.randn(shape, generator=g) * 0.05
        elif leaf == 'pos_emb':
            out[name] = torch.randn(shape, generator=g) * 0.1
        else:
            fan_in = int(np.prod(shape[1:]))
            out[name] = torch.randn(shape, generator=g) * (1.0 / math.sqrt(fan_in))
    return out
