"""H100-native `TransfuserBackbone` — drop-in for team_code_transfuser/transfuser.py:7-211.

Same constructor signature, same `forward(image, lidar, velocity) -> ((p2, p3, p4, p5), image_features_grid,
fused_features)` contract (NCHW fp32 in / out), and the same parameter / buffer names and shapes as the reference
(including the alias keys created by ImageCNN / LidarEncoder, transfuser.py:383-393, 475-486), so reference checkpoints
load unchanged. The nn.Conv2d / nn.BatchNorm2d / nn.Linear / nn.LayerNorm objects below are *parameter containers only*:
their forward is never called — every op runs through transfuser_b200.ops (hand-written sm_90a kernels, NHWC inside).

The RegNetY-3.2GF definition (timm 0.5.4 `regnety_032`: stem 32, widths 72/216/576/1512, depths 2/5/13/1, group width 24,
SE ratio 0.25) is restated from timm's published config; timm itself is not a dependency."""
import torch
from torch import nn

from . import ops

REGNETY_032 = dict(stem_width=32, widths=(72, 216, 576, 1512), depths=(2, 5, 13, 1), group_w=24, se_ratio=0.25)


class _ConvBn(nn.Module):
    """`conv` + `bn` (BatchNormAct2d in timm: the ReLU lives inside the norm layer)."""

    def __init__(self, cin, cout, k=1, stride=1, groups=1, act=True):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, stride=stride, padding=k // 2, groups=groups, bias=False)
        self.bn = nn.BatchNorm2d(cout)
        self.stride, self.groups, self.act = stride, groups, act

    def run(self, x, emit16=False, residual=None, pool=False):
        """emit16: the output is the operand of a tensor-core GEMM / conv next (bf16 mode: BatchNorm writes its bf16 copy too).
        residual: relu(bn(conv(x)) + residual) — the Bottleneck tail, add and ReLU fused into the BatchNorm passes."""
        y = ops.conv2d(x, self.conv.weight, None, self.stride, self.groups, bn_stats=self.bn.training)
        # bwd16: this conv has no bias / ReLU of its own, so BatchNorm's dx is exactly the dy its tensor-core dgrad / wgrad read
        return ops.batch_norm(y, self.bn, self.act or residual is not None, self.bn.training, emit16,
                              bwd16=self.conv.in_channels % 8 == 0, residual=residual, pool=pool)


class _SE(nn.Module):
    def __init__(self, channels, rd_channels):
        super().__init__()
        self.fc1 = nn.Conv2d(channels, rd_channels, 1, bias=True)
        self.fc2 = nn.Conv2d(rd_channels, channels, 1, bias=True)

    def run(self, x):
        # the gated output always feeds the 1x1 conv3 GEMM: emit its bf16 copy in the gating pass
        return ops.SEFn.apply(x, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias, True)


class _Bottleneck(nn.Module):
    def __init__(self, cin, cout, stride, group_w, se_ratio):
        super().__init__()
        self.conv1 = _ConvBn(cin, cout, 1)
        self.conv2 = _ConvBn(cout, cout, 3, stride=stride, groups=cout // group_w)
        self.se = _SE(cout, int(round(cin * se_ratio)))
        self.conv3 = _ConvBn(cout, cout, 1, act=False)
        self.downsample = _ConvBn(cin, cout, 1, stride=stride, act=False) if (cin != cout or stride != 1) else None
        nn.init.zeros_(self.conv3.bn.weight)  # timm zero_init_last_bn

    def run(self, x, emit16=True):
        """emit16: the block output feeds a 1x1 conv next (the following block's conv1, or the channel-change conv)."""
        y1 = self.conv1.run(x, emit16=self.conv2.stride == 1)
        c2 = self.conv2
        if ops.bn_se_ok(y1, c2.bn, self.se.fc1):
            # conv2.bn (+ReLU, + SE average pool) and the squeeze-excite module as one autograd node (ops.BNSEFn)
            t = ops.conv2d(y1, c2.conv.weight, None, c2.stride, c2.groups, bn_stats=True)
            y = ops.bn_se(t, c2.bn, self.se.fc1, self.se.fc2, bwd16=c2.conv.in_channels % 8 == 0)
        else:
            y = self.se.run(c2.run(y1, pool=True))            # SE pool inside conv2.bn
        sc = self.downsample.run(x) if self.downsample is not None else x
        return self.conv3.run(y, emit16=emit16, residual=sc)      # relu(conv3.bn(conv3(y)) + shortcut)


class _Stage(nn.Module):
    def __init__(self, cin, cout, depth, group_w, se_ratio):
        super().__init__()
        for i in range(depth):
            self.add_module('b%d' % (i + 1), _Bottleneck(cin if i == 0 else cout, cout, 2 if i == 0 else 1, group_w, se_ratio))

    def run(self, x, last16=True):
        """last16 = False when the stage output goes to a GPT fusion (token pooling / upsample-add), not straight into a conv."""
        blocks = list(self.children())
        for i, blk in enumerate(blocks):
            x = blk.run(x, emit16=last16 or i + 1 < len(blocks))
        return x


class _RegNet(nn.Module):
    """Parameter tree of timm's RegNet (names: stem.{conv,bn}, s1..s4.b{k}.{conv1,conv2,se,conv3,downsample})."""

    def __init__(self, cfg=REGNETY_032, in_chans=3):
        super().__init__()
        self.stem = _ConvBn(in_chans, cfg['stem_width'], 3, stride=2)
        self.feature_info = [dict(num_chs=cfg['stem_width'], reduction=2, module='stem')]
        prev = cfg['stem_width']
        for i, (w, d) in enumerate(zip(cfg['widths'], cfg['depths'])):
            self.add_module('s%d' % (i + 1), _Stage(prev, w, d, cfg['group_w'], cfg['se_ratio']))
            prev = w
            self.feature_info.append(dict(num_chs=w, reduction=2 ** (i + 2), module='s%d' % (i + 1)))
        self.num_features = prev
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                fan_out = m.kernel_size[0] * m.kernel_size[1] * m.out_channels // m.groups
                nn.init.normal_(m.weight, 0.0, (2.0 / fan_out) ** 0.5)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)


class ImageCNN(nn.Module):
    """transfuser.py:369-416 (regnet branch): `features` + the alias attributes the reference's forward goes through."""

    def __init__(self, architecture, normalize=True, out_features=512):
        super().__init__()
        if architecture != 'regnety_032':
            raise RuntimeError('transfuser_b200 implements the regnety_032 trunk only (train.py:50-53 default), got %r' % (architecture,))
        self.normalize = normalize
        f = self.features = _RegNet()
        f.conv1, f.bn1 = f.stem.conv, f.stem.bn
        f.layer1, f.layer2, f.layer3, f.layer4 = f.s1, f.s2, f.s3, f.s4


class LidarEncoder(nn.Module):
    """transfuser.py:431-488: same trunk, new `conv1` with `in_channels`, `stem.conv` deleted."""

    def __init__(self, architecture, in_channels=2, out_features=512):
        super().__init__()
        if architecture != 'regnety_032':
            raise RuntimeError('transfuser_b200 implements the regnety_032 trunk only, got %r' % (architecture,))
        m = self._model = _RegNet()
        old = m.stem.conv
        m.conv1, m.bn1 = m.stem.conv, m.stem.bn   # same registration order as the reference (transfuser.py:446-453)
        m.layer1, m.layer2, m.layer3, m.layer4 = m.s1, m.s2, m.s3, m.s4
        m.conv1 = nn.Conv2d(in_channels, old.out_channels, kernel_size=old.kernel_size, stride=old.stride, padding=old.padding, bias=False)
        del m.stem.conv


class SelfAttention(nn.Module):
    def __init__(self, n_embd, n_head, attn_pdrop, resid_pdrop):
        super().__init__()
        assert n_embd % n_head == 0
        self.key = nn.Linear(n_embd, n_embd)
        self.query = nn.Linear(n_embd, n_embd)
        self.value = nn.Linear(n_embd, n_embd)
        self.proj = nn.Linear(n_embd, n_embd)
        self.n_head, self.attn_pdrop, self.resid_pdrop = n_head, attn_pdrop, resid_pdrop


class Block(nn.Module):
    """transfuser.py:530-549: x + attn(ln1(x)); x + mlp(ln2(x)), ReLU MLP, three dropouts."""

    def __init__(self, n_embd, n_head, block_exp, attn_pdrop, resid_pdrop):
        super().__init__()
        self.ln1 = nn.LayerNorm(n_embd)
        self.ln2 = nn.LayerNorm(n_embd)
        self.attn = SelfAttention(n_embd, n_head, attn_pdrop, resid_pdrop)
        self.mlp = nn.Sequential(nn.Linear(n_embd, block_exp * n_embd), nn.ReLU(True), nn.Linear(block_exp * n_embd, n_embd),
                                 nn.Dropout(resid_pdrop))

    def _first_half(self, x, h, B, T):
        """h = ln1(x) -> (x + attn(h), mlp[0](ln2(x + attn(h))))."""
        a, training = self.attn, self.training
        p_att = a.attn_pdrop if training else 0.0
        y = ops.AttentionFn.apply(h, a.query.weight, a.query.bias, a.key.weight, a.key.bias, a.value.weight, a.value.bias,
                                  B, T, a.n_head, p_att, ops.next_seed())
        x, h = ops.add_dropout_ln(x, ops.linear(y, a.proj.weight, a.proj.bias), a.resid_pdrop, training, self.ln2, emit16=True)
        return x, ops.linear(h, self.mlp[0].weight, self.mlp[0].bias, relu=True)

    def run(self, x, B, T):
        x, h = self._first_half(x, ops.layer_norm(x, self.ln1, emit16=True), B, T)
        return ops.add_dropout(x, ops.linear(h, self.mlp[2].weight, self.mlp[2].bias), self.attn.resid_pdrop, self.training)

    def run_chained(self, x, h, B, T, next_ln, next_emit16):
        """As run(), with the LayerNorms moved onto the residual connections in front of them: x is the residual stream and
        h = ln1(x); returns the new residual stream and next_ln of it (the next block's ln1, or ln_f after the last block)."""
        x, h = self._first_half(x, h, B, T)
        return ops.add_dropout_ln(x, ops.linear(h, self.mlp[2].weight, self.mlp[2].bias), self.attn.resid_pdrop, self.training, next_ln,
                                  emit16=next_emit16)


class GPT(nn.Module):
    """transfuser.py:284-366."""

    def __init__(self, n_embd, n_head, block_exp, n_layer, img_vert_anchors, img_horz_anchors, lidar_vert_anchors,
                 lidar_horz_anchors, seq_len, embd_pdrop, attn_pdrop, resid_pdrop, config, use_velocity=True):
        super().__init__()
        self.n_embd, self.seq_len, self.config, self.use_velocity = n_embd, 1, config, bool(use_velocity)
        self.grid = (img_vert_anchors, img_horz_anchors, lidar_vert_anchors, lidar_horz_anchors)
        self.pos_emb = nn.Parameter(torch.zeros(1, img_vert_anchors * img_horz_anchors + lidar_vert_anchors * lidar_horz_anchors, n_embd))
        if self.use_velocity:
            self.vel_emb = nn.Linear(self.seq_len, n_embd)          # transfuser.py:306-309 (registered between pos_emb and the blocks)
        self.embd_pdrop = embd_pdrop
        self.drop = nn.Dropout(embd_pdrop)
        self.blocks = nn.Sequential(*[Block(n_embd, n_head, block_exp, attn_pdrop, resid_pdrop) for _ in range(n_layer)])
        self.ln_f = nn.LayerNorm(n_embd)
        self.block_size = self.seq_len
        self.apply(self._init_weights)

    def _init_weights(self, module):
        if isinstance(module, nn.Linear):
            module.weight.data.normal_(mean=self.config.gpt_linear_layer_init_mean, std=self.config.gpt_linear_layer_init_std)
            if module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(self.config.gpt_layer_norm_init_weight)

    def run(self, img, lid, velocity=None):
        """img / lid: NHWC stage features -> the same features with the upsampled GPT output added. velocity [B, 1]: the ego speed
        (only read with use_velocity: its embedding is added to every token before the embedding dropout, transfuser.py:352-355)."""
        ghi, gwi, ghl, gwl = self.grid
        B = img.shape[0]
        T = ghi * gwi + ghl * gwl
        p = self.embd_pdrop if self.training else 0.0
        if self.use_velocity:
            if velocity is None:
                raise RuntimeError('GPT(use_velocity=True) needs the velocity input')
            tok = ops.TokensFn.apply(img, lid, self.pos_emb, ghi, gwi, ghl, gwl, 0.0, 0)
            ve = ops.linear(velocity.reshape(B, self.seq_len).to(self.vel_emb.weight.dtype), self.vel_emb.weight, self.vel_emb.bias)
            tok = ops.dropout(ops.BcastAddTokensFn.apply(tok, ve), self.embd_pdrop, self.training)
        else:
            tok = ops.TokensFn.apply(img, lid, self.pos_emb, ghi, gwi, ghl, gwl, p, ops.next_seed())
        x = tok.view(B * T, self.n_embd)
        blocks = list(self.blocks)
        h = ops.layer_norm(x, blocks[0].ln1, emit16=True)
        for i, blk in enumerate(blocks):
            last = i + 1 == len(blocks)
            x, h = blk.run_chained(x, h, B, T, self.ln_f if last else blocks[i + 1].ln1, not last)
        x = h.view(B, T, self.n_embd)
        return ops.GptUpAddFn.apply(img, lid, x, ghi, gwi, ghl, gwl)


class TransfuserBackbone(nn.Module):
    """Multi-scale fusion transformer for image + LiDAR feature fusion (transfuser.py:7-211)."""

    def __init__(self, config, image_architecture='resnet34', lidar_architecture='resnet18', use_velocity=True):
        super().__init__()
        self.config = config
        self.image_encoder = ImageCNN(architecture=image_architecture, normalize=True, out_features=config.perception_output_features)
        if config.use_point_pillars:
            raise RuntimeError('PointPillars LiDAR encoder is out of scope (config.py:42 default False)')
        in_channels = 2 * config.lidar_seq_len + (1 if config.use_target_point_image else 0)
        self.lidar_encoder = self._make_lidar_encoder(lidar_architecture, in_channels)
        info = self.image_encoder.features.feature_info
        for i in range(1, 5):
            setattr(self, 'transformer%d' % i, GPT(
                n_embd=info[i]['num_chs'], n_head=config.n_head, block_exp=config.block_exp, n_layer=config.n_layer,
                img_vert_anchors=config.img_vert_anchors, img_horz_anchors=config.img_horz_anchors,
                lidar_vert_anchors=config.lidar_vert_anchors, lidar_horz_anchors=config.lidar_horz_anchors, seq_len=config.seq_len,
                embd_pdrop=config.embd_pdrop, attn_pdrop=config.attn_pdrop, resid_pdrop=config.resid_pdrop, config=config,
                use_velocity=use_velocity))
        c_last, c_out = info[4]['num_chs'], config.perception_output_features
        self.change_channel_conv_image = nn.Conv2d(c_last, c_out, (1, 1))
        self.change_channel_conv_lidar = nn.Conv2d(c_last, c_out, (1, 1))
        channel = config.bev_features_chanels
        self.up_conv5 = nn.Conv2d(channel, channel, (1, 1))
        self.up_conv4 = nn.Conv2d(channel, channel, (1, 1))
        self.up_conv3 = nn.Conv2d(channel, channel, (1, 1))
        self.c5_conv = nn.Conv2d(c_out, channel, (1, 1))
        self.two_streams = ops.TWO_STREAMS

    def _make_lidar_encoder(self, architecture, in_channels):
        return LidarEncoder(architecture=architecture, in_channels=in_channels, out_features=self.config.perception_output_features)

    def _bn_modules(self):
        if not hasattr(self, '_bn_cache'):
            object.__setattr__(self, '_bn_cache', [m for m in self.modules() if isinstance(m, nn.BatchNorm2d)])
        return self._bn_cache

    def forward_nhwc(self, image, lidar, taps=None, velocity=None):
        """image: NCHW 0..255, lidar: NCHW -> (p2..p5 NHWC), image grid NHWC, fused [B,512]. `taps` (optional dict) receives the
        per-stage fused feature maps (NHWC) for layer-by-layer parity checks. velocity [B, 1]: read by the GPTs with use_velocity."""
        if self.training:
            torch._foreach_add_([m.num_batches_tracked for m in self._bn_modules()], 1)
            ops.tick(image.device)
        ie, le = self.image_encoder.features, self.lidar_encoder._model
        x = ops.image_prep(image) if self.image_encoder.normalize else ops.nchw_to_nhwc(image)
        l = ops.nchw_to_nhwc(lidar)
        if not self.two_streams:
            x = ie.stem.run(x, emit16=True)
            l = ops.batch_norm(ops.conv2d(l, le.conv1.weight, None, 2, 1), le.bn1, True, le.bn1.training, emit16=True)
            for i in range(1, 5):
                x = getattr(ie, 's%d' % i).run(x, last16=False)
                l = getattr(le, 's%d' % i).run(l, last16=False)
                x, l = getattr(self, 'transformer%d' % i).run(x, l, velocity)
                if taps is not None:
                    taps['img_s%d' % i], taps['lid_s%d' % i] = x, l
        else:
            # The two trunks are independent between fusion points: the LiDAR trunk runs on a second stream (forward here,
            # backward automatically — autograd replays each node on its forward stream), so its small kernels fill the SMs the
            # image trunk leaves idle. Joins before each GPT; forks after it. Captured into the step's CUDA graph as branches.
            main = torch.cuda.current_stream()
            side = ops.side_stream(image.device)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                l = ops.batch_norm(ops.conv2d(l, le.conv1.weight, None, 2, 1), le.bn1, True, le.bn1.training, emit16=True)
            x = ie.stem.run(x, emit16=True)
            for i in range(1, 5):
                with torch.cuda.stream(side):
                    l = getattr(le, 's%d' % i).run(l, last16=False)
                x = getattr(ie, 's%d' % i).run(x, last16=False)
                main.wait_stream(side)
                ops.record_stream(l, main)
                x, l = getattr(self, 'transformer%d' % i).run(x, l, velocity)
                if taps is not None:
                    taps['img_s%d' % i], taps['lid_s%d' % i] = x, l
                if i < 4:
                    side.wait_stream(main)
                    ops.record_stream(l, side)
        x = ops.conv2d(x, self.change_channel_conv_image.weight, self.change_channel_conv_image.bias)
        l = ops.conv2d(l, self.change_channel_conv_lidar.weight, self.change_channel_conv_lidar.bias)
        fused = ops.add(ops.PoolHWFn.apply(x), ops.PoolHWFn.apply(l))
        f = self.config.bev_upsample_factor
        up = lambda t: ops.upsample(t, t.shape[1] * f, t.shape[2] * f, False, emit16=True)
        p5 = ops.conv2d(l, self.c5_conv.weight, self.c5_conv.bias, relu=True)
        p4 = ops.conv2d(up(p5), self.up_conv5.weight, self.up_conv5.bias, relu=True)
        p3 = ops.conv2d(up(p4), self.up_conv4.weight, self.up_conv4.bias, relu=True)
        p2 = ops.conv2d(up(p3), self.up_conv3.weight, self.up_conv3.bias, relu=True)
        return (p2, p3, p4, p5), x, fused

    def forward(self, image, lidar, velocity):
        feats, grid, fused = self.forward_nhwc(image, lidar, velocity=velocity)
        return tuple(ops.nhwc_to_nchw(f) for f in feats), ops.nhwc_to_nchw(grid), fused


class _PlainEncoder(nn.Module):
    """late_fusion.py:114-163: the timm trunk used whole (stem -> s1..s4); classifier parts replaced by empty Sequentials."""

    def __init__(self, architecture, attr, in_chans=3, normalize=True):
        super().__init__()
        if architecture != 'regnety_032':
            raise RuntimeError('transfuser_b200 implements the regnety_032 trunk only, got %r' % (architecture,))
        self.normalize = normalize
        net = _RegNet(in_chans=in_chans)
        net.fc, net.classifier, net.global_pool, net.head = nn.Sequential(), nn.Sequential(), nn.Sequential(), nn.Sequential()
        setattr(self, attr, net)
        object.__setattr__(self, '_net', net)

    def run(self, x):
        net = self._net
        x = net.stem.run(x, emit16=True)
        for i in range(1, 5):
            x = getattr(net, 's%d' % i).run(x)
        return x


class LateFusionBackbone(nn.Module):
    """H100-native drop-in for team_code_transfuser/late_fusion.py:5-111 (BASELINE config 5): two independent
    RegNetY trunks, 1x1 channel reduction, global pools summed, FPN top-down on the LiDAR grid. Same parameter names."""

    def __init__(self, config, image_architecture='resnet34', lidar_architecture='resnet18', use_velocity=0):
        super().__init__()
        self.config = config
        if config.use_point_pillars:
            raise RuntimeError('PointPillars LiDAR encoder is out of scope (config.py:42 default False)')
        if use_velocity:
            raise RuntimeError('use_velocity=True is not implemented (train.py:54 default is 0)')
        in_channels = 2 * config.lidar_seq_len + (1 if config.use_target_point_image else 0)
        self.image_encoder = _PlainEncoder(image_architecture, 'features', 3, normalize=True)
        self.lidar_encoder = _PlainEncoder(lidar_architecture, '_model', in_channels, normalize=False)
        self.norm_after_pool_img = nn.Sequential()
        self.norm_after_pool_lidar = nn.Sequential()
        self.use_velocity = use_velocity
        channel, c_out, c_last = config.bev_features_chanels, config.perception_output_features, REGNETY_032['widths'][-1]
        self.reduce_channels_conv_image = nn.Conv2d(c_last, c_out, (1, 1))
        self.reduce_channels_conv_lidar = nn.Conv2d(c_last, c_out, (1, 1))
        self.up_conv5 = nn.Conv2d(channel, channel, (1, 1))
        self.up_conv4 = nn.Conv2d(channel, channel, (1, 1))
        self.up_conv3 = nn.Conv2d(channel, channel, (1, 1))
        self.c5_conv = nn.Conv2d(c_out, channel, (1, 1))

    def _bn_modules(self):
        if not hasattr(self, '_bn_cache'):
            object.__setattr__(self, '_bn_cache', [m for m in self.modules() if isinstance(m, nn.BatchNorm2d)])
        return self._bn_cache

    def forward_nhwc(self, image, lidar):
        if self.training:
            torch._foreach_add_([m.num_batches_tracked for m in self._bn_modules()], 1)
            ops.tick(image.device)
        if ops.TWO_STREAMS:
            main, side = torch.cuda.current_stream(), ops.side_stream(image.device)
            l = ops.nchw_to_nhwc(lidar)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                l = self.lidar_encoder.run(l)
            x = self.image_encoder.run(ops.image_prep(image))
            main.wait_stream(side)
            ops.record_stream(l, main)
        else:
            x = self.image_encoder.run(ops.image_prep(image))
            l = self.lidar_encoder.run(ops.nchw_to_nhwc(lidar))
        x = ops.conv2d(x, self.reduce_channels_conv_image.weight, self.reduce_channels_conv_image.bias)
        l = ops.conv2d(l, self.reduce_channels_conv_lidar.weight, self.reduce_channels_conv_lidar.bias)
        fused = ops.add(ops.PoolHWFn.apply(x), ops.PoolHWFn.apply(l))
        f = self.config.bev_upsample_factor
        up = lambda t: ops.upsample(t, t.shape[1] * f, t.shape[2] * f, False, emit16=True)
        p5 = ops.conv2d(l, self.c5_conv.weight, self.c5_conv.bias, relu=True)
        p4 = ops.conv2d(up(p5), self.up_conv5.weight, self.up_conv5.bias, relu=True)
        p3 = ops.conv2d(up(p4), self.up_conv4.weight, self.up_conv4.bias, relu=True)
        p2 = ops.conv2d(up(p3), self.up_conv3.weight, self.up_conv3.bias, relu=True)
        return (p2, p3, p4, p5), x, fused

    def forward(self, image, lidar, velocity):
        feats, grid, fused = self.forward_nhwc(image, lidar)
        return tuple(ops.nhwc_to_nchw(f) for f in feats), ops.nhwc_to_nchw(grid), fused


class _GeoLidarEncoder(nn.Module):
    """geometric_fusion.py:353-403: like transfuser.py's LidarEncoder, but the whole `stem` is deleted after aliasing, so the
    stem's parameters live under `conv1` / `bn1` only."""

    def __init__(self, architecture, in_channels=2):
        super().__init__()
        if architecture != 'regnety_032':
            raise RuntimeError('transfuser_b200 implements the regnety_032 trunk only, got %r' % (architecture,))
        m = self._model = _RegNet()
        old = m.stem.conv
        m.conv1, m.bn1 = m.stem.conv, m.stem.bn
        m.layer1, m.layer2, m.layer3, m.layer4 = m.s1, m.s2, m.s3, m.s4
        m.conv1 = nn.Conv2d(in_channels, old.out_channels, kernel_size=old.kernel_size, stride=old.stride, padding=old.padding, bias=False)
        del m.stem


def _mlp3(hid):
    return nn.Sequential(nn.Linear(hid, hid), nn.ReLU(True), nn.Linear(hid, hid), nn.ReLU(True), nn.Linear(hid, hid), nn.ReLU(True))


class GeometricFusionBackbone(nn.Module):
    """H100-native drop-in for team_code_transfuser/geometric_fusion.py:7-296 (BASELINE config 4): at each of
    the 4 trunk scales, features of one modality are pooled to its anchor grid, gathered at 5 projected correspondences per
    cell of the other modality's grid, summed, passed through a 3-layer MLP and added back at full resolution.

    Same parameter names / shapes as the reference. Two exact-in-real-arithmetic reassociations keep the work on the
    anchor grids instead of the full maps (both ops are linear, bilinear weights sum to 1):
      avgpool(conv1x1(x))           -> conv1x1(avgpool(x))          (geometric_fusion.py:132-135)
      conv1x1(interpolate(enc))     -> interpolate(conv1x1(enc))    (geometric_fusion.py:150-151)
    so the 512-channel embeddings only ever exist as [B,5,22,512] / [B,8,8,512]. fp32 rounding differs at the 1e-6 level.
    The scale-4 image branch gathers from the scale-3 LiDAR embedding, as the reference does (geometric_fusion.py:277)."""

    def __init__(self, config, image_architecture='resnet34', lidar_architecture='resnet18', use_velocity=0):
        super().__init__()
        self.config = config
        if config.use_point_pillars:
            raise RuntimeError('PointPillars LiDAR encoder is out of scope (config.py:42 default False)')
        if use_velocity:
            raise RuntimeError('use_velocity=True is not implemented (train.py:54 default is 0)')
        if config.n_scale != 4:
            raise RuntimeError('n_scale=%r is not implemented (config.py default 4)' % (config.n_scale,))
        self.use_velocity = use_velocity
        in_channels = 2 * config.lidar_seq_len + (1 if config.use_target_point_image else 0)
        self.image_encoder = ImageCNN(architecture=image_architecture, normalize=True)
        self.lidar_encoder = _GeoLidarEncoder(architecture=lidar_architecture, in_channels=in_channels)
        widths, hid = REGNETY_032['widths'], config.n_embd
        for stem in ('image_conv', 'image_deconv', 'lidar_conv', 'lidar_deconv'):
            for i in range(4):
                cin, cout = (hid, widths[i]) if 'deconv' in stem else (widths[i], hid)
                setattr(self, '%s%d' % (stem, i + 1), nn.Conv2d(cin, cout, 1))
        for stem in ('image_projection', 'lidar_projection'):
            for i in range(4):
                setattr(self, '%s%d' % (stem, i + 1), _mlp3(hid))
        c_out = config.perception_output_features
        self.change_channel_conv_image = nn.Conv2d(widths[-1], c_out, (1, 1))
        self.change_channel_conv_lidar = nn.Conv2d(widths[-1], c_out, (1, 1))
        channel = config.bev_features_chanels
        self.up_conv5 = nn.Conv2d(channel, channel, (1, 1))
        self.up_conv4 = nn.Conv2d(channel, channel, (1, 1))
        self.up_conv3 = nn.Conv2d(channel, channel, (1, 1))
        self.c5_conv = nn.Conv2d(c_out, channel, (1, 1))

    def _bn_modules(self):
        if not hasattr(self, '_bn_cache'):
            object.__setattr__(self, '_bn_cache', [m for m in self.modules() if isinstance(m, nn.BatchNorm2d)])
        return self._bn_cache

    @staticmethod
    def _project(mlp, x):
        for j in (0, 2, 4):
            x = ops.linear(x, mlp[j].weight, mlp[j].bias, relu=True)
        return x

    def forward_nhwc(self, image, lidar, bev_points, img_points):
        """image NCHW 0..255, lidar NCHW, bev_points [B,8,8,5,2] / img_points [B,5,22,5,2] int64 (x, y) correspondences."""
        cfg = self.config
        if self.training:
            torch._foreach_add_([m.num_batches_tracked for m in self._bn_modules()], 1)
            ops.tick(image.device)
        ie, le = self.image_encoder.features, self.lidar_encoder._model
        x = ie.stem.run(ops.image_prep(image), emit16=True)
        l = ops.batch_norm(ops.conv2d(ops.nchw_to_nhwc(lidar), le.conv1.weight, None, 2, 1), le.bn1, True, le.bn1.training, emit16=True)
        ih, iw, lh, lw = cfg.img_vert_anchors, cfg.img_horz_anchors, cfg.lidar_vert_anchors, cfg.lidar_horz_anchors
        prev_lidar_embd = None
        for i in range(1, 5):
            x = getattr(ie, 's%d' % i).run(x, last16=False)
            l = getattr(le, 's%d' % i).run(l, last16=False)
            ic, lc = getattr(self, 'image_conv%d' % i), getattr(self, 'lidar_conv%d' % i)
            img_embd = ops.linear(ops.avgpool_grid(x, ih, iw), ic.weight, ic.bias)          # [B,5,22,512]
            # scale 4's LiDAR embedding is never read (the image branch gathers from scale 3's, geometric_fusion.py:277)
            lidar_embd = ops.linear(ops.avgpool_grid(l, lh, lw), lc.weight, lc.bias) if i < 4 else None   # [B,8,8,512]
            bev_enc = self._project(getattr(self, 'image_projection%d' % i), ops.gather_sum(img_embd, bev_points))
            img_enc = self._project(getattr(self, 'lidar_projection%d' % i),
                                    ops.gather_sum(prev_lidar_embd if i == 4 else lidar_embd, img_points))
            ld, idc = getattr(self, 'lidar_deconv%d' % i), getattr(self, 'image_deconv%d' % i)
            dl = ops.linear(bev_enc, ld.weight, ld.bias)                                    # [B,8,8,C_i]
            dx = ops.linear(img_enc, idc.weight, idc.bias)                                  # [B,5,22,C_i]
            if i < 4:
                dl = ops.upsample(dl, l.shape[1], l.shape[2], False)
                dx = ops.upsample(dx, x.shape[1], x.shape[2], False)
            l = ops.add(l, dl, emit16=True)       # feeds the next stage's 1x1 conv1 / the channel-change conv
            x = ops.add(x, dx, emit16=True)
            prev_lidar_embd = lidar_embd
        x = ops.conv2d(x, self.change_channel_conv_image.weight, self.change_channel_conv_image.bias)
        l = ops.conv2d(l, self.change_channel_conv_lidar.weight, self.change_channel_conv_lidar.bias)
        fused = ops.add(ops.PoolHWFn.apply(x), ops.PoolHWFn.apply(l))
        f = cfg.bev_upsample_factor
        up = lambda t: ops.upsample(t, t.shape[1] * f, t.shape[2] * f, False, emit16=True)
        p5 = ops.conv2d(l, self.c5_conv.weight, self.c5_conv.bias, relu=True)
        p4 = ops.conv2d(up(p5), self.up_conv5.weight, self.up_conv5.bias, relu=True)
        p3 = ops.conv2d(up(p4), self.up_conv4.weight, self.up_conv4.bias, relu=True)
        p2 = ops.conv2d(up(p3), self.up_conv3.weight, self.up_conv3.bias, relu=True)
        return (p2, p3, p4, p5), x, fused

    def forward(self, image, lidar, velocity, bev_points, img_points):
        feats, grid, fused = self.forward_nhwc(image, lidar, bev_points, img_points)
        return tuple(ops.nhwc_to_nchw(f) for f in feats), ops.nhwc_to_nchw(grid), fused


class latentTFBackbone(TransfuserBackbone):
    """H100-native drop-in for team_code_transfuser/latentTF.py:8-217: the TransFuser architecture with the two
    LiDAR histogram channels replaced by a fixed positional grid in [-1, 1] (latentTF.py:132-137; the target-point channel is
    kept). Same kernels and schedule as TransfuserBackbone; the only differences are the input assembly and the parameter
    names of the LiDAR stem (its encoder deletes the whole `stem`, latentTF.py:195-196)."""

    def _make_lidar_encoder(self, architecture, in_channels):
        return _GeoLidarEncoder(architecture=architecture, in_channels=in_channels)

    def _grid(self, lidar):
        key = (lidar.device, lidar.dtype, lidar.shape[2], lidar.shape[3])
        if getattr(self, '_grid_key', None) != key:
            cfg = self.config
            rows = torch.linspace(-1, 1, cfg.lidar_resolution_width, device=lidar.device, dtype=lidar.dtype)
            cols = torch.linspace(-1, 1, cfg.lidar_resolution_height, device=lidar.device, dtype=lidar.dtype)
            g = torch.stack((rows.view(-1, 1).expand(lidar.shape[2], lidar.shape[3]), cols.view(1, -1).expand(lidar.shape[2], lidar.shape[3])))
            object.__setattr__(self, '_grid_buf', g.unsqueeze(0).contiguous())
            object.__setattr__(self, '_grid_key', key)
        return self._grid_buf

    def forward_nhwc(self, image, lidar, taps=None, velocity=None):
        lidar = torch.cat((self._grid(lidar).expand(lidar.shape[0], -1, -1, -1), lidar[:, 2:]), dim=1)
        return super().forward_nhwc(image, lidar, taps, velocity)
