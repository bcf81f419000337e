"""H100-native `LidarCenterNet` training forward — drop-in for team_code_transfuser/model.py:538-805.

Same constructor and `forward(...) -> dict of the 11 scalar losses` contract (keys = config.detailed_losses), same
parameter names (`_model.*`, `seg_decoder.*`, `depth_decoder.*`, `pred_bev.*`, `head.*_head.*`, `join.*`, `decoder.*`,
`output.*`), so train.py's loop (`loss.backward()`, `optimizer.step()`, `state_dict()`) runs unchanged. The nn.* members
are parameter containers; all compute goes through transfuser_b200.ops (hand-written sm_90a kernels).
`forward_ego` (model.py:685-731: waypoints + decoded boxes for the driving agent) runs the same kernels in eval mode plus the
one-launch CenterNet decode; the agent-side control / visualisation members (control_pid, visualize_model_io) are out of scope."""
import numpy as np
import torch
from torch import nn

from . import ops
from .backbone import GeometricFusionBackbone, LateFusionBackbone, TransfuserBackbone, latentTFBackbone

HEAD_NAMES = ('heatmap_head', 'wh_head', 'offset_head', 'yaw_class_head', 'yaw_res_head', 'velocity_head', 'brake_head')
HEAD_LOSSES = ('loss_center_heatmap', 'loss_wh', 'loss_offset', 'loss_yaw_class', 'loss_yaw_res', 'loss_velocity', 'loss_brake')


def _conv_pair(cin, cmid, cout):
    return nn.Sequential(nn.Conv2d(cin, cmid, kernel_size=3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(cmid, cout, kernel_size=1))


def _run_pair(seq, x):
    y = ops.conv2d(x, seq[0].weight, seq[0].bias, relu=True)
    return ops.conv2d(y, seq[2].weight, seq[2].bias)


class LidarCenterNetHead(nn.Module):
    """Parameters of model.py:33-125 (seven conv3x3+ReLU+conv1x1 branches); targets + losses run in ops.CenterNetLossFn."""

    def __init__(self, in_channel, feat_channel, num_classes, train_cfg=None):
        super().__init__()
        self.num_classes = num_classes
        self.num_dir_bins = train_cfg.num_dir_bins
        self.heatmap_head = _conv_pair(in_channel, feat_channel, num_classes)
        self.wh_head = _conv_pair(in_channel, feat_channel, 2)
        self.offset_head = _conv_pair(in_channel, feat_channel, 2)
        self.yaw_class_head = _conv_pair(in_channel, feat_channel, self.num_dir_bins)
        self.yaw_res_head = _conv_pair(in_channel, feat_channel, 1)
        self.velocity_head = _conv_pair(in_channel, feat_channel, 1)
        self.brake_head = _conv_pair(in_channel, feat_channel, 2)
        self.train_cfg = train_cfg

    def run(self, feat):
        """feat NHWC -> [B, H, W, 21] raw predictions (heat logit | wh | offset | yaw class | yaw res | velocity | brake)."""
        return torch.cat([_run_pair(getattr(self, n), feat) for n in HEAD_NAMES], dim=3)

    def get_bboxes_nhwc(self, preds):
        """model.py:376-497 (get_bboxes with with_nms=False -> decode_heatmap) on the raw NHWC head output of `run`:
        list over the batch of (boxes [k,8] = x, y, w, h, yaw, velocity, brake, score; labels [k])."""
        cfg = self.train_cfg
        kernel = getattr(cfg, 'center_net_max_pooling_kernel', 3)
        if kernel != 3:
            raise RuntimeError('center_net_max_pooling_kernel=%r is not implemented (config.py:59 default 3)' % (kernel,))
        boxes, labels = ops.centernet_decode(preds, self.num_dir_bins, getattr(cfg, 'top_k_center_keypoints', 100), 4.0)
        return [(boxes[b], labels[b]) for b in range(boxes.shape[0])]


class _Decoder(nn.Module):
    """SegDecoder / DepthDecoder parameter tree (transfuser.py:214-281)."""

    def __init__(self, config, latent_dim, out_ch):
        super().__init__()
        self.config = config
        c1, c2, c3 = config.deconv_channel_num_1, config.deconv_channel_num_2, config.deconv_channel_num_3
        mk = lambda a, b, c, last_relu: nn.Sequential(*([nn.Conv2d(a, b, 3, 1, 1), nn.ReLU(True), nn.Conv2d(b, c, 3, 1, 1)] + ([nn.ReLU(True)] if last_relu else [])))
        self.deconv1 = mk(latent_dim, c1, c2, True)
        self.deconv2 = mk(c2, c3, c3, True)
        self.deconv3 = mk(c3, c3, out_ch, False)

    def run(self, x):
        cfg = self.config
        c = lambda seq, t, last_relu: ops.conv2d(ops.conv2d(t, seq[0].weight, seq[0].bias, relu=True), seq[2].weight, seq[2].bias, relu=last_relu)
        x = c(self.deconv1, x, True)
        x = ops.upsample(x, x.shape[1] * cfg.deconv_scale_factor_1, x.shape[2] * cfg.deconv_scale_factor_1, False, emit16=True)
        x = c(self.deconv2, x, True)
        x = ops.upsample(x, x.shape[1] * cfg.deconv_scale_factor_2, x.shape[2] * cfg.deconv_scale_factor_2, False, emit16=True)
        return c(self.deconv3, x, False)


class SegDecoder(_Decoder):
    def __init__(self, config, latent_dim=512):
        super().__init__(config, latent_dim, config.num_class)
        self.latent_dim, self.num_class = latent_dim, config.num_class


class DepthDecoder(_Decoder):
    def __init__(self, config, latent_dim=512):
        super().__init__(config, latent_dim, 1)
        self.latent_dim = latent_dim


class LidarCenterNet(nn.Module):
    def __init__(self, config, device, backbone, image_architecture='resnet34', lidar_architecture='resnet18', use_velocity=True):
        super().__init__()
        self.device = device
        self.config = config
        self.pred_len = config.pred_len
        self.use_target_point_image = config.use_target_point_image
        self.gru_concat_target_point = config.gru_concat_target_point
        self.use_point_pillars = config.use_point_pillars
        if self.use_point_pillars:
            raise RuntimeError('PointPillars is out of scope (config.py:42 default False)')
        if not self.gru_concat_target_point:
            raise RuntimeError('gru_concat_target_point=False is not implemented (config.py:31 default True)')
        # sizes the kernels hard-code (csrc/losses.cu: 12 yaw bins / 21 head channels; csrc/gru_adamw.cu: hidden size 64, 4 + 64 inputs)
        if config.num_dir_bins != 12:
            raise RuntimeError('num_dir_bins=%r is not implemented (the CenterNet loss kernels assume config.py default 12)' % (config.num_dir_bins,))
        if config.gru_hidden_size != 64:
            raise RuntimeError('gru_hidden_size=%r is not implemented (the GRU kernels assume config.py default 64)' % (config.gru_hidden_size,))
        if getattr(config, 'n_scale', 4) != 4:
            raise RuntimeError('n_scale=%r is not implemented (config.py default 4)' % (config.n_scale,))
        self.backbone = backbone
        if backbone == 'transFuser':
            self._model = TransfuserBackbone(config, image_architecture, lidar_architecture, use_velocity=use_velocity).to(self.device)
        elif backbone == 'late_fusion':
            self._model = LateFusionBackbone(config, image_architecture, lidar_architecture, use_velocity=use_velocity).to(self.device)
        elif backbone == 'geometric_fusion':
            self._model = GeometricFusionBackbone(config, image_architecture, lidar_architecture, use_velocity=use_velocity).to(self.device)
        elif backbone == 'latentTF':
            self._model = latentTFBackbone(config, image_architecture, lidar_architecture, use_velocity=use_velocity).to(self.device)
        else:
            raise RuntimeError('implemented backbones: "transFuser", "late_fusion", "geometric_fusion", "latentTF"; got %r' % (backbone,))
        if config.multitask:
            self.seg_decoder = SegDecoder(config, config.perception_output_features).to(self.device)
            self.depth_decoder = DepthDecoder(config, config.perception_output_features).to(self.device)
        channel = config.channel
        self.pred_bev = nn.Sequential(nn.Conv2d(channel, channel, kernel_size=(3, 3), stride=1, padding=(1, 1), bias=True),
                                      nn.ReLU(inplace=True),
                                      nn.Conv2d(channel, 3, kernel_size=(1, 1), stride=1, padding=0, bias=True)).to(self.device)
        self.head = LidarCenterNetHead(channel, channel, 1, train_cfg=config).to(self.device)
        self.i = 0
        self.join = nn.Sequential(nn.Linear(512, 256), nn.ReLU(inplace=True), nn.Linear(256, 128), nn.ReLU(inplace=True),
                                  nn.Linear(128, 64), nn.ReLU(inplace=True)).to(self.device)
        self.decoder = nn.GRUCell(input_size=4, hidden_size=config.gru_hidden_size).to(self.device)
        self.output = nn.Linear(config.gru_hidden_size, 3).to(self.device)
        self.register_buffer('_bev_class_weight', torch.tensor([1., 1., 3.], device=self.device), persistent=False)

    def forward_gru(self, z, target_point):
        for i in (0, 2, 4):
            z = ops.linear(z, self.join[i].weight, self.join[i].bias, relu=True)
        d = self.decoder
        pred_wp = ops.GRUFn.apply(z, target_point, d.weight_ih, d.weight_hh, d.bias_ih, d.bias_hh, self.output.weight, self.output.bias,
                                  self.pred_len, float(self.config.lidar_pos[0]))
        return pred_wp, None, None, None, None

    def _run_backbone(self, rgb, lidar_bev, bev_points, cam_points, ego_vel=None):
        if self.backbone == 'geometric_fusion':
            if bev_points is None or cam_points is None:
                raise RuntimeError('the geometric_fusion backbone needs bev_points and cam_points (train.py:281-288)')
            return self._model.forward_nhwc(rgb, lidar_bev, bev_points, cam_points)
        if self.backbone in ('transFuser', 'latentTF') and self._model.transformer1.use_velocity:   # (latentTF.py:144-195: same GPTs)
            return self._model.forward_nhwc(rgb, lidar_bev, velocity=ego_vel)      # model.py:753 passes ego_vel to the backbone
        return self._model.forward_nhwc(rgb, lidar_bev)

    def get_bbox_local_metric(self, bbox):
        """model.py:810-842: one decoded row (x, y, w, h, yaw, speed, brake, confidence; LiDAR-BEV pixels) -> (6x3 array: the
        4 corners, centre and velocity tip in the ego frame in metres; brake; confidence). Host numpy, as in the reference."""
        cfg = self.config
        x, y, w, h, yaw, speed, brake, confidence = bbox
        scale = cfg.bounding_box_divisor * cfg.pixels_per_meter
        w, h = w / scale, h / scale
        # inverse of utils.py:29-37's LiDAR -> BEV-image map  p = 8 * [[0,-1,16],[-1,0,32]] @ (X, Y, 1)
        ppm = 8.0
        cx = (32.0 * ppm - y) / ppm + cfg.lidar_pos[0]
        cy = -((16.0 * ppm - x) / ppm + cfg.lidar_pos[1])
        c, s_ = np.cos(yaw), np.sin(yaw)
        local = np.array([[-h, -w], [-h, w], [h, w], [h, -w], [0.0, 0.0], [0.0, h * speed * 0.5]], dtype=np.float64)
        out = np.ones((6, 3), dtype=np.float64)
        out[:, 0] = c * local[:, 0] - s_ * local[:, 1] + cx
        out[:, 1] = s_ * local[:, 0] + c * local[:, 1] + cy
        return out, brake, confidence

    @torch.no_grad()
    def forward_ego(self, rgb, lidar_bev, target_point, target_point_image, ego_vel, bev_points=None, cam_points=None, save_path=None,
                    expert_waypoints=None, stuck_detector=0, forced_move=False, num_points=None, rgb_back=None, debug=False):
        """model.py:685-731: (pred_wp [B,4,2], list of (corners, brake, confidence) for sample 0's boxes above
        config.bb_confidence_threshold). Debug visualisation (model.py:720-728) is not implemented."""
        if debug and save_path is not None:
            raise RuntimeError('forward_ego(debug=True) visualisation is out of scope')
        if self.use_target_point_image:
            lidar_bev = torch.cat((lidar_bev, target_point_image), dim=1)
        features, _, fused_features = self._run_backbone(rgb, lidar_bev, bev_points, cam_points, ego_vel)
        pred_wp, _, _, _, _ = self.forward_gru(fused_features, target_point)
        bboxes, _ = self.head.get_bboxes_nhwc(self.head.run(features[0]))[0]
        bboxes = bboxes[bboxes[:, -1] > self.config.bb_confidence_threshold]
        rotated_bboxes = [self.get_bbox_local_metric(b) for b in bboxes.cpu().numpy()]
        self.i += 1
        return pred_wp, rotated_bboxes

    def forward(self, rgb, lidar_bev, ego_waypoint, target_point, target_point_image, ego_vel, bev, label, depth, semantic,
                num_points=None, save_path=None, bev_points=None, cam_points=None):
        cfg = self.config
        loss = {}
        if self.use_target_point_image:
            lidar_bev = torch.cat((lidar_bev, target_point_image), dim=1)
        features, image_features_grid, fused_features = self._run_backbone(rgb, lidar_bev, bev_points, cam_points, ego_vel)
        two = ops.TWO_STREAMS and cfg.multitask
        if two:
            # auxiliary decoders (image grid -> 160x704 maps) on the second stream, concurrently with the BEV-side heads
            main, side = torch.cuda.current_stream(), ops.side_stream(rgb.device)
            # the two decoders are independent chains of mostly latency-bound launches (5x22 -> 160x704): one side stream each
            side2 = ops.side_stream2(rgb.device) if ops.DECODER_STREAMS else side
            side.wait_stream(main)
            ops.record_stream(image_features_grid, side)
            if side2 is not side:
                side2.wait_stream(main)
                ops.record_stream(image_features_grid, side2)
            with torch.cuda.stream(side):
                pred_semantic = self.seg_decoder.run(image_features_grid)
                loss_semantic = ops.CrossEntropyFn.apply(pred_semantic, semantic, None, 'count', float(cfg.ls_seg))
            with torch.cuda.stream(side2):
                pred_depth = self.depth_decoder.run(image_features_grid)
                loss_depth = ops.L1Fn.apply(pred_depth.view(pred_depth.shape[0], pred_depth.shape[1], pred_depth.shape[2]), depth, True, float(cfg.ls_depth))

        pred_wp, _, _, _, _ = self.forward_gru(fused_features, target_point)

        pred_bev = _run_pair(self.pred_bev, features[0])
        pred_bev = ops.upsample(pred_bev, cfg.bev_resolution_height, cfg.bev_resolution_width, True)
        w = self._bev_class_weight
        if w.device != pred_bev.device:
            w = self._bev_class_weight = w.to(pred_bev.device)
        loss['loss_wp'] = ops.L1Fn.apply(pred_wp, ego_waypoint, False, 1.0)
        loss['loss_bev'] = ops.CrossEntropyFn.apply(pred_bev, bev, w, 'wsum', 1.0)

        preds = self.head.run(features[0])
        H, W = preds.shape[1], preds.shape[2]
        head_losses = ops.CenterNetLossFn.apply(preds, label, float(W / cfg.lidar_resolution_width), float(H / cfg.lidar_resolution_height),
                                               cfg.num_dir_bins)
        for i, k in enumerate(HEAD_LOSSES):
            loss[k] = head_losses[i]

        if two:
            main.wait_stream(side)
            if side2 is not side:
                main.wait_stream(side2)
            loss_depth.record_stream(main)
            loss_semantic.record_stream(main)
            loss['loss_depth'], loss['loss_semantic'] = loss_depth, loss_semantic
        elif cfg.multitask:
            pred_semantic = self.seg_decoder.run(image_features_grid)
            pred_depth = self.depth_decoder.run(image_features_grid)
            loss['loss_depth'] = ops.L1Fn.apply(pred_depth.view(pred_depth.shape[0], pred_depth.shape[1], pred_depth.shape[2]), depth, True, float(cfg.ls_depth))
            loss['loss_semantic'] = ops.CrossEntropyFn.apply(pred_semantic, semantic, None, 'count', float(cfg.ls_seg))
        else:
            loss['loss_depth'] = torch.zeros_like(loss['loss_wp'])
            loss['loss_semantic'] = torch.zeros_like(loss['loss_wp'])
        self.i += 1
        return loss
