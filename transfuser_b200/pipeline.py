"""GPU input pipeline (SURVEY.md §8f rank 2): the device side of CARLA_Data.__getitem__
(team_code_transfuser/data.py:103-356) for a whole batch, fed with compact inputs.

The reference prepares every sample on CPU workers (numpy / OpenCV) and ships expanded tensors: fp32 RGB (1.35 MB), fp32
LiDAR histogram + target map (0.79 MB), float depth and int64 semantics (0.45 + 0.90 MB) per sample. Here the host ships
what is on disk — uint8 frames, raw points, one 4x4 pose transform, the target point — and three launches build the model
inputs in HBM (csrc/input_prep.cu, csrc/bev_hist.cu):

    batch = InputPipeline(config, device).prepare(raw)      # raw: dict of pinned host / device tensors, see prepare()
    losses = model(batch['rgb'], batch['lidar'], target_point_image=batch['target_point_image'], ...)

Host-side pieces that stay numpy, as in the reference (tiny, per sample): the pose algebra of align() (data.py:413-431) and
the augmentation draw. JPEG/PNG decoding, label parsing and the BEV-label rotation (skimage) are not part of this module."""
import numpy as np
import torch

from . import _lib

LIDAR_TO_VEHICLE = np.array([[0., 1., 0., 1.3], [-1., 0., 0., 0.0], [0., 0., 1., 2.5], [0., 0., 0., 1.]])   # utils.py:14-24


def align_transform(ego_matrix_0, ego_matrix_1, degree=0.0):
    """4x4 float64 matrix of align() (data.py:413-431): LiDAR frame of measurement 0 -> LiDAR frame of measurement 1, followed
    by the augmentation rotation by `degree`."""
    m0, m1 = np.asarray(ego_matrix_0, dtype=np.float64), np.asarray(ego_matrix_1, dtype=np.float64)
    T = np.linalg.inv(LIDAR_TO_VEHICLE) @ np.linalg.inv(m1) @ m0 @ LIDAR_TO_VEHICLE
    rad = np.deg2rad(degree)
    c, s = np.cos(rad), np.sin(rad)
    return np.array([[c, s, 0, 0], [-s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]]) @ T


def crop_shift_pixels(degree, img_width, scale):
    """data.py:219: horizontal crop shift that accompanies an augmentation yaw of `degree` (truncated like int())."""
    return int(degree / 60 * img_width / scale)


class InputPipeline:
    def __init__(self, config, device, crop=(160, 704)):
        self.device = torch.device(device)
        self.crop = tuple(crop)
        conv = getattr(config, 'converter', None)
        lut = np.zeros(256, dtype=np.uint8)
        if conv is not None:
            lut[:len(conv)] = np.uint8(conv)
        self.has_lut = conv is not None
        self.lut = torch.from_numpy(lut).to(self.device)

    def _require_cuda(self):
        if self.device.type != 'cuda':
            raise RuntimeError('InputPipeline needs a CUDA device (no CPU fallback)')

    def _dev(self, t, dtype):
        t = torch.as_tensor(t)
        if t.dtype != dtype:
            raise TypeError('expected %s, got %s' % (dtype, t.dtype))
        return t.to(self.device, non_blocking=True).contiguous()

    def _out(self, out, key, shape, dtype):
        """Destination tensor: the caller's preallocated one (e.g. a static CUDA-graph input buffer) or a fresh allocation."""
        t = None if out is None else out.get(key)
        if t is None:
            return torch.empty(shape, dtype=dtype, device=self.device)
        if tuple(t.shape) != tuple(shape) or t.dtype != dtype or not t.is_cuda or not t.is_contiguous():
            raise ValueError('out[%r] must be a contiguous CUDA %s tensor of shape %s' % (key, dtype, tuple(shape)))
        return t

    def prepare(self, raw, normalized_nhwc=False, out=None):
        """raw (host or device tensors):
             rgb [B,H,W,3] uint8 (RGB), optional depth [B,H,W,3] uint8, seg [B,H,W] uint8, crop_shift [B] int32 (host values),
             points [B,N,4] float32 (padded), optional n_valid [B] int32, transforms [B,4,4] float64 (align_transform),
             target_point [B,2] float64.
           Returns rgb [B,3,h,w] float32 0..255 (or, with normalized_nhwc, the normalised NHWC tensor the backbone consumes
           directly), lidar [B,2,256,256], target_point_image [B,1,256,256], target_point [B,2] float32, and depth [B,h,w] /
           semantic [B,h,w] int64 when their sources are given. `out` (optional dict) supplies preallocated destinations
           by the same keys, so the three launches can write straight into the static inputs of a captured training step."""
        self._require_cuda()
        res = {}
        rgb = self._dev(raw['rgb'], torch.uint8)
        B, H, W, _ = rgb.shape
        ch, cw = self.crop
        cs = raw.get('crop_shift')
        if isinstance(cs, torch.Tensor) and cs.is_cuda:
            # device-resident shifts (the static inputs of a captured training step): validated on the host when they were produced
            # (no device -> host read here: it would synchronise, and is illegal inside a CUDA-graph capture)
            if ch > H or cw > W or cs.dtype != torch.int32:
                raise ValueError('crop %s does not fit the %dx%d frame / crop_shift must be int32' % (self.crop, H, W))
            shift = cs.contiguous()
        else:
            shift_host = torch.as_tensor(cs if cs is not None else torch.zeros(B, dtype=torch.int32)).to('cpu', torch.int32)
            x0 = W // 2 - cw // 2 + shift_host
            if ch > H or cw > W or int(x0.min()) < 0 or int(x0.max()) + cw > W:
                raise ValueError('crop %s with shifts %s leaves the %dx%d frame' % (self.crop, shift_host.tolist(), H, W))
            shift = shift_host.to(self.device, non_blocking=True)
        depth = self._dev(raw['depth'], torch.uint8) if raw.get('depth') is not None else None
        seg = self._dev(raw['seg'], torch.uint8) if raw.get('seg') is not None else None
        if seg is not None and not self.has_lut:
            raise RuntimeError('config.converter is needed to map the semantic classes (data.py:36)')
        rgb_out = None if normalized_nhwc else self._out(out, 'rgb', (B, 3, ch, cw), torch.float32)
        rgb_norm = self._out(out, 'rgb', (B, ch, cw, 3), torch.float32) if normalized_nhwc else None
        depth_out = self._out(out, 'depth', (B, ch, cw), torch.float32) if depth is not None else None
        seg_out = self._out(out, 'semantic', (B, ch, cw), torch.int64) if seg is not None else None
        _lib.call('tfb_camera_prep', rgb, depth, seg, shift, self.lut, B, H, W, ch, cw, rgb_out, rgb_norm, depth_out, seg_out)
        if normalized_nhwc:
            rgb_norm._tfb_nhwc_normalized = True       # ops.image_prep passes such a tensor through untouched
        res['rgb'] = rgb_norm if normalized_nhwc else rgb_out
        if depth_out is not None:
            res['depth'] = depth_out
        if seg_out is not None:
            res['semantic'] = seg_out

        points = torch.as_tensor(raw['points'])
        if points.dim() != 3 or points.shape[2] != 4 or points.dtype not in (torch.float32, torch.float64):
            raise ValueError('points must be [B, N, 4] float32/float64')
        points = points.to(self.device, non_blocking=True).contiguous()
        T = self._dev(torch.as_tensor(raw['transforms']).reshape(B, 16), torch.float64)
        n_valid = self._dev(raw['n_valid'], torch.int32) if raw.get('n_valid') is not None else None
        counts = torch.empty((B, 2, 256, 256), dtype=torch.int32, device=self.device)
        lidar = self._out(out, 'lidar', (B, 2, 256, 256), torch.float32)
        _lib.call('tfb_bev_histogram_aligned', points, 1 if points.dtype == torch.float64 else 0, T, n_valid, B, points.shape[1], counts, lidar)
        res['lidar'] = lidar

        tp = self._dev(raw['target_point'], torch.float64)
        tpi = self._out(out, 'target_point_image', (B, 1, 256, 256), torch.float32)
        _lib.call('tfb_draw_target_point', tp, B, tpi)
        res['target_point_image'] = tpi
        tpf = self._out(out, 'target_point', (B, 2), torch.float32)
        tpf.copy_(tp)
        res['target_point'] = tpf
        return res
