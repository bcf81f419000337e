"""GPU input pipeline (SURVEY.md §8f rank 2): the device side of CARLA_Data.__getitem__
(team_code_transfuser/data.py:103-356) for a whole batch, fed with compact inputs.

The reference prepares every sample on CPU workers (numpy / OpenCV) and ships expanded tensors: fp32 RGB (1.35 MB), fp32
LiDAR histogram + target map (0.79 MB), float depth and int64 semantics (0.45 + 0.90 MB) per sample. Here the host ships
what is on disk — uint8 frames, raw points, one 4x4 pose transform, the target point — and three launches build the model
inputs in HBM (csrc/input_prep.cu, csrc/bev_hist.cu):

    batch = InputPipeline(config, device).prepare(raw)      # raw: dict of pinned host / device tensors, see prepare()
    losses = model(batch['rgb'], batch['lidar'], target_point_image=batch['target_point_image'], ...)

Host-side pieces that stay numpy, as in the reference (tiny, per sample): the pose algebra of align() (data.py:413-431) and
the augmentation draw. With the topdown plane and the matrix of bev_rotation_matrix, a fourth launch builds the rotated BEV label
(csrc/bev_label.cu, skimage's rotate in load_crop_bev_npy). With a per-sample seed, a fifth launch builds the geometric-fusion
LiDAR <-> camera correspondences of the sweep (csrc/correspondences.cu, lidar_bev_cam_correspondences). PNG decoding and label
parsing stay on the host (dataset.py)."""
import math

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


def _mat3(a, b):
    return [[(a[i][0] * b[0][j] + a[i][1] * b[1][j]) + a[i][2] * b[2][j] for j in range(3)] for i in range(3)]


def bev_rotation_matrix(degree, H, W):
    """The 2x3 float64 output -> input matrix of skimage.transform.rotate(image of H x W, degree) that load_crop_bev_npy
    (data.py:601) applies to the BEV label, as the [6] row-major input of tfb_bev_label_prep.

    skimage composes translate(-c) -> rotate(rad) -> translate(c), c = (W/2 - 0.5, H/2 - 0.5), as T1 . (R . T3). This computes
    it in scalar Python floats: rad = degree * (pi / 180) (np.deg2rad), math.cos / math.sin, and every entry of the two 3x3
    products as ((a0*b0 + a1*b1) + a2*b2). It equals skimage's matrix on a BLAS without fused multiply-add (numpy's `@` may go
    through an FMA dgemm, which would make the result depend on the host)."""
    degree = float(degree)
    cx, cy = W / 2. - 0.5, H / 2. - 0.5
    rad = degree * (math.pi / 180)
    t1 = [[math.cos(0.0), -math.sin(0.0), cx], [math.sin(0.0), math.cos(0.0), cy], [0.0, 0.0, 1.0]]
    t2 = [[math.cos(rad), -math.sin(rad), 0.0], [math.sin(rad), math.cos(rad), 0.0], [0.0, 0.0, 1.0]]
    t3 = [[math.cos(0.0), -math.sin(0.0), -cx], [math.sin(0.0), math.cos(0.0), -cy], [0.0, 0.0, 1.0]]
    m = _mat3(t1, _mat3(t2, t3))
    assert m[2] == [0.0, 0.0, 1.0], m[2]        # affine: the kernel's projective divide is by exactly 1
    return np.array(m[0] + m[1], dtype=np.float64)


def correspondence_constants():
    """The host constants of tfb_lidar_cam_correspondences, from the reference's own numpy expressions: [20] float64 = focal_x,
    focal_y (data.py:701-706), the left (-60 degrees) and right (+60 degrees) camera rotations row-major (data.py:740-745, 763-768),
    and the float32 z shift float32(2.5 - 2.3) (data.py:718: a float32 array plus a Python float)."""
    img_width, img_height, fov_width = 352, 160, 60
    fov_height = np.rad2deg(2.0 * np.arctan((img_height / img_width) * np.tan(0.5 * np.radians(fov_width))))
    focal_x = img_width / (2.0 * np.tan(np.deg2rad(fov_width) / 2.0))
    focal_y = img_height / (2.0 * np.tan(np.deg2rad(fov_height) / 2.0))
    rot = []
    for angle in (-60.0, 60.0):
        theta = np.radians(angle)
        rot += [np.cos(theta), -np.sin(theta), 0.0, np.sin(theta), np.cos(theta), 0.0, 0.0, 0.0, 1.0]
    return np.array([focal_x, focal_y] + rot, dtype=np.float64), np.float32(2.5 - 2.3)


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
        consts, self.corr_dz = correspondence_constants()
        self.corr_consts = torch.from_numpy(consts).to(self.device)

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
             target_point [B,2] float64, optional bev_u8 [B,H,W] uint8 (RGB plane 2 of topdown/encoded_*.png) with bev_matrix
             [B,6] float64 (bev_rotation_matrix of each sample's augmentation angle), optional corr_seed [B] int64 >= 0 (the
             geometric-fusion correspondences of the float32 sweep, data.py:675-842; the seed picks the entries of cells with
             more than 5 candidates, csrc/correspondences.cu).
           Returns rgb [B,3,h,w] float32 0..255 (or, with normalized_nhwc, the normalised NHWC tensor the backbone consumes
           directly), lidar [B,2,256,256], target_point_image [B,1,256,256], target_point [B,2] float32, and depth [B,h,w] /
           semantic [B,h,w] int64 when their sources are given, and the rotated BEV label bev [B,160,160] int64
           (load_crop_bev_npy, csrc/bev_label.cu) when bev_u8 is given, and bev_points [B,8,8,5,2] / cam_points [B,22,5,5,2] int64
           when corr_seed is given. `out` (optional dict) supplies preallocated destinations
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

        if (raw.get('bev_u8') is None) != (raw.get('bev_matrix') is None):
            raise ValueError('bev_u8 and bev_matrix go together')
        if raw.get('bev_u8') is not None:
            plane = self._dev(raw['bev_u8'], torch.uint8)
            m = torch.as_tensor(raw['bev_matrix'])
            if plane.dim() != 3 or plane.shape[0] != B or plane.shape[1] < 250 or plane.shape[2] < 330:
                raise ValueError('bev_u8 must be [B, H >= 250, W >= 330] uint8, got %s' % (tuple(plane.shape),))
            if tuple(m.shape) != (B, 6):
                raise ValueError('bev_matrix must be [B, 6] float64 (bev_rotation_matrix), got %s' % (tuple(m.shape),))
            if not m.is_cuda and not bool(torch.isfinite(m).all()):
                raise ValueError('bev_matrix holds a non-finite value')
            m = self._dev(m, torch.float64)
            bev_out = self._out(out, 'bev', (B, 160, 160), torch.int64)
            _lib.call('tfb_bev_label_prep', plane, m, B, plane.shape[1], plane.shape[2], bev_out)
            res['bev'] = bev_out

        if raw.get('corr_seed') is not None:
            if points.dtype != torch.float32:
                raise ValueError('the correspondences read a float32 sweep (the dtype dataset.CarlaRawDataset ships)')
            seed = self._dev(raw['corr_seed'], torch.int64)
            if tuple(seed.shape) != (B,):
                raise ValueError('corr_seed must be [B] int64, got %s' % (tuple(seed.shape),))
            N = points.shape[1]
            work = torch.empty((B, 6 * max(N, 1)), dtype=torch.int32, device=self.device)
            bev_pts = self._out(out, 'bev_points', (B, 8, 8, 5, 2), torch.int64)
            cam_pts = self._out(out, 'cam_points', (B, 22, 5, 5, 2), torch.int64)
            _lib.call('tfb_lidar_cam_correspondences', points, n_valid, seed, self.corr_consts, float(self.corr_dz), B, N, work, bev_pts, cam_pts)
            res['bev_points'], res['cam_points'] = bev_pts, cam_pts
        return res
