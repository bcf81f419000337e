"""Reader of the on-disk CARLA dataset (the layout the reference's CARLA_Data reads, team_code_transfuser/data.py:16-356) that
hands the GPU input pipeline its compact inputs instead of the expanded tensors:

    ds = CarlaRawDataset(roots, TrainConfig(), backbone='transFuser', max_points=40000)
    loader = DataLoader(ds, batch_size=B, num_workers=n, collate_fn=collate, pin_memory=True, drop_last=True)
    tr = Trainer(cfg, 'cuda', raw_inputs='dataset')
    for batch in loader: ... tr.step / tr.load + tr.replay

Per sample the host decodes the PNGs with OpenCV (as the reference does), draws the augmentation angle with the same
`random.random()` calls in the same order (data.py:213-220), parses the labels and waypoints in numpy, and ships uint8 frames,
the raw LiDAR sweep, the topdown plane that holds the two BEV channels, and float64 matrices. On the GPU (pipeline.InputPipeline)
the frames are cropped and shifted, the sweep is aligned and binned, the target point is drawn, and the BEV label is rotated
(csrc/bev_label.cu in place of skimage's rotate in load_crop_bev_npy).

Geometric fusion, with the correspondences built on the GPU:

    ds = CarlaRawDataset(roots, TrainConfig(), backbone='geometric_fusion', correspondences='gpu', max_points=40000)
    tr = Trainer(cfg, 'cuda', backbone='geometric_fusion', raw_inputs='dataset')

The reader does not compute the reference's host-side correspondences (lidar_bev_cam_correspondences, data.py:632-842, with
its random.sample calls), so backbone='geometric_fusion' alone is refused and correspondences='gpu' opts in: a sample then also
ships `corr_seed`, drawn with random.getrandbits(63) after the augmentation angle, and the correspondences are built on the GPU
from the same raw sweep (csrc/correspondences.cu). Cells with at most 5 candidates equal the reference's; in fuller cells the
seed picks the 5 entries where the reference calls random.sample. Those random.sample calls consume a reference worker's RNG
state and this draw consumes different state, so the first sample's angle is the reference's but later samples' angles of the
same worker diverge from a reference worker's.

Out of scope, and refused: seq_len > 1, PointPillars, the reference's host-side correspondences, the reference's in-memory
cache."""
import json
import os
import random
from pathlib import Path

import numpy as np
import torch

from . import pipeline

# data.py:14 -> utils.py:3-12, 29-37
_VEHICLE_TO_VIRTUAL_LIDAR = np.linalg.inv(np.array([[1., 0., 0., 1.3], [0., 1., 0., 0.], [0., 0., 1., 2.5], [0., 0., 0., 1.]]))
_LIDAR_TO_BEVIMAGE = np.array([[0, -1, 16], [-1, 0, 32], [0, 0, 1]], dtype=np.float32)
_LIDAR_TO_BEVIMAGE[:2, :] *= 8

MAX_BOXES = 20


def _read_json(path):
    with open(path, 'r') as f:
        return json.load(f)


def _imread(path, flags):
    import cv2
    img = cv2.imread(str(path), flags)
    if img is None:
        raise FileNotFoundError('cannot decode %s' % path)
    return img


def scale_image(image, scale, nearest=False):
    """scale_image_cv2 (data.py:521-524) / scale_seg (data.py:562-568)."""
    import cv2
    if nearest:
        if scale == 1:
            return image
        return cv2.resize(image, (int(image.shape[1] / scale), int(image.shape[0] / scale)), interpolation=cv2.INTER_NEAREST)
    return cv2.resize(image, (int(image.shape[1] // scale), int(image.shape[0] // scale)))


def parse_labels(labels, rad):
    """parse_labels(labels, rad) + get_bbox_label (data.py:472-514): {id: [x, y, w, h, yaw, speed, brake]} in BEV-image pixels
    of the boxes that stay strictly inside the 0..255 frame after the rotation and the clip, in the order of the file."""
    c, s = np.cos(rad), np.sin(rad)
    T = _LIDAR_TO_BEVIMAGE @ np.array([[c, s, 0], [-s, c, 0], [0, 0, 1]])
    boxes = {}
    for r in labels:
        dz, dx, dy = r['extent']
        x, y, z = r['position']
        pos = np.clip(T @ np.array([x, y, 1.0]).reshape([3, 1]), 0., 255.)
        px, py = pos[:2, 0]
        if r['num_points'] <= 1 or px <= 0.0 or px >= 255.0 or py <= 0.0 or py >= 255.0:
            continue
        boxes[r['id']] = np.array([px, py, dy * 8, dx * 8, r['yaw'] + rad, r['speed'], r['brake']])
    return boxes


def ego_waypoints(labels, rad):
    """get_waypoints -> transform_waypoints -> the ego's row -> rotated by the augmentation (data.py:277-305), float64 [pred_len, 2]."""
    ego = labels[0][0]
    track = [ego['ego_matrix']]
    for frame in labels[1:]:
        track += [r['ego_matrix'] for r in frame if r['id'] == ego['id']]
    track += [np.eye(4)] * (len(labels) - len(track))
    inv0 = np.linalg.inv(np.array(track[0]))
    wp = np.array([(_VEHICLE_TO_VIRTUAL_LIDAR @ inv0 @ np.array(m))[:2, 3] for m in track[1:]])
    R = np.array([[np.cos(rad), np.sin(rad)], [-np.sin(rad), np.cos(rad)]])
    return (R @ wp.T).T


def target_point(m, rad):
    """data.py:340-353: the route's next command point in the ego frame, with the augmentation yaw added to the heading."""
    theta = m['theta'] + rad
    R = np.array([[np.cos(np.pi / 2 + theta), -np.sin(np.pi / 2 + theta)], [np.sin(np.pi / 2 + theta), np.cos(np.pi / 2 + theta)]])
    return R.T.dot(np.array([m['x_command'] - m['x'], m['y_command'] - m['y']]))


class CarlaRawDataset(torch.utils.data.Dataset):
    def __init__(self, roots, config, backbone='transFuser', max_points=None, correspondences=None):
        if int(config.seq_len) != 1:
            raise NotImplementedError('CarlaRawDataset reads seq_len == 1 (the reference default) only')
        if correspondences not in (None, 'gpu'):
            raise ValueError("correspondences must be None or 'gpu'")
        self.geometric = backbone == 'geometric_fusion'
        if self.geometric and correspondences != 'gpu':
            raise NotImplementedError("the reference's host-side geometric-fusion correspondences are not produced by CarlaRawDataset; "
                                      "pass correspondences='gpu' to ship a per-sample seed and build them on the GPU "
                                      "(InputPipeline.prepare(corr_seed=))")
        if correspondences == 'gpu' and not self.geometric:
            raise ValueError("correspondences='gpu' is for backbone='geometric_fusion'")
        if getattr(config, 'use_point_pillars', False):
            raise NotImplementedError('PointPillars inputs are not produced by CarlaRawDataset')
        self.pred_len = int(config.pred_len)
        self.scale = config.scale
        self.img_width = config.img_width
        self.crop = tuple(config.img_resolution)
        self.augment = bool(config.augment)
        self.inv_augment_prob = config.inv_augment_prob
        self.aug_max_rotation = config.aug_max_rotation
        self.max_points = int(max_points if max_points is not None else config.max_lidar_points)
        self.frames = []            # (route directory, frame)
        # the route index of CARLA_Data.__init__ (data.py:46-85): every sub-directory of a root is a route; its first two and
        # last (pred_len + seq_len + 2) frames are skipped
        for root in roots:
            root = Path(root)
            for route in os.listdir(root):
                if os.path.isfile(os.path.join(root, route)):
                    continue
                n = len(os.listdir(root / route / 'lidar'))
                for seq in range(2, n - self.pred_len - 1 - 2):
                    self.frames.append((str(root / route), seq))

    def __len__(self):
        return len(self.frames)

    def draw_degree(self):
        """The augmentation draw of data.py:213-220, random.random() call for call."""
        degree = 0
        if self.augment and random.random() > self.inv_augment_prob:
            degree = (random.random() * 2. - 1.) * self.aug_max_rotation
        return degree

    def __getitem__(self, index):
        import cv2
        route, seq = self.frames[index]
        d = Path(route)
        labels = [_read_json(d / 'label_raw' / ('%04d.json' % (seq + i))) for i in range(1 + self.pred_len)]
        m = _read_json(d / 'measurements' / ('%04d.json' % seq))
        pts = np.load(str(d / 'lidar' / ('%04d.npy' % seq)), allow_pickle=True)[1]   # the reference's pickled layout: [.., XYZI]
        pts[:, 1] *= -1
        rgb = scale_image(cv2.cvtColor(_imread(d / 'rgb' / ('%04d.png' % seq), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB), self.scale)
        top = cv2.cvtColor(_imread(d / 'topdown' / ('encoded_%04d.png' % seq), cv2.IMREAD_UNCHANGED), cv2.COLOR_BGR2RGB)
        depth = scale_image(cv2.cvtColor(_imread(d / 'depth' / ('%04d.png' % seq), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB), self.scale)
        seg = scale_image(_imread(d / 'semantics' / ('%04d.png' % seq), cv2.IMREAD_UNCHANGED), self.scale, nearest=True)

        degree = self.draw_degree()
        corr_seed = random.getrandbits(63) if self.geometric else None    # after the angle: the angle stays the reference's
        rad = np.deg2rad(degree)
        if len(pts) > self.max_points:
            raise ValueError('%s/lidar/%04d.npy holds %d points, more than max_points = %d' % (route, seq, len(pts), self.max_points))
        points = np.zeros((self.max_points, 4), dtype=np.float32)
        points[:len(pts)] = pts
        boxes = parse_labels(labels[0], -rad)
        if len(boxes) > MAX_BOXES:
            raise ValueError('%s/label_raw/%04d.json: %d boxes survive the filters, at most %d fit the label' % (route, seq, len(boxes), MAX_BOXES))
        label = np.zeros((MAX_BOXES, 7), dtype=np.float32)
        if boxes:
            label[:len(boxes)] = np.array(list(boxes.values()))
        plane = np.ascontiguousarray(top[..., 2])
        sample = dict(
            rgb_u8=np.ascontiguousarray(rgb), depth_u8=np.ascontiguousarray(depth), seg_u8=np.ascontiguousarray(seg),
            bev_u8=plane, bev_matrix=pipeline.bev_rotation_matrix(degree, plane.shape[0], plane.shape[1]),
            points=points, n_valid=np.int32(len(pts)),
            transforms=pipeline.align_transform(m['ego_matrix'], m['ego_matrix'], degree),
            crop_shift=np.int32(pipeline.crop_shift_pixels(degree, self.img_width, self.scale)),
            target_point64=target_point(m, rad), ego_waypoint=ego_waypoints(labels, rad).astype(np.float32),
            label=label, ego_vel=np.array([m['speed']], dtype=np.float32), degree=np.float64(degree))
        if corr_seed is not None:
            sample['corr_seed'] = np.int64(corr_seed)
        return sample


def collate(samples):
    """Stacks CarlaRawDataset samples into a batch of host tensors (the keys of Trainer(raw_inputs='dataset'), plus the drawn
    angle `degree`). Called in the main process with a CUDA device present, the tensors are pinned; in a DataLoader worker
    they are not (a forked worker must not touch CUDA): pass pin_memory=True to the DataLoader, which pins them there."""
    out = {k: torch.from_numpy(np.stack([np.asarray(s[k]) for s in samples])) for k in samples[0]}
    if torch.utils.data.get_worker_info() is None and torch.cuda.is_available():
        out = {k: v.pin_memory() for k, v in out.items()}
    return out
