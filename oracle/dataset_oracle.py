"""ORACLE / TEST INFRASTRUCTURE ONLY — never imported by the product path.

numpy restatement of what CARLA_Data.__getitem__ (data.py:103-356) computes from the compact sample of
transfuser_b200.dataset.CarlaRawDataset, in the dtypes the training step consumes:
  bev_label            load_crop_bev_npy (data.py:586-612) of decode_pil_to_npy's channels 10 / 11 (data.py:844-856), with
                       skimage's rotate through the shim in oracle/shims/skimage
  expand               the camera crop / depth / classes, aligned LiDAR histogram and target-point map (pipeline_oracle,
                       bev_oracle) plus bev_label
Pinned against the reference itself through tests/golden/reference_dataset.npz (oracle/make_golden_dataset.py)."""
import os
import sys

import numpy as np

from oracle import bev_oracle, pipeline_oracle as PO
from oracle.make_golden_reference import digest  # noqa: F401  (sha256 of dtype, shape and bytes: the fixtures' digest)

SHIMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'shims')


def _shim_transform():
    if SHIMS not in sys.path:
        sys.path.insert(0, SHIMS)
    from skimage import transform
    return transform


def bev_channels(plane):
    """decode_pil_to_npy's channels 10 and 11 of RGB plane 2: bits 7 and 6, as float32 [H, W, 2]."""
    p = np.asarray(plane, dtype=np.uint8)
    return np.stack([(p >> 7) & 1, (p >> 6) & 1], axis=-1).astype(np.float32)


def bev_label(plane, degree):
    """int64 [160, 160] classes of load_crop_bev_npy."""
    bev = bev_channels(plane)
    shifted = np.zeros_like(bev)
    shifted[7:] = bev[:-7]
    rot = _shim_transform().rotate(shifted, degree)
    crop = np.moveaxis(rot[90:250, 170:330], -1, 0)
    stack = np.concatenate((np.zeros_like(crop[:1]), crop[:1], crop[:1] + crop[1:2]), axis=0)
    return np.argmax(stack, axis=0)


def expand(s, converter, crop=(160, 704)):
    """The expanded arrays of one compact sample: rgb uint8 [3,h,w], depth float32, semantic int64, lidar float32 [2,256,256],
    target_point_image float32 [1,256,256], bev int64 [160,160]."""
    shift = int(s['crop_shift'])
    pts = np.asarray(s['points'])[:int(s['n_valid'])]
    return dict(rgb=PO.crop_rgb(s['rgb_u8'], crop, shift),
                depth=PO.depth_from_rgb(PO.crop_rgb(s['depth_u8'], crop, shift)).astype(np.float32),
                semantic=PO.seg_classes(s['seg_u8'], converter, crop, shift).astype(np.int64),
                lidar=bev_oracle.lidar_to_histogram_features(PO.align_points(pts, s['transforms'])),
                target_point_image=PO.draw_target_point(s['target_point64']).astype(np.float32),
                bev=bev_label(s['bev_u8'], float(s['degree'])))


ANGLES = (0.0, 1e-9, -1e-9, 19.999, -19.999, 20.0, -20.0, 45.0, 90.0, 180.0)


def angle_sweep(n_random=200, seed=7):
    """The angles of the fixture's load_crop_bev_npy digests: the fixed edge values, then n_random seeded draws in [-200, 200)."""
    rng = np.random.default_rng(seed)
    return list(ANGLES) + [float(a) for a in rng.uniform(-200, 200, n_random)]


def sweep_planes():
    """The seeded 500 x 500 planes of the angle sweep: random bytes, and one with rectangles in bits 7 / 6 and stray lower bits."""
    rng = np.random.default_rng(99)
    noise = rng.integers(0, 256, (500, 500), dtype=np.uint8)
    rect = (rng.integers(0, 256, (500, 500), dtype=np.uint8) & 0x3f)
    for _ in range(20):
        r0, c0 = rng.integers(0, 460, 2)
        rect[r0:r0 + rng.integers(3, 40), c0:c0 + rng.integers(3, 40)] |= np.uint8(rng.choice([0x80, 0x40, 0xc0]))
    return {'noise': noise, 'rect': rect}
