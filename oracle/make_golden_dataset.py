"""Writes tests/golden/reference_dataset.npz by running the reference's data.py VERBATIM (CARLA_Data.__init__ / __getitem__ and
load_crop_bev_npy) behind the shims in oracle/shims (skimage.transform.rotate, ujson) on the routes of oracle/synthetic_route.py.

    python oracle/make_golden_dataset.py        # needs the reference checkout (oracle/ref_import.py)

numpy 2 dropped the np.string_ / np.float aliases data.py uses; this process restores them as np.bytes_ / float before the import.
Samples are keyed by (route, frame), not by index (os.listdir order is the host's); random.seed(seed_of(route, frame)) runs
before every sample, so the reader under test draws the same augmentation angle. Stored per sample, with and without
augmentation: digests of rgb, depth, semantic, lidar, target_point_image and bev in the dtypes the training step consumes
(uint8, float32, int64, float32, float32, int64), and the arrays label, ego_waypoint, target_point, speed and the drawn angle.
Also digests of load_crop_bev_npy over dataset_oracle.angle_sweep() on dataset_oracle.sweep_planes()."""
import importlib
import os
import random
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dataset_oracle as DO, ref_import, synthetic_route  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'reference_dataset.npz')


def seed_of(route, frame):
    return 1000 * sorted(r[0] for r in synthetic_route.ROUTES).index(route) + frame


def key(route, frame, aug):
    return '%s_%04d_aug%d' % (route, frame, aug)


def load_data_module():
    if not hasattr(np, 'string_'):
        np.string_ = np.bytes_
    if not hasattr(np, 'float'):
        np.float = float
    for p in (ref_import.REF_ROOT, ref_import.SHIMS):
        if p not in sys.path:
            sys.path.insert(0, p)
    return importlib.import_module('data'), importlib.import_module('config')


def main():
    data, config = load_data_module()
    out = {}
    tmp = tempfile.mkdtemp()
    root = synthetic_route.write_dataset(os.path.join(tmp, 'data'))
    for aug in (0, 1):
        cfg = config.GlobalConfig(setting='eval')
        cfg.augment = bool(aug)
        ds = data.CARLA_Data([root], cfg)
        for idx in range(len(ds)):
            lidar_path = str(ds.lidars[idx][0], encoding='utf-8')
            route = os.path.basename(os.path.dirname(os.path.dirname(lidar_path)))
            frame = int(os.path.basename(lidar_path)[:4])
            random.seed(seed_of(route, frame))
            d = ds[idx]
            k = key(route, frame, aug)
            out[k + '_rgb'] = DO.digest(d['rgb'])
            out[k + '_depth'] = DO.digest(d['depth'].astype(np.float32))
            out[k + '_semantic'] = DO.digest(d['semantic'].astype(np.int64))
            out[k + '_lidar'] = DO.digest(d['lidar'])
            out[k + '_target_point_image'] = DO.digest(d['target_point_image'].astype(np.float32))
            out[k + '_bev'] = DO.digest(d['bev'])
            out[k + '_label'] = d['label']
            out[k + '_ego_waypoint'] = d['ego_waypoint']
            out[k + '_target_point'] = d['target_point']
            out[k + '_speed'] = np.float64(d['speed'])
            random.seed(seed_of(route, frame))     # the angle __getitem__ drew, replayed (it is not part of its output)
            do = cfg.augment and random.random() > cfg.inv_augment_prob
            out[k + '_degree'] = np.float64((random.random() * 2. - 1.) * cfg.aug_max_rotation if do else 0.0)
        print('aug=%d: %d samples' % (aug, len(ds)))
    planes = DO.sweep_planes()
    angles = DO.angle_sweep()
    out['sweep_angles'] = np.array(angles)
    for name, plane in planes.items():
        noise = np.random.default_rng(5).integers(0, 256, (2,) + plane.shape, dtype=np.uint8)   # RGB planes 0 / 1: ignored
        bev = data.decode_pil_to_npy(np.concatenate([noise, plane[None]])).astype(np.uint8)
        out['sweep_%s' % name] = np.array([DO.digest(data.load_crop_bev_npy(bev, a)) for a in angles])
    shutil.rmtree(tmp)
    np.savez_compressed(GOLD, **out)
    print('wrote', GOLD, len(out), 'entries')


if __name__ == '__main__':
    main()
