"""Writes tests/golden/reference_correspondences.npz by running the reference's lidar_bev_cam_correspondences VERBATIM
(data.py:632-842, exec'd from data.py by oracle/ref_import.py) on oracle/correspondence_oracle.fixture_sweeps(), and the
reference's CARLA_Data.__getitem__ with backbone='geometric_fusion' (as oracle/make_golden_dataset.py does) on the routes of
oracle/synthetic_route.py with augmentation.

    python oracle/make_golden_correspondences.py        # needs the reference checkout (oracle/ref_import.py)

random.sample is replaced by a recorder that stores the population it is given, with the cell of the calling loop, and returns
its first k entries; the cell lists of cells with more than 5 candidates are stored in CSR form. Per sweep / sample key:
  _bev [8,8,5,2], _cam [22,5,5,2] int64      the reference's outputs (with the recorder's pop[:5] in cells with > 5 candidates)
  _pop_cell [K]                               cell of each recorded population: i * 8 + j (bev_points), 64 + i * 5 + j (cam_points)
  _pop_ptr [K + 1], _pop_val [T, 2] int64     the populations, concatenated
  _digest                                     digest of the sweep (fixture sweeps) / _degree the angle drawn (routes)"""
import copy
import os
import random
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import correspondence_oracle as CO, dataset_oracle as DO, ref_import, synthetic_route  # noqa: E402
from oracle.make_golden_dataset import key, load_data_module, seed_of  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'reference_correspondences.npz')


class Recorder:
    """Stands in for the `random` module: random() is the real one; sample(pop, k) records pop and returns pop[:k]."""

    def __init__(self):
        self.pops = []

    @staticmethod
    def random():
        return random.random()

    def sample(self, pop, k):
        f = sys._getframe(1).f_locals
        cell = (64 + f['i'] * 5 + f['j']) if 'bev_to_cam_points' in f else f['i'] * 8 + f['j']
        self.pops.append((cell, np.array(pop, dtype=np.int64).reshape(-1, 2)))
        return pop[:k]


def store(out, k, bev, cam, pops):
    out[k + '_bev'] = np.asarray(bev).astype(np.int64)
    out[k + '_cam'] = np.asarray(cam).astype(np.int64)
    out[k + '_pop_cell'] = np.array([c for c, _ in pops], dtype=np.int64)
    out[k + '_pop_ptr'] = np.cumsum([0] + [len(p) for _, p in pops]).astype(np.int64)
    out[k + '_pop_val'] = np.concatenate([p for _, p in pops]) if pops else np.zeros((0, 2), np.int64)


def main():
    out = {}
    fns = ref_import.load_data_fns(['lidar_bev_cam_correspondences', 'correspondences_at_one_scale'])
    fn = fns['lidar_bev_cam_correspondences']
    rec = Recorder()
    fn.__globals__.update(random=rec, deepcopy=copy.deepcopy)
    for name, sweep in CO.fixture_sweeps().items():
        rec.pops = []
        bev, cam = fn(sweep[:, :3].copy())
        store(out, 'sweep_' + name, bev, cam, rec.pops)
        out['sweep_%s_digest' % name] = DO.digest(sweep)
        print(name, len(sweep), 'points,', len(rec.pops), 'cells with > 5 candidates')

    data, config = load_data_module()
    rec = Recorder()
    data.random = rec
    tmp = tempfile.mkdtemp()
    root = synthetic_route.write_dataset(os.path.join(tmp, 'data'))
    cfg = config.GlobalConfig(setting='eval')
    cfg.augment = True
    cfg.backbone = 'geometric_fusion'
    ds = data.CARLA_Data([root], cfg)
    for idx in range(len(ds)):
        lidar_path = str(ds.lidars[idx][0], encoding='utf-8')
        route = os.path.basename(os.path.dirname(os.path.dirname(lidar_path)))
        frame = int(os.path.basename(lidar_path)[:4])
        random.seed(seed_of(route, frame))
        rec.pops = []
        d = ds[idx]
        k = key(route, frame, 1)
        store(out, k, d['bev_points'], d['cam_points'], rec.pops)
        random.seed(seed_of(route, frame))
        do = cfg.augment and random.random() > cfg.inv_augment_prob
        out[k + '_degree'] = np.float64((random.random() * 2. - 1.) * cfg.aug_max_rotation if do else 0.0)
    print('routes: %d samples' % len(ds))
    shutil.rmtree(tmp)
    np.savez_compressed(GOLD, **out)
    print('wrote', GOLD, len(out), 'entries')


if __name__ == '__main__':
    main()
