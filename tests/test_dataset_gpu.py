"""The BEV-label rotation (csrc/bev_label.cu) and the dataset-mode training step on the GPU:
- tfb_bev_label_prep bit for bit against the reference's load_crop_bev_npy over the fixture's angle sweep, and against the
  oracle on the edge-case planes (the same checks tests/test_dataset_reader.py runs through the CUDA emulation);
- InputPipeline.prepare on batches of dataset.CarlaRawDataset against the reference's CARLA_Data.__getitem__ on the generated
  routes (tests/golden/reference_dataset.npz);
- a captured Trainer(raw_inputs='dataset') step equal, loss for loss, to an eager raw_inputs=False step fed the pipeline's
  expanded outputs of the same batch; two fresh captured trainers from one seed give the same bits."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import dataset_oracle as DO
from oracle import synthetic_route
from oracle.make_golden_dataset import key, seed_of

from test_dataset_reader import GOLD, check_edge_planes, check_sweep

pytestmark = pytest.mark.gpu


def _cuda(t):
    return t.cuda()


def _call(name, *args):
    from transfuser_b200 import _lib
    _lib.call(name, *args)
    torch.cuda.synchronize()


def test_bev_label_kernel_sweep():
    check_sweep(_call, _cuda)


def test_bev_label_kernel_edge_planes():
    check_edge_planes(_call, _cuda)


@pytest.fixture(scope='module')
def routes(tmp_path_factory):
    return synthetic_route.write_dataset(str(tmp_path_factory.mktemp('carla') / 'data'))


def _batch(root, aug, idx=None, max_points=4000):
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.dataset import CarlaRawDataset, collate
    ds = CarlaRawDataset([root], TrainConfig(augment=bool(aug)), max_points=max_points)
    idx = range(len(ds)) if idx is None else idx
    samples, keys = [], []
    for i in idx:
        route, frame = ds.frames[i]
        random.seed(seed_of(os.path.basename(route), frame))
        samples.append(ds[i])
        keys.append(key(os.path.basename(route), frame, aug))
    return collate(samples), keys


def _raw(b):
    return dict(rgb=b['rgb_u8'], depth=b['depth_u8'], seg=b['seg_u8'], crop_shift=b['crop_shift'], points=b['points'], n_valid=b['n_valid'],
                transforms=b['transforms'], target_point=b['target_point64'], bev_u8=b['bev_u8'], bev_matrix=b['bev_matrix'])


@pytest.mark.parametrize('aug', [0, 1])
def test_pipeline_matches_reference_getitem(routes, aug):
    from transfuser_b200 import pipeline
    from transfuser_b200.config import TrainConfig
    g = np.load(GOLD)
    b, keys = _batch(routes, aug)
    out = pipeline.InputPipeline(TrainConfig(), 'cuda').prepare(_raw(b))
    torch.cuda.synchronize()
    assert out['bev'].dtype == torch.int64 and tuple(out['bev'].shape) == (len(keys), 160, 160)
    for i, k in enumerate(keys):
        got = dict(rgb=out['rgb'][i].cpu().numpy().astype(np.uint8), depth=out['depth'][i].cpu().numpy(),
                   semantic=out['semantic'][i].cpu().numpy(), lidar=out['lidar'][i].cpu().numpy(),
                   target_point_image=out['target_point_image'][i].cpu().numpy(), bev=out['bev'][i].cpu().numpy())
        for name, v in got.items():
            assert DO.digest(v) == str(g['%s_%s' % (k, name)]), (k, name)


def test_pipeline_without_bev_is_unchanged(routes):
    from transfuser_b200 import pipeline
    from transfuser_b200.config import TrainConfig
    b, _ = _batch(routes, 1, idx=[0, 1])
    raw = _raw(b)
    pipe = pipeline.InputPipeline(TrainConfig(), 'cuda')
    full = pipe.prepare(raw)
    del raw['bev_u8'], raw['bev_matrix']
    plain = pipe.prepare(raw)
    assert 'bev' not in plain and set(full) == set(plain) | {'bev'}
    for k in plain:
        assert torch.equal(plain[k], full[k]), k
    with pytest.raises(ValueError):
        pipe.prepare(dict(_raw(b), bev_matrix=None))
    with pytest.raises(ValueError):
        pipe.prepare(dict(_raw(b), bev_u8=b['bev_u8'][:, :249]))
    bad = b['bev_matrix'].clone()
    bad[0, 2] = float('nan')
    with pytest.raises(ValueError):
        pipe.prepare(dict(_raw(b), bev_matrix=bad))


def _trainer(mode, gemm_mode='bf16'):
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    torch.manual_seed(0)
    return Trainer(TrainConfig(), torch.device('cuda', 0), gemm_mode=gemm_mode, seed=0, raw_inputs=mode)


def _bits(losses):
    return {k: float(v.detach()) for k, v in losses.items()}


def test_captured_dataset_step_equals_expanded_eager_step(routes, monkeypatch):
    """Three steps on one batch: the dataset-mode trainer runs two eager warm-up steps and captures, then replays once; the
    expanded-input trainer runs three eager steps on the pipeline's outputs of that batch (the LiDAR histogram handed in as
    computed by the pipeline). The 11 losses of the third step are equal bit for bit."""
    from transfuser_b200 import pipeline, trainer as trainer_mod
    from transfuser_b200.config import TrainConfig
    b, _ = _batch(routes, 1, idx=[0, 3])
    tr = _trainer('dataset')
    assert tr.capture(b), tr.graph_error
    tr.replay()
    torch.cuda.synchronize()
    got = _bits(tr.last_losses)
    del tr

    p = pipeline.InputPipeline(TrainConfig(), 'cuda').prepare({k: v.cuda() for k, v in _raw(b).items()})
    d = dict(rgb=p['rgb'], points=b['points'].cuda(), target_point_image=p['target_point_image'], target_point=p['target_point'],
             ego_vel=b['ego_vel'].cuda(), ego_waypoint=b['ego_waypoint'].cuda(), bev=p['bev'], semantic=p['semantic'], depth=p['depth'],
             label=b['label'].cuda())
    monkeypatch.setattr(trainer_mod.bev, 'lidar_to_histogram_features_batched', lambda pts: p['lidar'])
    tr = _trainer(False)
    for _ in range(3):
        tr.step(d)
    torch.cuda.synchronize()
    want = _bits(tr.last_losses)
    assert list(got) == list(want) and len(got) == 11
    for k in want:
        assert np.float32(got[k]).view(np.int32) == np.float32(want[k]).view(np.int32), (k, got[k], want[k])
    assert all(np.isfinite(v) for v in got.values())


def test_captured_dataset_step_is_reproducible(routes):
    b, _ = _batch(routes, 1, idx=[1, 2])
    runs = []
    for _ in range(2):
        tr = _trainer('dataset')
        assert tr.capture(b), tr.graph_error
        losses = []
        for _ in range(3):
            tr.replay()
            losses.append(torch.stack(list(tr.last_losses.values())).clone())
        torch.cuda.synchronize()
        total = tr.flat.total
        idx = torch.from_numpy(np.unique(np.random.default_rng(0).integers(0, total, size=1 << 16))).cuda()
        runs.append((torch.stack(losses).cpu(), tr.flat.flat[idx].float().cpu(), tr.flat.grad[idx].float().cpu()))
        del tr
    for a, c in zip(*runs):
        assert torch.equal(a.view(torch.int32), c.view(torch.int32))
    assert float(runs[0][2].abs().sum()) > 0
