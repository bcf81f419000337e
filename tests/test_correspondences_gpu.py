"""The geometric-fusion correspondences on the GPU (csrc/correspondences.cu):
- tfb_lidar_cam_correspondences bit for bit against the oracle's selection rule (oracle/correspondence_oracle.py) on every
  fixture sweep and at batch 1 / 12 with n_valid in {0, partial, max_points}; two launches give the same bits;
- InputPipeline.prepare on CarlaRawDataset(backbone='geometric_fusion', correspondences='gpu') batches against the verbatim
  reference's __getitem__ (tests/golden/reference_correspondences.npz): cells with at most 5 candidates equal, fuller cells hold a sub-multiset of the
  recorded population;
- a captured Trainer(backbone='geometric_fusion', raw_inputs='dataset') step equal, loss for loss, to an eager raw_inputs=False
  step fed the pipeline's outputs and the same correspondences; two fresh captured trainers give the same bits;
- GeometricFusionBackbone fed the reference's [B,22,5,5,2] camera layout equals the same memory viewed as [B,5,22,5,2]."""
from collections import Counter

import numpy as np
import pytest
import torch

from oracle import correspondence_oracle as CO
from oracle import synthetic_route

from test_correspondences import GOLD, cell_key, check_fixture_sweeps, geometric_samples, run_kernel, shipped

pytestmark = pytest.mark.gpu


def _call(name, *args):
    from transfuser_b200 import _lib
    _lib.call(name, *args)
    torch.cuda.synchronize()


def _cuda(t):
    return t.cuda()


def test_kernel_fixture_sweeps():
    check_fixture_sweeps(_call, _cuda)


@pytest.mark.parametrize('B', [1, 12])
def test_kernel_batches_and_n_valid(B):
    """max_points = 40000: sample 0 uses all of it, sample 1 none, the others part (random and fixture sweeps); two launches
    give identical bits."""
    sweeps = CO.fixture_sweeps()
    N = 40000
    pool = [sweeps['rand40k'], sweeps['rand20k'][:13000], sweeps['pile'], sweeps['boundary'], CO.random_sweep(31000, 9)]
    chosen = [sweeps['rand40k']] if B == 1 else [sweeps['rand40k'], np.zeros((0, 4), np.float32)] + [pool[(i + 1) % len(pool)] for i in range(B - 2)]
    pts, nv = shipped(chosen, N=N)
    seeds = [(i * 0x9E3779B97F4A7C15 + 17) & ((1 << 63) - 1) for i in range(B)]
    bev, cam = run_kernel(_call, _cuda, pts, nv, seeds)
    for i, s in enumerate(chosen):
        wb, wc = CO.correspondences(s, seeds[i])
        assert np.array_equal(bev[i], wb) and np.array_equal(cam[i], wc), i
    bev2, cam2 = run_kernel(_call, _cuda, pts, nv, seeds)
    assert np.array_equal(bev, bev2) and np.array_equal(cam, cam2)


@pytest.fixture(scope='module')
def routes(tmp_path_factory):
    return synthetic_route.write_dataset(str(tmp_path_factory.mktemp('carla') / 'data'))


def _batch(root, idx=None):
    from transfuser_b200.dataset import collate
    samples = geometric_samples(root, idx)
    return collate([s for _, s in samples]), [k for k, _ in samples]


def _raw(b):
    return dict(rgb=b['rgb_u8'], depth=b['depth_u8'], seg=b['seg_u8'], crop_shift=b['crop_shift'], points=b['points'], n_valid=b['n_valid'],
                transforms=b['transforms'], target_point=b['target_point64'], bev_u8=b['bev_u8'], bev_matrix=b['bev_matrix'],
                corr_seed=b['corr_seed'])


def test_pipeline_matches_reference_getitem(routes):
    from transfuser_b200 import pipeline
    from transfuser_b200.config import TrainConfig
    g = np.load(GOLD)
    b, keys = _batch(routes)
    pipe = pipeline.InputPipeline(TrainConfig(), 'cuda')
    out = pipe.prepare(_raw(b))
    torch.cuda.synchronize()
    assert out['bev_points'].dtype == torch.int64 and tuple(out['bev_points'].shape) == (len(keys), 8, 8, 5, 2)
    assert tuple(out['cam_points'].shape) == (len(keys), 22, 5, 5, 2)
    full = 0
    for i, k in enumerate(keys):
        got = {'bev': out['bev_points'][i].cpu().numpy(), 'cam': out['cam_points'][i].cpu().numpy()}
        pops = {cell_key(int(c)): g[k + '_pop_val'][g[k + '_pop_ptr'][q]:g[k + '_pop_ptr'][q + 1]] for q, c in enumerate(g[k + '_pop_cell'])}
        for name, shape in (('bev', (8, 8)), ('cam', (22, 5))):
            want = g['%s_%s' % (k, name)]
            for i0 in range(shape[0]):
                for j0 in range(shape[1]):
                    pop = pops.get((name, i0, j0))
                    if pop is None:
                        assert np.array_equal(got[name][i0, j0], want[i0, j0]), (k, name, i0, j0)
                    else:
                        have = Counter(map(tuple, got[name][i0, j0].tolist()))
                        assert not have - Counter(map(tuple, pop.tolist())), (k, name, i0, j0)
                        full += 1
    assert full > 0
    # preallocated destinations, and the outputs without corr_seed are unchanged
    dst = {'bev_points': torch.full((len(keys), 8, 8, 5, 2), -1, dtype=torch.int64, device='cuda'),
           'cam_points': torch.full((len(keys), 22, 5, 5, 2), -1, dtype=torch.int64, device='cuda')}
    again = pipe.prepare(_raw(b), out=dst)
    assert again['bev_points'] is dst['bev_points'] and torch.equal(dst['bev_points'], out['bev_points'])
    assert torch.equal(dst['cam_points'], out['cam_points'])
    raw = _raw(b)
    del raw['corr_seed']
    plain = pipe.prepare(raw)
    assert set(out) == set(plain) | {'bev_points', 'cam_points'}
    for k in plain:
        assert torch.equal(plain[k], out[k]), k
    with pytest.raises(ValueError):
        pipe.prepare(dict(_raw(b), points=b['points'].double()))
    with pytest.raises(ValueError):
        pipe.prepare(dict(_raw(b), corr_seed=b['corr_seed'][:1]))


def _trainer(mode):
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    torch.manual_seed(0)
    return Trainer(TrainConfig(), torch.device('cuda', 0), gemm_mode='bf16', seed=0, raw_inputs=mode, backbone='geometric_fusion')


def _bits(losses):
    return {k: float(v.detach()) for k, v in losses.items()}


def test_captured_geometric_dataset_step_equals_eager_step(routes, monkeypatch):
    """As tests/test_dataset_gpu.py does for the transFuser backbone: two eager warm-up steps, capture, one replay of the
    dataset-mode trainer against three eager steps of the expanded-input trainer fed the pipeline's outputs of the same batch,
    the correspondences included. The 11 losses of the third step are equal bit for bit."""
    from transfuser_b200 import pipeline, trainer as trainer_mod
    from transfuser_b200.config import TrainConfig
    b, _ = _batch(routes, idx=[0, 3])
    tr = _trainer('dataset')
    assert 'corr_seed' in tr.input_keys and 'bev_points' not in tr.input_keys
    assert tr.capture(b), tr.graph_error
    tr.replay()
    torch.cuda.synchronize()
    got = _bits(tr.last_losses)
    del tr

    p = pipeline.InputPipeline(TrainConfig(), 'cuda').prepare({k: v.cuda() for k, v in _raw(b).items()})
    d = dict(rgb=p['rgb'], points=b['points'].cuda(), target_point_image=p['target_point_image'], target_point=p['target_point'],
             ego_vel=b['ego_vel'].cuda(), ego_waypoint=b['ego_waypoint'].cuda(), bev=p['bev'], semantic=p['semantic'], depth=p['depth'],
             label=b['label'].cuda(), bev_points=p['bev_points'], cam_points=p['cam_points'])
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


def test_captured_geometric_dataset_step_is_reproducible(routes):
    b, _ = _batch(routes, idx=[1, 2])
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


def test_backbone_reads_reference_camera_layout():
    """[B,22,5,5,2] (what the reference's dataset and the pipeline produce) and the same memory viewed as [B,5,22,5,2] give the
    same bits: the backbone reads the correspondences flat, as geometric_fusion.py:147 does."""
    from oracle import torch_oracle as O
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    torch.manual_seed(0)
    net = LidarCenterNet(TrainConfig(), 'cuda', 'geometric_fusion', 'regnety_032', 'regnety_032', use_velocity=False).cuda().eval()
    batch = {k: v.cuda() for k, v in O.synthetic_batch(2, seed=5).items()}
    g = torch.Generator().manual_seed(3)
    cam = torch.stack([torch.randint(0, 8, (2, 22, 5, 5), generator=g), torch.randint(0, 8, (2, 22, 5, 5), generator=g)], -1).cuda()
    bev = torch.stack([torch.randint(0, 22, (2, 8, 8, 5), generator=g), torch.randint(0, 5, (2, 8, 8, 5), generator=g)], -1).cuda()
    lidar = torch.cat((batch['lidar'], batch['target_point_image']), dim=1)
    outs = []
    with torch.no_grad():
        for c in (cam, cam.view(2, 5, 22, 5, 2)):
            feats, grid, fused = net._model(batch['rgb'], lidar, batch['ego_vel'], bev, c)
            outs.append([t.clone() for t in feats] + [grid.clone(), fused.clone()])
    torch.cuda.synchronize()
    for a, c in zip(*outs):
        assert torch.equal(a, c)
