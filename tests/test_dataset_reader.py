"""The on-disk dataset reader (transfuser_b200/dataset.py) and the BEV-label rotation (csrc/bev_label.cu), on the CPU:
- the skimage shim (oracle/shims/skimage/transform.py) against scipy.ndimage, and pipeline.bev_rotation_matrix against its matrix;
- the reader plus the oracle expansions (oracle/dataset_oracle.py) against the reference's own CARLA_Data.__getitem__ on the
  generated routes (tests/golden/reference_dataset.npz, oracle/make_golden_dataset.py), with and without augmentation;
- tfb_bev_label_prep executed unchanged through the CUDA emulation (tests/cuda_emul/bev_label_emul.py), bit for bit against
  the reference's load_crop_bev_npy over the fixture's angle sweep and against the oracle on edge-case planes;
- the error cases. tests/test_dataset_gpu.py runs the kernel and the pipeline on the device."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import dataset_oracle as DO
from oracle import synthetic_route
from oracle.make_golden_dataset import key, seed_of

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_dataset.npz')
ULP32 = 2.0 ** -23


def _transform():
    return DO._shim_transform()


# ---------------------------------------------------------------- the skimage shim and the host matrix

@pytest.mark.parametrize('angle', [0.0, 7.3, -19.999, 90.0, 200.0])
def test_shim_rotate_matches_scipy_affine_transform(angle):
    from scipy import ndimage
    rng = np.random.default_rng(3)
    img = rng.random((37, 53, 2))
    img[0, 0, 0], img[1, 1, 1] = 0.0, 1.0
    T = _transform()
    M = T.rotation_matrix(angle, 37, 53)
    got = T.rotate(img, angle)
    # scipy maps output (row, col) to input matrix @ (row, col) + offset; grid-constant: zero outside, bilinear inside
    A = np.array([[M[1, 1], M[1, 0]], [M[0, 1], M[0, 0]]])
    for ch in range(2):
        want = ndimage.affine_transform(img[..., ch], A, offset=(M[1, 2], M[0, 2]), order=1, mode='grid-constant', cval=0.0)
        want = np.clip(want, img.min(), img.max())
        assert np.abs(got[..., ch] - want).max() <= 1e-12, angle


def test_shim_rotate_identity_at_zero():
    img = np.random.default_rng(4).random((21, 30, 2)).astype(np.float32)
    assert np.array_equal(_transform().rotate(img, 0.0), img.astype(np.float64))


@pytest.mark.parametrize('shape', [(500, 500), (260, 340), (333, 517)])
def test_bev_rotation_matrix_equals_shim_bitwise(shape):
    from transfuser_b200 import pipeline
    for a in DO.angle_sweep(n_random=50):
        want = _transform().rotation_matrix(a, *shape)
        got = pipeline.bev_rotation_matrix(a, *shape)
        assert got.dtype == np.float64 and got.shape == (6,)
        assert np.array_equal(got.view(np.int64), want[:2].reshape(6).view(np.int64)), a
        assert list(want[2]) == [0.0, 0.0, 1.0]


# ---------------------------------------------------------------- the reader against the reference

@pytest.fixture(scope='module')
def routes(tmp_path_factory):
    return synthetic_route.write_dataset(str(tmp_path_factory.mktemp('carla') / 'data'))


def _cfg(**kw):
    from transfuser_b200.config import TrainConfig
    return TrainConfig(**kw)


def _samples(root, aug):
    from transfuser_b200.dataset import CarlaRawDataset
    ds = CarlaRawDataset([root], _cfg(augment=bool(aug)), max_points=4000)
    for idx, (route, frame) in enumerate(ds.frames):
        random.seed(seed_of(os.path.basename(route), frame))
        yield os.path.basename(route), frame, ds[idx]


def _close32(got, want):
    want = np.asarray(want, dtype=np.float64)
    return np.all(np.abs(np.asarray(got, np.float64) - want) <= ULP32 * np.maximum(np.abs(want), 2.0 ** -126))


@pytest.mark.parametrize('aug', [0, 1])
def test_reader_matches_reference_getitem(routes, aug):
    from transfuser_b200.config import TrainConfig
    g = np.load(GOLD)
    seen = 0
    for route, frame, s in _samples(routes, aug):
        k = key(route, frame, aug)
        assert float(s['degree']) == float(g[k + '_degree']), k
        assert s['rgb_u8'].dtype == np.uint8 and s['bev_u8'].dtype == np.uint8 and s['bev_matrix'].dtype == np.float64
        e = DO.expand(s, TrainConfig.converter)
        for name in ('rgb', 'depth', 'semantic', 'lidar', 'target_point_image', 'bev'):
            assert DO.digest(e[name]) == str(g['%s_%s' % (k, name)]), (k, name)
        assert s['label'].dtype == np.float32 and _close32(s['label'], g[k + '_label']), k
        assert s['ego_waypoint'].dtype == np.float32 and _close32(s['ego_waypoint'], g[k + '_ego_waypoint']), k
        assert _close32(s['target_point64'], g[k + '_target_point']), k
        assert s['ego_vel'].tolist() == [float(g[k + '_speed'])]
        assert int(s['n_valid']) <= 4000 and not s['points'][int(s['n_valid']):].any()
        seen += 1
    assert seen == sum(1 for n in g.files if n.endswith('_aug%d_bev' % aug)) == 11


def test_reader_collate(routes):
    from transfuser_b200.dataset import CarlaRawDataset, collate
    ds = CarlaRawDataset([routes], _cfg(), max_points=4000)
    random.seed(0)
    b = collate([ds[0], ds[3]])
    want = dict(rgb_u8=((2, 160, 960, 3), torch.uint8), depth_u8=((2, 160, 960, 3), torch.uint8), seg_u8=((2, 160, 960), torch.uint8),
                bev_u8=((2, 500, 500), torch.uint8), bev_matrix=((2, 6), torch.float64), points=((2, 4000, 4), torch.float32),
                n_valid=((2,), torch.int32), transforms=((2, 4, 4), torch.float64), crop_shift=((2,), torch.int32),
                target_point64=((2, 2), torch.float64), ego_waypoint=((2, 4, 2), torch.float32), label=((2, 20, 7), torch.float32),
                ego_vel=((2, 1), torch.float32), degree=((2,), torch.float64))
    assert {k: (tuple(v.shape), v.dtype) for k, v in b.items()} == want


def test_reader_draw_matches_reference_order():
    """random.random() call for call as data.py:216-218: no draw without augmentation, one draw when it is skipped."""
    from transfuser_b200.dataset import CarlaRawDataset
    ds = CarlaRawDataset([], _cfg())
    for seed in range(50):
        random.seed(seed)
        a, b, c = random.random(), random.random(), random.random()
        random.seed(seed)
        assert ds.draw_degree() == ((b * 2. - 1.) * 20 if a > 0.1 else 0)
        assert random.random() == (c if a > 0.1 else b)
    ds.augment = False
    random.seed(1)
    ds.draw_degree()
    after = random.random()
    random.seed(1)
    assert after == random.random()


def test_reader_errors(routes, tmp_path):
    import json
    import shutil
    from transfuser_b200.dataset import CarlaRawDataset
    with pytest.raises(NotImplementedError):
        CarlaRawDataset([routes], _cfg(seq_len=2))
    with pytest.raises(NotImplementedError):
        CarlaRawDataset([routes], _cfg(), backbone='geometric_fusion')
    with pytest.raises(NotImplementedError):
        CarlaRawDataset([routes], _cfg(use_point_pillars=True))
    with pytest.raises(ValueError, match='max_points'):
        CarlaRawDataset([routes], _cfg(), max_points=1000)[0]        # never truncated: that would change the histogram
    # 21 boxes that survive the filters: the reference fails to pad them into its [20, 7] label too
    root = tmp_path / 'data'
    shutil.copytree(os.path.join(routes, 'route_a'), root / 'route_a')
    f = root / 'route_a' / 'label_raw' / '0005.json'
    boxes = json.loads(f.read_text())
    boxes.append(dict(boxes[1], id=99))
    f.write_text(json.dumps(boxes))
    ds = CarlaRawDataset([str(root)], _cfg(augment=False), max_points=4000)
    with pytest.raises(ValueError, match='at most 20'):
        ds[ds.frames.index((str(root / 'route_a'), 5))]


# ---------------------------------------------------------------- the kernel through the emulation

def edge_planes():
    """(name, [B, H, W] uint8 planes): all-zero, all-ones, single pixels, stray bits only, random (at a non-square size too)."""
    H, W = 500, 500
    zero = np.zeros((H, W), np.uint8)
    single = []
    for (r, c, v) in ((250, 250, 0x80), (160, 249, 0x40), (492, 10, 0xc0), (100, 300, 0x80), (0, 0, 0xc0)):
        p = zero.copy()
        p[r, c] = v
        single.append(p)
    stray = np.random.default_rng(8).integers(0, 64, (H, W), dtype=np.uint8)
    dropped = zero.copy()
    dropped[493:] = 0xc0                                              # only the rows the 7-row shift drops
    rnd = np.random.default_rng(9).integers(0, 256, (2, 270, 350), dtype=np.uint8)
    return [('zero', np.stack([zero])), ('ones', np.stack([np.full((H, W), 255, np.uint8)])), ('single', np.stack(single)),
            ('stray', np.stack([stray, dropped])), ('random_small', rnd)]


def run_kernel(call, planes, angles, to_dev=lambda t: t):
    """tfb_bev_label_prep on planes[b] rotated by angles[b] -> int64 numpy [B, 160, 160]."""
    from transfuser_b200 import pipeline
    planes = np.ascontiguousarray(planes)
    B, H, W = planes.shape
    m = torch.from_numpy(np.stack([pipeline.bev_rotation_matrix(a, H, W) for a in angles]))
    out = to_dev(torch.full((B, 160, 160), -1, dtype=torch.int64))
    call('tfb_bev_label_prep', to_dev(torch.from_numpy(planes)), to_dev(m), B, H, W, out)
    return out.cpu().numpy()


def check_sweep(call, to_dev=lambda t: t):
    """Every angle of the fixture's sweep on its two planes: digests equal to the reference's load_crop_bev_npy."""
    g = np.load(GOLD)
    angles = [float(a) for a in g['sweep_angles']]
    for name, plane in DO.sweep_planes().items():
        got = run_kernel(call, np.broadcast_to(plane, (len(angles),) + plane.shape), angles, to_dev)
        for a, o, want in zip(angles, got, g['sweep_%s' % name]):
            assert DO.digest(o) == str(want), (name, a)


def check_edge_planes(call, to_dev=lambda t: t, angles=(0.0, 1e-9, -19.999, 20.0, 45.0, 90.0, 180.0)):
    for name, planes in edge_planes():
        for a in angles:
            got = run_kernel(call, planes, [a] * len(planes), to_dev)
            for b in range(len(planes)):
                want = DO.bev_label(planes[b], a)
                assert np.array_equal(got[b], want), (name, b, a)
            if name in ('zero', 'stray'):
                assert not got.any()


def test_oracle_matches_reference_sweep_sample():
    g = np.load(GOLD)
    angles = [float(a) for a in g['sweep_angles']]
    for name, plane in DO.sweep_planes().items():
        for i in list(range(10)) + [10, 77, 209]:
            assert DO.digest(DO.bev_label(plane, angles[i])) == str(g['sweep_%s' % name][i]), (name, angles[i])


def test_bev_label_kernel_emulated_sweep():
    from cuda_emul import bev_label_emul
    check_sweep(bev_label_emul.call)


def test_bev_label_kernel_emulated_edge_planes():
    from cuda_emul import bev_label_emul
    check_edge_planes(bev_label_emul.call)


def test_bev_label_argument_checks_emulated():
    from cuda_emul import bev_label_emul
    m = torch.zeros(1, 6, dtype=torch.float64)
    out = torch.zeros(1, 160, 160, dtype=torch.int64)
    for H, W in ((249, 500), (500, 329)):
        with pytest.raises(RuntimeError, match='argument check'):
            bev_label_emul.call('tfb_bev_label_prep', torch.zeros(1, H, W, dtype=torch.uint8), m, 1, H, W, out)
    with pytest.raises(RuntimeError, match='argument check'):
        bev_label_emul.call('tfb_bev_label_prep', torch.zeros(1, 500, 500, dtype=torch.uint8), m, 0, 500, 500, out)
