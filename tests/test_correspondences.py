"""The geometric-fusion correspondences (csrc/correspondences.cu, oracle/correspondence_oracle.py) on the CPU:
- the oracle's per-cell candidate lists against the populations the verbatim reference handed random.sample, element for
  element, and its cells with at most 5 candidates against the reference's outputs (tests/golden/reference_correspondences.npz,
  oracle/make_golden_correspondences.py), on the fixture sweeps and on the routes through CARLA_Data.__getitem__;
- tfb_lidar_cam_correspondences executed unchanged through the CUDA emulation (tests/cuda_emul/correspondences_emul.py), bit for
  bit against the oracle on every fixture sweep, cells with more than 5 candidates included;
- the selection rule's frequencies on a 12-candidate cell;
- the reader in geometric mode (the sweep and the angle of the reference) and its error cases.
tests/test_correspondences_gpu.py runs the kernel, the pipeline and the training step on the device."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import correspondence_oracle as CO
from oracle import synthetic_route
from oracle.make_golden_dataset import key, seed_of

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, 'golden', 'reference_correspondences.npz')
DATASET_GOLD = os.path.join(HERE, 'golden', 'reference_dataset.npz')


def cell_key(c):
    return ('bev', c // 8, c % 8) if c < 64 else ('cam', (c - 64) // 5, (c - 64) % 5)


def check_against_reference(g, k, lists):
    """The oracle's lists of sweep / sample k against the recorded populations and outputs of the verbatim reference."""
    cells, ptr, val = g[k + '_pop_cell'], g[k + '_pop_ptr'], g[k + '_pop_val']
    assert {cell_key(int(c)) for c in cells} == {c for c, l in lists.items() if len(l[0]) > 5}, k
    for q, c in enumerate(cells):
        assert np.array_equal(lists[cell_key(int(c))][2], val[ptr[q]:ptr[q + 1]]), (k, cell_key(int(c)))
    bev, cam = g[k + '_bev'], g[k + '_cam']
    for (name, i, j), (view, _, vals) in lists.items():
        want = (bev if name == 'bev' else cam)[i, j]
        if len(view) <= 5:
            assert np.array_equal(want[:len(vals)], vals) and not want[len(vals):].any(), (k, name, i, j)
        else:
            assert np.array_equal(want, vals[:5]), (k, name, i, j)       # the recorder returned pop[:5]
    for name, out in (('bev', bev), ('cam', cam)):          # cells without candidates hold zeros
        empty = [(i, j) for i in range(out.shape[0]) for j in range(out.shape[1]) if (name, i, j) not in lists]
        assert all(not out[i, j].any() for i, j in empty), (k, name)


def test_oracle_matches_reference_on_fixture_sweeps():
    g = np.load(GOLD)
    from oracle import dataset_oracle as DO
    sweeps = CO.fixture_sweeps()
    assert {'rand20k', 'rand40k', 'empty', 'boundary', 'out_of_range', 'pile'} <= set(sweeps)
    for name, sweep in sweeps.items():
        assert DO.digest(sweep) == str(g['sweep_%s_digest' % name]), name
        lists = CO.cell_lists(sweep)
        check_against_reference(g, 'sweep_' + name, lists)
        if name in ('empty', 'out_of_range'):
            assert not lists
        if name != 'empty' and name != 'out_of_range':
            assert any(len(v[0]) > 5 for v in lists.values()), name
        if name in ('pile', 'boundary'):
            assert any(len(v[0]) <= 5 for v in lists.values()), name


@pytest.fixture(scope='module')
def routes(tmp_path_factory):
    return synthetic_route.write_dataset(str(tmp_path_factory.mktemp('carla') / 'data'))


def geometric_samples(root, idx=None, max_points=4000):
    """(key, sample) of CarlaRawDataset(backbone='geometric_fusion', correspondences='gpu') with augmentation, seeded as the fixture was."""
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.dataset import CarlaRawDataset
    ds = CarlaRawDataset([root], TrainConfig(augment=True), backbone='geometric_fusion', correspondences='gpu', max_points=max_points)
    out = []
    for i in (range(len(ds)) if idx is None else idx):
        route, frame = ds.frames[i]
        random.seed(seed_of(os.path.basename(route), frame))
        out.append((key(os.path.basename(route), frame, 1), ds[i]))
    return out


def disk_sweep(s):
    """The on-disk sweep of a geometric sample: the shipped points with y negated back."""
    pts = s['points'][:int(s['n_valid'])].copy()
    pts[:, 1] *= -1
    return pts


def test_reader_geometric_mode_matches_reference(routes):
    """The reader ships the reference's sweep (the oracle's lists from it equal the reference's populations), the angle the
    reference drew (reference_dataset.npz and this fixture's _degree), and a 63-bit seed drawn after the angle."""
    g, gd = np.load(GOLD), np.load(DATASET_GOLD)
    samples = geometric_samples(routes)
    assert len(samples) == 11
    for k, s in samples:
        assert float(s['degree']) == float(g[k + '_degree']) == float(gd[k + '_degree']), k
        check_against_reference(g, k, CO.cell_lists(disk_sweep(s)))
        assert s['corr_seed'].dtype == np.int64 and 0 <= int(s['corr_seed']) < 2 ** 63
        route, frame = k.split('_aug')[0].rsplit('_', 1)
        random.seed(seed_of(route, int(frame)))
        if random.random() > 0.1:
            random.random()
        assert int(s['corr_seed']) == random.getrandbits(63), k


def test_reader_collate_geometric(routes):
    from transfuser_b200.dataset import collate
    b = collate([s for _, s in geometric_samples(routes, idx=[0, 3])])
    assert b['corr_seed'].dtype == torch.int64 and tuple(b['corr_seed'].shape) == (2,)
    from transfuser_b200.trainer import DATASET_KEYS
    assert set(DATASET_KEYS) | {'corr_seed', 'degree'} == set(b)


def test_reader_geometric_opt_in(routes):
    """backbone='geometric_fusion' alone is refused (the reference's host-side correspondences are not produced);
    correspondences='gpu' opts in and ships the seed; seq_len > 1 and PointPillars stay refused in geometric mode."""
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.dataset import CarlaRawDataset
    with pytest.raises(NotImplementedError, match="correspondences='gpu'"):
        CarlaRawDataset([routes], TrainConfig(), backbone='geometric_fusion')
    with pytest.raises(NotImplementedError):
        CarlaRawDataset([routes], TrainConfig(seq_len=2), backbone='geometric_fusion', correspondences='gpu')
    with pytest.raises(NotImplementedError):
        CarlaRawDataset([routes], TrainConfig(use_point_pillars=True), backbone='geometric_fusion', correspondences='gpu')
    with pytest.raises(ValueError):
        CarlaRawDataset([routes], TrainConfig(), correspondences='gpu')
    with pytest.raises(ValueError):
        CarlaRawDataset([routes], TrainConfig(), backbone='geometric_fusion', correspondences='cpu')
    assert 'corr_seed' in CarlaRawDataset([routes], TrainConfig(), backbone='geometric_fusion', correspondences='gpu', max_points=4000)[0]
    assert 'corr_seed' not in CarlaRawDataset([routes], TrainConfig(), max_points=4000)[0]


# ---------------------------------------------------------------- the kernel

def shipped(sweeps, N=None):
    """[B, N, 4] float32 as the reader ships sweeps (y negated, zero padded) and n_valid [B] int32."""
    N = max(len(s) for s in sweeps) if N is None else N
    pts = np.zeros((len(sweeps), max(N, 1), 4), np.float32)[:, :N]
    for b, s in enumerate(sweeps):
        pts[b, :len(s)] = s
        pts[b, :len(s), 1] *= -1
    return torch.from_numpy(np.ascontiguousarray(pts)), torch.tensor([len(s) for s in sweeps], dtype=torch.int32)


def run_kernel(call, to_dev, points, n_valid, seeds):
    """tfb_lidar_cam_correspondences -> (bev_points, cam_points) int64 numpy; outputs start as garbage (every element is written)."""
    from transfuser_b200 import pipeline
    consts, dz = pipeline.correspondence_constants()
    B, N = points.shape[0], points.shape[1]
    bev = to_dev(torch.full((B, 8, 8, 5, 2), -7, dtype=torch.int64))
    cam = to_dev(torch.full((B, 22, 5, 5, 2), -7, dtype=torch.int64))
    work = to_dev(torch.full((B, 6 * max(N, 1)), -1, dtype=torch.int32))
    call('tfb_lidar_cam_correspondences', to_dev(points), None if n_valid is None else to_dev(n_valid), to_dev(torch.as_tensor(seeds, dtype=torch.int64)),
         to_dev(torch.from_numpy(consts)), float(dz), B, N, work, bev, cam)
    return bev.cpu().numpy(), cam.cpu().numpy()


SEEDS = [0, 1, 2 ** 63 - 1, 0x5DEECE66D, 123456789123456789]


def check_fixture_sweeps(call, to_dev=lambda t: t, names=None):
    sweeps = CO.fixture_sweeps()
    names = list(sweeps) if names is None else names
    for q, name in enumerate(names):
        seed = SEEDS[q % len(SEEDS)]
        pts, nv = shipped([sweeps[name]])
        bev, cam = run_kernel(call, to_dev, pts, nv, [seed])
        want_bev, want_cam = CO.correspondences(sweeps[name], seed)
        assert np.array_equal(bev[0], want_bev) and np.array_equal(cam[0], want_cam), name


def test_constants_equal_the_oracle():
    from transfuser_b200 import pipeline
    consts, dz = pipeline.correspondence_constants()
    fx, fy, rl, rr = CO.constants()
    want = np.array([fx, fy] + list(rl.ravel()) + list(rr.ravel()))
    assert np.array_equal(consts.view(np.int64), want.view(np.int64)) and dz == np.float32(2.5 - 2.3)
    assert 304.8 < fx < 304.9


def test_kernel_emulated_fixture_sweeps():
    from cuda_emul import correspondences_emul
    check_fixture_sweeps(correspondences_emul.call)


def test_kernel_emulated_batch_and_n_valid():
    """A batch of three: n_valid cuts sample 0's sweep, sample 1 is empty, sample 2 uses the whole buffer; a null n_valid
    reads every point."""
    from cuda_emul import correspondences_emul
    sweeps = CO.fixture_sweeps()
    a, b = sweeps['pile'], sweeps['boundary']
    pts, nv = shipped([a, np.zeros((0, 4), np.float32), b], N=max(len(a), len(b)))
    pts[1, :50] = torch.from_numpy(a[:50])          # beyond n_valid = 0: ignored
    nv[0] = 700
    seeds = [5, 6, 7]
    bev, cam = run_kernel(correspondences_emul.call, lambda t: t, pts, nv, seeds)
    for i, sweep in enumerate([a[:700], np.zeros((0, 4), np.float32), b]):
        wb, wc = CO.correspondences(sweep, seeds[i])
        assert np.array_equal(bev[i], wb) and np.array_equal(cam[i], wc), i
    pts, _ = shipped([b])
    bev, cam = run_kernel(correspondences_emul.call, lambda t: t, pts, None, [9])
    wb, wc = CO.correspondences(b, 9)
    assert np.array_equal(bev[0], wb) and np.array_equal(cam[0], wc)


def test_kernel_argument_checks_emulated():
    from cuda_emul import correspondences_emul
    pts, nv = shipped([CO.fixture_sweeps()['pile'][:10]])
    for B, N in ((0, 10), (1, -1), (1, 1 << 20)):
        with pytest.raises(RuntimeError, match='argument check'):
            correspondences_emul.call('tfb_lidar_cam_correspondences', pts, nv, torch.zeros(1, dtype=torch.int64), torch.zeros(20, dtype=torch.float64),
                                      0.2, B, N, torch.zeros(60, dtype=torch.int32), torch.zeros(640, dtype=torch.int64), torch.zeros(1100, dtype=torch.int64))


def test_selection_rule_frequencies():
    """One cell with 12 candidates, 6000 seeds: each candidate is among the 5 selected with rate 5/12 and first with rate 1/12
    (chi-square, 11 degrees of freedom, p = 0.001 bound 31.26); the five slots are distinct."""
    view = np.array([0] * 3 + [1] * 6 + [2] * 3)
    index = np.array([3, 50, 900, 3, 4, 5, 6, 70, 800, 2, 60, 61])
    vals = np.stack([np.arange(12), np.zeros(12, np.int64)], 1)
    lists = {('bev', 2, 3): (view, index, vals)}
    n = 6000
    inc, first = np.zeros(12), np.zeros(12)
    for s in range(n):
        bev, _ = CO.select(lists, (s * 0x9E3779B97F4A7C15) & ((1 << 63) - 1))
        got = bev[2, 3, :, 0]
        assert len(set(got.tolist())) == 5
        inc[got] += 1
        first[got[0]] += 1
    for counts, p in ((inc, 5 / 12), (first, 1 / 12)):
        e = n * p
        chi2 = float(((counts - e) ** 2 / e).sum()) if p == 1 / 12 else float(((counts - e) ** 2 / (e * (1 - p))).sum())
        assert chi2 < 31.26, (counts, chi2)
    # at most 5 candidates: the reference's order whatever the seed
    small = {('cam', 4, 1): (view[:5], index[:5], vals[:5])}
    for s in (0, 1, 2 ** 62):
        _, cam = CO.select(small, s)
        assert cam[4, 1, :, 0].tolist() == [0, 1, 2, 3, 4]
