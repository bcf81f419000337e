"""BEV histogram: oracle vs the reference function's outputs / committed fixtures (CPU), CUDA kernel vs oracle (GPU, bit-exact)."""
import os

import numpy as np
import pytest
import torch

from oracle import bev_oracle
from oracle.make_golden_reference import GOLD as REF_GOLD, digest

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'bev_hist.npz')


def test_oracle_matches_golden_fixture():
    g = np.load(GOLD)
    for key in [k for k in g.files if k.startswith('out_')]:
        _, dt, seed, n = key.split('_')
        pts = bev_oracle.synthetic_points(int(n), int(seed), np.dtype(dt).type)
        assert np.array_equal(bev_oracle.lidar_to_histogram_features(pts), g[key]), key


def test_oracle_matches_reference_function():
    """Bit-exact against the reference's lidar_to_histogram_features (data.py:446-470) on the same inputs (digests of its
    outputs, oracle/make_golden_reference.py)."""
    g = np.load(REF_GOLD)
    for dt in (np.float32, np.float64):
        for seed, n in ((0, 40000), (1, 1000), (2, 0), (3, 64)):
            pts = bev_oracle.synthetic_points(n, seed, dt)
            if n == 0:
                pts = pts.reshape(0, 4)
            assert digest(bev_oracle.lidar_to_histogram_features(pts)) == str(g['bev_%s_%d_%d' % (np.dtype(dt).name, seed, n)]), (dt, seed, n)


@pytest.mark.gpu
@pytest.mark.parametrize('dt', [np.float32, np.float64])
def test_cuda_matches_oracle_bit_exact(dt):
    from transfuser_b200 import bev
    for seed, n in ((0, 40000), (1, 1000), (3, 64), (4, 1), (5, 123457)):
        pts = bev_oracle.synthetic_points(n, seed, dt)
        got = bev.lidar_to_histogram_features(pts)
        assert got.dtype == np.float32 and got.shape == (2, 256, 256)
        assert np.array_equal(got, bev_oracle.lidar_to_histogram_features(pts)), (dt, seed, n)


@pytest.mark.gpu
def test_cuda_golden_fixture_and_batch_ragged():
    from transfuser_b200 import bev
    g = np.load(GOLD)
    for key in [k for k in g.files if k.startswith('out_')]:
        _, dt, seed, n = key.split('_')
        pts = bev_oracle.synthetic_points(int(n), int(seed), np.dtype(dt).type)
        assert np.array_equal(bev.lidar_to_histogram_features(pts), g[key]), key
    # ragged batch: per-sample point counts, padding rows must be ignored; empty sample -> all zeros
    ns = [40000, 0, 17, 25000]
    batch = np.zeros((len(ns), 40000, 4), dtype=np.float32)
    batch[:] = 3.0  # padding that WOULD land inside the grid if it were counted
    want = []
    for i, n in enumerate(ns):
        pts = bev_oracle.synthetic_points(n, 10 + i, np.float32) if n else np.zeros((0, 4), np.float32)
        batch[i, :n] = pts
        want.append(bev_oracle.lidar_to_histogram_features(pts))
    got = bev.lidar_to_histogram_features_batched(torch.from_numpy(batch).cuda(), torch.tensor(ns, dtype=torch.int32).cuda())
    assert np.array_equal(got.cpu().numpy(), np.stack(want))
    assert got[1].abs().sum().item() == 0


@pytest.mark.gpu
def test_cuda_full_size_properties():
    """Size-independent properties at the bench size (B=10 x 40k points): counts are additive under concatenation
    below the clip, values lie in {0,.2,..,1}, and point order does not matter."""
    from transfuser_b200 import bev
    pts = torch.from_numpy(np.stack([bev_oracle.synthetic_points(40000, 100 + i, np.float32, edge_cases=False) for i in range(10)])).cuda()
    out = bev.lidar_to_histogram_features_batched(pts)
    vals = torch.unique(out)
    assert set(np.round(vals.cpu().numpy() * 5).astype(int).tolist()) <= {0, 1, 2, 3, 4, 5}
    perm = torch.randperm(40000, device='cuda')
    assert torch.equal(out, bev.lidar_to_histogram_features_batched(pts[:, perm].contiguous()))
    half_a = bev.lidar_to_histogram_features_batched(pts[:, :20000].contiguous())
    half_b = bev.lidar_to_histogram_features_batched(pts[:, 20000:].contiguous())
    summed = torch.clamp(torch.round((half_a + half_b) * 5), max=5) / 5
    unclipped = (half_a < 1) & (half_b < 1)
    assert torch.equal(torch.round(out[unclipped] * 5), torch.round(summed[unclipped] * 5))
