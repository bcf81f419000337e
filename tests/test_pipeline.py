"""GPU input pipeline (SURVEY.md §8f rank 2; data.py:103-356). CPU: the numpy oracle against the outputs of the reference's own
functions (exec'd from data.py with the real OpenCV; tests/golden/reference_checks.npz) and against the committed fixture;
host-side pose algebra of the product against the reference. GPU: the three kernels against the oracle — bytes / indices / histogram counts bit-exact."""
import os

import numpy as np
import pytest
import torch

from oracle import pipeline_oracle as PO
from oracle import bev_oracle
from oracle.make_golden_reference import GOLD as REF_GOLD, digest, sample_index

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'pipeline_golden.npz')
DEV = 'cuda'   # the emulated re-runs (tests/test_widen_emulated.py, tools/emulated_module_checks.py) switch this to 'cpu'


def _sync():
    if DEV == 'cuda':
        torch.cuda.synchronize()


CONVERTER = [0, 1, 2, 3, 4, 5, 6, 4, 3, 0, 2, 1, 5, 6, 0, 1, 2, 3, 4, 5, 6, 0, 1]    # any 23-entry map to 7 classes


def _oracle_sample(f, crop=(160, 704), scale=1, img_width=320):
    shift = int(f['degree'] / 60 * img_width / scale)
    T = PO.align_transform(f['ego_matrix_0'], f['ego_matrix_1'], f['degree'])
    rgb = PO.crop_rgb(f['rgb'], crop, shift)
    return dict(rgb=rgb.astype(np.float32), rgb_norm=PO.normalize_nhwc(rgb),
                depth=PO.depth_from_rgb(PO.crop_rgb(f['depth'], crop, shift)).astype(np.float32),
                semantic=PO.seg_classes(f['seg'], CONVERTER, crop, shift).astype(np.int64),
                lidar=bev_oracle.lidar_to_histogram_features(PO.align_points(f['points'], T)),
                target_point_image=PO.draw_target_point(f['target_point']).astype(np.float32), T=T, shift=shift)


def test_pipeline_oracle_matches_reference_functions():
    """Bit-exact against the reference's align / lidar_to_histogram_features / crop_image_cv2 / get_depth / crop_seg /
    draw_target_point on the same inputs (digests of their outputs, oracle/make_golden_reference.py)."""
    g = np.load(REF_GOLD)
    for seed in range(6):
        f = PO.synthetic_frame(seed)
        shift = f['degree'] / 60 * 320 / 1                                   # data.py:219, config.img_width 320 (float; the crops apply int())
        T = PO.align_transform(f['ego_matrix_0'], f['ego_matrix_1'], f['degree'])
        got_pts = PO.align_points(f['points'], T)
        assert got_pts.dtype == np.float64 and digest(got_pts) == str(g['pipe_%d_align' % seed]), seed
        assert digest(bev_oracle.lidar_to_histogram_features(got_pts)) == str(g['pipe_%d_lidar' % seed]), seed
        assert digest(PO.crop_rgb(f['rgb'], (160, 704), shift)) == str(g['pipe_%d_rgb' % seed]), seed
        assert digest(PO.depth_from_rgb(PO.crop_rgb(f['depth'], (160, 704), shift))) == str(g['pipe_%d_depth' % seed]), seed
        assert digest(PO.seg_classes(f['seg'], CONVERTER, (160, 704), shift)) == str(g['pipe_%d_seg' % seed]), seed
    for tp, want in zip(g['target_points'], g['target_point_images']):
        assert digest(PO.draw_target_point(tp)) == str(want), tp


def test_pipeline_oracle_matches_golden():
    g = np.load(GOLD)
    for seed in (0, 1):
        o = _oracle_sample(PO.synthetic_frame(seed, H=40, W=240), crop=(32, 176), img_width=80)
        for k in ('rgb', 'depth', 'semantic', 'lidar', 'target_point_image'):
            assert np.array_equal(o[k], g['%s_%d' % (k, seed)]), (k, seed)


def test_product_pose_algebra_matches_reference():
    """transfuser_b200.pipeline.align_transform (host numpy, like the reference) applied the reference's way == align()
    (a seeded sample of align()'s points, and the digest of the histogram of all of them)."""
    from transfuser_b200 import pipeline
    g = np.load(REF_GOLD)
    for seed in range(4):
        f = PO.synthetic_frame(seed)
        T = pipeline.align_transform(f['ego_matrix_0'], f['ego_matrix_1'], f['degree'])
        got = PO.align_points(f['points'], T)
        assert np.allclose(got[sample_index(len(got), seed)], g['pipe_%d_align_sample' % seed], rtol=0, atol=1e-9)
        assert digest(bev_oracle.lidar_to_histogram_features(got)) == str(g['pipe_%d_lidar' % seed])
    assert pipeline.crop_shift_pixels(-13.7, 320, 1) == int(-13.7 / 60 * 320 / 1)


def test_pipeline_rejects_bad_inputs_on_host():
    from transfuser_b200 import pipeline
    from transfuser_b200.config import TrainConfig
    with pytest.raises(RuntimeError):
        pipeline.InputPipeline(TrainConfig(), 'cpu').prepare({})


def _raw_batch(seeds):
    from transfuser_b200 import pipeline
    fs = [PO.synthetic_frame(s) for s in seeds]
    raw = dict(rgb=torch.from_numpy(np.stack([f['rgb'] for f in fs])), depth=torch.from_numpy(np.stack([f['depth'] for f in fs])),
               seg=torch.from_numpy(np.stack([f['seg'] for f in fs])),
               crop_shift=torch.tensor([pipeline.crop_shift_pixels(f['degree'], 320, 1) for f in fs], dtype=torch.int32),
               points=torch.from_numpy(np.stack([f['points'] for f in fs])),
               transforms=torch.from_numpy(np.stack([pipeline.align_transform(f['ego_matrix_0'], f['ego_matrix_1'], f['degree']) for f in fs])),
               target_point=torch.from_numpy(np.stack([f['target_point'] for f in fs])))
    return fs, raw


@pytest.mark.gpu
def test_input_pipeline_matches_oracle():
    from transfuser_b200 import pipeline
    from transfuser_b200.config import TrainConfig
    fs, raw = _raw_batch([0, 1, 2])
    pipe = pipeline.InputPipeline(TrainConfig(converter=CONVERTER), DEV)
    out = pipe.prepare(raw)
    outn = pipe.prepare(raw, normalized_nhwc=True)
    _sync()
    for b, f in enumerate(fs):
        o = _oracle_sample(f)
        assert np.array_equal(out['rgb'][b].cpu().numpy(), o['rgb'])
        assert np.array_equal(out['semantic'][b].cpu().numpy(), o['semantic'])
        assert np.array_equal(out['depth'][b].cpu().numpy(), o['depth'])
        assert np.array_equal(out['target_point_image'][b].cpu().numpy(), o['target_point_image'])
        assert np.array_equal(out['lidar'][b].cpu().numpy(), o['lidar'])
        assert np.allclose(outn['rgb'][b].cpu().numpy(), o['rgb_norm'], rtol=1e-6, atol=1e-6)
    # the normalised NHWC form is what the backbone's own prep kernel produces from the float NCHW form
    from transfuser_b200 import ops
    assert torch.equal(ops.image_prep(out['rgb']), outn['rgb']) and ops.image_prep(outn['rgb']) is outn['rgb']


@pytest.mark.gpu
def test_target_point_map_borders_and_overflow():
    from transfuser_b200 import _lib
    pts = [(x, y) for x in (-16.2, -16.0, 15.9, 16.0, 16.1, 0.3) for y in (-1.4, -1.3, 30.6, 30.7, 30.8, 7.77)] + [(1e12, -1e12), (float('nan'), 0.0)]
    tp = torch.tensor(pts, dtype=torch.float64, device=DEV)
    out = torch.empty((len(pts), 1, 256, 256), dtype=torch.float32, device=DEV)
    _lib.call('tfb_draw_target_point', tp, len(pts), out)
    for i, p in enumerate(pts):
        assert np.array_equal(out[i].cpu().numpy(), PO.draw_target_point(np.array(p)).astype(np.float32)), p


@pytest.mark.gpu
def test_aligned_histogram_identity_transform_equals_plain_histogram():
    """Property at full size (40k points): with the identity transform the fused kernel is the plain histogram kernel on the
    float64 copy of the cloud — align() returns float64 (data.py:440: float64 matrix @ points), so the z split `<= -2.3` is a
    float64 comparison there, while a float32 cloud is compared in float32 (a point at z = float32(-2.3) lands in different
    channels; first hardware run of round 2 showed exactly that one cell)."""
    from transfuser_b200 import _lib, bev
    pts = torch.from_numpy(np.stack([bev_oracle.synthetic_points(40000, s, np.float32) for s in (3, 4)])).to(DEV)
    want = bev.lidar_to_histogram_features_batched(pts.double())
    for i in range(2):   # and the float64 oracle (the reference's numpy semantics) agrees
        assert np.array_equal(want[i].cpu().numpy(), bev_oracle.lidar_to_histogram_features(pts[i].double().cpu().numpy()))
    T = torch.eye(4, dtype=torch.float64, device=DEV).reshape(1, 16).repeat(2, 1).contiguous()
    counts = torch.empty((2, 2, 256, 256), dtype=torch.int32, device=DEV)
    got = torch.empty((2, 2, 256, 256), dtype=torch.float32, device=DEV)
    _lib.call('tfb_bev_histogram_aligned', pts, 0, T, None, 2, 40000, counts, got)
    assert torch.equal(got, want)
