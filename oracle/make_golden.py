"""ORACLE / TEST INFRASTRUCTURE ONLY. Generates the committed fixtures under tests/golden/ by executing the REFERENCE
itself (imported verbatim from a reference checkout via oracle/ref_import.py) on seeded inputs. Run in the build container:
    python oracle/make_golden.py [bev] [model] [pipeline]
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import bev_oracle, ref_import  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')


def make_bev():
    ref = ref_import.load_histogram_fn()
    out = {}
    for dt in ('float32', 'float64'):
        for seed, n in ((0, 40000), (7, 2000)):
            pts = bev_oracle.synthetic_points(n, seed, np.dtype(dt).type)
            out['out_%s_%d_%d' % (dt, seed, n)] = ref(pts)
    np.savez_compressed(os.path.join(GOLD, 'bev_hist.npz'), **out)
    print('wrote bev_hist.npz', {k: float(v.sum()) for k, v in out.items()})


def make_pipeline():
    """Input-preparation fixtures from the reference's own data.py functions (real OpenCV), plus the exhaustive check of the
    target-point stamp that oracle/pipeline_oracle.py and csrc/input_prep.cu embed."""
    import cv2
    from oracle import pipeline_oracle as PO
    fn = ref_import.load_data_fns(['align', 'draw_target_point', 'crop_image_cv2', 'crop_seg', 'get_depth', 'lidar_to_histogram_features'])
    img = np.zeros((256, 256), np.uint8)
    cv2.circle(img, (128, 128), radius=5, color=(255, 255, 255), thickness=3)
    st = img[121:136, 121:136] > 0
    assert tuple(int(''.join('1' if v else '0' for v in r[::-1]), 2) for r in st) == PO.STAMP
    for py in range(257):
        for px in range(257):
            im = np.zeros((256, 256), np.uint8)
            cv2.circle(im, (px, py), radius=5, color=(255, 255, 255), thickness=3)
            exp = np.zeros((272, 272), bool)
            exp[py + 1:py + 16, px + 1:px + 16] = st
            assert np.array_equal(im > 0, exp[8:264, 8:264]), (px, py)
    conv = [0, 1, 2, 3, 4, 5, 6, 4, 3, 0, 2, 1, 5, 6, 0, 1, 2, 3, 4, 5, 6, 0, 1]
    out = {}
    crop, H, W = (32, 176), 40, 240                      # a small frame keeps the (incompressible, random) fixture small
    for seed in (0, 1):
        f = PO.synthetic_frame(seed, H=H, W=W)
        shift = f['degree'] / 60 * (W // 3) / 1          # data.py:219 with img_width = one camera's width
        pts = fn['align'](f['points'], dict(ego_matrix=f['ego_matrix_0']), dict(ego_matrix=f['ego_matrix_1']), degree=f['degree'])
        out['lidar_%d' % seed] = fn['lidar_to_histogram_features'](pts)
        out['rgb_%d' % seed] = fn['crop_image_cv2'](f['rgb'], crop=crop, crop_shift=shift).astype(np.float32)
        out['depth_%d' % seed] = fn['get_depth'](fn['crop_image_cv2'](f['depth'], crop=crop, crop_shift=shift)).astype(np.float32)
        out['semantic_%d' % seed] = np.uint8(conv)[fn['crop_seg'](f['seg'], crop=crop, crop_shift=shift)].astype(np.int64)
        out['target_point_image_%d' % seed] = fn['draw_target_point'](f['target_point']).astype(np.float32)
    np.savez_compressed(os.path.join(GOLD, 'pipeline_golden.npz'), **out)
    print('wrote pipeline_golden.npz; stamp verified over 257x257 centres')


if __name__ == '__main__':
    what = sys.argv[1:] or ['bev', 'model', 'pipeline']
    os.makedirs(GOLD, exist_ok=True)
    if 'bev' in what:
        make_bev()
    if 'model' in what:
        from oracle import make_golden_model
        make_golden_model.main()
    if 'pipeline' in what:
        make_pipeline()
