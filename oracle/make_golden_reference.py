"""ORACLE / TEST INFRASTRUCTURE ONLY. Runs the VERBATIM reference (oracle/ref_import.py) on the seeded weights / inputs of the
tests that compare against it and stores what they compare with as tests/golden/reference_checks.npz, so that those tests
run from the repository alone:
    python oracle/make_golden_reference.py        (needs a reference checkout, see oracle/ref_import.py)

Bit-exact comparisons of large arrays are stored as SHA-256 digests of (dtype, shape, bytes); tolerance comparisons of large
tensors as their norm plus a seeded sample of SAMPLE elements; everything else verbatim."""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import bev_oracle, ref_import, torch_oracle as O  # noqa: E402
from oracle import pipeline_oracle as PO  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'reference_checks.npz')
SAMPLE = 4096


def digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(('%s%s' % (a.dtype.str, a.shape)).encode() + a.tobytes()).hexdigest()


def sample_index(n, seed=0):
    return np.unique(np.random.default_rng(seed).integers(0, n, size=min(SAMPLE, n)))


def shrink(t):
    """(norm, seeded sample) of a tensor: what a relative-error comparison against it needs."""
    f = t.detach().double().reshape(-1).numpy()
    return np.array([np.linalg.norm(f)]), f[sample_index(f.size)]


# the reference model configurations of the tests: (backbone, n_layer or None for the reference default, use_velocity)
MODELS = {'transFuser': ('transFuser', 4, False), 'late_fusion': ('late_fusion', None, False), 'geometric_fusion': ('geometric_fusion', None, False),
          'latentTF': ('latentTF', 4, False), 'transFuser_vel': ('transFuser', 4, True)}


def reference(m, key, seed=None, drop0=False):
    backbone, n_layer, vel = MODELS[key]
    cfg = m['config'].GlobalConfig(setting='eval')
    cfg.use_target_point_image = True
    if n_layer:
        cfg.n_layer = n_layer
    if drop0:
        cfg.embd_pdrop = cfg.attn_pdrop = cfg.resid_pdrop = 0.0
    torch.manual_seed(0)
    ref = m['model'].LidarCenterNet(cfg, 'cpu', backbone, 'regnety_032', 'regnety_032', use_velocity=vel)
    if seed is not None:
        names = [(n, tuple(p.shape)) for n, p in list(ref.named_parameters()) + list(ref.named_buffers())]
        ref.load_state_dict(O.deterministic_state(names, seed=seed), strict=False)
    return ref, cfg


def config_attrs(m):
    """The reference's GlobalConfig(setting='eval') with use_target_point_image = True, as JSON: every public attribute whose
    value JSON can hold (the product modules are built from it in tests/test_widen.py)."""
    import json
    cfg = m['config'].GlobalConfig(setting='eval')
    cfg.use_target_point_image = True
    out = {}
    for k in dir(cfg):
        if k.startswith('_'):
            continue
        v = getattr(cfg, k)
        try:
            json.dumps(v)
        except TypeError:
            continue
        out[k] = v
    return json.dumps(out, sort_keys=True)


def losses_of(ref, batch, **kw):
    with torch.no_grad():
        want = ref(batch['rgb'], batch['lidar'], ego_waypoint=batch['ego_waypoint'], target_point=batch['target_point'],
                   target_point_image=batch['target_point_image'], ego_vel=batch['ego_vel'], bev=batch['bev'], label=batch['label'],
                   depth=batch['depth'], semantic=batch['semantic'], **kw)
    return np.array(list(want.keys())), np.array([float(v) for v in want.values()], dtype=np.float64)


def main():
    m = ref_import.load()
    out = {}
    out['reference_config_json'] = np.array(config_attrs(m))
    # state_dict contracts (key order and shapes) of every backbone the product offers as a drop-in
    for key in MODELS:
        ref, _ = reference(m, key)
        sd = ref.state_dict()
        out['sd_%s_keys' % key] = np.array(list(sd.keys()))
        out['sd_%s_shapes' % key] = np.array(['x'.join(map(str, v.shape)) for v in sd.values()])

    # whole-model losses: tests/test_oracle.py
    from oracle.make_golden_model import WEIGHT_SEED
    ref, _ = reference(m, 'transFuser', WEIGHT_SEED, drop0=True)
    out['loss_transFuser_names'], out['loss_transFuser'] = losses_of(ref.train(), O.synthetic_batch(1, seed=2))
    ref, _ = reference(m, 'late_fusion', 6)
    out['loss_late_fusion_names'], out['loss_late_fusion'] = losses_of(ref.train(), O.synthetic_batch(1, seed=4))
    ref, _ = reference(m, 'geometric_fusion', 8)
    b = O.synthetic_batch(2, seed=5)
    b['bev_points'], b['cam_points'] = O.synthetic_correspondences(2, seed=5)
    out['loss_geometric_fusion_names'], out['loss_geometric_fusion'] = losses_of(ref.train(), b, bev_points=b['bev_points'], cam_points=b['cam_points'])
    ref, _ = reference(m, 'latentTF', 12)
    for mode in (True, False):
        ref.train(mode)
        for mod in ref.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
        b = O.synthetic_batch(2, seed=7)
        b['rgb'], b['lidar'] = b['rgb'].clone(), b['lidar'].clone()
        out['loss_latentTF_%d_names' % mode], out['loss_latentTF_%d' % mode] = losses_of(ref, b)

    # CenterNet decode and forward_ego (eval mode): tests/test_oracle.py
    ref, _ = reference(m, 'transFuser', 3)
    ref.eval()
    g = torch.Generator().manual_seed(21)
    for case in range(3):
        B = 2
        heat = torch.rand(B, 1, 64, 64, generator=g)
        if case == 1:
            heat = (heat * 8).round() / 8
        if case == 2:
            heat = heat * (heat > 0.995)
        preds = [heat] + [torch.randn(B, c, 64, 64, generator=g) for c in (2, 2, 12, 1, 1, 2)]
        want = ref.head.get_bboxes(*[[p] for p in preds])
        for bi in range(B):
            out['decode_%d_%d_boxes' % (case, bi)] = want[bi][0].numpy()
            out['decode_%d_%d_labels' % (case, bi)] = want[bi][1].numpy()
    ref, _ = reference(m, 'transFuser', 9)
    ref.eval()
    batch = O.synthetic_batch(1, seed=6)
    with torch.no_grad():
        wp, boxes = ref.forward_ego(batch['rgb'], batch['lidar'], batch['target_point'], batch['target_point_image'], batch['ego_vel'])
    out['ego_wp'] = wp.numpy()
    out['ego_boxes'] = np.stack([b[0] for b in boxes])
    out['ego_brake'] = np.array([float(b[1]) for b in boxes])
    out['ego_conf'] = np.array([float(b[2]) for b in boxes])

    # host box geometry: tests/test_widen.py
    ref, _ = reference(m, 'late_fusion')
    rng = np.random.default_rng(5)
    rows, metric, brake, conf = [], [], [], []
    for _ in range(20):
        row = np.concatenate([rng.uniform(0, 256, 2), rng.uniform(1, 40, 2), rng.uniform(-np.pi, np.pi, 1), rng.uniform(0, 8, 1),
                              rng.integers(0, 2, 1), rng.uniform(0.3, 1, 1)]).astype(np.float32)
        a, ab, ac = ref.get_bbox_local_metric(row)
        rows.append(row); metric.append(a); brake.append(float(ab)); conf.append(float(ac))
    out['bbox_rows'], out['bbox_metric'], out['bbox_brake'], out['bbox_conf'] = np.stack(rows), np.stack(metric), np.array(brake), np.array(conf)

    # use_velocity backbone outputs, built and run with float64 as the default dtype like the test: tests/test_host_logic.py
    torch.set_default_dtype(torch.float64)
    for train in (True, False):
        ref, _ = reference(m, 'transFuser_vel', 12, drop0=True)
        ref = ref.double().train(train)
        batch = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in O.synthetic_batch(2, seed=13).items()}
        lidar = torch.cat((batch['lidar'], batch['target_point_image']), dim=1)
        with torch.no_grad():
            feats, grid, fused = ref._model(batch['rgb'], lidar.clone(), batch['ego_vel'])
        for i, t in enumerate(list(feats) + [grid, fused]):
            out['vel_%d_%d_shape' % (train, i)] = np.array(t.shape)
            out['vel_%d_%d_norm' % (train, i)], out['vel_%d_%d_sample' % (train, i)] = shrink(t)
    torch.set_default_dtype(torch.float32)

    # BEV histogram and input preparation, bit-exact: tests/test_bev.py, tests/test_pipeline.py
    hist = ref_import.load_histogram_fn()
    for dt in (np.float32, np.float64):
        for seed, n in ((0, 40000), (1, 1000), (2, 0), (3, 64)):
            pts = bev_oracle.synthetic_points(n, seed, dt)
            if n == 0:
                pts = pts.reshape(0, 4)
            out['bev_%s_%d_%d' % (np.dtype(dt).name, seed, n)] = np.array(digest(hist(pts)))
    fn = ref_import.load_data_fns(['align', 'draw_target_point', 'crop_image_cv2', 'crop_seg', 'get_depth', 'lidar_to_histogram_features'])
    conv = [0, 1, 2, 3, 4, 5, 6, 4, 3, 0, 2, 1, 5, 6, 0, 1, 2, 3, 4, 5, 6, 0, 1]
    for seed in range(6):
        f = PO.synthetic_frame(seed)
        shift = f['degree'] / 60 * 320 / 1
        pts = fn['align'](f['points'], dict(ego_matrix=f['ego_matrix_0']), dict(ego_matrix=f['ego_matrix_1']), degree=f['degree'])
        out['pipe_%d_align' % seed] = np.array(digest(pts))
        out['pipe_%d_align_sample' % seed] = pts[sample_index(len(pts), seed)]
        out['pipe_%d_lidar' % seed] = np.array(digest(fn['lidar_to_histogram_features'](pts)))
        out['pipe_%d_rgb' % seed] = np.array(digest(fn['crop_image_cv2'](f['rgb'], crop=(160, 704), crop_shift=shift)))
        out['pipe_%d_depth' % seed] = np.array(digest(fn['get_depth'](fn['crop_image_cv2'](f['depth'], crop=(160, 704), crop_shift=shift))))
        out['pipe_%d_seg' % seed] = np.array(digest(np.uint8(conv)[fn['crop_seg'](f['seg'], crop=(160, 704), crop_shift=shift)]))
    rng = np.random.default_rng(0)
    tps = [rng.uniform(-40, 40, 2) for _ in range(300)] + [np.array([x, y]) for x in (-16.2, -16.0, 15.9, 16.0, 16.1) for y in (-1.4, -1.3, 30.6, 30.7, 30.8)]
    tps += [np.array([1e12, -1e12]), np.array([0.0, 0.0])]
    out['target_points'] = np.stack(tps)
    out['target_point_images'] = np.array([digest(fn['draw_target_point'](tp)) for tp in tps])

    np.savez_compressed(GOLD, **out)
    print('wrote %s (%d bytes, %d arrays)' % (GOLD, os.path.getsize(GOLD), len(out)))


if __name__ == '__main__':
    main()
