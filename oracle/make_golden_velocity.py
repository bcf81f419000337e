"""ORACLE / TEST INFRASTRUCTURE ONLY. Runs the VERBATIM reference (oracle/ref_import.py) with use_velocity=True for the four
backbones and stores what tests/test_velocity.py and tests/test_velocity_gpu.py compare with as
tests/golden/reference_velocity.npz:
    python oracle/make_golden_velocity.py        (needs a reference checkout, see oracle/ref_import.py)

Per backbone: the state_dict keys and shapes; in float64, the backbone outputs (norm + seeded sample, as make_golden_reference.py
stores them) in train mode with dropout 0 and in eval mode, and the forward_ego waypoints of one eval batch; in float32, the 11
losses of the whole model on a seeded batch and the gradients of every vel_emb* parameter under the loss weights of config.py."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import, torch_oracle as O  # noqa: E402
from oracle.make_golden_reference import shrink  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'reference_velocity.npz')
# backbone -> n_layer (None: the reference default), as oracle/make_golden_reference.py builds them
BACKBONES = {'transFuser': 4, 'late_fusion': None, 'geometric_fusion': None, 'latentTF': 4}
WEIGHT_SEED = 31
BATCH_SEED = 17


def reference(m, backbone, seed=None):
    cfg = m['config'].GlobalConfig(setting='eval')
    cfg.use_target_point_image = True
    if BACKBONES[backbone]:
        cfg.n_layer = BACKBONES[backbone]
    cfg.embd_pdrop = cfg.attn_pdrop = cfg.resid_pdrop = 0.0
    torch.manual_seed(0)
    ref = m['model'].LidarCenterNet(cfg, 'cpu', backbone, 'regnety_032', 'regnety_032', use_velocity=True)
    if seed is not None:
        names = [(n, tuple(p.shape)) for n, p in list(ref.named_parameters()) + list(ref.named_buffers())]
        ref.load_state_dict(O.deterministic_state(names, seed=seed), strict=False)
    return ref, cfg


def batch_of(B, seed, backbone):
    b = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in O.synthetic_batch(B, seed=seed).items()}
    if backbone == 'geometric_fusion':
        b['bev_points'], b['cam_points'] = O.synthetic_correspondences(B, seed=seed)
    return b


def geo_kw(b):
    return dict(bev_points=b['bev_points'], cam_points=b['cam_points']) if 'bev_points' in b else {}


def main():
    m = ref_import.load()
    out = {}
    for backbone in BACKBONES:
        ref, _ = reference(m, backbone)
        sd = ref.state_dict()
        out['sd_%s_keys' % backbone] = np.array(list(sd.keys()))
        out['sd_%s_shapes' % backbone] = np.array(['x'.join(map(str, v.shape)) for v in sd.values()])

    torch.set_default_dtype(torch.float64)
    for backbone in BACKBONES:
        # backbone outputs, train (dropout 0) and eval
        for train in (True, False):
            ref, _ = reference(m, backbone, WEIGHT_SEED)
            ref = ref.double().train(train)
            b = batch_of(2, BATCH_SEED, backbone)
            lidar = torch.cat((b['lidar'], b['target_point_image']), dim=1)
            args = (b['bev_points'], b['cam_points']) if backbone == 'geometric_fusion' else ()
            with torch.no_grad():
                feats, grid, fused = ref._model(b['rgb'], lidar.clone(), b['ego_vel'], *args)
            for i, t in enumerate(list(feats) + [grid, fused]):
                key = '%s_out_%d_%d' % (backbone, train, i)
                out[key + '_shape'] = np.array(t.shape)
                out[key + '_norm'], out[key + '_sample'] = shrink(t)
        # whole-model losses and the vel_emb* gradients (train mode, dropout 0), in float32: the reference's BEV loss makes its
        # class-weight tensor in float32 (model.py:762-763)
        torch.set_default_dtype(torch.float32)
        ref, cfg = reference(m, backbone, WEIGHT_SEED)
        ref = ref.train()
        b = {k: (v.float() if v.dtype.is_floating_point else v) for k, v in batch_of(2, BATCH_SEED + 1, backbone).items()}
        loss = ref(b['rgb'], b['lidar'], ego_waypoint=b['ego_waypoint'], target_point=b['target_point'],
                   target_point_image=b['target_point_image'], ego_vel=b['ego_vel'], bev=b['bev'], label=b['label'],
                   depth=b['depth'], semantic=b['semantic'], **geo_kw(b))
        w = dict(zip(cfg.detailed_losses, cfg.detailed_losses_weights))
        out['%s_loss_names' % backbone] = np.array(list(loss.keys()))
        out['%s_losses' % backbone] = np.array([float(v) for v in loss.values()], dtype=np.float64)
        sum(w[k] * v for k, v in loss.items()).backward()
        vel = [(n, p) for n, p in ref.named_parameters() if '.vel_emb' in n]
        out['%s_grad_names' % backbone] = np.array([n for n, _ in vel])
        for n, p in vel:
            out['%s_grad_%s' % (backbone, n)] = p.grad.double().numpy()
        torch.set_default_dtype(torch.float64)
        # forward_ego waypoints (eval)
        ref, _ = reference(m, backbone, WEIGHT_SEED)
        ref = ref.double().eval()
        b = batch_of(1, BATCH_SEED + 2, backbone)
        with torch.no_grad():
            wp, _ = ref.forward_ego(b['rgb'], b['lidar'], b['target_point'], b['target_point_image'], b['ego_vel'], **geo_kw(b))
        out['%s_ego_wp' % backbone] = wp.double().numpy()
        print(backbone, 'done', flush=True)
    torch.set_default_dtype(torch.float32)
    np.savez_compressed(GOLD, **out)
    print('wrote %s (%d bytes, %d arrays)' % (GOLD, os.path.getsize(GOLD), len(out)))


if __name__ == '__main__':
    main()
