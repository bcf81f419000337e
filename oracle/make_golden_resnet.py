"""ORACLE / TEST INFRASTRUCTURE ONLY. Runs the VERBATIM reference (oracle/ref_import.py) with its default ResNet trunks
(image resnet34, LiDAR resnet18; model.py:545) and stores what tests/test_resnet_trunks.py compares with as
tests/golden/reference_resnet.npz, so that those tests run from the repository alone:
    python oracle/make_golden_resnet.py        (needs a reference checkout, see oracle/ref_import.py)

Stored: the state_dict keys and shapes of transFuser and late_fusion, the 11 losses of both at seeded weights and batch with
dropout 0, the parameter-gradient norms of transFuser for the weighted loss sum, and the exception type the reference raises
when geometric_fusion / latentTF are asked for ResNet trunks."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import, timm_resnet, torch_oracle as O  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'reference_resnet.npz')
TRUNKS = ('resnet34', 'resnet18')
# (backbone, weight seed, batch seed) of the loss checks
LOSS_CASES = {'transFuser': (31, 32), 'late_fusion': (33, 34)}


def reference(m, backbone, seed=None):
    cfg = m['config'].GlobalConfig(setting='eval')
    cfg.use_target_point_image = True
    cfg.n_layer = 4
    cfg.embd_pdrop = cfg.attn_pdrop = cfg.resid_pdrop = 0.0
    torch.manual_seed(0)
    with timm_resnet.with_resnets(sys.modules['timm']):       # the reference's `import timm` is the regnety_032 shim
        ref = m['model'].LidarCenterNet(cfg, 'cpu', backbone, *TRUNKS, use_velocity=False)
    if seed is not None:
        names = [(n, tuple(p.shape)) for n, p in list(ref.named_parameters()) + list(ref.named_buffers())]
        ref.load_state_dict(O.deterministic_state(names, seed=seed), strict=False)
    return ref, cfg


def main():
    m = ref_import.load()
    out = {'trunks': np.array(TRUNKS)}
    for backbone, (wseed, bseed) in LOSS_CASES.items():
        ref, cfg = reference(m, backbone, wseed)
        sd = ref.state_dict()
        out['sd_%s_keys' % backbone] = np.array(list(sd.keys()))
        out['sd_%s_shapes' % backbone] = np.array(['x'.join(map(str, v.shape)) for v in sd.values()])
        ref.train()
        b = O.synthetic_batch(1, seed=bseed)
        losses = ref(b['rgb'], b['lidar'], ego_waypoint=b['ego_waypoint'], target_point=b['target_point'],
                     target_point_image=b['target_point_image'], ego_vel=b['ego_vel'], bev=b['bev'], label=b['label'],
                     depth=b['depth'], semantic=b['semantic'])
        out['loss_%s_names' % backbone] = np.array(list(losses.keys()))
        out['loss_%s' % backbone] = np.array([float(v) for v in losses.values()], dtype=np.float64)
        if backbone == 'transFuser':
            w = dict(zip(cfg.detailed_losses, cfg.detailed_losses_weights))
            sum(w[k] * v for k, v in losses.items()).backward()
            named = [(n, p.grad) for n, p in ref.named_parameters() if p.grad is not None]
            out['grad_transFuser_names'] = np.array([n for n, _ in named])
            out['grad_transFuser_norms'] = np.array([float(g.double().norm()) for _, g in named])
    for backbone in ('geometric_fusion', 'latentTF'):
        try:
            reference(m, backbone)
            raised = ''
        except Exception as e:          # noqa: BLE001 (the type is the datum)
            raised = type(e).__name__
        out['raises_%s' % backbone] = np.array(raised)
    np.savez_compressed(GOLD, **out)
    print('wrote %s (%d bytes, %d arrays)' % (GOLD, os.path.getsize(GOLD), len(out)))


if __name__ == '__main__':
    main()
