"""CPU: the oracle restatement (oracle/torch_oracle.py) against the committed fixtures produced by the VERBATIM reference
(tests/golden/model_golden.npz, tests/golden/reference_checks.npz: oracle/make_golden_model.py, oracle/make_golden_reference.py);
plus the structural cross-check of the timm shim against torchvision's RegNetY-3.2GF and the C-ABI export check."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import ref_import, torch_oracle as O
from oracle.make_golden_reference import GOLD as REF_GOLD

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'model_golden.npz')
REF = np.load(REF_GOLD)


def ref_names(key):
    """(name, shape) of every state_dict entry of the reference module `key` (oracle/make_golden_reference.py MODELS), in order."""
    return [(str(n), tuple(int(d) for d in str(s).split('x') if d)) for n, s in zip(REF['sd_%s_keys' % key], REF['sd_%s_shapes' % key])]


def assert_same_state_dict(mine, key):
    assert [(k, tuple(v.shape)) for k, v in mine.state_dict().items()] == ref_names(key)   # drop-in checkpoint contract


def assert_losses(got, key, tol, floor):
    names, want = REF['loss_%s_names' % key], REF['loss_%s' % key]
    assert [str(n) for n in names] == list(got.keys())
    for k, w in zip(names, want):
        assert abs(float(w) - float(got[str(k)])) <= tol * max(abs(float(w)), floor), (key, str(k), float(w), float(got[str(k)]))


def _product_container():
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    return LidarCenterNet(TrainConfig(), 'cpu', 'transFuser', 'regnety_032', 'regnety_032', use_velocity=False)


def test_oracle_reproduces_reference_golden():
    from oracle.make_golden_model import BATCH, BATCH_SEED, WEIGHT_SEED
    g = np.load(GOLD)
    net = _product_container()  # parameter names / shapes only (the product's forward needs the GPU)
    names = [(n, tuple(p.shape)) for n, p in list(net.named_parameters()) + list(net.named_buffers()) if not n.startswith('_bev')]
    st = O.deterministic_state(names, seed=WEIGHT_SEED)
    P = {k: v.clone().requires_grad_(v.dtype.is_floating_point and 'running' not in k) for k, v in st.items()}
    # alias keys of the reference state_dict are not needed by the oracle (it reads stem./s1../conv1 names)

    class C(O.Cfg):
        embd_pdrop = attn_pdrop = resid_pdrop = 0.0
    losses = O.forward(P, O.synthetic_batch(BATCH, seed=BATCH_SEED), C, train=True)
    assert list(losses.keys()) == list(g['loss_names'])
    for k, want in zip(g['loss_names'], g['losses']):
        assert abs(float(losses[k]) - want) <= 1e-5 * max(abs(want), 1e-6), (k, float(losses[k]), want)
    from transfuser_b200.config import TrainConfig
    w = dict(zip(TrainConfig.detailed_losses, TrainConfig.detailed_losses_weights))
    sum(w[k] * v for k, v in losses.items()).backward()
    for k, want in zip(g['grad_keys'], g['grad_norms']):
        assert abs(float(P[str(k)].grad.double().norm()) - want) <= 1e-3 * want, k
    assert np.allclose(P['_model.image_encoder.features.stem.bn.running_mean'].detach().numpy(), g['stem_running_mean'], rtol=1e-5, atol=1e-6)


def test_oracle_and_state_dict_match_verbatim_reference():
    from oracle.make_golden_model import WEIGHT_SEED
    mine = _product_container()
    assert_same_state_dict(mine, 'transFuser')
    P = O.deterministic_state(ref_names('transFuser'), seed=WEIGHT_SEED)
    mine.load_state_dict(P, strict=True)
    batch = O.synthetic_batch(1, seed=2)

    class C(O.Cfg):
        embd_pdrop = attn_pdrop = resid_pdrop = 0.0
    with torch.no_grad():
        got = O.forward(P, batch, C, train=True)
    assert_losses(got, 'transFuser', 1e-6, 1e-6)


def test_timm_shim_matches_torchvision_regnet_structure():
    """The un-vendored timm 0.5.4 `regnety_032` restatement has the stage widths / depths / group counts / SE sizes and the
    parameter count of torchvision's independent RegNetY-3.2GF definition."""
    import sys
    sys.path.insert(0, ref_import.SHIMS)
    import timm
    import torchvision
    shim = timm.create_model('regnety_032')
    tv = torchvision.models.regnet_y_3_2gf(weights=None)
    n_shim = sum(p.numel() for p in shim.parameters())
    n_tv = sum(p.numel() for p in tv.parameters())
    assert n_shim == n_tv, (n_shim, n_tv)
    shapes_shim = sorted(tuple(p.shape) for p in shim.parameters())
    shapes_tv = sorted(tuple(p.shape) for p in tv.parameters())
    assert shapes_shim == shapes_tv


def test_c_abi_library_exports_every_declared_symbol():
    from transfuser_b200 import _lib
    decls = _lib.parse_header()
    assert len(decls) >= 40
    cdll = ctypes.CDLL(_lib.LIB_PATH)
    missing = [n for n in decls if not hasattr(cdll, n)]
    assert not missing, missing
    assert cdll.tfb_abi_version() == 1


def test_late_fusion_oracle_and_state_dict_match_verbatim_reference():
    """BASELINE config 5 (late_fusion.py): drop-in key set of the product module + oracle restatement vs the reference."""
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    mine = LidarCenterNet(TrainConfig(), 'cpu', 'late_fusion', 'regnety_032', 'regnety_032', use_velocity=False)
    assert_same_state_dict(mine, 'late_fusion')
    P = O.deterministic_state(ref_names('late_fusion'), seed=6)
    batch = O.synthetic_batch(1, seed=4)
    with torch.no_grad():
        got = O.forward(P, batch, O.Cfg, train=True, backbone_name='late_fusion')
    assert_losses(got, 'late_fusion', 1e-6, 1e-6)


def test_geometric_fusion_oracle_matches_verbatim_reference():
    """BASELINE config 4 (geometric_fusion.py): oracle restatement vs the reference module, batch 2 so that the
    reference's B x B gather + diagonal (geometric_fusion.py:145-147) is exercised with distinct per-sample indices."""
    P = O.deterministic_state(ref_names('geometric_fusion'), seed=8)
    batch = O.synthetic_batch(2, seed=5)
    batch['bev_points'], batch['cam_points'] = O.synthetic_correspondences(2, seed=5)
    with torch.no_grad():
        got = O.forward(P, batch, O.Cfg, train=True, backbone_name='geometric_fusion')
    # fp32: the gather-sum adds the 5 correspondences in a different order than the reference's diagonal/permute/sum
    assert_losses(got, 'geometric_fusion', 1e-4, 1e-3)


def test_decode_heatmap_oracle_matches_reference_head():
    """model.py:376-497 (get_bboxes / decode_heatmap) on seeded maps with plateaus, saturated peaks and border maxima."""
    g = torch.Generator().manual_seed(21)
    for case in range(3):
        B = 2
        heat = torch.rand(B, 1, 64, 64, generator=g)
        if case == 1:
            heat = (heat * 8).round() / 8            # plateaus: equal neighbours are all kept by (hmax == heat)
        if case == 2:
            heat = heat * (heat > 0.995)             # fewer than k peaks: the tail of the top-k is zeros
        preds = [heat] + [torch.randn(B, c, 64, 64, generator=g) for c in (2, 2, 12, 1, 1, 2)]
        got_boxes, got_labels = O.decode_heatmap(preds, 12)
        for b in range(B):
            wb, wl = torch.from_numpy(REF['decode_%d_%d_boxes' % (case, b)]), torch.from_numpy(REF['decode_%d_%d_labels' % (case, b)])
            keep = wb[:, -1] > 0                     # rows with score 0 are an arbitrary choice among equal zeros
            if case != 1:                            # (ties between equal positive scores are ordered arbitrarily by topk)
                assert torch.equal(wb[keep], got_boxes[b][keep]) and torch.equal(wl[keep], got_labels[b][keep])
            else:
                assert torch.equal(wb[:, -1], got_boxes[b][:, -1])


def test_forward_ego_oracle_matches_verbatim_reference():
    """model.py:685-731 in eval mode (running-stat BN, no dropout): waypoints, decoded boxes, ego-frame box corners."""
    batch = O.synthetic_batch(1, seed=6)
    P = O.deterministic_state(ref_names('transFuser'), seed=9)
    with torch.no_grad():
        got_wp, got_boxes, raw = O.forward_ego(P, batch, O.Cfg)
    assert torch.allclose(torch.from_numpy(REF['ego_wp']), got_wp, rtol=1e-5, atol=1e-5)
    boxes = list(zip(REF['ego_boxes'], REF['ego_brake'], REF['ego_conf']))
    assert len(boxes) == len(got_boxes) and len(boxes) > 0, (len(boxes), len(got_boxes), float(raw[0, 0, -1]))
    for (a, abrake, aconf), (b, bbrake, bconf) in zip(boxes, got_boxes):
        assert np.allclose(a, b, rtol=1e-5, atol=1e-5) and abrake == bbrake and abs(aconf - bconf) < 1e-6


def test_latent_tf_oracle_matches_verbatim_reference():
    """latentTF.py (positional grid instead of the LiDAR histogram): the 11 training losses, eval mode for the dropouts."""
    P = O.deterministic_state(ref_names('latentTF'), seed=12)
    for mode in (True, False):        # the train-mode pass updates P's BatchNorm running statistics, as it does the reference's
        batch = O.synthetic_batch(2, seed=7)
        with torch.no_grad():
            got = O.forward(P, batch, O.Cfg, train=mode, backbone_name='latentTF')
        assert_losses(got, 'latentTF_%d' % mode, 1e-5, 1e-3)
