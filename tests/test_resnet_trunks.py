"""The ResNet-18 / ResNet-34 trunks (the reference's default image / LiDAR trunks, model.py:545) on the CPU: the timm restatement
(oracle/timm_resnet.py) against torchvision, the product's parameter tree and the CPU oracle against tests/golden/reference_resnet.npz (made by running the
verbatim reference, oracle/make_golden_resnet.py), and the trunk combinations that must keep raising."""
import os

import numpy as np
import pytest
import torch

from oracle import resnet_oracle as R, timm_resnet, torch_oracle as O
from transfuser_b200 import LidarCenterNet
from transfuser_b200.config import TrainConfig

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_resnet.npz'))
TRUNKS = tuple(GOLD['trunks'])
LOSS_CASES = {'transFuser': (31, 32), 'late_fusion': (33, 34)}       # (weight seed, batch seed), as oracle/make_golden_resnet.py


def _state(backbone):
    net = LidarCenterNet(TrainConfig(), 'cpu', backbone, *TRUNKS, use_velocity=False)
    return net, {k: v for k, v in net.state_dict().items() if not k.startswith('_bev')}


@pytest.mark.parametrize('name', ['resnet18', 'resnet34'])
def test_timm_shim_matches_torchvision(name):
    """torchvision and timm name the BasicBlock ResNet parameters alike (conv1, bn1, layer{i}.{k}.{conv1,bn1,conv2,bn2,downsample})."""
    import torchvision
    timm = timm_resnet
    shim = timm.create_model(name)
    tv = getattr(torchvision.models, name)(weights=None)
    a = [(n, tuple(p.shape)) for n, p in shim.named_parameters()]
    b = [(n, tuple(p.shape)) for n, p in tv.named_parameters()]
    assert a == b
    assert sum(p.numel() for p in shim.parameters()) == sum(p.numel() for p in tv.parameters())
    assert [f['num_chs'] for f in shim.feature_info] == [64, 64, 128, 256, 512] and shim.num_features == 512
    x = torch.randn(1, 3, 64, 96)
    assert shim(x).shape == (1, 1000)
    assert timm.create_model(name, in_chans=3).conv1.in_channels == 3 and timm.create_model(name, in_chans=5).conv1.in_channels == 5


@pytest.mark.parametrize('backbone', ['transFuser', 'late_fusion'])
def test_state_dict_matches_reference(backbone):
    net, sd = _state(backbone)
    assert list(sd) == list(GOLD['sd_%s_keys' % backbone])
    assert ['x'.join(map(str, v.shape)) for v in sd.values()] == list(GOLD['sd_%s_shapes' % backbone])
    other, _ = _state(backbone)
    other.load_state_dict(net.state_dict(), strict=True)
    trunk = net._model.image_encoder._net if backbone == 'late_fusion' else net._model.image_encoder.features
    assert [f['num_chs'] for f in trunk.feature_info] == [64, 64, 128, 256, 512] and trunk.num_features == 512
    # timm init: zero last BatchNorm scale of every BasicBlock
    assert float(trunk.layer1.get_submodule("0").bn2.weight.abs().sum()) == 0.0


def test_default_arguments_build_resnet_trunks():
    net = LidarCenterNet(TrainConfig(), 'cpu', 'transFuser')
    m = net._model
    assert m.image_encoder.features.conv1.weight.shape == (64, 3, 7, 7)
    assert m.lidar_encoder._model.conv1.weight.shape == (64, 3, 7, 7)
    assert len(list(m.image_encoder.features.layer3.children())) == 6 and len(list(m.lidar_encoder._model.layer3.children())) == 2
    assert isinstance(m.change_channel_conv_image, torch.nn.Sequential) and not list(m.change_channel_conv_image.parameters())


@pytest.mark.parametrize('backbone', ['geometric_fusion', 'latentTF'])
def test_stemless_lidar_encoders_raise(backbone):
    """The reference deletes the LiDAR trunk's `stem`, which a timm ResNet does not have: it fails, and so does the product."""
    assert str(GOLD['raises_%s' % backbone]) == 'AttributeError'
    with pytest.raises(RuntimeError, match='geometric_fusion.py:404'):
        LidarCenterNet(TrainConfig(), 'cpu', backbone, *TRUNKS, use_velocity=False)


@pytest.mark.parametrize('backbone', ['transFuser', 'late_fusion', 'geometric_fusion'])
@pytest.mark.parametrize('trunks,match', [(('regnety_032', 'resnet18'), 'cannot be combined'), (('resnet34', 'regnety_032'), 'cannot be combined'),
                                          (('resnet50', 'resnet50'), 'Bottleneck'), (('resnet34', 'resnet26'), 'Bottleneck'),
                                          (('convnext_tiny', 'convnext_tiny'), 'ConvNeXt')])
def test_unsupported_trunks_raise(backbone, trunks, match):
    with pytest.raises(RuntimeError, match=match):
        LidarCenterNet(TrainConfig(), 'cpu', backbone, *trunks, use_velocity=False)


def _fixture_state(backbone, seed):
    names = [(k, tuple(int(d) for d in s.split('x')) if s else ()) for k, s in zip(GOLD['sd_%s_keys' % backbone], GOLD['sd_%s_shapes' % backbone])]
    P = O.deterministic_state(names, seed=seed)
    for k, v in P.items():
        if v.dtype.is_floating_point and 'running' not in k:
            v.requires_grad_()
    return P


@pytest.mark.parametrize('backbone', list(LOSS_CASES))
def test_oracle_matches_reference(backbone):
    """The CPU oracle's ResNet trunks (oracle/resnet_oracle.py) reproduce the reference's losses (and, for transFuser, its parameter-gradient norms)."""
    wseed, bseed = LOSS_CASES[backbone]
    P = _fixture_state(backbone, wseed)
    losses = R.forward(P, O.synthetic_batch(1, seed=bseed), TRUNKS, O.Cfg, train=True, backbone_name=backbone)
    want = dict(zip(GOLD['loss_%s_names' % backbone], GOLD['loss_%s' % backbone]))
    assert list(losses) == list(want)
    for k, v in want.items():
        assert abs(float(losses[k]) - v) <= 1e-6 * max(abs(v), 1e-6), (k, float(losses[k]), v)
    if backbone != 'transFuser':
        return
    c = TrainConfig()
    w = dict(zip(c.detailed_losses, c.detailed_losses_weights))
    sum(w[k] * losses[k] for k in losses).backward()
    names = list(GOLD['grad_transFuser_names'])
    assert len(names) > 400
    for n, gn in zip(names, GOLD['grad_transFuser_norms']):
        if n.endswith('attn.key.bias'):
            continue            # the true gradient is identically zero (softmax shift invariance): both sides are rounding noise
        assert abs(float(P[n].grad.double().norm()) - gn) <= 1e-3 * gn, (n, float(P[n].grad.norm()), gn)
