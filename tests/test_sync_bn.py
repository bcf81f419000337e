"""Synchronized BatchNorm without a GPU: the converted model's BatchNorm bookkeeping, and the sync kernels through the CPU emulation
of csrc/norm.cu for 1, 2, 3 and 8 simulated ranks with unequal row counts (tests/sync_bn_check.py)."""
import pytest
import torch

import sync_bn_check
from cuda_emul import loader


class _Stop(Exception):
    pass


@pytest.mark.parametrize('backbone', ['transFuser', 'late_fusion', 'geometric_fusion', 'latentTF'])
def test_convert_sync_batchnorm(backbone, monkeypatch):
    """convert_sync_batchnorm (train.py:133, submission_agent.py:92) keeps the state_dict keys and tensors; _bn_modules finds every
    BatchNorm once per counter, and the step's bookkeeping advances each num_batches_tracked exactly once; flat-buffer views stay."""
    from transfuser_b200 import ops, optim
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.model import LidarCenterNet
    net = LidarCenterNet(TrainConfig(), 'cpu', backbone, 'regnety_032', 'regnety_032').train()
    flat = optim.flatten(net)
    keys = list(net.state_dict())
    before = {k: v for k, v in net.state_dict().items()}
    net = torch.nn.SyncBatchNorm.convert_sync_batchnorm(net)
    assert list(net.state_dict()) == keys
    assert all(v is before[k] or v.data_ptr() == before[k].data_ptr() for k, v in net.state_dict().items())
    for p in net.parameters():                       # the converter reuses the Parameters: still views of the flat buffer
        assert p.data_ptr() >= flat.flat.data_ptr() and p.data_ptr() < flat.flat.data_ptr() + flat.flat.numel() * 4
    bb = net._model
    bns = [m for m in bb.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)]
    assert bns and all(isinstance(m, torch.nn.SyncBatchNorm) for m in bns)
    counters = {id(m.num_batches_tracked) for m in bns}
    found = bb._bn_modules()
    assert len(found) == len(counters) and {id(m.num_batches_tracked) for m in found} == counters
    # the training forward's first action: advance the counters, then the step tick (stopped there)
    monkeypatch.setattr(ops, 'tick', lambda dev: (_ for _ in ()).throw(_Stop()))
    cfg = net.config if hasattr(net, 'config') else TrainConfig()
    x, v = torch.zeros(1, 3, 8, 8), torch.zeros(1, 1)
    lidar = torch.zeros(1, 3, cfg.lidar_resolution_width, cfg.lidar_resolution_height)
    with pytest.raises(_Stop):
        if backbone == 'geometric_fusion':
            bb.forward_nhwc(x, lidar, None, None, velocity=v)
        else:
            bb.forward_nhwc(x, lidar, velocity=v)
    assert all(m.num_batches_tracked.item() == 1 for m in bns)


@pytest.mark.parametrize('world', [1, 2, 3, 8])
@pytest.mark.parametrize('variant', ['plain', 'relu', 'residual', 'pool'])
@pytest.mark.parametrize('from_stats', [0, 1])
def test_sync_kernels_emulated(world, variant, from_stats):
    lib = loader.emul()
    sync_bn_check.run(lib.call, 'cpu', world, variant, from_stats)


def test_sync_wide_channels_emulated():
    """C > 128 channel quads: the 2-D statistics / reduction grids rather than the flat ones."""
    lib = loader.emul()
    sync_bn_check.run(lib.call, 'cpu', 3, 'relu', 0, C=520, hw=2)
