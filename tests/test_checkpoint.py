"""Checkpoint compatibility (SURVEY.md §8f rank 3): the reference's model_%d.pth / optimizer_%d.pth formats
(train.py:179-183, 381-384; submission_agent.py:92-96) load into, and are produced by, the product classes. CPU only."""
import io

import numpy as np
import pytest
import torch
from torch import nn

from oracle import torch_oracle as O
from transfuser_b200 import checkpoint, optim


class _Tiny(nn.Module):
    def __init__(self):
        super().__init__()
        self.a = nn.Linear(5, 7)
        self.bn = nn.BatchNorm1d(7)
        self.b = nn.Linear(7, 3, bias=False)
        self.alias = self.a            # registered twice, like the reference's s1 / layer1

    def forward(self, x):
        return self.b(self.bn(self.a(x))).sum()


def _adamw_reference_run(steps):
    torch.manual_seed(0)
    ref = _Tiny()
    opt = torch.optim.AdamW(ref.parameters(), lr=3e-3, weight_decay=0.02)
    for i in range(steps):
        opt.zero_grad()
        ref(torch.randn(4, 5)).backward()
        opt.step()
    return ref, opt


def test_optimizer_state_round_trip_with_torch_adamw():
    ref, opt = _adamw_reference_run(3)
    mine = _Tiny()
    mine.load_state_dict(ref.state_dict())
    fp = optim.flatten(mine)
    fused = optim.FusedAdamW(mine.parameters(), lr=1e-4)
    buf = io.BytesIO()
    torch.save(opt.state_dict(), buf)
    buf.seek(0)
    checkpoint.load_optimizer(fused, buf)
    assert fused._step == 3 and fused.param_groups[0]['lr'] == 3e-3 and fused.param_groups[0]['weight_decay'] == 0.02
    for i, (p, o) in enumerate(zip(fp.params, fp.offsets)):
        st = opt.state_dict()['state'][i]
        assert torch.equal(fused._m[o:o + p.numel()].view(p.shape), st['exp_avg'])
        assert torch.equal(fused._v[o:o + p.numel()].view(p.shape), st['exp_avg_sq'])
    # and back: torch.optim.AdamW resumes from what the fused optimizer writes
    again = torch.optim.AdamW(_Tiny().parameters(), lr=1.0)
    again.load_state_dict(fused.state_dict())
    a, b = again.state_dict(), opt.state_dict()
    assert a['param_groups'][0]['lr'] == 3e-3 and a['param_groups'][0]['params'] == b['param_groups'][0]['params']
    for i in b['state']:
        assert float(a['state'][i]['step']) == float(b['state'][i]['step'])
        assert torch.equal(a['state'][i]['exp_avg'], b['state'][i]['exp_avg']) and torch.equal(a['state'][i]['exp_avg_sq'], b['state'][i]['exp_avg_sq'])


def test_optimizer_state_rejects_mismatches():
    _, opt = _adamw_reference_run(1)
    mine = _Tiny()
    optim.flatten(mine)
    fused = optim.FusedAdamW(mine.parameters())
    sd = opt.state_dict()
    sd['state'][0]['step'] = torch.tensor(5.0)
    with pytest.raises(ValueError):
        fused.load_state_dict(sd)
    sd = opt.state_dict()
    sd['param_groups'][0]['params'] = sd['param_groups'][0]['params'][:-1]
    with pytest.raises(ValueError):
        fused.load_state_dict(sd)
    fresh = optim.FusedAdamW(mine.parameters())
    assert fresh.state_dict()['state'] == {}      # like torch before the first step


def test_model_checkpoint_prefix_aliases_and_flat_views():
    torch.manual_seed(1)
    src = _Tiny()
    sd = {'module.' + k: v for k, v in src.state_dict().items()}           # DDP-wrapped save (train.py:383)
    dst = _Tiny()
    fp = optim.flatten(dst)
    missing, unexpected = checkpoint.load_model(dst, sd)
    assert not missing and not unexpected
    for k, v in src.state_dict().items():
        assert torch.equal(dst.state_dict()[k], v)
    # parameters are still views of the flat buffer after the load (load_state_dict copies in place)
    for p, o in zip(fp.params, fp.offsets):
        assert p.data_ptr() == fp.flat.data_ptr() + 4 * o
    # a de-duplicated checkpoint (only one name per aliased tensor) is completed from the alias
    partial = {k: v for k, v in src.state_dict().items() if not k.startswith('alias.')}
    missing, unexpected = checkpoint.load_model(_Tiny(), partial)
    assert not missing and not unexpected
    # unprefixed keys that merely start with 'module' are left alone
    assert checkpoint.clean_state_dict({'module.a': 1, 'b': 2}) == {'module.a': 1, 'b': 2}
    buf = io.BytesIO()
    checkpoint.save_model(src, buf, module_prefix=True)
    buf.seek(0)
    assert all(k.startswith('module.') for k in torch.load(buf))


def test_reference_ddp_checkpoint_loads_strict_into_product_model():
    """A state dict with the verbatim reference module's keys and shapes (tests/golden/reference_checks.npz) and the DDP prefix,
    as models_2022.zip's files have, loads strict=True into the product module, and the agent's own loading code (k[7:],
    strict=False) finds every key it expects in what we save, and no other."""
    from oracle.make_golden_reference import GOLD
    g = np.load(GOLD)
    names = [(str(n), tuple(int(d) for d in str(s).split('x') if d)) for n, s in zip(g['sd_transFuser_keys'], g['sd_transFuser_shapes'])]
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    src = LidarCenterNet(TrainConfig(), 'cpu', 'transFuser', 'regnety_032', 'regnety_032', use_velocity=False)
    own = [(n, tuple(p.shape)) for n, p in list(src.named_parameters()) + list(src.named_buffers())]
    src.load_state_dict(O.deterministic_state(own, seed=2), strict=False)       # seeded by parameter name, aliases share the tensor
    ref_sd = {k: src.state_dict()[k] for k, _ in names}                          # the reference's keys, in its order
    mine = LidarCenterNet(TrainConfig(), 'cpu', 'transFuser', 'regnety_032', 'regnety_032', use_velocity=False)
    missing, unexpected = checkpoint.load_model(mine, {'module.' + k: v for k, v in ref_sd.items()}, strict=True)
    assert not missing and not unexpected
    a = mine.state_dict()
    assert all(torch.equal(a[k], v) for k, v in ref_sd.items())
    buf = io.BytesIO()
    checkpoint.save_model(mine, buf, module_prefix=True)
    buf.seek(0)
    state_dict = torch.load(buf)
    state_dict = {k[7:]: v for k, v in state_dict.items()}                  # submission_agent.py:95
    assert set(state_dict) == set(ref_sd) and all(tuple(state_dict[k].shape) == s for k, s in names)


def test_parameters_without_gradient_are_left_to_the_optimizer_untouched():
    """torch.optim.AdamW skips parameters whose .grad is None (config 4's lidar_conv4 never gets one): the fused optimizer's
    launch spans exclude them."""
    assert optim.subtract_spans(0, 1000, []) == [(0, 1000)]
    assert optim.subtract_spans(0, 1000, [(0, 64)]) == [(64, 1000)]
    assert optim.subtract_spans(0, 1000, [(128, 64), (960, 64)]) == [(0, 128), (192, 960)]
    assert optim.subtract_spans(512, 1024, [(128, 64), (448, 128), (1000, 64)]) == [(576, 1000)]
    assert optim.subtract_spans(0, 64, [(0, 64)]) == []
    net = _Tiny()
    fp = optim.flatten(net)
    net.b.weight.grad = torch.ones_like(net.b.weight)
    spans = fp.gather_stragglers()
    got = {o for o, _ in spans}
    want = {o for p, o in zip(fp.params, fp.offsets) if p is not net.b.weight}
    assert got == want and all(n % optim.ALIGN == 0 for _, n in spans)
