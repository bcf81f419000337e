"""use_velocity=True on the H100:
- tfb_vel_emb_add / tfb_vel_emb_bwd against the header's formula and summation order (the shapes of tests/test_velocity.py), on
  NaN-prefilled, sentinel-guarded outputs, repeated launches giving the same bits;
- every backbone with velocity: the 11 losses and the vel_emb* gradients against the CPU oracle (simt mode, tests/test_widen.py's
  bounds) and the losses against the bf16-operand oracle (bf16 mode, tests/test_bf16.py's bounds; gradients finite and non-zero);
- Trainer(use_velocity=True): a captured step equals its eager twin loss for loss and gradient for gradient, two captured trainers
  from one seed give the same bits, Validator replay equals its eager step; one raw_inputs='dataset' step equals its eager twin;
- forward_ego with velocity against the verbatim reference's waypoints (tests/golden/reference_velocity.npz)."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

if __name__ == '__main__':          # _check_trainer in a process of its own (test_trainer_with_velocity_captured_equals_eager)
    sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__))), os.path.dirname(os.path.abspath(__file__))]

from oracle import torch_oracle as O  # noqa: E402
from oracle import velocity_oracle as VO  # noqa: E402
from test_correspondences_gpu import _batch as _dataset_batch, _raw, routes  # noqa: F401  (fixture)
from test_velocity import BACKBONES, KERNEL_CASES, WEIGHT_SEED, BATCH_SEED, _bwd_order, _embedding, _gold, _inputs

pytestmark = pytest.mark.gpu
SENTINEL = 12345.0
PAD = 64


@pytest.fixture(autouse=True)
def _release_device_memory():
    """Trainers, captured graphs and validators form reference cycles: collect them after each test, so that the trainers of
    four backbones do not pile up on the device over the module."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _guarded(shape):
    """A NaN-filled view of `shape` inside a sentinel-filled buffer (PAD floats on each side)."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * PAD,), SENTINEL, device='cuda')
    view = buf[PAD:PAD + n].view(shape)
    view.fill_(float('nan'))
    return buf, view


def _intact(buf, n):
    return bool((buf[:PAD] == SENTINEL).all()) and bool((buf[PAD + n:] == SENTINEL).all())


def _bits(t):
    return t.detach().float().contiguous().cpu().numpy().view(np.int32)


@pytest.mark.parametrize('Ts,C,B', KERNEL_CASES)
def test_vel_emb_kernels_match_header_formula(Ts, C, B):
    from transfuser_b200 import _lib
    v, w, bias, xs = _inputs(Ts, C, B, seed=C + B + sum(Ts))
    e = _embedding(v, w, bias)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    outs = []
    for _ in range(2):
        guarded = [_guarded(x.shape) for x in xs]
        x1, y1, T1 = (cu(xs[1]), guarded[1][1], Ts[1]) if len(Ts) == 2 else (None, None, 0)
        _lib.call('tfb_vel_emb_add', cu(v), cu(w), cu(bias), cu(xs[0]), guarded[0][1], Ts[0], x1, y1, T1, B, C)
        torch.cuda.synchronize()
        assert all(_intact(buf, x.size) for (buf, _), x in zip(guarded, xs))
        outs.append([_bits(y) for _, y in guarded])
    for k, x in enumerate(xs):
        assert np.array_equal(outs[0][k], (x + e[:, None, :]).view(np.int32)), k
        assert np.array_equal(outs[0][k], outs[1][k])

    _, _, _, dys = _inputs(Ts, C, B, seed=7 * C + B)
    grads = []
    for _ in range(3):
        (bw, dw), (bb, db) = _guarded((C, 1)), _guarded((C,))
        d1, T1 = (cu(dys[1]), Ts[1]) if len(Ts) == 2 else (None, 0)
        _lib.call('tfb_vel_emb_bwd', cu(v), cu(dys[0]), Ts[0], d1, T1, B, C, dw, db)
        torch.cuda.synchronize()
        assert _intact(bw, C) and _intact(bb, C)
        grads.append((_bits(dw).reshape(-1), _bits(db)))
    assert all(np.array_equal(a, c) for g in grads[1:] for a, c in zip(grads[0], g))
    want_dw, want_db = _bwd_order(v, dys)
    assert np.array_equal(grads[0][1], want_db.view(np.int32))
    dwf = grads[0][0].view(np.float32)
    eps = 2.0 ** -24
    scale = (np.abs(v.astype(np.float64))[:, None] * sum(np.abs(d.astype(np.float64)).sum(1) for d in dys)).sum(0)
    assert np.all(np.abs(dwf - want_dw) <= 2 * eps * scale)


def _seeded_net(backbone, dev='cpu'):
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig

    class C(TrainConfig):
        embd_pdrop = attn_pdrop = resid_pdrop = 0.0
    net = LidarCenterNet(C, dev, backbone, 'regnety_032', 'regnety_032', use_velocity=True)
    names = [(n, tuple(p.shape)) for n, p in list(net.named_parameters()) + list(net.named_buffers()) if not n.startswith('_bev')]
    net.load_state_dict(O.deterministic_state(names, seed=WEIGHT_SEED), strict=False)
    return net, C


def _host_batch(B, seed, backbone):
    b = O.synthetic_batch(B, seed=seed)
    if backbone == 'geometric_fusion':
        b['bev_points'], b['cam_points'] = O.synthetic_correspondences(B, seed=seed)
    return b


def _losses(net, cb):
    return net(cb['rgb'], cb['lidar'], ego_waypoint=cb['ego_waypoint'], target_point=cb['target_point'],
               target_point_image=cb['target_point_image'], ego_vel=cb['ego_vel'], bev=cb['bev'], label=cb['label'],
               depth=cb['depth'], semantic=cb['semantic'], bev_points=cb.get('bev_points'), cam_points=cb.get('cam_points'))


@pytest.mark.parametrize('backbone', BACKBONES)
def test_model_with_velocity_matches_oracle(backbone):
    from transfuser_b200 import gemm

    class OC(O.Cfg):
        embd_pdrop = attn_pdrop = resid_pdrop = 0.0
    net, C = _seeded_net(backbone)
    batch = _host_batch(2, BATCH_SEED + 1, backbone)
    w = dict(zip(C.detailed_losses, C.detailed_losses_weights))
    P = {k: v.clone().requires_grad_(v.dtype.is_floating_point and 'running' not in k) for k, v in net.state_dict().items()}
    ref = VO.forward(P, batch, OC, train=True, backbone_name=backbone)
    sum(w[k] * ref[k] for k in ref).backward()
    Pq = {k: v.detach().clone() for k, v in P.items()}
    O.BF16_OPERANDS[0] = True
    try:
        with torch.no_grad():
            ref16 = VO.forward(Pq, batch, OC, train=True, backbone_name=backbone)
    finally:
        O.BF16_OPERANDS[0] = False
    cb = {k: v.cuda() for k, v in batch.items()}
    vel_names = [n for n, _ in net.named_parameters() if '.vel_emb' in n]
    assert vel_names
    for mode in ('simt', 'bf16'):
        gemm.set_mode(mode)
        m, _ = _seeded_net(backbone)
        m = m.cuda().train()
        out = _losses(m, cb)
        want = ref if mode == 'simt' else ref16
        for k in want:
            a, b = out[k].item(), want[k].item()
            # bf16: tests/test_bf16.py's 5 %, except the SmoothL1 yaw residual over a handful of pixels, which one flipped bf16
            # rounding upstream moves by 5-20 % (smoke() bounds it at 35 %; geometric fusion measured 5.8 % here)
            bound = (1e-3 * max(abs(b), 1e-6) if mode == 'simt' else
                     0.35 * abs(b) if k == 'loss_yaw_res' else 5e-2 * max(abs(b), 0.1))
            assert abs(a - b) <= bound, (mode, k, a, b)
        sum(w[k] * out[k] for k in out).backward()
        named = dict(m.named_parameters())
        for n in vel_names:
            g = named[n].grad
            assert bool(torch.isfinite(g).all()) and float(g.abs().sum()) > 0, (mode, n)
            e = _rel(g, P[n].grad)
            print('%s %s %s: grad rel err vs fp32 oracle %.2e' % (backbone, mode, n, e))
            # simt: tests/test_widen.py's gradient bound (measured 0.5-1.7 % at batch 2). bf16: the oracle restates the forward
            # rounding only, and these sums over every token / pixel cancel: transformer1's moved 140 % from the fp32 oracle's
            # In geometric fusion scales 1-3 feed a train-mode BatchNorm, which removes a per-channel constant: the bias gradient is 0
            # in real arithmetic there, so it is held to the scale of the per-sample sums, |dW| / max |v|, instead of its own norm
            if mode == 'simt':
                if n.endswith('.bias'):
                    ref_w = P[n[:-len('bias')] + 'weight'].grad
                    scale = max(P[n].grad.norm().item(), ref_w.norm().item() / batch['ego_vel'].abs().max().item())
                    assert (g.double().cpu() - P[n].grad.double()).norm().item() < 5e-2 * scale, (mode, n, e)
                else:
                    assert e < 5e-2, (mode, n, e)
        del m
    gemm.set_mode('simt')


def _trainer(backbone, raw_inputs=False):
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    torch.manual_seed(0)
    return Trainer(TrainConfig(), torch.device('cuda', 0), gemm_mode='bf16', seed=0, backbone=backbone, raw_inputs=raw_inputs,
                   use_velocity=True)


def _state(tr):
    return torch.stack(list(tr.last_losses.values())).detach().clone(), tr.flat.grad.detach().clone(), tr.flat.flat.detach().clone()


def _same_bits(a, b):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))


@pytest.mark.parametrize('backbone', BACKBONES)
def test_trainer_with_velocity_captured_equals_eager(backbone):
    """Runs _check_trainer in a fresh process: three full trainers and a validator per backbone would otherwise stay resident on
    the device for the rest of the session."""
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), backbone], cwd=os.path.dirname(here), capture_output=True, text=True,
                       timeout=1200)
    print(r.stdout[-2000:], r.stderr[-4000:])
    assert r.returncode == 0 and 'TRAINER OK' in r.stdout


def _check_trainer(backbone):
    from bench import make_host_batch
    from transfuser_b200.trainer import Validator
    host = make_host_batch(2, seed=5, torch=torch, np=np, backbone=backbone)
    runs = []
    for captured in (True, True, False):
        tr = _trainer(backbone)
        if captured:
            assert tr.capture(host), tr.graph_error          # two eager warm-up steps inside
            tr.replay()
        else:
            d = {k: v.cuda() for k, v in host.items()}
            for _ in range(3):
                tr.step(d)
        torch.cuda.synchronize()
        runs.append(_state(tr))
        if captured and len(runs) == 1:
            vel = [p for n, p in tr.net.named_parameters() if '.vel_emb' in n]
            assert vel and all(float(p.grad.abs().sum()) > 0 for p in vel)
            val = Validator(tr)
            assert val.capture(host)
            val.replay()
            torch.cuda.synchronize()
            replayed = {k: v.clone() for k, v in val.static_losses.items()}
            eager = val.step(host)
            torch.cuda.synchronize()
            assert list(replayed) == list(eager)
            for k in eager:
                assert torch.equal(replayed[k].view(torch.int32), eager[k].view(torch.int32)), k
            del val, replayed, eager
        del tr
        gc.collect()
    assert _same_bits(runs[0], runs[1])               # two captured trainers from one seed
    assert _same_bits(runs[0], runs[2])               # captured = eager, loss for loss and gradient for gradient
    assert all(np.isfinite(runs[0][0].cpu().numpy()))
    print('TRAINER OK')


def test_dataset_step_with_velocity_equals_eager_twin(routes, monkeypatch):
    """A captured Trainer(raw_inputs='dataset', use_velocity=True) step against three eager steps of the expanded-input trainer fed
    the pipeline's outputs of the same batch (its ego_vel [B, 1] included): the 11 losses are equal bit for bit."""
    from transfuser_b200 import pipeline, trainer as trainer_mod
    from transfuser_b200.config import TrainConfig
    b, _ = _dataset_batch(routes, idx=[0, 3])
    assert tuple(b['ego_vel'].shape) == (2, 1)
    tr = _trainer('geometric_fusion', 'dataset')
    assert tr.capture(b), tr.graph_error
    tr.replay()
    torch.cuda.synchronize()
    got = torch.stack(list(tr.last_losses.values())).clone()
    del tr
    p = pipeline.InputPipeline(TrainConfig(), 'cuda').prepare({k: v.cuda() for k, v in _raw(b).items()})
    d = dict(rgb=p['rgb'], points=b['points'].cuda(), target_point_image=p['target_point_image'], target_point=p['target_point'],
             ego_vel=b['ego_vel'].cuda(), ego_waypoint=b['ego_waypoint'].cuda(), bev=p['bev'], semantic=p['semantic'], depth=p['depth'],
             label=b['label'].cuda(), bev_points=p['bev_points'], cam_points=p['cam_points'])
    monkeypatch.setattr(trainer_mod.bev, 'lidar_to_histogram_features_batched', lambda pts: p['lidar'])
    tr = _trainer('geometric_fusion')
    for _ in range(3):
        tr.step(d)
    torch.cuda.synchronize()
    want = torch.stack(list(tr.last_losses.values()))
    assert got.shape == (11,) and torch.equal(got.view(torch.int32), want.view(torch.int32))
    assert bool(torch.isfinite(got).all())


@pytest.mark.parametrize('backbone', BACKBONES)
def test_forward_ego_with_velocity_matches_reference(backbone):
    """The fixture's weights and batch were drawn with float64 as the default dtype (the seeded draws depend on it): drawn the
    same way here, then run in float32."""
    g = _gold()
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        net, _ = _seeded_net(backbone)
        host = _host_batch(1, BATCH_SEED + 2, backbone)
    finally:
        torch.set_default_dtype(old)
    net = net.float().cuda().eval()
    b = {k: (v.float() if v.dtype.is_floating_point else v).cuda() for k, v in host.items()}
    kw = dict(bev_points=b['bev_points'], cam_points=b['cam_points']) if backbone == 'geometric_fusion' else {}
    wp, _ = net.forward_ego(b['rgb'], b['lidar'], b['target_point'], b['target_point_image'], b['ego_vel'], **kw)
    assert _rel(wp, torch.from_numpy(g['%s_ego_wp' % backbone])) < 1e-3


if __name__ == '__main__':
    _check_trainer(sys.argv[1])
