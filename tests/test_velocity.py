"""use_velocity=True (the ego-speed input) on every backbone, checked without a GPU:
- the state_dict contract of the verbatim reference with velocity (tests/golden/reference_velocity.npz, oracle/make_golden_velocity.py);
- the modules' host wiring in float64 with torch stand-ins for the kernels (as tests/test_host_logic.py does) against the reference's
  backbone outputs and forward_ego waypoints, and the oracle's velocity terms against the reference's losses and vel_emb* gradients;
- tfb_vel_emb_add / tfb_vel_emb_bwd through the CPU emulation of their CUDA source, against the formula and summation order the
  header states."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import torch_oracle as O
from oracle import velocity_oracle as VO
from oracle.make_golden_reference import sample_index
from oracle.make_golden_velocity import BATCH_SEED, GOLD, WEIGHT_SEED
from test_host_logic import fp64, torch_ops  # noqa: F401  (fixtures)

BACKBONES = ('transFuser', 'late_fusion', 'geometric_fusion', 'latentTF')


def _gold():
    return np.load(GOLD)


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def _net(backbone):
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    return LidarCenterNet(TrainConfig(embd_pdrop=0.0, attn_pdrop=0.0, resid_pdrop=0.0), 'cpu', backbone, 'regnety_032', 'regnety_032',
                          use_velocity=True)


def _reference_names(backbone):
    g = _gold()
    return [(str(n), tuple(int(d) for d in str(s).split('x') if d)) for n, s in zip(g['sd_%s_keys' % backbone], g['sd_%s_shapes' % backbone])]


@pytest.mark.parametrize('backbone', BACKBONES)
def test_state_dict_matches_reference_with_velocity(backbone):
    """Keys, order and shapes equal the reference's with use_velocity=True; a reference-shaped state dict loads strictly."""
    net = _net(backbone)
    names = _reference_names(backbone)
    assert [(k, tuple(v.shape)) for k, v in net.state_dict().items()] == names
    assert any('vel_emb' in n for n, _ in names)
    net.load_state_dict(O.deterministic_state(names, seed=3), strict=True)


@pytest.mark.parametrize('backbone', BACKBONES)
def test_default_construction_builds(backbone):
    """LidarCenterNet's default is use_velocity=True (model.py:545), as the reference's; geometric_fusion and latentTF are built
    with RegNet trunks, the only ones their LiDAR encoders accept."""
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    trunks = ('regnety_032', 'regnety_032') if backbone in ('geometric_fusion', 'latentTF') else ()
    net = LidarCenterNet(TrainConfig(), 'cpu', backbone, *trunks)
    assert any('vel_emb' in n for n, _ in net.named_parameters())


@pytest.fixture
def vel_torch_ops(torch_ops, monkeypatch):
    """torch_ops plus a torch stand-in for the speed-embedding node."""
    def vel_emb_add(velocity, emb, *xs):
        e = F.linear(velocity.reshape(-1, 1), emb.weight, emb.bias)
        ys = tuple(x + e.view((e.shape[0],) + (1,) * (x.dim() - 2) + (e.shape[1],)) for x in xs)
        return ys[0] if len(ys) == 1 else ys
    monkeypatch.setattr(torch_ops, 'vel_emb_add', vel_emb_add)
    return torch_ops


def _seeded(backbone):
    net = _net(backbone)
    own = [(n, tuple(p.shape)) for n, p in list(net.named_parameters()) + list(net.named_buffers()) if not n.startswith('_bev')]
    net.load_state_dict(O.deterministic_state(own, seed=WEIGHT_SEED), strict=False)
    return net.double()


def _batch(B, seed, backbone):
    b = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in O.synthetic_batch(B, seed=seed).items()}
    if backbone == 'geometric_fusion':
        b['bev_points'], b['cam_points'] = O.synthetic_correspondences(B, seed=seed)
    return b


@pytest.mark.parametrize('backbone', BACKBONES)
@pytest.mark.parametrize('train', [True, False])
def test_backbone_outputs_match_reference(vel_torch_ops, fp64, backbone, train):
    """The product module (host wiring, kernels replaced by torch) and the oracle equal the verbatim reference's backbone outputs
    within 1e-9 relative; a speed 3 m/s higher moves the fused vector."""
    g = _gold()
    net = _seeded(backbone).train(train)
    b = _batch(2, BATCH_SEED, backbone)
    lidar = torch.cat((b['lidar'], b['target_point_image']), dim=1)
    geo = (b['bev_points'], b['cam_points']) if backbone == 'geometric_fusion' else ()
    P = {k: v.clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        mine = net._model(b['rgb'], lidar.clone(), b['ego_vel'], *geo)
        faster = net._model(b['rgb'], lidar.clone(), b['ego_vel'] + 3.0, *geo)
        oracle = VO.run_backbone(P, b, O.Cfg, train, None, None, backbone)
    mine = list(mine[0]) + [mine[1], mine[2]]
    faster = list(faster[0]) + [faster[1], faster[2]]
    oracle = list(oracle[0]) + [oracle[1], oracle[2]]
    for i, (x, y) in enumerate(zip(mine, oracle)):
        key = '%s_out_%d_%d' % (backbone, train, i)
        assert tuple(x.shape) == tuple(g[key + '_shape']), (i, x.shape)
        want = torch.from_numpy(g[key + '_sample'])
        for name, t in (('module', x), ('oracle', y)):
            f = t.double().reshape(-1)
            got = f[torch.from_numpy(sample_index(f.numel()))]
            assert _rel(got, want) < 1e-9, (name, i, _rel(got, want))
            assert abs(f.norm().item() - float(g[key + '_norm'][0])) <= 1e-9 * float(g[key + '_norm'][0]), (name, i)
    assert _rel(faster[-1], mine[-1]) > 1e-6         # the fused vector: every backbone adds the embedding upstream of it


@pytest.mark.parametrize('backbone', BACKBONES)
def test_forward_ego_matches_reference(vel_torch_ops, fp64, backbone):
    g = _gold()
    net = _seeded(backbone).eval()
    b = _batch(1, BATCH_SEED + 2, backbone)
    kw = dict(bev_points=b['bev_points'], cam_points=b['cam_points']) if backbone == 'geometric_fusion' else {}
    wp, _ = net.forward_ego(b['rgb'], b['lidar'], b['target_point'], b['target_point_image'], b['ego_vel'], **kw)
    assert _rel(wp, torch.from_numpy(g['%s_ego_wp' % backbone])) < 1e-9


@pytest.mark.parametrize('backbone', BACKBONES)
def test_oracle_losses_and_velocity_gradients_match_reference(backbone):
    """velocity_oracle.forward (float32, as the reference's whole-model forward runs) against the reference's
    11 losses and vel_emb* gradients on the same weights and batch."""
    from transfuser_b200.config import TrainConfig
    g = _gold()
    net = _net(backbone)
    own = [(n, tuple(p.shape)) for n, p in list(net.named_parameters()) + list(net.named_buffers()) if not n.startswith('_bev')]
    P = {k: v.clone().requires_grad_(v.dtype.is_floating_point and 'running' not in k)
         for k, v in O.deterministic_state(own, seed=WEIGHT_SEED).items()}
    b = {k: v.float() if v.dtype.is_floating_point else v for k, v in _batch(2, BATCH_SEED + 1, backbone).items()}

    class C(O.Cfg):
        embd_pdrop = attn_pdrop = resid_pdrop = 0.0
    loss = VO.forward(P, b, C, train=True, backbone_name=backbone)
    assert list(loss) == [str(n) for n in g['%s_loss_names' % backbone]]
    for k, want in zip(loss, g['%s_losses' % backbone]):
        assert abs(loss[k].item() - want) <= 1e-3 * max(abs(want), 1e-3), (k, loss[k].item(), want)
    cfg = TrainConfig()
    w = dict(zip(cfg.detailed_losses, cfg.detailed_losses_weights))
    sum(w[k] * v for k, v in loss.items()).backward()
    names = [str(n) for n in g['%s_grad_names' % backbone]]
    assert names == [n for n in P if '.vel_emb' in n] and names
    for n in names:
        # float32 on both sides, batch 2 through train-mode BatchNorms: the scale-1 embedding of geometric fusion differs by 1.7 %.
        # Geometric fusion's scales 1-3 feed a train-mode BatchNorm, which removes a per-channel constant, so their bias gradient is
        # 0 in real arithmetic: it is held to the scale of the per-sample sums, |dW| / max |v|, instead of its own norm
        want = torch.from_numpy(g['%s_grad_%s' % (backbone, n)])
        scale = want.norm().item()
        if n.endswith('.bias'):
            ref_w = torch.from_numpy(g['%s_grad_%sweight' % (backbone, n[:-len('bias')])])
            scale = max(scale, ref_w.norm().item() / b['ego_vel'].abs().max().item())
        assert (P[n].grad.double() - want).norm().item() < 5e-2 * scale, (n, _rel(P[n].grad, want))


# ------------------------------------------------------------------ the kernels through the CPU emulation
VROWS = 16        # thread rows of tfb_vel_emb_bwd: the partial sums over t = r, r + 16, ... (see the header)

KERNEL_CASES = [((1,), 72, 1), ((174,), 1512, 10), ((110,), 216, 12), ((64,), 512, 10), ((1,), 576, 12),
                ((64, 110), 576, 12), ((64, 110), 72, 1), ((1, 174), 216, 10), ((110, 64), 1512, 12), ((174, 1), 512, 1)]


def _inputs(Ts, C, B, seed):
    """Speeds with at most 16 significant bits, so that v * w + bias is exact in float64 and one rounding to float32 is the
    header's fmaf (the float64 sum is checked to be exact below)."""
    rng = np.random.default_rng(seed)
    v = (np.round(rng.uniform(0, 12, B) * 4096) / 4096).astype(np.float32)
    w = (rng.standard_normal(C) * 0.3).astype(np.float32)
    bias = (rng.standard_normal(C) * 0.1).astype(np.float32)
    xs = [rng.standard_normal((B, T, C)).astype(np.float32) for T in Ts]
    return v, w, bias, xs


def _embedding(v, w, bias):
    p = v.astype(np.float64)[:, None] * w.astype(np.float64)[None, :]          # exact: 24 x 16 significant bits
    s = p + bias.astype(np.float64)[None, :]
    assert np.array_equal(s - p, np.broadcast_to(bias.astype(np.float64), s.shape)) and np.array_equal(s - bias.astype(np.float64), p)
    return s.astype(np.float32)                                                 # one rounding of the exact value: fmaf


def _emul():
    from cuda_emul import loader
    return loader.emul()


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


@pytest.mark.parametrize('Ts,C,B', KERNEL_CASES)
def test_vel_emb_add_emulated_equals_formula(Ts, C, B):
    lib = _emul()
    v, w, bias, xs = _inputs(Ts, C, B, seed=C + B + sum(Ts))
    e = _embedding(v, w, bias)
    ys = [torch.full(x.shape, float('nan')) for x in xs]
    x1, y1, T1 = (_t(xs[1]), ys[1], Ts[1]) if len(Ts) == 2 else (None, None, 0)
    lib.call('tfb_vel_emb_add', _t(v), _t(w), _t(bias), _t(xs[0]), ys[0], Ts[0], x1, y1, T1, B, C)
    for x, y in zip(xs, ys):
        want = x + e[:, None, :]                                                 # float32 add
        assert np.array_equal(y.numpy().view(np.int32), want.view(np.int32))


def _bwd_order(v, dys):
    """tfb_vel_emb_bwd's summation order (include/tfb200.h), in float32: returns (dw, dbias); dw's fmaf taken in float64
    then rounded (double rounding: checked against a bound, not bit for bit)."""
    B, C = dys[0].shape[0], dys[0].shape[2]
    f = np.float32
    db = np.zeros(C, f)
    dw = np.zeros(C, f)
    for b in range(B):
        S = []
        for d in dys:
            parts = []
            for r in range(VROWS):
                p = np.zeros(C, f)
                for t in range(r, d.shape[1], VROWS):
                    p = (p + d[b, t]).astype(f)
                parts.append(p)
            s = np.zeros(C, f)
            for p in parts:
                s = (s + p).astype(f)
            S.append(s)
        s = S[0] if len(S) == 1 else (S[0] + S[1]).astype(f)
        db = (db + s).astype(f)
        dw = (v[b].astype(np.float64) * s.astype(np.float64) + dw.astype(np.float64)).astype(f)
    return dw, db


@pytest.mark.parametrize('Ts,C,B', KERNEL_CASES)
def test_vel_emb_bwd_emulated_is_fixed_order_sum(Ts, C, B):
    lib = _emul()
    v, _, _, dys = _inputs(Ts, C, B, seed=7 * C + B)
    d1, T1 = (_t(dys[1]), Ts[1]) if len(Ts) == 2 else (None, 0)
    outs = []
    for _ in range(2):
        dw, db = torch.full((C, 1), float('nan')), torch.full((C,), float('nan'))
        lib.call('tfb_vel_emb_bwd', _t(v), _t(dys[0]), Ts[0], d1, T1, B, C, dw, db)
        outs.append((dw.numpy().reshape(-1).copy(), db.numpy().copy()))
    assert all(np.array_equal(a.view(np.int32), c.view(np.int32)) for a, c in zip(*outs))      # the same bits on every call
    dw, db = outs[0]
    want_dw, want_db = _bwd_order(v, dys)
    assert np.array_equal(db.view(np.int32), want_db.view(np.int32))                         # the header's order, bit for bit
    # within the fp32 accumulation bound of the float64 sums: n sequential roundings of partial sums of |terms|
    s64 = sum(d.astype(np.float64).sum(1) for d in dys)                                     # [B, C]
    a64 = sum(np.abs(d.astype(np.float64)).sum(1) for d in dys)
    n = max(Ts) // VROWS + 1 + VROWS + 2 + B
    eps = 2.0 ** -24
    assert np.all(np.abs(db - s64.sum(0)) <= n * eps * a64.sum(0))
    vw = v.astype(np.float64)[:, None]
    assert np.all(np.abs(dw - (vw * s64).sum(0)) <= (n + 1) * eps * (np.abs(vw) * a64).sum(0))
    assert np.all(np.abs(dw - want_dw) <= 2 * eps * (np.abs(vw) * a64).sum(0))


def test_vel_emb_entry_points_reject_bad_arguments():
    lib = _emul()
    x = torch.zeros(2, 3, 8)
    v, w, b = torch.zeros(2), torch.zeros(8), torch.zeros(8)
    with pytest.raises(RuntimeError):
        lib.call('tfb_vel_emb_add', v, w, b, x, torch.empty_like(x), 3, x, None, 3, 2, 8)      # second input without its output
    with pytest.raises(RuntimeError):
        lib.call('tfb_vel_emb_bwd', v, x, 3, None, 4, 2, 8, w, b)                              # T1 > 0 without dy1
