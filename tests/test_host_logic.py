"""Host-side wiring of the product modules, checked WITHOUT a GPU: every `transfuser_b200.ops` entry the modules call is
replaced, for the duration of one test, by a plain fp32 torch stand-in with the same NHWC contract, and the module's output is
compared with the oracle. This exercises exactly the Python that runs on the GPU box (parameter names, scale loops, the
pool-before-embed / upsample-after-deconv reassociations, the scale-3/scale-4 quirk, the decode plumbing of forward_ego) —
the CUDA kernels themselves are covered by the `-m gpu` tests. Nothing here is importable by the product."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import torch_oracle as O


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


@pytest.fixture
def torch_ops(monkeypatch):
    from transfuser_b200 import ops

    def conv2d(x, w, bias=None, stride=1, groups=1, relu=False, bn_stats=False):      # bn_stats: epilogue-statistics hint
        y = F.conv2d(_nchw(x), w, bias, stride=stride, padding=w.shape[2] // 2, groups=groups)
        return _nhwc(F.relu(y) if relu else y)

    def batch_norm(x, bn, relu, training, emit16=False, bwd16=False, residual=None, pool=False):    # emit16 / bwd16: bf16-sidecar hints
        y = F.batch_norm(_nchw(x), bn.running_mean, bn.running_var, bn.weight, bn.bias, training, bn.momentum, bn.eps)
        if residual is not None:
            y = y + _nchw(residual)               # the Bottleneck tail: relu(bn(x) + shortcut)
        return _nhwc(F.relu(y) if relu else y)

    def linear(x, w, bias=None, relu=False):
        y = F.linear(x, w.view(w.shape[0], -1), bias)
        return F.relu(y) if relu else y

    def gather_sum(emb, pts):
        B = emb.shape[0]
        rows = [emb[b][pts[b, ..., 1], pts[b, ..., 0]].sum(2) for b in range(B)]      # [H,W,5,C] -> [H,W,C]
        return torch.stack(rows)

    def se(x, w1, b1, w2, b2, emit16=False):
        s = x.mean((1, 2))
        s = torch.sigmoid(F.linear(F.relu(F.linear(s, w1.view(w1.shape[0], -1), b1)), w2.view(w2.shape[0], -1), b2))
        return x * s[:, None, None, :]

    def gru(z, tp, w_ih, w_hh, b_ih, b_hh, w_out, b_out, steps, x_shift):
        P = {'decoder.weight_ih': w_ih, 'decoder.weight_hh': w_hh, 'decoder.bias_ih': b_ih, 'decoder.bias_hh': b_hh,
             'output.weight': w_out, 'output.bias': b_out}
        for i in (0, 2, 4):   # gru_waypoints applies the join MLP itself: feed it identities so only the GRU part runs
            n = z.shape[1]
            P['join.%d.weight' % i], P['join.%d.bias' % i] = torch.eye(n), torch.zeros(n)

        class C(O.Cfg):
            pred_len, lidar_pos_x = steps, x_shift
        return O.gru_waypoints(P, z, tp, C)      # z >= 0 after the model's own ReLU, so relu(eye @ z) == z

    def decode(preds, num_dir_bins, k=100, ratio=4.0):
        p = _nchw(preds)
        nb = num_dir_bins
        maps = [p[:, 0:1].sigmoid(), p[:, 1:3], p[:, 3:5], p[:, 5:5 + nb], p[:, 5 + nb:6 + nb], p[:, 6 + nb:7 + nb], p[:, 7 + nb:9 + nb]]
        return O.decode_heatmap(maps, nb, k=k, ratio=ratio, stable=True)

    def image_prep(img):
        mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
        std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
        return _nhwc(((img / 255.0) - mean) / std)

    def tokens(img, lid, pos_emb, ghi, gwi, ghl, gwl, p, seed):
        B, C = img.shape[0], img.shape[3]
        pool = lambda t, gh, gw: _nhwc(F.adaptive_avg_pool2d(_nchw(t), (gh, gw))).reshape(B, gh * gw, C)
        return torch.cat((pool(img, ghi, gwi), pool(lid, ghl, gwl)), dim=1) + pos_emb

    def attention(h, wq, bq, wk, bk, wv, bv, B, T, nh, p, seed):
        C = h.shape[1]
        split = lambda w, b: F.linear(h, w, b).view(B, T, nh, C // nh).transpose(1, 2)
        q, k, v = split(wq, bq), split(wk, bk), split(wv, bv)
        att = F.softmax((q @ k.transpose(-2, -1)) * (1.0 / (C // nh) ** 0.5), dim=-1)
        return (att @ v).transpose(1, 2).reshape(B * T, C)

    def gpt_up_add(img, lid, x, ghi, gwi, ghl, gwl):
        B, n_img = x.shape[0], ghi * gwi
        # transfuser.py:363-364: token-major buffers re-interpreted as NCHW without permuting back
        xi = x[:, :n_img].contiguous().view(B, -1, ghi, gwi)
        xl = x[:, n_img:].contiguous().view(B, -1, ghl, gwl)
        up = lambda t, ref: _nhwc(F.interpolate(t, size=ref.shape[1:3], mode='bilinear', align_corners=False))
        return img + up(xi, img), lid + up(xl, lid)

    class _Apply:
        def __init__(self, fn):
            self.apply = fn

    monkeypatch.setattr(ops, 'conv2d', conv2d)
    monkeypatch.setattr(ops, 'batch_norm', batch_norm)
    monkeypatch.setattr(ops, 'linear', linear)
    monkeypatch.setattr(ops, 'gather_sum', gather_sum)
    monkeypatch.setattr(ops, 'avgpool_grid', lambda x, gh, gw: _nhwc(F.adaptive_avg_pool2d(_nchw(x), (gh, gw))))
    monkeypatch.setattr(ops, 'upsample', lambda x, Ho, Wo, ac=False, emit16=False: _nhwc(F.interpolate(_nchw(x), (Ho, Wo), mode='bilinear', align_corners=ac)))
    monkeypatch.setattr(ops, 'add', lambda a, b, relu=False, emit16=False: F.relu(a + b) if relu else a + b)
    monkeypatch.setattr(ops, 'image_prep', image_prep)
    monkeypatch.setattr(ops, 'nchw_to_nhwc', _nhwc)
    monkeypatch.setattr(ops, 'nhwc_to_nchw', lambda t: _nchw(t).contiguous())
    monkeypatch.setattr(ops, 'tick', lambda device: None)
    monkeypatch.setattr(ops, 'SEFn', _Apply(se))
    monkeypatch.setattr(ops, 'PoolHWFn', _Apply(lambda x: x.mean((1, 2))))
    monkeypatch.setattr(ops, 'GRUFn', _Apply(gru))
    monkeypatch.setattr(ops, 'centernet_decode', decode)
    monkeypatch.setattr(ops, 'TWO_STREAMS', False)
    monkeypatch.setattr(ops, 'BN_SE_FUSED', False)      # (the Bottleneck then goes through ops.batch_norm + ops.SEFn, stubbed above)
    monkeypatch.setattr(ops, 'TokensFn', _Apply(tokens))
    monkeypatch.setattr(ops, 'AttentionFn', _Apply(attention))
    monkeypatch.setattr(ops, 'GptUpAddFn', _Apply(gpt_up_add))
    monkeypatch.setattr(ops, 'layer_norm', lambda x, ln, emit16=False: F.layer_norm(x, (x.shape[-1],), ln.weight, ln.bias, ln.eps))
    monkeypatch.setattr(ops, 'dropout', lambda x, p, training: x)       # the tests run with all dropout probabilities at 0
    monkeypatch.setattr(ops, 'BcastAddTokensFn', _Apply(lambda tok, v: tok + v[:, None, :]))

    def add_dropout_ln(res, x, p, training, ln, emit16=False):
        xnew = res + x
        return xnew, F.layer_norm(xnew, (xnew.shape[-1],), ln.weight, ln.bias, ln.eps)

    monkeypatch.setattr(ops, 'add_dropout_ln', add_dropout_ln)
    monkeypatch.setattr(ops, 'next_seed', lambda: 0)
    return ops


@pytest.fixture
def fp64():
    """The comparisons run in float64: the product's reassociations (pool <-> 1x1, 1x1 <-> upsample) are exact in real
    arithmetic, so fp64 shows wiring errors at 1e-9 while fp32 train-mode BatchNorm at batch 2 amplifies rounding to ~2e-4."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


def _build(backbone, seed):
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    net = LidarCenterNet(TrainConfig(embd_pdrop=0.0, attn_pdrop=0.0, resid_pdrop=0.0), 'cpu', backbone, 'regnety_032', 'regnety_032', use_velocity=False)
    names = [(n, tuple(p.shape)) for n, p in list(net.named_parameters()) + list(net.named_buffers()) if not n.startswith('_bev')]
    net.load_state_dict(O.deterministic_state(names, seed=seed), strict=False)
    return net.double()


def _batch(B, seed):
    return {k: (v.double() if v.dtype.is_floating_point else v) for k, v in O.synthetic_batch(B, seed=seed).items()}


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize('train', [True, False])
def test_geometric_fusion_module_wiring(torch_ops, fp64, train):
    """GeometricFusionBackbone.forward (NCHW contract) vs oracle.backbone_geometric_fusion: FPN levels, image grid, fused vector.
    The reassociated order (pool -> 1x1, 1x1 -> upsample) must agree with the reference order to fp32 rounding."""
    net = _build('geometric_fusion', 8)
    net.train(train)
    batch = _batch(2, 5)
    bev_pts, cam_pts = O.synthetic_correspondences(2, seed=5)
    lidar = torch.cat((batch['lidar'], batch['target_point_image']), dim=1)
    P = {k: v.clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        want_feats, want_grid, want_fused = O.backbone_geometric_fusion(P, batch['rgb'], lidar, bev_pts, cam_pts, O.Cfg, train)
        feats, grid, fused = net._model(batch['rgb'], lidar, batch['ego_vel'], bev_pts, cam_pts)
    assert len(feats) == 4
    for a, b in zip(feats, want_feats):
        assert a.shape == b.shape and _rel(a, b) < 1e-9, _rel(a, b)
    assert grid.shape == want_grid.shape and _rel(grid, want_grid) < 1e-9
    assert _rel(fused, want_fused) < 1e-9
    if train:
        assert int(net.state_dict()['_model.lidar_encoder._model.bn1.num_batches_tracked']) == 1


def test_late_fusion_module_wiring(torch_ops, fp64):
    net = _build('late_fusion', 6).train()
    batch = _batch(2, 8)
    lidar = torch.cat((batch['lidar'], batch['target_point_image']), dim=1)
    P = {k: v.clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        want_feats, want_grid, want_fused = O.backbone_late_fusion(P, batch['rgb'], lidar, O.Cfg, True)
        feats, grid, fused = net._model(batch['rgb'], lidar, batch['ego_vel'])
    assert _rel(feats[0], want_feats[0]) < 1e-9 and _rel(grid, want_grid) < 1e-9 and _rel(fused, want_fused) < 1e-9


@pytest.mark.parametrize('backbone', ['transFuser', 'latentTF'])
@pytest.mark.parametrize('train', [True, False])
def test_transfuser_family_module_wiring(torch_ops, fp64, backbone, train):
    """TransfuserBackbone / latentTFBackbone (single-stream schedule) vs the oracle, incl. the per-stage taps."""
    net = _build(backbone, 4)
    net.train(train)
    batch = _batch(2, 11)
    lidar = torch.cat((batch['lidar'], batch['target_point_image']), dim=1)
    P = {k: v.clone() for k, v in net.state_dict().items()}
    fn = O.backbone if backbone == 'transFuser' else O.backbone_latent_tf
    with torch.no_grad():
        want_feats, want_grid, want_fused = fn(P, batch['rgb'], lidar.clone(), O.Cfg, train)
        feats, grid, fused = net._model(batch['rgb'], lidar, batch['ego_vel'])
    for a, b in zip(feats, want_feats):
        assert a.shape == b.shape and _rel(a, b) < 1e-9, _rel(a, b)
    assert _rel(grid, want_grid) < 1e-9 and _rel(fused, want_fused) < 1e-9


@pytest.mark.parametrize('train', [True, False])
def test_transfuser_with_velocity_matches_verbatim_reference(torch_ops, fp64, train):
    """use_velocity=True (transfuser.py:306-309, 352-355: a Linear(1, n_embd) embedding of the ego speed added to every token of all
    four GPTs): same state_dict keys as the verbatim reference, strict load, and the same backbone outputs (their norms and a
    seeded sample of their elements, tests/golden/reference_checks.npz)."""
    from oracle.make_golden_reference import GOLD, sample_index
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    g = np.load(GOLD)
    names = [(str(n), tuple(int(d) for d in str(s).split('x') if d)) for n, s in zip(g['sd_transFuser_vel_keys'], g['sd_transFuser_vel_shapes'])]
    net = LidarCenterNet(TrainConfig(embd_pdrop=0.0, attn_pdrop=0.0, resid_pdrop=0.0), 'cpu', 'transFuser', 'regnety_032', 'regnety_032',
                         use_velocity=True)
    a = {k: v for k, v in net.state_dict().items() if not k.startswith('_bev')}
    assert [(k, tuple(v.shape)) for k, v in a.items()] == names
    assert '_model.transformer3.vel_emb.weight' in a and a['_model.transformer3.vel_emb.weight'].shape == (576, 1)
    own = [(n, tuple(p.shape)) for n, p in list(net.named_parameters()) + list(net.named_buffers()) if not n.startswith('_bev')]
    net.load_state_dict(O.deterministic_state(own, seed=12), strict=False)      # seeded by parameter name, aliases share the tensor
    net = net.double().train(train)
    batch = _batch(2, 13)
    lidar = torch.cat((batch['lidar'], batch['target_point_image']), dim=1)
    with torch.no_grad():
        feats, grid, fused = net._model(batch['rgb'], lidar, batch['ego_vel'])
        # the velocity really enters: a different speed moves the outputs
        _, grid2, _ = net._model(batch['rgb'], lidar, batch['ego_vel'] + 3.0) if not train else (None, None, None)
    for i, x in enumerate(list(feats) + [grid, fused]):
        f = x.double().reshape(-1)
        want = torch.from_numpy(g['vel_%d_%d_sample' % (train, i)])
        assert tuple(x.shape) == tuple(g['vel_%d_%d_shape' % (train, i)]), i
        assert _rel(f[torch.from_numpy(sample_index(f.numel()))], want) < 1e-9, (i, _rel(f[torch.from_numpy(sample_index(f.numel()))], want))
        assert abs(f.norm().item() - float(g['vel_%d_%d_norm' % (train, i)][0])) <= 1e-9 * float(g['vel_%d_%d_norm' % (train, i)][0]), i
    if not train:
        assert _rel(grid2, grid) > 1e-6


@pytest.mark.parametrize('backbone', ['late_fusion', 'geometric_fusion', 'latentTF'])
def test_forward_ego_wiring(torch_ops, fp64, backbone):
    """LidarCenterNet.forward_ego (eval): waypoints, thresholded boxes of sample 0, host box geometry vs oracle.forward_ego."""
    net = _build(backbone, 9).eval()
    batch = _batch(1, 6)
    kw = {}
    if backbone == 'geometric_fusion':
        batch['bev_points'], batch['cam_points'] = O.synthetic_correspondences(1, seed=6)
        kw = dict(bev_points=batch['bev_points'], cam_points=batch['cam_points'])
    P = {k: v.clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        want_wp, want_boxes, _ = O.forward_ego(P, batch, O.Cfg, backbone_name=backbone)
    wp, boxes = net.forward_ego(batch['rgb'], batch['lidar'], batch['target_point'], batch['target_point_image'], batch['ego_vel'], **kw)
    assert _rel(wp, want_wp) < 1e-9
    assert len(boxes) == len(want_boxes) and len(boxes) > 0
    for (a, ab, ac), (b, bb, bc) in zip(boxes, want_boxes):
        assert np.allclose(a, b, rtol=1e-6, atol=1e-6) and ab == bb and abs(ac - bc) < 1e-9
    assert net.i == 1
