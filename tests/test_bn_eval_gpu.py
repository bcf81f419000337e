"""Eval-mode BatchNorm in the tensor-core epilogues and the captured validation (`-m gpu`):
- tfb_gemm_bf16_tc_bn_eval / tfb_conv3x3_tc_bn_eval equal the plain launch + tfb_bn_apply bit for bit (fp32 and bf16 outputs) on
  the RegNetY-032 and ResNet-18/34 trunk shapes, NaN-prefilled and sentinel-guarded;
- the whole model in bf16 eval mode gives the same losses and forward_ego outputs with the epilogue path on and patched off;
- Validator: graph replay = eager steps, finish() = Engine.validate + log_losses restated, and no effect on training."""
import pickle

import numpy as np
import pytest
import torch

from tc_ref import Guarded

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _call(name, *a):
    from transfuser_b200 import _lib
    _lib.call(name, *a)


def _bn_params(C, g):
    mean = torch.randn(C, generator=g).to(DEV)
    var = (torch.rand(C, generator=g) * 2 + 0.05).to(DEV)
    gamma = torch.randn(C, generator=g).to(DEV)                     # about half negative
    beta = torch.randn(C, generator=g).to(DEV)
    return mean, torch.rsqrt(var + 1e-5), gamma, beta


VARIANTS = [(False, False, False), (False, True, True), (True, True, True), (True, False, False)]   # (residual, relu, sidecar)


def _compare(fused, plain, shape, C, params, g):
    """fused(y, res, relu, y16) vs plain(y0) + tfb_bn_apply, for every VARIANT, twice each."""
    mean, invstd, gamma, beta = params
    M = int(np.prod(shape[:-1]))
    res = torch.randn(shape, generator=g).to(DEV)
    y0 = Guarded(shape, torch.float32)
    plain(y0.reset())
    assert not torch.isnan(y0.t).any() and y0.tail_ok()
    for with_res, relu, side in VARIANTS:
        r = res if with_res else None
        ref, ref16 = Guarded(shape, torch.float32), Guarded(shape, torch.bfloat16)
        _call('tfb_bn_apply', y0.t, ref.reset(), M, C, gamma, beta, mean, invstd, int(relu), ref16.reset() if side else None, r)
        for _ in range(2):
            out, out16 = Guarded(shape, torch.float32), Guarded(shape, torch.bfloat16)
            out16.reset()
            fused(out.reset(), r, int(relu), out16.t if side else None)
            torch.cuda.synchronize()
            assert out.tail_ok() and out16.tail_ok()
            assert torch.equal(out.bits(), ref.bits()), (shape, with_res, relu, side)
            if side:
                assert torch.equal(out16.bits(), ref16.bits()), (shape, with_res, relu, side)
            else:
                assert torch.isnan(out16.t.float()).all()


# 1x1 convs / downsample GEMMs of the trunks (Cin, Cout) at row counts on and off the 128-row tile
GEMM_SHAPES = [(32, 72), (72, 72), (72, 216), (216, 216), (216, 576), (576, 576), (576, 1512), (1512, 1512), (64, 128), (128, 256),
               (256, 512)]


@pytest.mark.parametrize('M', [1000, 1568, 128])
@pytest.mark.parametrize('K,N', GEMM_SHAPES)
def test_gemm_bn_eval_bits(K, N, M):
    g = torch.Generator().manual_seed(K * 7919 + N * 31 + M)
    x = torch.randn(M, K, generator=g).to(DEV).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV).to(torch.bfloat16)
    params = _bn_params(N, g)
    plain = lambda y: _call('tfb_gemm_bf16_tc', 0, 1, M, N, K, x, K, w, K, y, N, None, 0, 1.0, 0.0, 1)
    fused = lambda y, r, relu, y16: _call('tfb_gemm_bf16_tc_bn_eval', M, N, K, x, K, w, K, y, N, *params, r, relu, y16)
    _compare(fused, plain, (M, N), N, params, g)


# 3x3 convs of the trunks (Cin, Cout, groups, stride): RegNetY-032 grouped (group width 24, stride 1 and 2), ResNet dense
CONV_SHAPES = [(72, 72, 3, 1), (72, 72, 3, 2), (216, 216, 9, 1), (216, 216, 9, 2), (576, 576, 24, 1), (576, 576, 24, 2),
               (1512, 1512, 63, 1), (1512, 1512, 63, 2), (64, 64, 1, 1), (64, 128, 1, 2), (128, 128, 1, 1), (128, 256, 1, 2),
               (256, 256, 1, 1), (256, 512, 1, 2), (512, 512, 1, 1), (32, 32, 1, 1), (16, 16, 1, 1)]


@pytest.mark.parametrize('Cin,Cout,groups,stride', CONV_SHAPES)
def test_conv3x3_bn_eval_bits(Cin, Cout, groups, stride):
    from transfuser_b200 import ops
    g = torch.Generator().manual_seed(Cin * 131 + Cout + groups * 17 + stride)
    N, H, W = 2, 19, 37                       # neither a multiple of the 8 x 16 tile
    x16 = torch.randn(N, H, W, Cin, generator=g).to(DEV).to(torch.bfloat16)
    w = (torch.randn(Cout, Cin // groups, 3, 3, generator=g) / (9 * Cin / groups) ** 0.5).to(DEV)
    plan = ops._conv_tc_plan(Cin, Cout, groups)
    assert plan is not None
    wp = ops._packed_current(w, plan, 0, groups).wp
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    params = _bn_params(Cout, g)
    a = (N, H, W, Cin, Cout, plan['NB'], plan['KC'], plan['c_step'], plan['nchunks'], plan['nb_real'], plan['gblocks'])
    plain = lambda y: _call('tfb_conv3x3_tc_strided', x16, wp, None, y, *a, 0, stride, None)
    fused = lambda y, r, relu, y16: _call('tfb_conv3x3_tc_bn_eval', x16, wp, y, *a, stride, *params, r, relu, y16)
    _compare(fused, plain, (N, Ho, Wo, Cout), Cout, params, g)


def test_bn_eval_argument_checks():
    C = 12
    x = torch.zeros(64, 16, dtype=torch.bfloat16, device=DEV)
    w = torch.zeros(C, 16, dtype=torch.bfloat16, device=DEV)
    y = torch.zeros(64 * C + 4, device=DEV)
    p = [torch.zeros(C, device=DEV) for _ in range(4)]
    with pytest.raises(RuntimeError, match='argument check'):       # N % 4
        _call('tfb_gemm_bf16_tc_bn_eval', 64, 10, 16, x, 16, w, 16, y, 12, *p, None, 0, None)
    with pytest.raises(RuntimeError, match='argument check'):       # misaligned residual
        _call('tfb_gemm_bf16_tc_bn_eval', 64, C, 16, x, 16, w, 16, y, C, *p, y[1:], 0, None)
    with pytest.raises(RuntimeError, match='argument check'):       # misaligned output
        _call('tfb_gemm_bf16_tc_bn_eval', 64, C, 16, x, 16, w, 16, y[2:], C, *p, None, 0, None)


# ------------------------------------------------------------------ the model
MODELS = [('transFuser', 'regnety_032', 'regnety_032'), ('transFuser', 'resnet34', 'resnet18'), ('late_fusion', 'resnet34', 'resnet18'),
          ('geometric_fusion', 'regnety_032', 'regnety_032'), ('latentTF', 'regnety_032', 'regnety_032')]   # (their LiDAR trunk needs a stem)


def _randomise_bn(tr, seed):
    from transfuser_b200 import gemm
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in tr.net.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                C = m.num_features
                m.running_mean.copy_(torch.randn(C, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(C, generator=g) + 0.5)
                m.weight.copy_(torch.randn(C, generator=g))
                m.bias.copy_(torch.randn(C, generator=g) * 0.1)
    gemm.attach_bf16_weights(tr.flat)


def _trainer(backbone='transFuser', img='regnety_032', lid='regnety_032', raw=False, seed=0):
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    torch.manual_seed(seed)
    return Trainer(TrainConfig(), torch.device('cuda', 0), gemm_mode='bf16', seed=seed, backbone=backbone, image_architecture=img,
                   lidar_architecture=lid, raw_inputs=raw)


def _host(B, seed, backbone='transFuser'):
    from bench import make_host_batch
    return make_host_batch(B, seed=seed, torch=torch, np=np, backbone=backbone)


def _bits(losses):
    return torch.stack([v.reshape(()) for v in losses.values()]).view(torch.int32).cpu()


@pytest.mark.parametrize('backbone,img,lid', MODELS)
def test_model_eval_same_bits_with_epilogue_bn(backbone, img, lid, monkeypatch):
    from transfuser_b200 import _lib, ops
    from transfuser_b200.trainer import Validator
    tr = _trainer(backbone, img, lid)
    _randomise_bn(tr, 3)
    val = Validator(tr)
    batch = {k: v.cuda() for k, v in _host(2, 5, backbone).items()}
    fused_calls = []
    real = _lib.call

    def spy(name, *a):
        if name.endswith('_bn_eval'):
            fused_calls.append(name)
        return real(name, *a)
    monkeypatch.setattr(_lib, 'call', spy)
    monkeypatch.setattr(ops, 'call', spy)

    def run():
        lib = _lib.lib()
        n0 = lib.launches
        losses = val.step(batch)
        torch.cuda.synchronize()
        n = lib.launches - n0
        tr.net.eval()
        with torch.no_grad():
            d, lidar = tr.expand_inputs(batch)
            wp, boxes = tr.net.forward_ego(d['rgb'], lidar, d['target_point'], d['target_point_image'], d['ego_vel'], d.get('bev_points'),
                                           d.get('cam_points'))
        tr.net.train()
        return _bits(losses), wp.clone(), boxes, n
    run()                                     # first use: every 3x3 conv weight is packed once per call
    fused_calls.clear()
    on = run()
    nf = len(fused_calls)
    assert nf > 0
    with monkeypatch.context() as m:
        m.setattr(ops, 'bn_epilogue_path', lambda *a: None)
        fused_calls.clear()
        off = run()
        assert not fused_calls
    assert torch.equal(on[0], off[0])
    assert torch.equal(on[1].view(torch.int32), off[1].view(torch.int32))
    assert pickle.dumps(on[2]) == pickle.dumps(off[2])
    # val.step: one fused launch per batch norm replaces a conv + tfb_bn_apply pair; forward_ego runs the same trunks
    assert off[3] - on[3] == nf // 2, (off[3], on[3], nf)


def test_validator_graph_launches_and_fused_count(monkeypatch):
    """The captured graph has exactly as many launches fewer as there are epilogue BatchNorms."""
    from transfuser_b200 import ops
    from transfuser_b200.trainer import Validator
    tr = _trainer()
    host = _host(2, 7)
    counts = []
    for on in (True, False):
        with monkeypatch.context() as m:
            if not on:
                m.setattr(ops, 'bn_epilogue_path', lambda *a: None)
            val = Validator(tr)
            val.capture(host)
            counts.append(val.graph_launches)
            val.replay()
            counts.append(_bits(val.static_losses))
    nf = sum(1 for _ in _fused_sites(tr))
    assert counts[2] - counts[0] == nf, (counts[0], counts[2], nf)
    assert torch.equal(counts[1], counts[3])


def _fused_sites(tr):
    """The trunk BatchNorms the epilogue path covers (everything but the stems)."""
    from transfuser_b200 import backbone as B
    for m in tr.net.modules():
        if isinstance(m, B._Bottleneck):
            yield from ('conv1', 'conv2', 'conv3') + (('downsample',) if m.downsample is not None else ())
        elif isinstance(m, B._BasicBlock):
            yield from ('conv1', 'conv2') + (('downsample',) if m.downsample is not None else ())


def _restated_validate(per_batch, weights):
    order = list(per_batch[0])
    detailed = {k: 0.0 for k in order}
    loss_epoch = 0.0
    for losses in per_batch:
        loss = np.float32(0.0)
        for k in order:
            wv = np.float32(weights[k]) * np.float32(losses[k])
            loss = np.float32(loss + wv)
            detailed[k] += float(wv)
        loss_epoch += float(loss)
    n = len(per_batch)
    return dict({'loss_total': loss_epoch / n}, **{k: v / n for k, v in detailed.items()})


def test_validator_graph_equals_eager_and_engine_validate():
    from transfuser_b200.trainer import Validator
    tr = _trainer()
    _randomise_bn(tr, 4)
    batches = [_host(2, s) for s in (11, 12, 13)] + [_host(1, 14)]        # the last, smaller batch runs eagerly
    val = Validator(tr)
    val.capture(batches[0])
    for b in batches[:3]:
        val.load(b)
        val.replay()
    val.step(batches[3])
    acc_graph = val.acc.clone()
    means = val.finish()
    eager = Validator(tr)
    per_batch = [{k: v.item() for k, v in eager.step(b).items()} for b in batches]
    assert torch.equal(acc_graph.view(torch.int64), eager.acc.view(torch.int64))
    assert means == _restated_validate(per_batch, tr.weights)
    for b in batches[:3]:                                                  # a second validation of the same weights
        val.load(b)
        val.replay()
    val.step(batches[3])
    assert val.finish() == means


def test_validator_oracle_simt_and_bf16():
    """Validator losses against the oracle's eval-mode forward with non-trivial running statistics."""
    from oracle import torch_oracle as O
    from transfuser_b200 import gemm
    from transfuser_b200.trainer import Validator
    host = _host(2, 21)
    b = O.synthetic_batch(2, seed=21)

    class C(O.Cfg):
        embd_pdrop = attn_pdrop = resid_pdrop = 0.0
    for mode, bf16_ops, tol in (('simt', False, 2e-3), ('bf16', True, 5e-2)):
        tr = _trainer()
        gemm.set_mode(mode)
        _randomise_bn(tr, 9)
        P = {k: v.detach().cpu().clone() for k, v in tr.net.state_dict().items()}
        val = Validator(tr)
        got = {k: v.item() for k, v in val.step(host).items()}
        with torch.no_grad():
            b['lidar'] = tr.expand_inputs({k: v.cuda() for k, v in host.items()})[1].cpu()    # the BEV histogram of the sweep
        O.BF16_OPERANDS[0] = bf16_ops
        try:
            with torch.no_grad():
                ref = {k: v.item() for k, v in O.forward(P, b, C, train=False).items()}
        finally:
            O.BF16_OPERANDS[0] = False
        for k in ref:
            t = 0.35 if (mode == 'bf16' and k == 'loss_yaw_res') else tol
            assert abs(got[k] - ref[k]) <= t * max(abs(ref[k]), 1e-6), (mode, k, got[k], ref[k])
    gemm.set_mode('bf16')


def test_validation_leaves_training_unchanged():
    from transfuser_b200.trainer import Validator
    host = _host(2, 31)
    vb = [_host(2, 32), _host(2, 33)]
    runs = []
    for validate in (False, True):
        tr = _trainer(seed=0)
        assert tr.capture(host), tr.graph_error
        val = Validator(tr) if validate else None
        for i in range(4):
            tr.replay()
            if validate and i in (1, 2):
                if val.graph is None:
                    val.capture(vb[0])
                for b in vb:
                    val.load(b)
                    val.replay()
                means = val.finish()
                if i == 2:
                    eager = Validator(tr)
                    for b in vb:
                        eager.step(b)
                    assert eager.finish() == means      # the captured re-pack saw the weights of the latest training step
        torch.cuda.synchronize()
        bufs = torch.cat([b.detach().double().flatten() for n, b in tr.net.named_buffers() if 'running' in n])
        runs.append((tr.flat.flat.clone(), tr.flat.grad.clone(), bufs, tr.opt._m.clone(), tr.opt._v.clone()))
        del tr, val
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int64 if a.dtype == torch.float64 else torch.int32),
                           b.view(torch.int64 if b.dtype == torch.float64 else torch.int32))
