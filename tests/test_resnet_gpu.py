"""The ResNet-18 / ResNet-34 trunks on the GPU: the stem kernels (csrc/resnet_stem.cu) by their C-ABI entry points, TransFuser and
late fusion with (resnet34, resnet18) against the CPU oracle, and the reproducibility of a captured training step."""
import numpy as np
import pytest
import torch

from oracle import resnet_oracle as R, torch_oracle as O
from test_model import Cfg, rel
from test_resnet_stem_emulated import check_pool, check_stem, pool_case, stem_case

pytestmark = pytest.mark.gpu
TRUNKS = ('resnet34', 'resnet18')


def _call(name, *args):
    from transfuser_b200 import _lib
    return _lib.call(name, *args)


def _cuda(t):
    return t.cuda()


@pytest.mark.parametrize('N,Cin,H,W', [(2, 3, 160, 704), (2, 3, 256, 256), (1, 2, 37, 45), (2, 4, 9, 7)])
def test_stem_conv_gpu(N, Cin, H, W):
    check_stem(_call, *stem_case(N, Cin, 64, H, W, seed=H + W + Cin), to_dev=_cuda)


@pytest.mark.parametrize('N,C,H,W', [(2, 64, 80, 352), (2, 64, 128, 128), (3, 8, 5, 7)])
def test_maxpool_gpu(N, C, H, W):
    x, dy = pool_case(N, C, H, W, seed=H * W)
    runs = [check_pool(_call, x, dy, to_dev=_cuda) for _ in range(2)]
    for a, b in zip(*runs):                 # every launch repeated gives the same bits
        assert torch.equal(a.cpu().view(torch.uint8), b.cpu().view(torch.uint8))


def build(backbone='transFuser', seed=1):
    from transfuser_b200 import LidarCenterNet
    net = LidarCenterNet(Cfg, 'cpu', backbone, *TRUNKS, use_velocity=False)
    names = [(n, tuple(p.shape)) for n, p in list(net.named_parameters()) + list(net.named_buffers()) if not n.startswith('_bev')]
    net.load_state_dict(O.deterministic_state(names, seed=seed), strict=False)
    return net


def _oracle(net, batch, dtype, backbone='transFuser', bf16_operands=False, grads=True):
    class C(O.Cfg):
        embd_pdrop = attn_pdrop = resid_pdrop = 0.0
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    O.BF16_OPERANDS[0] = bf16_operands
    try:
        P = {k: (v.clone().to(dtype) if v.dtype.is_floating_point else v.clone()) for k, v in net.state_dict().items()}
        for k, v in P.items():
            if grads and v.dtype.is_floating_point and 'running' not in k:
                v.requires_grad_()
        b = {k: (v.to(dtype) if v.dtype.is_floating_point else v) for k, v in batch.items()}
        taps = {}
        with torch.set_grad_enabled(grads):
            losses = R.forward(P, b, TRUNKS, C, train=True, taps=taps, backbone_name=backbone)
            if grads:
                w = dict(zip(Cfg.detailed_losses, Cfg.detailed_losses_weights))
                sum(w[k] * losses[k] for k in losses).backward()
    finally:
        torch.set_default_dtype(old)
        O.BF16_OPERANDS[0] = False
    return P, losses, taps


def _run(net, cb):
    return net(cb['rgb'], cb['lidar'], ego_waypoint=cb['ego_waypoint'], target_point=cb['target_point'],
               target_point_image=cb['target_point_image'], ego_vel=cb['ego_vel'], bev=cb['bev'], label=cb['label'],
               depth=cb['depth'], semantic=cb['semantic'])


_CACHE = {}


@pytest.mark.parametrize('mode', ['simt', 'bf16x6', 'bf16'])
def test_transfuser_resnet_matches_oracle(mode):
    """simt / bf16x6: per-stage taps and the 11 losses within 1e-3 of the fp32 oracle, gradients against the fp64 oracle by the
    percentile rules of tests/test_model.py. bf16: the losses within smoke()'s bounds of the oracle with bf16 tensor-core operands."""
    from transfuser_b200 import gemm
    torch.manual_seed(0)
    net = build()
    batch = O.synthetic_batch(2, seed=3)
    if 'runs' not in _CACHE:
        _CACHE['runs'] = (_oracle(net, batch, torch.float32), _oracle(net, batch, torch.float64))
    (P, ref, taps), (P64, _, _) = _CACHE['runs']
    if mode == 'bf16':
        _, ref, _ = _oracle(net, batch, torch.float32, bf16_operands=True, grads=False)
    w = dict(zip(Cfg.detailed_losses, Cfg.detailed_losses_weights))
    old = gemm.MODE
    gemm.set_mode(mode)
    try:
        net = net.cuda().train()
        cb = {k: v.cuda() for k, v in batch.items()}
        if mode != 'bf16':
            mine = {}
            net._model.forward_nhwc(cb['rgb'], torch.cat((cb['lidar'], cb['target_point_image']), dim=1), taps=mine)
            torch.cuda.synchronize()
            for k in sorted(mine):
                e = rel(mine[k].permute(0, 3, 1, 2), taps[k])
                print('[%s] activation %-8s rel err %.2e' % (mode, k, e))
                assert e < 1e-3, (k, e)
            net.load_state_dict({k: v.detach().float() for k, v in build().state_dict().items()}, strict=False)   # undo the BN stat update
        out = _run(net, cb)
        assert list(out) == list(ref)
        for k in ref:
            a, b = out[k].item(), ref[k].item()
            tol = (0.35 if k == 'loss_yaw_res' else 5e-2) if mode == 'bf16' else 1e-3
            print('[%s] %-22s oracle %.7f cuda %.7f rel %.2e' % (mode, k, b, a, abs(a - b) / max(abs(b), 1e-12)))
            assert abs(a - b) <= tol * max(abs(b), 1e-6), (k, a, b)
        sum(w[k] * out[k] for k in out).backward()
        if mode == 'bf16':
            assert all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)
            return
        rows = [(rel(p.grad, P64[n].grad), rel(P[n].grad, P64[n].grad)) for n, p in net.named_parameters() if not n.endswith('attn.key.bias')]
        e, eo = np.array([r[0] for r in rows]), np.array([r[1] for r in rows])
        q = lambda a, p: float(np.percentile(a, p))
        print('[%s] cuda-vs-fp64: median %.2e p95 %.2e max %.2e | oracle32-vs-fp64: median %.2e p95 %.2e max %.2e'
              % (mode, q(e, 50), q(e, 95), e.max(), q(eo, 50), q(eo, 95), eo.max()))
        assert q(e, 50) <= max(1e-3, 2 * q(eo, 50))
        assert q(e, 95) <= max(1e-3, 2 * q(eo, 95))
        assert (e > max(1e-3, 5 * q(eo, 95))).sum() <= 0.01 * len(e)
        assert e.max() < 0.5
        sd = net.state_dict()
        worst = max((rel(sd[k], P[k]), k) for k in P if 'running' in k and ('.bn1.' in k or '.layer1.' in k or '.layer4.' in k))
        assert worst[0] < 1e-4, worst
    finally:
        gemm.set_mode(old)


def test_late_fusion_resnet_matches_oracle():
    net = build('late_fusion', seed=6)
    batch = O.synthetic_batch(2, seed=8)
    P, ref, _ = _oracle(net, batch, torch.float32, backbone='late_fusion')
    net = net.cuda().train()
    out = _run(net, {k: v.cuda() for k, v in batch.items()})
    for k in ref:
        assert abs(out[k].item() - ref[k].item()) <= 1e-3 * max(abs(ref[k].item()), 1e-6), (k, out[k].item(), ref[k].item())
    w = dict(zip(Cfg.detailed_losses, Cfg.detailed_losses_weights))
    sum(w[k] * out[k] for k in out).backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in net.parameters())


def test_captured_resnet_step_is_reproducible():
    """A captured bf16 training step with ResNet trunks, replayed 3 times, run twice from the same seed: identical bits for the
    losses, the parameters and the gradients."""
    from bench import make_host_batch
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    dev = torch.device('cuda', 0)
    host = make_host_batch(2, seed=5, torch=torch, np=np)
    runs = []
    for _ in range(2):
        torch.manual_seed(0)
        tr = Trainer(TrainConfig(), dev, gemm_mode='bf16', seed=0, image_architecture=TRUNKS[0], lidar_architecture=TRUNKS[1])
        assert tr.capture(host), tr.graph_error
        losses = [tr.replay().clone() for _ in range(3)]
        torch.cuda.synchronize()
        runs.append((torch.stack(losses).cpu(), tr.flat.flat.cpu(), tr.flat.grad.cpu()))
        del tr
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert bool(torch.isfinite(runs[0][0]).all()) and float(runs[0][2].abs().sum()) > 0
