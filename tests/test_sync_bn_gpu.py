"""Synchronized BatchNorm on the H100: the sync kernels for simulated ranks, the captured Trainer step with a one-rank NCCL group
(byte-identical to the step without sync), two processes over gloo against one full-batch process, and NCCL with two GPUs."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import sync_bn_check

pytestmark = pytest.mark.gpu
JOIN_S = 900
PG_TIMEOUT = __import__('datetime').timedelta(seconds=600)


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _spawn(fn, world, *args):
    """Runs fn(rank, world, port, out, *args) in `world` spawned processes; joins with a timeout and kills what is still alive."""
    ctx = mp.get_context('spawn')
    out = ctx.Manager().dict()
    port = _free_port()
    ps = [ctx.Process(target=fn, args=(r, world, port, out) + args) for r in range(world)]
    for p in ps:
        p.start()
    for p in ps:
        p.join(JOIN_S)
    alive = [p for p in ps if p.is_alive()]
    for p in alive:
        p.kill()
        p.join(10)
    assert not alive, 'a rank did not finish within %d s' % JOIN_S
    assert all(p.exitcode == 0 for p in ps), [(p.exitcode, out.get('error%d' % r)) for r, p in enumerate(ps)]
    return dict(out)


def _init(rank, world, port, backend):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(0 if torch.cuda.device_count() < world else rank)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=PG_TIMEOUT)


@pytest.mark.parametrize('world', [1, 2, 3, 8])
@pytest.mark.parametrize('variant', ['plain', 'relu', 'residual', 'pool'])
@pytest.mark.parametrize('from_stats', [0, 1])
def test_sync_kernels_simulated_ranks(world, variant, from_stats):
    from transfuser_b200 import _lib
    sync_bn_check.run(_lib.call, 'cuda', world, variant, from_stats, C=72, hw=40)
    sync_bn_check.run(_lib.call, 'cuda', world, variant, from_stats, C=1512, hw=3)
    if world == 1:      # rank 0 holds 3 samples: M = 4200 rows, the flat statistics / reduction kernels
        sync_bn_check.run(_lib.call, 'cuda', world, variant, from_stats, C=72, hw=1400)


def _snapshot(tr, loss):
    net = tr.net
    return dict(loss=loss.detach().cpu().clone(), flat=tr.flat.flat.detach().cpu().clone(),
                grad=tr.flat.grad.detach().cpu().clone() if getattr(tr.flat, 'grad', None) is not None else None,
                bufs=torch.cat([b.detach().double().flatten().cpu() for b in net.buffers()]))


CONFIGS = [('transFuser', 'regnety_032', 'regnety_032', 'bf16'), ('transFuser', 'regnety_032', 'regnety_032', 'simt'),
           ('transFuser', 'resnet34', 'resnet18', 'bf16'), ('late_fusion', 'regnety_032', 'regnety_032', 'bf16'),
           ('geometric_fusion', 'regnety_032', 'regnety_032', 'bf16')]


def _world1_worker(rank, world, port, out):
    try:
        import numpy as np
        from bench import make_host_batch
        from transfuser_b200.config import TrainConfig
        from transfuser_b200.trainer import Trainer
        _init(rank, world, port, 'nccl')
        for ci, (backbone, ia, la, mode) in enumerate(CONFIGS):
            host = make_host_batch(2, seed=7, torch=torch, np=np, backbone=backbone)
            snaps = {}
            for sync in (False, True):
                torch.manual_seed(0)
                tr = Trainer(TrainConfig(), 'cuda', gemm_mode=mode, backbone=backbone, image_architecture=ia, lidar_architecture=la,
                             sync_batch_norm=sync)
                assert tr.capture(host), tr.graph_error
                for _ in range(2):
                    tr.load(host)
                    loss = tr.replay()
                torch.cuda.synchronize()
                snaps[sync] = _snapshot(tr, loss)
                if sync and ci == 0:
                    # eager steps of a fresh synchronized trainer: the same bits as the replays
                    torch.manual_seed(0)
                    te = Trainer(TrainConfig(), 'cuda', gemm_mode=mode, backbone=backbone, image_architecture=ia, lidar_architecture=la,
                                 sync_batch_norm=True)
                    dev = {k: v.cuda() for k, v in host.items()}
                    for _ in range(4):          # the two warm-up steps of capture() + the two replays
                        le = te.step(dev)
                    torch.cuda.synchronize()
                    e = _snapshot(te, le)
                    assert all(torch.equal(e[k], snaps[True][k]) for k in ('loss', 'flat', 'bufs')), 'eager != replay'
                del tr
            for k in ('loss', 'flat', 'grad', 'bufs'):
                a, b = snaps[False][k], snaps[True][k]
                assert (a is None and b is None) or torch.equal(a, b), (backbone, ia, mode, k)
        out['ok'] = True
        dist.destroy_process_group()
    except Exception as e:  # noqa: BLE001
        import traceback
        out['error%d' % rank] = traceback.format_exc()[-3000:]
        raise


def test_world1_nccl_captured_step_bitwise():
    """With one rank the synchronized step is the unsynchronized step, byte for byte (losses, parameters, gradients, buffers)."""
    assert _spawn(_world1_worker, 1).get('ok')


def _backbone(sync):
    from transfuser_b200 import gemm
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.model import LidarCenterNet
    gemm.set_mode('simt')
    torch.manual_seed(0)
    cfg = TrainConfig()
    cfg.embd_pdrop = cfg.attn_pdrop = cfg.resid_pdrop = 0.0     # dropout masks depend on the batch a rank holds
    net = LidarCenterNet(cfg, 'cuda', 'transFuser', 'regnety_032', 'regnety_032').train()
    if sync:
        net = torch.nn.SyncBatchNorm.convert_sync_batchnorm(net)
    return net


def _inputs(B):
    g = torch.Generator().manual_seed(11)
    img = (torch.rand(B, 3, 160, 704, generator=g) * 255).cuda()
    lid = torch.rand(B, 3, 256, 256, generator=g).cuda()
    return img, lid


def _run_taps(net, img, lid):
    taps = {}
    net._model.forward_nhwc(img, lid, taps=taps, velocity=torch.zeros(img.shape[0], 1, device='cuda'))
    obj = sum(t.double().sum() for t in taps.values())
    obj.backward()
    return taps


def _gloo_worker(rank, world, port, out, sync):
    try:
        _init(rank, world, port, 'gloo')
        net = _backbone(sync)
        img, lid = _inputs(2 * world)
        rows = slice(2 * rank, 2 * rank + 2)
        taps = _run_taps(net, img[rows].contiguous(), lid[rows].contiguous())
        grads = torch.cat([p.grad.flatten() if p.grad is not None else torch.zeros_like(p).flatten() for p in net.parameters()])
        dist.all_reduce(grads)
        out['taps%d' % rank] = {k: v.detach().cpu() for k, v in taps.items()}
        out['grad%d' % rank] = grads.cpu()
        out['bufs%d' % rank] = torch.cat([b.double().flatten() for n, b in net.named_buffers() if 'running' in n]).cpu()
        dist.destroy_process_group()
    except Exception:  # noqa: BLE001
        import traceback
        out['error%d' % rank] = traceback.format_exc()[-3000:]
        raise


def test_two_ranks_gloo_match_full_batch():
    """Two processes on one GPU (gloo, eager, simt): each rank's taps are its rows of the full-batch run, the running statistics are
    the same bits on both ranks (and differ without sync), and the all-reduced gradient of a summed objective is the full batch's."""
    r = _spawn(_gloo_worker, 2, True)
    plain = _spawn(_gloo_worker, 2, False)
    net = _backbone(False)
    img, lid = _inputs(4)
    full = {k: v.detach() for k, v in _run_taps(net, img, lid).items()}
    gfull = torch.cat([p.grad.flatten() if p.grad is not None else torch.zeros_like(p).flatten() for p in net.parameters()]).cpu()
    for rank in range(2):
        for k, v in full.items():
            part = v[2 * rank:2 * rank + 2].cpu()
            err = (r['taps%d' % rank][k] - part).abs().max() / part.abs().max()
            assert err < 1e-4, (rank, k, err.item())
    assert torch.equal(r['bufs0'], r['bufs1'])
    assert not torch.equal(plain['bufs0'], plain['bufs1'])
    err = (r['grad0'] - gfull).abs().max() / gfull.abs().max()
    assert err < 1e-3, err.item()


def _nccl2_worker(rank, world, port, out):
    try:
        import numpy as np
        from bench import make_host_batch
        from transfuser_b200.config import TrainConfig
        from transfuser_b200.trainer import Trainer
        _init(rank, world, port, 'nccl')
        host = make_host_batch(2, seed=20 + rank, torch=torch, np=np)
        res = []
        for graph in (False, True):
            torch.manual_seed(0)
            tr = Trainer(TrainConfig(), 'cuda', sync_batch_norm=True)
            if graph:
                assert tr.capture(host), tr.graph_error
                for _ in range(2):
                    tr.load(host)
                    loss = tr.replay()
            else:
                dev = {k: v.cuda() for k, v in host.items()}
                for _ in range(4):
                    loss = tr.step(dev)
            torch.cuda.synchronize()
            res.append(_snapshot(tr, loss))
        assert all(torch.equal(res[0][k], res[1][k]) for k in ('loss', 'flat', 'bufs'))
        out['bufs%d' % rank] = res[1]['bufs']
        dist.destroy_process_group()
    except Exception:  # noqa: BLE001
        import traceback
        out['error%d' % rank] = traceback.format_exc()[-3000:]
        raise


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL world 2 needs two GPUs')
def test_world2_nccl_captured_equals_eager():
    r = _spawn(_nccl2_worker, 2)
    assert torch.equal(r['bufs0'], r['bufs1'])
