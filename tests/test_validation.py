"""Validation bookkeeping without a GPU: tfb_val_accumulate (run through the CPU emulation of csrc/losses.cu) against a restatement
of the reference's Engine.validate loop (train.py:333-340), and trainer.average_over_ranks under gloo with two ranks against
log_losses' aggregate (train.py:344-379)."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from cuda_emul import loader
from transfuser_b200.config import TrainConfig

# the model's loss-dict order (model.py: wp, bev, the seven head terms, depth, semantic)
ORDER = ['loss_wp', 'loss_bev', 'loss_center_heatmap', 'loss_wh', 'loss_offset', 'loss_yaw_class', 'loss_yaw_res', 'loss_velocity',
         'loss_brake', 'loss_depth', 'loss_semantic']


def _reference_validate(batches, weights):
    """train.py:333-340: fp32 products of the (fp32-cast) weight and the loss, the total an fp32 running sum in loss-dict order,
    the per-key and epoch sums Python floats."""
    detailed = {k: 0.0 for k in ORDER}
    loss_epoch, n = 0.0, 0
    for losses in batches:
        loss = np.float32(0.0)
        for k in ORDER:
            wv = np.float32(weights[k]) * np.float32(losses[k])
            loss = np.float32(loss + wv)
            detailed[k] += float(wv)
        n += 1
        loss_epoch += float(loss)
    return detailed, loss_epoch, n


def test_val_accumulate_emulated_matches_engine_validate():
    lib = loader.emul()
    cfg = TrainConfig()
    weights = dict(zip(cfg.detailed_losses, cfg.detailed_losses_weights))
    assert sorted(weights) == sorted(ORDER) and 0.2 in weights.values() and 0.0 in weights.values()
    rng = np.random.default_rng(7)
    batches = []
    for b in range(9):
        scale = (1e-8, 1e4, 1.0)[b % 3]               # losses around 1e-8, 1e4 and 1, and mixes of them
        vals = (rng.random(len(ORDER)) * scale * 10.0 ** rng.integers(-2, 3, len(ORDER))).astype(np.float32)
        if b == 4:
            vals[::2] = np.float32(1e-8) * np.float32(1.0 + rng.random())
            vals[1::2] = np.float32(1e4) * np.float32(1.0 + rng.random())
        batches.append(dict(zip(ORDER, vals.tolist())))
    acc = torch.zeros(len(ORDER) + 2, dtype=torch.float64)
    w32 = torch.tensor([weights[k] for k in ORDER], dtype=torch.float32)
    for losses in batches:
        vals = [torch.tensor([losses[k]], dtype=torch.float32) for k in ORDER]
        table = torch.tensor([v.data_ptr() for v in vals], dtype=torch.int64)
        lib.call('tfb_val_accumulate', table, w32, len(ORDER), acc)
    detailed, loss_epoch, n = _reference_validate(batches, weights)
    got = acc.tolist()
    for i, k in enumerate(ORDER):
        assert got[i] == detailed[k], (k, got[i], detailed[k])
    assert got[len(ORDER)] == loss_epoch and got[len(ORDER) + 1] == n


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_means(rank):
    g = np.random.default_rng(100 + rank)
    return [float(v) for v in g.random(len(ORDER) + 1) * 10.0 ** g.integers(-6, 4, len(ORDER) + 1)]


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from transfuser_b200.trainer import average_over_ranks
    got = average_over_ranks(torch.tensor(_rank_means(rank), dtype=torch.float64))
    out.put((rank, got.tolist()))
    dist.destroy_process_group()


def test_average_over_ranks_world2_gloo_equals_log_losses():
    world, port = 2, _free_port()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    res = dict(q.get(timeout=5) for _ in range(world))
    gathered = [_rank_means(r) for r in range(world)]
    # log_losses: sum(gathered_loss) / len(gathered_loss) for the total, then per key 0.0 + rank 0 + rank 1 ..., / world_size
    want = [sum(g[0] for g in gathered) / world]
    for i in range(1, len(ORDER) + 1):
        v = 0.0
        for r in range(world):
            v += gathered[r][i]
        want.append(v / world)
    for r in range(world):
        assert res[r] == want, (r, res[r], want)


def test_average_over_ranks_single_process_is_identity():
    from transfuser_b200.trainer import average_over_ranks
    m = torch.tensor(_rank_means(0), dtype=torch.float64)
    assert torch.equal(average_over_ranks(m), m)
