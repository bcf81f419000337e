"""Per-step cost of synchronized BatchNorm: the captured training step (transFuser, RegNetY-032, bf16, batch per GPU as --batch) with
sync_batch_norm off and on, the two replayed alternately in one process, medians of CUDA-event timings.

    python tools/syncbn_step.py --batch 10 --rounds 5 --steps 10                         # world 1 (one-rank NCCL group)
    python -m torch.distributed.run --nproc_per_node 2 tools/syncbn_step.py --batch 10   # two GPUs or more

Prints one JSON line per rank 0 with the card name and power limit next to the numbers."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import gpu_identity, make_host_batch  # noqa: E402
from transfuser_b200.config import TrainConfig  # noqa: E402
from transfuser_b200.trainer import Trainer  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('syncbn_step.py measures on a GPU; none is visible')
    if 'RANK' not in os.environ:
        os.environ.update(RANK='0', WORLD_SIZE='1', LOCAL_RANK='0', MASTER_ADDR='127.0.0.1', MASTER_PORT='29561')
    rank, local = int(os.environ['RANK']), int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    dist.init_process_group('nccl')
    host = make_host_batch(a.batch, seed=3 + rank, torch=torch, np=np)
    trs = {}
    for sync in (False, True):
        torch.manual_seed(0)
        trs[sync] = Trainer(TrainConfig(), 'cuda', sync_batch_norm=sync)
        if not trs[sync].capture(host):
            raise SystemExit('capture failed: %s' % trs[sync].graph_error)
    times = {False: [], True: []}
    for r in range(a.rounds + 1):                      # round 0 is warm-up
        for sync in (False, True):
            tr = trs[sync]
            tr.load(host)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                tr.replay()
            e1.record()
            torch.cuda.synchronize()
            if r > 0:
                times[sync].append(e0.elapsed_time(e1) / a.steps)
    off, on = statistics.median(times[False]), statistics.median(times[True])
    if rank == 0:
        print(json.dumps(dict(world=dist.get_world_size(), batch_per_gpu=a.batch, step_ms_sync_off=round(off, 3), step_ms_sync_on=round(on, 3),
                              delta_ms=round(on - off, 3), rounds_off=[round(t, 3) for t in times[False]], rounds_on=[round(t, 3) for t in times[True]],
                              gpu=gpu_identity(local), graph_launches=trs[True].graph_launches - trs[False].graph_launches)), flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
