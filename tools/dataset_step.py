"""Training from the on-disk dataset, measured on the GPU. Writes two synthetic routes at full size (160 x 960 camera frames,
500 x 500 topdown, 20-30k LiDAR points per sweep; oracle/synthetic_route.py) to a temporary directory and reports, as one JSON line:
  - reader:  dataset.CarlaRawDataset + collate through a DataLoader, batch B, samples/s and samples/s per worker for each worker
             count (two passes over the data; the first, which also warms the page cache, is not timed);
  - kernel:  tfb_bev_label_prep at batch B, CUDA events over a CUDA graph of 200 launches;
  - step:    Trainer(raw_inputs='dataset') against Trainer(raw_inputs=True) fed the same batch with the BEV label the pipeline
             made, both captured, bf16, rounds alternated; ms per step;
  - the card's name and power limit.
    python tools/dataset_step.py [--batch 10] [--workers 1,4] [--rounds 3] [--steps 20]"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import gpu_identity  # noqa: E402
from oracle import synthetic_route  # noqa: E402


def reader_rate(root, batch, workers):
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.dataset import CarlaRawDataset, collate
    ds = CarlaRawDataset([root], TrainConfig(), max_points=40000)
    loader = torch.utils.data.DataLoader(ds, batch_size=batch, num_workers=workers, collate_fn=collate, pin_memory=True,
                                         drop_last=True, persistent_workers=True, shuffle=True)
    for _ in loader:
        pass
    t0, n = time.perf_counter(), 0
    for b in loader:
        n += len(b['bev_u8'])
    dt = time.perf_counter() - t0
    return n / dt, loader


def kernel_us(batch, dev):
    from transfuser_b200 import _lib
    n = 200
    plane = torch.randint(0, 256, (batch, 500, 500), dtype=torch.uint8, device=dev)
    from transfuser_b200 import pipeline
    m = torch.from_numpy(np.stack([pipeline.bev_rotation_matrix(a, 500, 500) for a in np.linspace(-20, 20, batch)])).to(dev)
    out = torch.empty((batch, 160, 160), dtype=torch.int64, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _lib.call('tfb_bev_label_prep', plane, m, batch, 500, 500, out)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            _lib.call('tfb_bev_label_prep', plane, m, batch, 500, 500, out)
    g.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / n)
    return sorted(times)[len(times) // 2], times


def make_trainer(mode, dev):
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    torch.manual_seed(0)
    return Trainer(TrainConfig(), dev, gemm_mode='bf16', lr=1e-4, seed=0, raw_inputs=mode)


def time_replays(tr, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        tr.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=10)
    ap.add_argument('--workers', default='1,4')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/dataset_step.py measures on a GPU; none is visible')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    tmp = tempfile.mkdtemp()
    try:
        root = synthetic_route.write_dataset(os.path.join(tmp, 'data'), routes=(('route_a', 21, 24), ('route_b', 22, 24)),
                                             n_points=(20000, 30000))
        out = {'gpu': gpu_identity(0), 'batch': args.batch, 'reader': {}}
        batch = None
        for w in [int(x) for x in args.workers.split(',')]:
            rate, loader = reader_rate(root, args.batch, w)
            out['reader']['workers_%d' % w] = {'samples_per_s': round(rate, 1), 'samples_per_s_per_worker': round(rate / w, 1)}
            if batch is None:
                batch = next(iter(loader))
            del loader
        us, all_us = kernel_us(args.batch, dev)
        out['bev_label_prep_us'] = {'median': round(us, 2), 'runs': [round(x, 2) for x in all_us]}

        from transfuser_b200 import pipeline
        from transfuser_b200.config import TrainConfig
        p = pipeline.InputPipeline(TrainConfig(), dev).prepare({'rgb': batch['rgb_u8'], 'points': batch['points'], 'transforms': batch['transforms'],
                                                                'target_point': batch['target_point64'], 'bev_u8': batch['bev_u8'],
                                                                'bev_matrix': batch['bev_matrix']})
        raw_batch = dict(batch, bev=p['bev'].cpu().pin_memory())
        trainers = {}
        for mode, b in (('dataset', batch), ('raw', raw_batch)):
            tr = make_trainer('dataset' if mode == 'dataset' else True, dev)
            assert tr.capture(b), tr.graph_error
            for _ in range(3):
                tr.replay()
            trainers[mode] = tr
        torch.cuda.synchronize()
        times = {k: [] for k in trainers}
        for _ in range(args.rounds):
            for k, tr in trainers.items():
                times[k].append(time_replays(tr, args.steps))
        out['step_ms'] = {k: {'runs': [round(x, 3) for x in v], 'median': round(sorted(v)[len(v) // 2], 3)} for k, v in times.items()}
        out['graph_launches'] = {k: tr.graph_launches for k, tr in trainers.items()}
        print(json.dumps(out), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()
