"""The geometric-fusion correspondences, measured. Reports one JSON line:
  - kernel:  tfb_lidar_cam_correspondences at batch B with 40k-point sweeps (random, oracle/correspondence_oracle.py), CUDA events
             over a CUDA graph of 200 launches, median of 5 replays; with the card's name and power limit;
  - step:    Trainer(backbone='geometric_fusion', raw_inputs='dataset') against Trainer(raw_inputs=True) fed the same batch with the
             BEV label and the correspondences the pipeline made, both captured, bf16, rounds alternated; ms per step (medians);
  - host:    the reference's lidar_bev_cam_correspondences per sample on the host's CPU, on the same sweeps, when a reference
             checkout is present (oracle/ref_import.py; --host-only measures just that, without a GPU).
    python tools/correspondence_step.py [--batch 12] [--points 40000] [--rounds 5] [--steps 20] [--host-only]"""
import argparse
import copy
import json
import os
import random
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from oracle import correspondence_oracle as CO, ref_import, synthetic_route  # noqa: E402


def host_reference_ms(sweeps):
    """ms per sample of the verbatim reference function (random.sample as in the reference), one call per sweep."""
    if not ref_import.available():
        return None
    fn = ref_import.load_data_fns(['lidar_bev_cam_correspondences', 'correspondences_at_one_scale'])['lidar_bev_cam_correspondences']
    fn.__globals__.update(random=random, deepcopy=copy.deepcopy)
    times = []
    for s in sweeps:
        w = s[:, :3].copy()
        t0 = time.perf_counter()
        fn(w)
        times.append((time.perf_counter() - t0) * 1e3)
    return {'median': round(sorted(times)[len(times) // 2], 2), 'runs': [round(t, 2) for t in times]}


def kernel_us(sweeps, dev, n=200):
    from transfuser_b200 import _lib, pipeline
    B, N = len(sweeps), max(len(s) for s in sweeps)
    pts = np.zeros((B, N, 4), np.float32)
    for b, s in enumerate(sweeps):
        pts[b, :len(s)] = s
        pts[b, :len(s), 1] *= -1
    points = torch.from_numpy(pts).to(dev)
    nv = torch.tensor([len(s) for s in sweeps], dtype=torch.int32, device=dev)
    seed = torch.arange(B, dtype=torch.int64, device=dev) * 7919 + 1
    consts, dz = pipeline.correspondence_constants()
    consts = torch.from_numpy(consts).to(dev)
    work = torch.empty((B, 6 * N), dtype=torch.int32, device=dev)
    bev = torch.empty((B, 8, 8, 5, 2), dtype=torch.int64, device=dev)
    cam = torch.empty((B, 22, 5, 5, 2), dtype=torch.int64, device=dev)
    args = (points, nv, seed, consts, float(dz), B, N, work, bev, cam)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _lib.call('tfb_lidar_cam_correspondences', *args)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            _lib.call('tfb_lidar_cam_correspondences', *args)
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
    return {'median': round(sorted(times)[len(times) // 2], 2), 'runs': [round(t, 2) for t in times]}


def step_ms(root, batch, dev, rounds, steps):
    from dataset_step import time_replays
    from transfuser_b200 import pipeline
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.dataset import CarlaRawDataset, collate
    from transfuser_b200.trainer import Trainer
    ds = CarlaRawDataset([root], TrainConfig(), backbone='geometric_fusion', correspondences='gpu', max_points=40000)
    random.seed(0)
    b = collate([ds[i % len(ds)] for i in range(batch)])
    p = pipeline.InputPipeline(TrainConfig(), dev).prepare({'rgb': b['rgb_u8'], 'points': b['points'], 'n_valid': b['n_valid'],
                                                            'transforms': b['transforms'], 'target_point': b['target_point64'],
                                                            'bev_u8': b['bev_u8'], 'bev_matrix': b['bev_matrix'], 'corr_seed': b['corr_seed']})
    raw_b = dict(b, bev=p['bev'].cpu().pin_memory(), bev_points=p['bev_points'].cpu().pin_memory(), cam_points=p['cam_points'].cpu().pin_memory())
    trainers = {}
    for mode, bb in (('dataset', b), ('raw', raw_b)):
        torch.manual_seed(0)
        tr = Trainer(TrainConfig(), dev, gemm_mode='bf16', lr=1e-4, seed=0, raw_inputs='dataset' if mode == 'dataset' else True,
                     backbone='geometric_fusion')
        assert tr.capture(bb), tr.graph_error
        for _ in range(3):
            tr.replay()
        trainers[mode] = tr
    torch.cuda.synchronize()
    times = {k: [] for k in trainers}
    for _ in range(rounds):
        for k, tr in trainers.items():
            times[k].append(time_replays(tr, steps))
    out = {k: {'runs': [round(x, 3) for x in v], 'median': round(sorted(v)[len(v) // 2], 3)} for k, v in times.items()}
    return out, {k: tr.graph_launches for k, tr in trainers.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=12)
    ap.add_argument('--points', type=int, default=40000)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--host-only', action='store_true')
    args = ap.parse_args()
    sweeps = [CO.random_sweep(args.points, 100 + b) for b in range(args.batch)]
    out = {'batch': args.batch, 'points': args.points, 'host_reference_ms_per_sample': host_reference_ms(sweeps)}
    if args.host_only:
        import platform
        out['cpu'] = platform.processor() or platform.machine()
        print(json.dumps(out), flush=True)
        return
    if not torch.cuda.is_available():
        raise SystemExit('tools/correspondence_step.py measures on a GPU; none is visible (--host-only measures the host side)')
    from bench import gpu_identity
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    out['gpu'] = gpu_identity(0)
    out['kernel_us'] = kernel_us(sweeps, dev)
    tmp = tempfile.mkdtemp()
    try:
        root = synthetic_route.write_dataset(os.path.join(tmp, 'data'), routes=(('route_a', 21, 24),), n_points=(20000, 30000))
        out['step_ms'], out['graph_launches'] = step_ms(root, args.batch, dev, args.rounds, args.steps)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
