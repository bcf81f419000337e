"""ms / step of the bench workload (BASELINE configs[1]: TransFuser, batch 10, all heads, dropout 0.1, bf16, raw inputs, captured
CUDA graph) with each trunk pair, regnety_032 x 2 and resnet34 / resnet18, alternated in one process. Every round builds a fresh
Trainer from the same seed, runs the warm-up and the capture, and times STEPS replays with CUDA events; the losses and a seeded
sample of the gradients after the last replay must be byte-identical across the rounds of a pair. Prints one JSON line.
    python tools/arch_step.py [--rounds 3] [--steps 20]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import gpu_identity, make_host_batch  # noqa: E402

PAIRS = {'regnety_032': ('regnety_032', 'regnety_032'), 'resnet34/resnet18': ('resnet34', 'resnet18')}


def one_round(trunks, host, steps, dev):
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    torch.manual_seed(0)
    tr = Trainer(TrainConfig(), dev, gemm_mode='bf16', lr=1e-4, seed=0, raw_inputs=True, image_architecture=trunks[0],
                 lidar_architecture=trunks[1])
    d = {k: v.to(dev) for k, v in host.items()}
    for _ in range(3):
        tr.step(d)
    assert tr.capture(host), tr.graph_error
    for _ in range(2):
        tr.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = tr.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    g = tr.flat.grad
    idx = torch.from_numpy(np.random.default_rng(0).integers(0, g.numel(), 4096)).to(dev)
    sig = (loss.detach().float().cpu().numpy().tobytes(), g[idx].cpu().numpy().tobytes(), tr.flat.flat[idx].cpu().numpy().tobytes())
    del tr
    torch.cuda.empty_cache()
    return ms, sig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--batch', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/arch_step.py measures on a GPU; none is visible')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    host = make_host_batch(args.batch, seed=100, torch=torch, np=np, raw=True)
    times = {k: [] for k in PAIRS}
    sigs = {k: [] for k in PAIRS}
    for _ in range(args.rounds):
        for name, trunks in PAIRS.items():
            ms, sig = one_round(trunks, host, args.steps, dev)
            times[name].append(ms)
            sigs[name].append(sig)
    out = {'gpu': gpu_identity(0), 'batch': args.batch, 'steps_per_round': args.steps, 'rounds': args.rounds, 'pairs': {}}
    for name in PAIRS:
        t = sorted(times[name])
        out['pairs'][name] = {'ms_per_step': [round(x, 3) for x in times[name]], 'median_ms': round(t[len(t) // 2], 3),
                              'samples_per_s': round(args.batch * 1e3 / t[len(t) // 2], 2),
                              'rounds_byte_identical': all(s == sigs[name][0] for s in sigs[name])}
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
