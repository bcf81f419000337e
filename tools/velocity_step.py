"""Time the captured training step with use_velocity on and off, per backbone at its BASELINE batch (transFuser 10, geometric
fusion 12, late fusion 16), alternated in rounds in one process. Each setting gets a fresh Trainer from the same seed and the
same host batch. Reports the median ms per replay (CUDA events), the launches per captured graph, and the card name and power
limit read in the same run. Writes tools_out/velocity_step.json.

    python tools/velocity_step.py [--rounds 5] [--iters 20]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = [('transFuser', 10), ('geometric_fusion', 12), ('late_fusion', 16)]   # BASELINE.json configs[1..4] batches


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return 'unknown (%s)' % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    from bench import make_host_batch
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    assert torch.cuda.is_available(), 'tools/velocity_step.py measures on the GPU'
    dev = torch.device('cuda', 0)
    out = dict(card=_card(), configs=[])
    for backbone, B in CONFIGS:
        host = make_host_batch(B, seed=3, torch=torch, np=np, backbone=backbone)
        trs = {}
        for vel in (False, True):
            torch.manual_seed(0)
            tr = Trainer(TrainConfig(), dev, gemm_mode='bf16', seed=0, backbone=backbone, use_velocity=vel)
            assert tr.capture(host), tr.graph_error
            trs[vel] = tr
        times = {False: [], True: []}
        for _ in range(args.rounds):
            for vel in (False, True):
                tr = trs[vel]
                tr.replay()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    tr.replay()
                e1.record()
                torch.cuda.synchronize()
                times[vel].append(e0.elapsed_time(e1) / args.iters)
        row = dict(backbone=backbone, batch=B,
                   off_ms=round(float(np.median(times[False])), 3), on_ms=round(float(np.median(times[True])), 3),
                   off_rounds=[round(t, 3) for t in times[False]], on_rounds=[round(t, 3) for t in times[True]],
                   off_launches=trs[False].graph_launches, on_launches=trs[True].graph_launches)
        row['delta_ms'] = round(row['on_ms'] - row['off_ms'], 3)
        out['configs'].append(row)
        print(json.dumps(row), flush=True)
        del trs
        torch.cuda.empty_cache()
    print('card:', out['card'])
    os.makedirs(os.path.join(ROOT, 'tools_out'), exist_ok=True)
    with open(os.path.join(ROOT, 'tools_out', 'velocity_step.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
