"""Time one validation batch three ways, alternated in rounds in one process, per trunk configuration:
  eager    the reference-style loop: eval-mode forward, then one .item() per loss and one for the total (train.py:333-340);
  unfused  the captured Validator with the eval-mode BatchNorms as separate launches (ops.bn_epilogue_path patched to None);
  fused    the captured Validator with the BatchNorms in the tensor-core conv / GEMM epilogues.
Reports the median ms per batch (CUDA events), the launches per captured graph, whether the three give the same loss bits, and the
card name and power limit read in the same run. Writes tools_out/eval_step.json.

    python tools/eval_step.py [--rounds 5] [--iters 10]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = [('regnety_032', 'regnety_032', 10), ('resnet34', 'resnet18', 10)]   # BASELINE configs[1]: batch 10, RegNetY x 2


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return 'unknown (%s)' % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=10)
    args = ap.parse_args()
    from bench import make_host_batch
    from transfuser_b200 import ops
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer, Validator
    assert torch.cuda.is_available(), 'tools/eval_step.py measures on the GPU'
    dev = torch.device('cuda', 0)
    card = _card()
    out = dict(card=card, configs=[])
    real_path = ops.bn_epilogue_path
    for img, lid, B in CONFIGS:
        torch.manual_seed(0)
        tr = Trainer(TrainConfig(), dev, gemm_mode='bf16', seed=0, image_architecture=img, lidar_architecture=lid)
        host = make_host_batch(B, seed=3, torch=torch, np=np)
        batch = {k: v.to(dev) for k, v in host.items()}
        vals, bits = {}, {}
        for name in ('unfused', 'fused'):
            ops.bn_epilogue_path = real_path if name == 'fused' else (lambda *a: None)
            v = Validator(tr)
            v.capture(host)
            v.load(host)
            v.replay()
            bits[name] = torch.stack([x.reshape(()) for x in v.static_losses.values()]).view(torch.int32).cpu()
            vals[name] = v
        ops.bn_epilogue_path = real_path

        def eager():
            was = tr.net.training
            tr.net.eval()
            with torch.no_grad():
                d, lidar = tr.expand_inputs(batch)
                losses = tr.forward_losses(d, lidar)
                loss = torch.tensor(0.0, device=dev)
                for k, x in losses.items():
                    loss += tr.weights[k] * x
                    float(tr.weights[k] * x.item())
                float(loss.item())
            tr.net.train(was)
            return losses
        el = eager()
        bits['eager'] = torch.stack([x.reshape(()) for x in el.values()]).view(torch.int32).cpu()
        arms = dict(eager=eager, unfused=vals['unfused'].replay, fused=vals['fused'].replay)
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                fn()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) / args.iters)
        res = dict(image=img, lidar=lid, batch=B, card=card,
                   ms_median={k: round(float(np.median(v)), 3) for k, v in times.items()},
                   ms_range={k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                   graph_launches=dict(unfused=vals['unfused'].graph_launches, fused=vals['fused'].graph_launches),
                   same_loss_bits=bool(torch.equal(bits['eager'], bits['fused']) and torch.equal(bits['unfused'], bits['fused'])))
        print(json.dumps(res), flush=True)
        out['configs'].append(res)
        del tr, vals
        torch.cuda.empty_cache()
    os.makedirs(os.path.join(ROOT, 'tools_out'), exist_ok=True)
    with open(os.path.join(ROOT, 'tools_out', 'eval_step.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
