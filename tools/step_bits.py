"""Digests of one captured bf16 training step per backbone, for showing that a change leaves the bits of the benchmark path alone.

    python tools/step_bits.py OUT.json [--root TREE] [--batch B]
    python tools/step_bits.py --compare A.json B.json

For each backbone a Trainer (bf16 tensor-core mode, raw inputs, the seeded batch of bench.py) captures its step into a CUDA graph
and replays it once. The script records the weighted loss and the 11 loss terms as fp32 bit patterns, and SHA-256 digests of the
whole flat gradient and parameter buffers after the step. --root imports the package from another tree (an older build, say), so
two builds can be run from the same script and compared with --compare."""
import argparse
import hashlib
import json
import os
import sys


def digests(root, batch):
    sys.path.insert(0, root)
    import numpy as np
    import torch
    from bench import make_host_batch
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    import transfuser_b200
    assert os.path.dirname(os.path.dirname(os.path.abspath(transfuser_b200.__file__))) == os.path.abspath(root)
    out = {}
    for backbone in ('transFuser', 'late_fusion', 'geometric_fusion', 'latentTF'):
        torch.manual_seed(0)
        tr = Trainer(TrainConfig(), 'cuda', gemm_mode='bf16', lr=1e-4, seed=0, backbone=backbone, raw_inputs=True)
        host = make_host_batch(batch, seed=100, torch=torch, np=np, backbone=backbone, raw=True)
        assert tr.capture(host), tr.graph_error
        loss = tr.replay()
        torch.cuda.synchronize()
        bits = lambda t: '%08x' % (t.detach().float().reshape(1).view(torch.int32).item() & 0xFFFFFFFF)
        sha = lambda t: hashlib.sha256(t.detach().cpu().numpy().tobytes()).hexdigest()
        out[backbone] = dict(loss=bits(loss), terms={k: bits(v) for k, v in tr.last_losses.items()},
                             grad=sha(tr.flat.grad), params=sha(tr.flat.flat), n=int(tr.flat.total))
        print(backbone, out[backbone]['loss'], out[backbone]['grad'][:16], out[backbone]['params'][:16], flush=True)
        del tr
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out', nargs='?')
    ap.add_argument('--root', default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument('--batch', type=int, default=10)
    ap.add_argument('--compare', nargs=2, metavar='JSON')
    a = ap.parse_args()
    if a.compare:
        x, y = (json.load(open(p)) for p in a.compare)
        same = x == y
        for bb in sorted(set(x) | set(y)):
            print('%-18s %s' % (bb, 'identical' if x.get(bb) == y.get(bb) else 'DIFFERENT'))
        sys.exit(0 if same else 1)
    res = digests(a.root, a.batch)
    with open(a.out, 'w') as f:
        json.dump(res, f, indent=1, sort_keys=True)


if __name__ == '__main__':
    main()
