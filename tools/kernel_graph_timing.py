"""Per-kernel time of the training step WITHOUT host launch gaps (run on the GPU box):
    python tools/kernel_graph_timing.py [entry point, default tfb_gemm_bf16_tc] [--batch 10]
Runs one eager step, records every call of the chosen C-ABI entry point with its arguments (tensors kept alive), captures exactly
those launches — in their original order, same operands — into ONE CUDA graph and times the replay with CUDA events. The eager
per-call timing of bench.py includes the ~15 us Python launch path whenever the GPU is ahead of the host, which inflates the
average of kernels shorter than that; this number does not. Writes tools_out/kernel_graph_timing_<name>.txt."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from transfuser_b200 import _lib  # noqa: E402
from transfuser_b200.config import TrainConfig  # noqa: E402
from transfuser_b200.trainer import Trainer  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('name', nargs='?', default='tfb_gemm_bf16_tc')
    ap.add_argument('--batch', type=int, default=10)
    ap.add_argument('--replays', type=int, default=20)
    a = ap.parse_args()
    import numpy as np
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    tr = Trainer(TrainConfig(), dev, gemm_mode='bf16')
    host = bench.make_host_batch(a.batch, 0, torch, np)
    d = {k: v.to(dev) for k, v in host.items()}
    for _ in range(2):
        tr.step(d)
    torch.cuda.synchronize()
    lib = _lib.lib()
    calls, orig = [], lib.call

    def rec(name, *args):
        if name == a.name:
            calls.append(args)
        return orig(name, *args)
    lib.call = rec
    tr.step(d)
    torch.cuda.synchronize()
    lib.call = orig
    if not calls:
        print('no calls of', a.name)
        return
    work = [_lib.Profiler._work(a.name, c) for c in calls]
    flops, byts = sum(w[0] for w in work), sum(w[1] for w in work)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for c in calls:
            orig(a.name, *c)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for c in calls:
            orig(a.name, *c)
    for _ in range(3):
        g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(a.replays):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.replays
    pk, how = bench.peaks()
    lines = ['%s: %d launches per step, %.3f ms per step in a dedicated graph, %.2f us per launch' % (a.name, len(calls), ms, 1e3 * ms / len(calls))]
    if flops > 0:
        tf = flops / (ms * 1e-3) / 1e12
        lines.append('algorithmic %.2f GFLOP per step -> %.1f TFLOP/s = %.4f of the %s bf16 peak %.1f' % (flops / 1e9, tf, tf / pk['bf16_tflops_sustained'], how, pk['bf16_tflops_sustained']))
    if byts > 0:
        gb = byts / (ms * 1e-3) / 1e9
        lines.append('algorithmic %.1f MB per step -> %.1f GB/s = %.4f of the HBM peak %.1f' % (byts / 1e6, gb, gb / pk['hbm_gbs'], pk['hbm_gbs']))
    print('\n'.join(lines))
    os.makedirs(os.path.join(ROOT, 'tools_out'), exist_ok=True)
    open(os.path.join(ROOT, 'tools_out', 'kernel_graph_timing_%s.txt' % a.name), 'w').write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
