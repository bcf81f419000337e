"""Per-shape timing of the 3x3 weight gradients of the bench step (measurement tool, not product code).

Records every bf16 tensor-core 3x3 wgrad of one eager training step (bench.py's default workload: TransFuser RegNetY-3.2GF, batch
10), then times each distinct shape two ways, each in a CUDA graph of its own (REPS calls per replay, CUDA events around replays):
im2col + the batched wgrad GEMM, and the same GEMM gathering its tiles from the activation (tfb_conv3x3_tc_wgrad). Prints one JSON
line per shape: the count per step, microseconds per call, the gathered path's algorithmic bytes (bf16 x and dy read, fp32 dW
written) and its achieved rate against the H100 SXM data-sheet HBM bandwidth (3.35 TB/s).

    python tools/wgrad_shapes.py [--batch 10]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0
REPS = 20


def record(batch):
    import numpy as np
    import torch
    import bench
    from transfuser_b200 import ops
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    dev = torch.device('cuda', 0)
    shapes = {}
    orig = ops._conv_wgrad_tc

    def spy(x, g16, w, groups, stride, implicit=False):
        key = (tuple(x.shape), w.shape[0], g16.shape[-1], groups, stride, implicit)
        shapes[key] = shapes.get(key, 0) + 1
        return orig(x, g16, w, groups, stride, implicit)

    ops._conv_wgrad_tc = spy
    try:
        host = bench.make_host_batch(batch, seed=100, torch=torch, np=np, backbone='transFuser', raw=True)
        tr = Trainer(TrainConfig(), dev, gemm_mode='bf16', lr=1e-4, seed=0, backbone='transFuser', raw_inputs=True)
        tr.step({k: v.to(dev) for k, v in host.items()})
        torch.cuda.synchronize()
    finally:
        ops._conv_wgrad_tc = orig
    return shapes


def time_shape(key):
    import torch
    from transfuser_b200 import ops
    (N, H, W, Cin), Cout, ldg, groups, stride, _ = key
    dev = torch.device('cuda', 0)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    x = torch.randn(N, H, W, Cin, device=dev)
    x16 = x.bfloat16()
    g16 = torch.zeros(N, Ho, Wo, ldg, device=dev, dtype=torch.bfloat16)
    g16[..., :Cout] = torch.randn(N, Ho, Wo, Cout, device=dev).bfloat16()
    w = torch.zeros(Cout, Cin // groups, 3, 3, device=dev)
    res = {}
    for implicit in (False, True):
        def run():
            ops._COL_CACHE.clear()
            ops._attach16(x, x16)
            ops._conv_wgrad_tc(x, g16, w, groups, stride, implicit)
        s = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(s):
            for _ in range(3):
                run()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                for _ in range(REPS):
                    run()
            for _ in range(3):
                g.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
        res[implicit] = e0.elapsed_time(e1) * 1e3 / (10 * REPS)
    nbytes = 2.0 * (N * H * W * Cin + N * Ho * Wo * ldg) + 4.0 * Cout * (Cin // groups) * 9
    return res[False], res[True], nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=10)
    args = ap.parse_args()
    import torch
    from transfuser_b200 import ops
    torch.cuda.set_device(0)
    shapes = record(args.batch)
    ops.WGRAD_STREAM = False                     # time each path by itself, with the grid cap the step gives the GEMM
    tot = [0.0, 0.0]
    from transfuser_b200 import _lib
    for key, count in sorted(shapes.items(), key=lambda kv: -kv[0][0][0] * kv[0][0][1] * kv[0][0][2] * kv[0][0][3]):
        _lib.call('tfb_gemm_set_max_ctas', ops.WGRAD_MAX_CTAS)
        try:
            t_col, t_imp, nbytes = time_shape(key)
        finally:
            _lib.call('tfb_gemm_set_max_ctas', 0)
        tot[0] += count * t_col
        tot[1] += count * t_imp
        (N, H, W, Cin), Cout, ldg, groups, stride, implicit = key
        print(json.dumps({'x': [N, H, W, Cin], 'Cout': Cout, 'ldg': ldg, 'groups': groups, 'stride': stride, 'implicit_site': implicit,
                          'count': count, 'im2col_gemm_us': round(t_col, 2), 'implicit_us': round(t_imp, 2), 'implicit_MB': round(nbytes / 1e6, 2),
                          'implicit_GBs': round(nbytes / t_imp / 1e3, 1), 'of_hbm_peak': round(nbytes / t_imp / 1e3 / HBM_GBS, 3)}), flush=True)
    print(json.dumps({'total_per_step_us': {'im2col_gemm': round(tot[0], 1), 'implicit': round(tot[1], 1)}}), flush=True)


if __name__ == '__main__':
    main()
