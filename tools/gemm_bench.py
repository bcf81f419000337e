"""Micro-benchmark of the tensor-core GEMM on the shapes of the training step (CUDA events, L2 flushed between launches)."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from transfuser_b200 import _lib

SHAPES = [  # (ta, tb, M, N, K, splits, tag)
    (0, 1, 1740, 1512, 1512, 1, 'gpt4 proj fwd'), (0, 0, 1740, 1512, 1512, 1, 'gpt4 proj dgrad'), (1, 0, 1512, 1512, 1740, 1, 'gpt4 proj wgrad'),
    (0, 1, 1740, 6048, 1512, 1, 'gpt4 fc1 fwd'), (0, 1, 1740, 1512, 6048, 1, 'gpt4 fc2 fwd'), (1, 0, 6048, 1512, 1740, 1, 'gpt4 fc1 wgrad'),
    (0, 1, 4400, 576, 576, 1, 's3 1x1 fwd'), (1, 0, 576, 576, 4400, 2, 's3 1x1 wgrad'), (0, 1, 70400, 72, 72, 1, 's1 1x1 fwd'),
    (0, 1, 17600, 216, 216, 1, 's2 1x1 fwd'), (0, 1, 1740, 2304, 576, 1, 'gpt3 fc1 fwd'),
]
flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
out = []
for ta, tb, M, N, K, splits, tag in SHAPES:
    a = torch.randn((K, M) if ta else (M, K), device='cuda').bfloat16()
    b = torch.randn((N, K) if tb else (K, N), device='cuda').bfloat16()
    c = torch.empty(M, N, device='cuda')
    ts = []
    for it in range(8):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.call('tfb_gemm_bf16_tc', ta, tb, M, N, K, a, a.stride(0), b, b.stride(0), c, N, None, 0, 1.0, 0.0, splits)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    t = sorted(ts[2:])[len(ts[2:]) // 2]
    ref = (a.float().t() if ta else a.float()) @ (b.float().t() if tb else b.float())     # same bf16 operands, fp32 product
    err = ((c - ref).norm() / ref.norm()).item()
    line = '%-18s ta%d tb%d M%6d N%5d K%5d  %8.1f us  %7.1f TF/s  rel err %.1e%s' % (
        tag, ta, tb, M, N, K, t * 1e3, 2.0 * M * N * K / (t * 1e-3) / 1e12, err, '' if err < 1e-3 else '  <-- WRONG')
    print(line, flush=True)
    out.append(line)
os.makedirs('tools_out', exist_ok=True)
open('tools_out/gemm_bench_%s.txt' % (os.environ.get('TFB_GEMM_BN') or ('model' + os.environ['TFB_GEMM_TILE_MODEL'] if 'TFB_GEMM_TILE_MODEL' in os.environ else 'auto')), 'w').write('\n'.join(out) + '\n')
