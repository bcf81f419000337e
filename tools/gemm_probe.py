"""Diagnostic (not a test): prints the error of every GEMM mode on a few shapes without stopping at the first failure."""
import sys
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from transfuser_b200 import _lib

torch.manual_seed(0)
res = []
for (M, N, K) in [(128, 64, 32), (128, 128, 32), (128, 128, 64), (256, 128, 256), (300, 72, 72), (1740, 1512, 1512)]:
    for ta, tb in [(0, 1), (0, 0), (1, 0), (1, 1)]:
        a = torch.randn((K, M) if ta else (M, K), device='cuda')
        b = torch.randn((N, K) if tb else (K, N), device='cuda')
        ref = (a.double().t() if ta else a.double()) @ (b.double().t() if tb else b.double())
        for name in ('tfb_gemm_f32_simt', 'tfb_gemm_tf32_tc', 'tfb_gemm_bf16_tc'):
            out = torch.full((M, N), float('nan'), device='cuda')
            try:
                if name == 'tfb_gemm_f32_simt':
                    _lib.call(name, ta, tb, M, N, K, a, a.stride(0), b, b.stride(0), out, N, None, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0)
                elif name == 'tfb_gemm_tf32_tc':
                    _lib.call(name, ta, tb, M, N, K, a, a.stride(0), b, b.stride(0), out, N, None, 0, 1.0, 0.0, 1)
                else:
                    if a.stride(0) % 8 or b.stride(0) % 8:
                        continue
                    ah, bh = a.bfloat16(), b.bfloat16()
                    ref_h = (ah.double().t() if ta else ah.double()) @ (bh.double().t() if tb else bh.double())
                    _lib.call(name, ta, tb, M, N, K, ah, ah.stride(0), bh, bh.stride(0), out, N, None, 0, 1.0, 0.0, 1)
                torch.cuda.synchronize()
                r = ref_h if name.endswith('bf16_tc') else ref
                err = ((out.double() - r).norm() / r.norm()).item()
                nan = int(torch.isnan(out).sum())
            except Exception as e:  # noqa
                err, nan = repr(e), -1
            line = '%-18s M=%5d N=%5d K=%5d ta=%d tb=%d  relerr=%s nan=%s' % (name, M, N, K, ta, tb, err, nan)
            print(line, flush=True)
            res.append(line)
os.makedirs('tools_out', exist_ok=True)
open('tools_out/gemm_probe.txt', 'w').write('\n'.join(res) + '\n')
