"""Where the fixed-order cross-CTA sums of a training step go (run on the GPU box):
    python tools/fold_attribution.py [--batch 10] [--out DIR]
For every C-ABI entry point whose launches end in an ordered fold (split-K tiles, BatchNorm statistics of the GEMM / conv
epilogues, norm.cu column reductions, squeeze-excite pooling), records its calls of one eager step, replays exactly those launches in
a dedicated CUDA graph (kernel_graph_timing.graph_ms) and prints the time per step, next to the fold size of each launch: partial
rows x outputs and the bytes of partials, from the shapes and the launchers' grid / split choices. Writes DIR/fold_attribution.txt
(default tools_out/)."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

import kernel_graph_timing as kgt  # noqa: E402
from transfuser_b200 import _lib  # noqa: E402

NAMES = ('tfb_gemm_bf16_tc_stats', 'tfb_conv3x3_tc_strided', 'tfb_gemm_bf16_tc', 'tfb_gemm_bf16_tc_wgrad_batched', 'tfb_bn_fwd',
         'tfb_bn_fwd_stats', 'tfb_bn_bwd', 'tfb_bn_bwd_se', 'tfb_colsum', 'tfb_grad_prep', 'tfb_layernorm_bwd', 'tfb_add_dropout_ln_bwd',
         'tfb_pool_hw_fwd', 'tfb_se_bwd_reduce')


def cdiv(a, b):
    return -(-a // b)


def pick_bn(M, N, zs, step, sms, num_kb=0, auto=False):
    """(tile width, splits) as gemm_tc.cu's pick_bn chooses them."""
    nmax, mt, best = cdiv(N, step) * step, cdiv(M, 128), None
    for bn in range(step, 193, step):
        use = min(bn, nmax)
        tiles = mt * cdiv(N, use) * zs
        s = 1
        if auto and num_kb > 0:
            s = max(1, min(sms // tiles, num_kb // 4))
            kbs = cdiv(num_kb, s)
            s = cdiv(num_kb, kbs)
            cost = cdiv(tiles * s, sms) * (kbs * (128 + use) + 6 * 256 + (4 * use if s > 1 else 0))
        else:
            cost = cdiv(tiles, sms) * (128 + use + 64)
        if best is None or cost < best[0] or (cost == best[0] and use > best[1]):
            best = (cost, use, s)
        if use == nmax:
            break
    return best[1], best[2]


def colreduce_rows(M, C, sms, flat_ok=True):
    """(partial rows, slabs) of norm.cu's launch_colreduce for a 16-byte aligned [M, C] matrix."""
    if flat_ok and C % 4 == 0 and C // 4 <= 128 and M >= 4096:
        return max(1, min(cdiv(M, (256 // (C // 4)) * 8), 4 * sms)), 1
    slabs = cdiv(C // 4, 32) if C % 4 == 0 else cdiv(C, 32)
    return max(1, min(cdiv(4 * sms, slabs), cdiv(M, 128), 65535)), slabs


def pool_rows(N, HW, C, sms):
    if C // 4 <= 128 and HW >= 1024:
        return max(1, min(cdiv(HW, (256 // (C // 4)) * 16), cdiv(4 * sms, N)))
    return min(cdiv(HW, 256), 32)


def folds(name, a, sms, cap):
    """[(what, partial rows, outputs, bytes of partials)] of one call."""
    wsms = cap if 0 < cap < sms else sms
    if name == 'tfb_gemm_bf16_tc_stats':
        M, N = a[0], a[1]
        bn, _ = pick_bn(M, N, 1, 32, wsms)
        rows = min(cdiv(M, 128) * cdiv(N, bn), wsms)
        return [('BN statistics', rows, 2 * N, 4 * rows * 2 * N)]
    if name == 'tfb_conv3x3_tc_strided':
        N, H, W, Cx, Cy, NB, KC, c_step, nchunks, nb_real, gblocks, relu, stride, stats = a[4:18]
        if stats is None:
            return []
        Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
        total = cdiv(Wo, 16) * cdiv(Ho, 8) * N * gblocks
        stage = 128 * KC * 2 + NB * KC * 2
        smem = (6 if NB <= 64 else 4) * stage + 256 + 8 * 576 * 4 + 1024 + (2 * Cy + 8 * 2 * 256) * 4
        rows = min(total, sms * (2 if smem <= 110 * 1024 else 1))
        return [('BN statistics', rows, 2 * Cy, 4 * rows * 2 * Cy)]
    if name in ('tfb_gemm_bf16_tc', 'tfb_gemm_bf16_tc_wgrad_batched'):
        if name == 'tfb_gemm_bf16_tc':
            tb, M, N, K, relu, beta, splits = a[1], a[2], a[3], a[4], a[12], a[14], a[15]
            nbatch, step = 1, 64 if tb == 0 else 32
            auto = splits <= 0 and not relu and beta in (0.0, 1.0)
        else:
            M, N, K, nbatch, splits = a[0], a[1], a[2], a[12], a[13]
            step, auto = 64, splits <= 0
        num_kb = cdiv(K, 64)
        if auto:
            _, splits = pick_bn(M, N, nbatch, step, wsms, num_kb, True)
        splits = min(max(splits, 1), num_kb)
        splits = cdiv(num_kb, cdiv(num_kb, splits))
        if splits <= 1:
            return []
        return [('split-K', splits, nbatch * M * N, 4 * splits * nbatch * M * N)]
    if name in ('tfb_bn_fwd', 'tfb_bn_bwd', 'tfb_bn_bwd_se', 'tfb_colsum', 'tfb_grad_prep', 'tfb_layernorm_bwd', 'tfb_add_dropout_ln_bwd'):
        i = {'tfb_bn_fwd': 2, 'tfb_bn_bwd': 3, 'tfb_bn_bwd_se': 3, 'tfb_colsum': 2, 'tfb_grad_prep': 6, 'tfb_layernorm_bwd': 3,
             'tfb_add_dropout_ln_bwd': 5}[name]      # position of M (rows); C follows
        M, C = a[i], a[i + 1]
        nsums = C if name in ('tfb_colsum', 'tfb_grad_prep') else 2 * C
        out = []
        if name == 'tfb_grad_prep':
            if a[4] is not None:
                out.append(('bias gradient', colreduce_rows(M, C, sms, False)[0], C, 8 * colreduce_rows(M, C, sms, False)[0] * C))
        elif name in ('tfb_layernorm_bwd', 'tfb_add_dropout_ln_bwd'):
            rows = max(1, min(cdiv(M, 64), 64))
            out.append(('LayerNorm parameter gradients', rows, nsums, 8 * rows * nsums))
        else:
            rows = colreduce_rows(M, C, sms, name != 'tfb_colsum' or a[1] == C)[0]
            out.append(('column reduction', rows, nsums, 8 * rows * nsums))
        if name == 'tfb_bn_fwd' and a[16] is not None:
            rows = min(cdiv(M // a[17], 256), 32)
            out.append(('SE pooling', rows, a[17] * C, 4 * rows * a[17] * C))
        return out
    if name == 'tfb_bn_fwd_stats':
        if a[16] is None:
            return []
        M, C, pb = a[2], a[3], a[17]
        rows = pool_rows(pb, M // pb, C, sms)
        return [('SE pooling', rows, pb * C, 4 * rows * pb * C)]
    if name in ('tfb_pool_hw_fwd', 'tfb_se_bwd_reduce'):
        N, HW, C = a[2:5] if name == 'tfb_pool_hw_fwd' else a[3:6]
        rows = min(cdiv(HW, 256), 32) if name == 'tfb_pool_hw_fwd' else pool_rows(N, HW, C, sms)
        return [('SE pooling' if name == 'tfb_pool_hw_fwd' else 'SE gate gradient', rows, N * C, 4 * rows * N * C)]
    return []


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=10)
    ap.add_argument('--replays', type=int, default=20)
    ap.add_argument('--out', default=os.path.join(ROOT, 'tools_out'))
    a = ap.parse_args()
    tr, d = kgt.trainer(a.batch)
    calls = kgt.record(lambda: (tr.step(d), torch.cuda.synchronize()), set(NAMES) | {'tfb_gemm_set_max_ctas'})
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    props = torch.cuda.get_device_properties(0)
    lines = ['%s, %d SMs, batch %d' % (props.name, sms, a.batch), '',
             '%-32s %8s %12s %14s %14s  %s' % ('entry point', 'launches', 'ms per step', 'fold MB/step', 'largest fold', 'rows x outputs')]
    detail, total_ms = [], 0.0
    for name in NAMES:
        cap, mine = 0, []
        for n, c in calls:        # each launch with the weight-gradient grid cap in force when it was made
            if n == 'tfb_gemm_set_max_ctas':
                cap = c[0]
                mine.append((n, c))
            elif n == name:
                mine.append((n, c))
                for what, rows, outs, byts in folds(n, c, sms, cap):
                    detail.append((name, what, rows, outs, byts))
        launches = [(n, c) for n, c in mine if n == name]
        if not launches:
            continue
        while mine and mine[-1][0] == 'tfb_gemm_set_max_ctas':
            mine.pop()
        ms = kgt.graph_ms(mine, a.replays)
        _lib.lib().call('tfb_gemm_set_max_ctas', 0)
        total_ms += ms
        fl = [x for x in detail if x[0] == name]
        big = max(fl, key=lambda x: x[4]) if fl else None
        lines.append('%-32s %8d %12.3f %14.2f %14s  %s' % (name, len(launches), ms, sum(x[4] for x in fl) / 1e6,
                                                           '%.2f MB' % (big[4] / 1e6) if big else '-', '%d x %d' % (big[2], big[3]) if big else '-'))
    lines.append('%-32s %8s %12.3f' % ('all of the above', '', total_ms))
    lines += ['', 'per launch: entry point, fold, partial rows x outputs, MB of partials']
    lines += ['  %-32s %-30s %5d x %-8d %8.3f' % (n, w, r, o, b / 1e6) for n, w, r, o, b in detail]
    print('\n'.join(lines))
    os.makedirs(a.out, exist_ok=True)
    open(os.path.join(a.out, 'fold_attribution.txt'), 'w').write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
