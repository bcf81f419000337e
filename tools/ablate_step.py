"""Critical-path attribution for the captured multi-stream training step (measurement tool, not product code).

The step runs on several streams inside one CUDA graph, so the sum of kernel times (36.7 ms single-stream) says little about where
the 26 ms of the captured step go. This tool answers "how much shorter would the step be if entry point X cost nothing": for each
ablation set it starts a fresh process, builds the Trainer, makes the listed C-ABI entry points return without launching, captures the step and times
graph replays. The step's RESULTS are garbage under ablation (outputs left uninitialised) — only the time is read; there is no
data-dependent control flow in the step, so the remaining launches are the same ones.

    python tools/ablate_step.py                      # the default sets below
    python tools/ablate_step.py tfb_bn_bwd tfb_se_mlp_bwd+tfb_se_bwd_reduce     # '+' joins entry points into one set
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT_SETS = [
    '', 'tfb_bn_bwd', 'tfb_bn_fwd_stats+tfb_bn_fwd',
    'tfb_se_mlp_bwd+tfb_se_bwd_reduce+tfb_se_bwd_apply+tfb_se_scale_fwd+tfb_gemm_small_m',
    'tfb_gemm_bf16_tc+tfb_gemm_bf16_tc_stats+tfb_gemm_bf16_tc_out16', 'tfb_conv3x3_tc+tfb_conv3x3_tc_strided',
    'tfb_layernorm_bwd+tfb_layernorm_fwd+tfb_dropout+tfb_add_dropout_ln_fwd+tfb_add_dropout_ln_bwd+tfb_attn_fwd_tc+tfb_attn_bwd_tc',
    'tfb_grad_prep+tfb_cast_bf16+tfb_dilate2+tfb_subsample2+tfb_colsum',
    'tfb_im2col3x3_bf16+tfb_gemm_bf16_tc_wgrad_batched', 'tfb_conv3x3_tc_wgrad', 'tfb_upsample_bilinear_bwd+tfb_upsample_bilinear_fwd+tfb_gpt_up_add_fwd+tfb_gpt_up_add_bwd',
]


def one(s):
    import numpy as np
    import torch
    import bench
    from transfuser_b200 import _lib
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer

    dev = torch.device('cuda', 0)
    torch.cuda.set_device(0)
    skip = set()
    orig = _lib._Lib.call

    def call(self, name, *args):
        if name in skip:
            return None
        return orig(self, name, *args)

    _lib._Lib.call = call
    host = bench.make_host_batch(10, seed=100, torch=torch, np=np, backbone='transFuser', raw=True)
    tr = Trainer(TrainConfig(), dev, gemm_mode='bf16', lr=1e-4, seed=0, backbone='transFuser', raw_inputs=True)
    for _ in range(3):
        tr.step({k: v.to(dev, non_blocking=True) for k, v in host.items()})       # un-ablated warm-up (allocator, caches)
    skip.update(x for x in s.split('+') if x)
    if not tr.capture(host):
        return {'ablate': s, 'error': tr.graph_error}
    for _ in range(3):
        tr.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        tr.replay()
    e1.record()
    torch.cuda.synchronize()
    return {'ablate': s or '(nothing)', 'ms_per_step': round(e0.elapsed_time(e1) / 10, 3), 'launches': tr.graph_launches}


def main():
    """One process per ablation set (a second Trainer in the same process does not reproduce the first one's step time), the
    un-ablated step first and last."""
    import subprocess
    if len(sys.argv) == 3 and sys.argv[1] == '--one':
        print('RESULT ' + json.dumps(one(sys.argv[2])), flush=True)
        return
    sets = sys.argv[1:] or DEFAULT_SETS
    base = None
    for s in sets + ['']:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), '--one', s], capture_output=True, text=True, timeout=300)
        line = [l for l in r.stdout.splitlines() if l.startswith('RESULT ')]
        if not line:
            print(json.dumps({'ablate': s, 'error': r.stderr[-300:]}), flush=True)
            continue
        d = json.loads(line[-1][7:])
        if not s and base is None:
            base = d.get('ms_per_step')
        if base is not None and 'ms_per_step' in d:
            d['saved_ms'] = round(base - d['ms_per_step'], 3)
        print(json.dumps(d), flush=True)


if __name__ == '__main__':
    main()
