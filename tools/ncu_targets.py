"""Representative launches of every hot kernel of the training step at its batch-10 shapes, for ONE `ncu --set full` capture:
    ncu --set full --clock-control none --import-source on -o tools_out/kernels python tools/ncu_targets.py
Each section runs forward + backward of a product op (C-ABI kernels through transfuser_b200.ops), so the capture holds the real
kernels with the real operand shapes: GPT GEMMs (C = 1512), trunk 1x1 GEMMs with BatchNorm statistics in the epilogue, grouped 3x3
convs (stride 1 and 2), fused attention, BatchNorm forward / backward, squeeze-excite, AdamW, BEV histogram, bilinear upsample."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from transfuser_b200 import _lib, bev, gemm, ops
from oracle import bev_oracle

torch.manual_seed(0)
dev = 'cuda'
gemm.set_mode('bf16')
B = 10


def rnd(*s, scale=1.0):
    return (torch.randn(*s, device=dev) * scale)


def fb(out, *inputs):
    g = torch.autograd.grad(out.sum() if out.dim() == 0 else (out * torch.randn_like(out)).sum(), [t for t in inputs if t.requires_grad], allow_unused=True)
    torch.cuda.synchronize()
    return g


warm = int(os.environ.get('WARM', '1'))
SECTIONS = set(os.environ.get('SECTIONS', 'gpt,trunk,attn,decoder,ln,bev,adamw').split(','))
for it in range(1 + warm):
    ops.tick(dev)
    # --- GPT block GEMMs, C = 1512, M = B*174 ---
    M, C = B * 174, 1512
    x = rnd(M, C).requires_grad_()
    for N in ((C, 4 * C) if 'gpt' in SECTIONS else ()):
        w = rnd(N, C, scale=0.02).requires_grad_()
        b = rnd(N, scale=0.1).requires_grad_()
        fb(ops.linear(x, w, b, relu=(N != C)), x, w, b)
    if 'gpt' in SECTIONS:
        w = rnd(C, 4 * C, scale=0.02).requires_grad_()
        x4 = rnd(M, 4 * C).requires_grad_()
        fb(ops.linear(x4, w, None), x4, w)
    # --- trunk stage 3 / stage 1 bottleneck pieces: 1x1 conv (+BN stats in the epilogue) + BN + ReLU, grouped 3x3 (s1, s2), SE ---
    for (H, W, Cc) in (((10, 44, 576), (40, 176, 72), (20, 88, 216)) if 'trunk' in SECTIONS else ()):
        xm = rnd(B, H, W, Cc).requires_grad_()
        w1 = rnd(Cc, Cc, 1, 1, scale=Cc ** -0.5).requires_grad_()
        bn = torch.nn.BatchNorm2d(Cc).to(dev).train()
        y = ops.batch_norm(ops.conv2d(xm, w1, None, 1, 1, False, bn_stats=True), bn, True, True, emit16=True, bwd16=True)
        w3 = rnd(Cc, 24, 3, 3, scale=(24 * 9) ** -0.5).requires_grad_()
        bn2 = torch.nn.BatchNorm2d(Cc).to(dev).train()
        y2 = ops.batch_norm(ops.conv2d(y, w3, None, 1, Cc // 24, False, bn_stats=True), bn2, True, True, pool=True, bwd16=True)
        se = [rnd(Cc // 4, Cc, 1, 1, scale=Cc ** -0.5).requires_grad_(), rnd(Cc // 4, scale=0.1).requires_grad_(),
              rnd(Cc, Cc // 4, 1, 1, scale=(Cc // 4) ** -0.5).requires_grad_(), rnd(Cc, scale=0.1).requires_grad_()]
        y3 = ops.SEFn.apply(y2, *se, True)
        w5 = rnd(Cc, 24, 3, 3, scale=(24 * 9) ** -0.5).requires_grad_()
        y4 = ops.conv2d(y3, w5, None, 2, Cc // 24, False, bn_stats=True)          # stride-2 grouped conv on the tensor cores
        fb(y4, xm, w1, w3, w5, bn.weight, bn2.weight, *se)
    # --- fused attention, all four head sizes ---
    for hs in ((378, 144, 54, 18) if 'attn' in SECTIONS else ()):
        Cc = 4 * hs
        h = rnd(B * 174, Cc).requires_grad_()
        flat = torch.cat([rnd(Cc * Cc, scale=Cc ** -0.5) for _ in range(3)] + [rnd(Cc, scale=0.1) for _ in range(3)]).contiguous()
        ws = [flat[i * Cc * Cc:(i + 1) * Cc * Cc].view(Cc, Cc).requires_grad_() for i in range(3)]
        bs = [flat[3 * Cc * Cc + i * Cc:3 * Cc * Cc + (i + 1) * Cc].requires_grad_() for i in range(3)]
        fb(ops.AttentionFn.apply(h, ws[0], bs[0], ws[1], bs[1], ws[2], bs[2], B, 174, 4, 0.1, 7), h, *ws)
    # --- decoder-size maps: 3x3 conv 32 -> 32 at 160 x 704, bilinear upsample x4 ---
    if 'decoder' in SECTIONS:
        xm = rnd(B, 40, 176, 64).requires_grad_()
        up = ops.upsample(xm, 160, 704, False, emit16=True)
        w = rnd(32, 64, 3, 3, scale=(64 * 9) ** -0.5).requires_grad_()
        bb = rnd(32, scale=0.1).requires_grad_()
        fb(ops.conv2d(up, w, bb, relu=True), xm, w, bb)
    # --- LayerNorm, residual add + dropout on GPT tokens ---
    if 'ln' in SECTIONS:
        t = rnd(B * 174, 1512).requires_grad_()
        ln = torch.nn.LayerNorm(1512).to(dev)
        fb(ops.add_dropout(t, ops.layer_norm(t, ln, emit16=True), 0.1, True), t, ln.weight)
    # --- BEV histogram (10 x 40k points) ---
    if 'bev' in SECTIONS:
        pts = torch.from_numpy(np.stack([bev_oracle.synthetic_points(40000, s, np.float32, edge_cases=False) for s in range(B)])).to(dev)
        bev.lidar_to_histogram_features_batched(pts)
    torch.cuda.synchronize()
# --- fused AdamW over a 168 M-element flat buffer (once) ---
if 'adamw' in SECTIONS:
    n = 168_000_000
    p, g, m, v = (torch.zeros(n, device=dev) for _ in range(4))
    p16 = torch.empty(n, dtype=torch.bfloat16, device=dev)
    step_dev = torch.ones(1, dtype=torch.int32, device=dev)
    _lib.call('tfb_adamw_step', p, g, m, v, n, 1e-4, 0.9, 0.999, 1e-8, 1e-2, 1, step_dev, 1.0, p16, 0, None)
    torch.cuda.synchronize()
print('ncu targets done')
