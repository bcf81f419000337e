"""The per-op parity tests of tests/test_ops.py (forward and backward of every exact-fp32 kernel through the product's autograd
wrappers, against plain fp32 torch ops) executed in this container WITHOUT a GPU: the same test functions, with the C-ABI calls
routed to the CPU emulation of the unchanged kernel sources (tests/cuda_emul/: one OS thread per CUDA thread, barriers for
__syncthreads / warp shuffles, launches rewritten to emul_launch). The tensor-core kernels (wgmma / TMA) cannot be emulated;
everything in the exact-fp32 ("simt") numerics mode can. The `-m gpu` run of test_ops.py on an H100 remains the parity test proper:
this run checks the kernel source's indexing, control flow and arithmetic, not the device compiler. Test infrastructure only."""
import math

import pytest
import torch
import torch.nn.functional as F

import test_ops as T
from cuda_emul import loader
from test_ops import (test_attention, test_batchnorm_add_relu_fused, test_batchnorm_squeeze_excite_one_node, test_batchnorm_train, test_batchnorm_with_se_pool, test_conv2d, test_gpt_tokens_and_view_quirk, test_gru_waypoints,  # noqa: F401
                      test_image_prep_and_layout, test_layernorm_linear_dropout, test_losses, test_se_add_pool, test_residual_dropout_layernorm_fused, test_se_fused_mlp_backward, test_small_m_gemm,
                      test_upsample)


@pytest.fixture(autouse=True)
def _emulated_kernels(monkeypatch):
    lib = loader.patch_product(monkeypatch)
    monkeypatch.setattr(T, 'DEV', 'cpu')
    monkeypatch.setattr(T, 'DROPOUT_N', 1 << 16)
    monkeypatch.setattr(T, 'LN_ROWS', 37)
    monkeypatch.setattr(T, 'ATT_T', 46)
    del T.SKIPPED_ON_EMULATOR[:]
    yield
    assert lib.log or T.SKIPPED_ON_EMULATOR, 'the test did not reach the emulated C-ABI'


def test_gpt_with_velocity_embedding():
    """(CPU emulation only: written after the round's GPU budget was spent, so it is kept out of the `-m gpu` module.)
    GPT.forward with use_velocity=True (transfuser.py:346-364): tokens + pos_emb + vel_emb(velocity) for every token, one Block,
    ln_f, the view quirk and the upsample-add — the product module (kernels through the C-ABI) against the same nn.Parameters driven
    through plain torch ops, outputs and gradients incl. vel_emb's."""
    from transfuser_b200.backbone import GPT

    class Cfg:
        gpt_linear_layer_init_mean, gpt_linear_layer_init_std, gpt_layer_norm_init_weight = 0.0, 0.02, 1.0
    C, B, nh = 32, 2, 4
    torch.manual_seed(0)
    g = GPT(C, nh, 4, 1, 2, 3, 2, 2, 1, 0.0, 0.0, 0.0, Cfg, use_velocity=True).to(T.DEV).train()
    with torch.no_grad():
        g.pos_emb.copy_(T.rnd(1, 10, C, seed=1, scale=0.1))
        g.vel_emb.weight.copy_(T.rnd(C, 1, seed=2, scale=0.3))
        g.vel_emb.bias.copy_(T.rnd(C, seed=3, scale=0.1))
        for i, p in enumerate(g.blocks.parameters()):
            if p.dim() == 2:
                p.copy_(T.rnd(*p.shape, seed=10 + i, scale=p.shape[1] ** -0.5))
    img, lid, vel = T.rnd(B, C, 4, 6, seed=4), T.rnd(B, C, 4, 4, seed=5), T.rnd(B, 1, seed=6).abs() * 5
    im, lm = T.nhwc(img).requires_grad_(), T.nhwc(lid).requires_grad_()
    oi, ol = g.run(im, lm, vel)
    # the same parameters through torch
    ir, lr = img.clone().requires_grad_(), lid.clone().requires_grad_()
    tok = torch.cat((F.adaptive_avg_pool2d(ir, (2, 3)).permute(0, 2, 3, 1).reshape(B, -1, C),
                     F.adaptive_avg_pool2d(lr, (2, 2)).permute(0, 2, 3, 1).reshape(B, -1, C)), dim=1)
    x = g.pos_emb + tok + g.vel_emb(vel).unsqueeze(1)
    blk = g.blocks[0]
    a = blk.attn
    h = blk.ln1(x)
    NT = 10
    q, k, v = [f(h).view(B, NT, nh, C // nh).transpose(1, 2) for f in (a.query, a.key, a.value)]
    att = F.softmax((q @ k.transpose(-2, -1)) * (1.0 / math.sqrt(C // nh)), dim=-1)
    x = x + a.proj((att @ v).transpose(1, 2).reshape(B, NT, C))
    x = x + blk.mlp(blk.ln2(x))
    x = g.ln_f(x)
    ref_i = ir + F.interpolate(x[:, :6, :].contiguous().view(B, -1, 2, 3), size=(4, 6), mode='bilinear', align_corners=False)
    ref_l = lr + F.interpolate(x[:, 6:, :].contiguous().view(B, -1, 2, 2), size=(4, 4), mode='bilinear', align_corners=False)
    assert T.rel(T.nchw(oi), ref_i) < T.TOL and T.rel(T.nchw(ol), ref_l) < T.TOL
    params = [g.vel_emb.weight, g.vel_emb.bias, g.pos_emb, a.proj.weight, blk.mlp[0].weight, g.ln_f.weight]
    gi, gl = T.rnd(B, C, 4, 6, seed=7), T.rnd(B, C, 4, 4, seed=8)
    want = torch.autograd.grad([ref_i, ref_l], [ir, lr] + params, [gi, gl])
    got = torch.autograd.grad([oi, ol], [im, lm] + params, [T.nhwc(gi), T.nhwc(gl)])
    assert T.rel(T.nchw(got[0]), want[0]) < T.TOL and T.rel(T.nchw(got[1]), want[1]) < T.TOL
    for name, x1, x2 in zip(('vel_emb.weight', 'vel_emb.bias', 'pos_emb', 'proj.weight', 'mlp.0.weight', 'ln_f.weight'), got[2:], want[2:]):
        assert T.rel(x1, x2) < T.TOL, (name, T.rel(x1, x2))
    # without the input the module refuses to run; the default module has no such parameter
    with pytest.raises(RuntimeError):
        g.run(im, lm)
    assert not hasattr(GPT(C, nh, 4, 1, 2, 3, 2, 2, 1, 0.0, 0.0, 0.0, Cfg, use_velocity=False), 'vel_emb')
