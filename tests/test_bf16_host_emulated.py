"""The bf16 tensor-core mode of the product, end to end on the CPU: every CUDA-core kernel runs for real on the emulation
(tests/cuda_emul/), only the three tensor-core entry points are replaced by torch stand-ins written from their C-ABI contract
(tests/cuda_emul/tc_standins.py). This exercises what no other CPU test reaches — the host logic that exists only in bf16 mode:
bf16 sidecars forward and backward, the packed-weight registry and the once-per-step batched pack, the (channel, tap) im2col feeding
the batched wgrad GEMM that writes PyTorch-layout gradients into the flat buffer, the q|k|v pack, the bf16 weight mirror — and
compares the result with the same modules in the exact-fp32 ('simt') mode within the bf16 tolerance of tests/test_bf16.py. A layout
or wiring error shows up as an O(1) difference. Test infrastructure only; the `-m gpu` tests remain the parity tests proper."""
import pytest
import torch
import torch.nn as nn

from cuda_emul import loader, tc_standins
from transfuser_b200 import _lib

TOL = 3e-2     # forward, bf16 operands (8 mantissa bits) through a few layers with batch-statistics BatchNorm (test_bf16.py: 2e-2 per op)
# Gradients against the fp32 mode carry ReLU-mask flips (a bf16-perturbed pre-activation near 0 flips its mask; with the random-sign
# upstream gradients used here one flipped element moves a column sum by ~10 %), so that comparison only has to separate "noise" from
# "wrong layout" (a permuted tap / channel order gives a relative error >= 1). The tight gradient check is bf16-mode against bf16-mode
# with every host-side option of DESIGN.md 4b switched off (the configuration the `-m gpu` tests run).
GRAD_TOL_VS_FP32 = 0.25
TOL_VS_PLAIN_BF16 = 3e-3    # (the fused BatchNorm + squeeze-excite backward forms dy*gate + dpool/HW with one fma inside BatchNorm's passes: 1e-7 differences, a few flipped bf16 roundings downstream)
FLAGS = ('SIDECARS', 'SE_FUSED_BWD', 'SE_POOL_FUSED', 'QKV_FUSED', 'BN_ADD_FUSED', 'PACK_BATCHED')   # the numerically EQUIVALENT options (BN_STATS_FUSED, CONV_S2_TC, ATTN_FUSED change roundings: they stay on in both runs)


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


@pytest.fixture()
def lib(monkeypatch):
    emul = loader.patch_product(monkeypatch)
    wrapped = tc_standins.WithTensorCoreStandins(emul)
    monkeypatch.setattr(_lib, '_LIB', wrapped)
    from transfuser_b200 import ops
    ops._PACKS.clear()
    ops._PACK_STATE.update(sig=None, table=None)
    ops._BWD16.clear()
    yield wrapped


class _Net(nn.Module):
    """A RegNetY stage in miniature (stride-2 block with downsample shortcut + identity block, SE, grouped 3x3 convs) between a stem-like
    conv and a decoder-like head: every conv flavour of the training step."""

    def __init__(self):
        super().__init__()
        from transfuser_b200.backbone import _ConvBn, _Stage
        self.stem = _ConvBn(32, 48, 3, stride=1)
        self.stage = _Stage(48, 72, 2, 24, 0.25)
        self.head3 = nn.Conv2d(72, 64, 3, padding=1)
        self.head1 = nn.Conv2d(64, 16, 1)
        self.narrow = nn.Conv2d(64, 7, 3, padding=1)      # 7 output channels: dy zero-padded to 8 for the tensor-core wgrad
        with torch.no_grad():
            for m in self.modules():
                if isinstance(m, nn.BatchNorm2d):
                    m.weight.uniform_(0.5, 1.5)             # (timm zero-inits conv3.bn.weight: keep every path alive)
                    m.bias.uniform_(-0.2, 0.2)

    def forward(self, x):
        from transfuser_b200 import ops
        if self.training:
            ops.tick(x.device)
        y = self.stage.run(self.stem.run(x, emit16=True))
        h = ops.conv2d(y, self.head3.weight, self.head3.bias, relu=True)
        return ops.conv2d(h, self.head1.weight, self.head1.bias), ops.conv2d(h, self.narrow.weight, self.narrow.bias)


def _run(net, x, r1, r2):
    a, b = net(x)
    loss = (a * r1).sum() + (b * r2).sum()
    params = [p for p in net.parameters()]
    grads = torch.autograd.grad(loss, [x] + params)
    return [a.detach(), b.detach()] + [g.detach().clone() for g in grads]


def test_conv_trunk_bf16_mode_matches_fp32_mode(lib):
    from transfuser_b200 import gemm, ops, optim
    torch.manual_seed(0)
    ref = _Net().train()
    state = {k: v.clone() for k, v in ref.state_dict().items()}
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 32, 32, 32, generator=g)       # 2 x 16 x 16 = 512 pixels after the stage: the tensor-core wgrad's minimum
    r1, r2 = torch.randn(2, 16, 16, 16, generator=g), torch.randn(2, 16, 16, 7, generator=g)
    want = _run(ref, x.clone().requires_grad_(True), r1, r2)                       # exact-fp32 mode (conftest default)

    gemm.set_mode('bf16')
    net = _Net().train()
    net.load_state_dict(state)
    fp = optim.flatten(net)
    gemm.attach_bf16_weights(fp)
    lib.log.clear()
    got = _run(net, x.clone().requires_grad_(True), r1, r2)
    log1 = list(lib.log)
    names = ['head1 out', 'narrow out', 'dx'] + [n for n, _ in net.named_parameters()]
    for i, (n, a, b) in enumerate(zip(names, got, want)):
        assert rel(a, b) < (TOL if i < 2 else GRAD_TOL_VS_FP32), (n, rel(a, b))
    # the tensor cores were used for every conv flavour, and the bf16-only host paths were taken
    assert log1.count('tfb_conv3x3_tc') >= 6 and log1.count('tfb_gemm_bf16_tc') >= 12 and log1.count('tfb_gemm_bf16_tc_wgrad_batched') >= 4
    assert 'tfb_im2col3x3_bf16' in log1 and 'tfb_cast_bf16_pad' in log1
    # BatchNorm statistics come out of the producing epilogues (1x1 GEMMs, grouped 3x3 incl. the stride-2 one): one BN launch, no reduction
    assert log1.count('tfb_gemm_bf16_tc_stats') >= 5 and log1.count('tfb_conv3x3_tc_strided') >= 3 and log1.count('tfb_bn_fwd_stats') >= 8
    assert log1.count('tfb_bn_fwd') == 0 and log1.count('tfb_conv2d_fwd') == 0
    # every weight gradient sits in its span of the flat buffer (the batched wgrad GEMM wrote PyTorch layout in place)
    grads = dict(zip([n for n, _ in net.named_parameters()], got[3:]))
    for (n, p), o in zip(((n, p) for n, p in net.named_parameters()), [dict(zip(map(id, fp.params), fp.offsets))[id(p)] for p in net.parameters()]):
        if p.dim() == 4 and p.shape[-1] == 3 and p.shape[0] % 8 == 0 and p.shape[1] % 8 == 0:
            assert torch.equal(fp.grad[o:o + p.numel()].view(p.shape), grads[n]), n
    # second step on the same weights: packed weights now come from ONE batched launch, results identical
    for p in net.parameters():
        p.grad = None
    lib.log.clear()
    again = _run(net, x.clone().requires_grad_(True), r1, r2)
    log2 = list(lib.log)
    assert log1.count('tfb_conv3x3_pack_weights') > 0 and log1.count('tfb_conv3x3_pack_weights_batched') == 0
    assert log2.count('tfb_conv3x3_pack_weights') == 0 and log2.count('tfb_conv3x3_pack_weights_batched') == 1
    for n, a, b in zip(names, again[:3], got[:3]):
        assert torch.equal(a, b), n
    # every host-side option off: the plain bf16 path. Same operands, so everything agrees tightly (sidecars / packs: same bits;
    # fused SE backward: fp32 summation order only)
    old = {f: getattr(ops, f) for f in FLAGS}
    try:
        for f in FLAGS:
            setattr(ops, f, False)
        for p in net.parameters():
            p.grad = None
        lib.log.clear()
        plain = _run(net, x.clone().requires_grad_(True), r1, r2)
        log3 = list(lib.log)
    finally:
        for f in FLAGS:
            setattr(ops, f, old[f])
    for n, a, b in zip(names, again, plain):
        assert rel(a, b) < TOL_VS_PLAIN_BF16, (n, rel(a, b))
    assert torch.equal(again[0], plain[0]) and torch.equal(again[1], plain[1])     # forward: bit-identical
    assert log3.count('tfb_cast_bf16') - log2.count('tfb_cast_bf16') >= 6          # sidecars replace these passes
    assert log3.count('tfb_grad_prep') + log3.count('tfb_cast_bf16') - log2.count('tfb_grad_prep') - log2.count('tfb_cast_bf16') >= 12
    assert len(log3) - len(log2) >= 35, (len(log3), len(log2))                     # C-ABI calls saved on this two-block miniature (121 -> 82)


def test_gpt_block_bf16_mode_matches_fp32_mode(lib):
    from transfuser_b200 import gemm, optim
    from transfuser_b200.backbone import Block
    C, nh, B, T = 32, 4, 2, 16
    torch.manual_seed(2)
    ref = Block(C, nh, 4, 0.0, 0.0).train()
    state = {k: v.clone() for k, v in ref.state_dict().items()}
    g = torch.Generator().manual_seed(3)
    x, r = torch.randn(B * T, C, generator=g), torch.randn(B * T, C, generator=g)

    def run(blk):
        xi = x.clone().requires_grad_(True)
        y = blk.run(xi, B, T)
        grads = torch.autograd.grad((y * r).sum(), [xi] + list(blk.parameters()))
        return [y.detach()] + [t.detach().clone() for t in grads]
    want = run(ref)
    gemm.set_mode('bf16')
    blk = Block(C, nh, 4, 0.0, 0.0).train()
    blk.load_state_dict(state)
    fp = optim.flatten(blk)
    gemm.attach_bf16_weights(fp)
    lib.log.clear()
    got = run(blk)
    names = ['y', 'dx'] + [n for n, _ in blk.named_parameters()]
    for i, (n, a, b) in enumerate(zip(names, got, want)):
        if n == 'attn.key.bias':
            continue                                       # true gradient 0 (softmax shift invariance)
        assert rel(a, b) < (TOL if i == 0 else GRAD_TOL_VS_FP32), (n, rel(a, b))
    # q|k|v as one GEMM in forward, dgrad and wgrad (3) + proj (3) + two MLP layers (6); LayerNorm outputs reach them as sidecars
    assert lib.log.count('tfb_gemm_bf16_tc') + lib.log.count('tfb_gemm_bf16_tc_out16') == 12 and lib.log.count('tfb_gemm_bf16_tc_out16') == 1
    assert lib.log.count('tfb_cast_bf16') == 1             # MLP hidden -> mlp.2 only: no LayerNorm-output casts, and the fused attention
    assert lib.log.count('tfb_attn_fwd_tc') == 1 and lib.log.count('tfb_attn_bwd_tc') == 1   # writes the bf16 copies of y and dqkv itself
    assert lib.log.count('tfb_colsum') == 1                # (the three bias gradients: one column reduction over dqkv)
    assert lib.log.count('tfb_gemm_f32_simt') == 0 and lib.log.count('tfb_softmax_fwd') == 0   # no T x T tensor in HBM
    from transfuser_b200 import ops
    old = {f: getattr(ops, f) for f in FLAGS}
    try:
        for f in FLAGS:
            setattr(ops, f, False)
        for p in blk.parameters():
            p.grad = None
        plain = run(blk)
    finally:
        for f in FLAGS:
            setattr(ops, f, old[f])
    for n, a, b in zip(names, got, plain):
        if n != 'attn.key.bias':
            assert rel(a, b) < TOL_VS_PLAIN_BF16, (n, rel(a, b))


def test_shared_input_im2col_is_built_once(lib):
    """The CenterNet heads / BEV head convolve the same p2 map: in backward the bf16 im2col matrix of a shared input is built by the
    first wgrad and reused by the others (same weight gradients as separate im2cols)."""
    from transfuser_b200 import gemm, ops
    gemm.set_mode('bf16')
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 16, 16, 64, generator=g).requires_grad_(True)
    ws = [(torch.randn(64, 64, 3, 3, generator=g) / 24).requires_grad_(True) for _ in range(3)]
    bs = [torch.randn(64, generator=g).requires_grad_(True) for _ in range(3)]
    rs = [torch.randn(2, 16, 16, 64, generator=g) for _ in range(3)]

    def run():
        ops.tick('cpu')
        lib.log.clear()
        loss = sum((ops.conv2d(x, w, b, relu=True) * r).sum() for w, b, r in zip(ws, bs, rs))
        n_cast_fwd = lib.log.count('tfb_cast_bf16')
        grads = torch.autograd.grad(loss, [x] + ws + bs)
        assert n_cast_fwd <= 1                      # the shared input is cast to bf16 once (ops._as16 keeps the copy on the tensor)
        return [t.clone() for t in grads], lib.log.count('tfb_im2col3x3_bf16')
    got, n_shared = run()
    assert n_shared == 1
    orig = ops._COL_CACHE
    try:
        class _Never(dict):
            def get(self, k, d=None):
                return None
        ops._COL_CACHE = _Never()
        want, n_sep = run()
    finally:
        ops._COL_CACHE = orig
    assert n_sep == 3
    for a, b in zip(got, want):
        assert torch.equal(a, b)
