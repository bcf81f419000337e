"""TEST INFRASTRUCTURE ONLY. torch stand-ins for the tensor-core entry points (wgmma / TMA: not emulable), written from the
CONTRACT in include/tfb200.h — operand layouts, leading dimensions, column windows, the packed-weight format of csrc/conv_pack.cu —
so that the product's bf16-mode host path (sidecars, packed weights, q|k|v packs, im2col + batched wgrad, flat gradients) can run
end to end on the CPU emulation with every CUDA-core kernel real and only the MMA itself replaced. They check what the real
kernels require (16-byte alignment, leading dimensions % 8) and compute in fp32 from the bf16 operands, like the hardware does."""
import torch
import torch.nn.functional as F

TC_NAMES = ('tfb_gemm_bf16_tc', 'tfb_gemm_bf16_tc_stats', 'tfb_gemm_bf16_tc_out16', 'tfb_conv3x3_tc', 'tfb_conv3x3_tc_strided', 'tfb_gemm_bf16_tc_wgrad_batched', 'tfb_attn_fwd_tc', 'tfb_attn_bwd_tc')


def _mat(t, rows, cols, ld):
    assert t.data_ptr() % 16 == 0 and ld % 8 == 0, 'TMA: 16-byte aligned base and leading dimension'
    return torch.as_strided(t, (rows, cols), (ld, 1))


def gemm_bf16_tc(ta, tb, M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, splits):
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16 and C.dtype == torch.float32
    a = _mat(A, K, M, lda).t() if ta else _mat(A, M, K, lda)
    b = _mat(B, N, K, ldb).t() if tb else _mat(B, K, N, ldb)
    out = torch.as_strided(C, (M, N), (ldc, 1))
    r = alpha * (a.float() @ b.float())
    if bias is not None:
        r = r + torch.as_strided(bias, (N,), (1,))
    if beta != 0.0:
        r = r + beta * out
    assert not (relu and splits > 1)
    out.copy_(r.clamp_min(0) if relu else r)


def gemm_bf16_tc_stats(M, N, K, A, lda, B, ldb, C, ldc, stats):
    gemm_bf16_tc(0, 1, M, N, K, A, lda, B, ldb, C, ldc, None, 0, 1.0, 0.0, 1)
    out = torch.as_strided(C, (M, N), (ldc, 1)).double()
    st = torch.as_strided(stats, (2, N), (N, 1))
    st[0] += out.sum(0)
    st[1] += (out * out).sum(0)


def gemm_bf16_tc_wgrad_batched(M, N, K, A, lda, a_step, B, ldb, b_step, C, ldc, c_bstride, nbatch, splits):
    assert A.data_ptr() % 16 == 0 and B.data_ptr() % 16 == 0 and lda % 8 == 0 and ldb % 8 == 0 and a_step % 8 == 0 and b_step % 8 == 0
    for b in range(nbatch):
        a = torch.as_strided(A, (K, M), (lda, 1), A.storage_offset() + b * a_step)
        bb = torch.as_strided(B, (K, N), (ldb, 1), B.storage_offset() + b * b_step)
        torch.as_strided(C, (M, N), (ldc, 1), C.storage_offset() + b * c_bstride).copy_(a.float().t() @ bb.float())


def conv3x3_tc(x16, wp, bias, y, N, H, W, Cx, Cy, NB, KC, c_step, nchunks, nb_real, gblocks, relu):
    conv3x3_tc_strided(x16, wp, bias, y, N, H, W, Cx, Cy, NB, KC, c_step, nchunks, nb_real, gblocks, relu, 1, None)


def conv3x3_tc_strided(x16, wp, bias, y, N, H, W, Cx, Cy, NB, KC, c_step, nchunks, nb_real, gblocks, relu, stride, stats):
    """y = conv3x3(x16, packed weights; pad 1, stride 1 or 2): block gb reads channels gb*c_step + chunk*KC + kk, writes channels gb*nb_real + j; tap t
    multiplies the input pixel shifted by (t/3 - 1, t%3 - 1); out-of-image pixels and channels >= Cx read as zero."""
    assert x16.dtype == torch.bfloat16 and wp.dtype == torch.bfloat16 and Cx % 8 == 0 and x16.data_ptr() % 16 == 0 and wp.data_ptr() % 16 == 0
    wpk = torch.as_strided(wp, (gblocks, nchunks, 9, NB, KC), (nchunks * 9 * NB * KC, 9 * NB * KC, NB * KC, KC, 1)).float()
    dense = torch.zeros(Cy, Cx, 9)
    for gb in range(gblocks):
        for ch in range(nchunks):
            for j in range(min(nb_real, NB)):
                oc = gb * nb_real + j
                if oc >= Cy:
                    continue
                rc0 = gb * c_step + ch * KC
                n = max(0, min(KC, Cx - rc0))
                if n:
                    dense[oc, rc0:rc0 + n] += wpk[gb, ch, :, j, :n].t()
    xin = torch.as_strided(x16, (N, H, W, Cx), (H * W * Cx, W * Cx, Cx, 1)).float().permute(0, 3, 1, 2)
    out = F.conv2d(xin, dense.view(Cy, Cx, 3, 3), None if bias is None else torch.as_strided(bias, (Cy,), (1,)), padding=1, stride=stride)
    out = out.clamp_min(0) if relu else out
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    torch.as_strided(y, (N, Ho, Wo, Cy), (Ho * Wo * Cy, Wo * Cy, Cy, 1)).copy_(out.permute(0, 2, 3, 1))
    if stats is not None:
        assert bias is None and not relu and Cy % 4 == 0 and nb_real % 4 == 0
        st = torch.as_strided(stats, (2, Cy), (Cy, 1))
        st[0] += out.double().sum((0, 2, 3))
        st[1] += (out.double() ** 2).sum((0, 2, 3))


def _attn_keep(seed_dev, seed_off, B, nh, T, p_drop):
    """The dropout keep-scale of csrc/attn_tc.cu (drop_scale): [B, nh, T, T], 0 or 1/(1-p)."""
    if p_drop <= 0.0:
        return torch.ones(B, nh, T, T)
    seed = (int(seed_dev.view(-1)[0].item()) if seed_dev is not None else 0) + int(seed_off)
    lo, hi, M = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF, 0xFFFFFFFF
    x = (torch.arange(B * nh * T * T, dtype=torch.int64) * 0x9E3779B1 + lo) & M
    x = ((x ^ (x >> 16)) * 0x85EBCA6B) & M
    x = x ^ hi
    x = ((x ^ (x >> 13)) * 0xC2B2AE35) & M
    x = x ^ (x >> 16)
    u = (x >> 8).float() * (1.0 / 16777216.0)
    return torch.where(u < p_drop, torch.zeros(()), torch.full((), 1.0 / (1.0 - p_drop))).view(B, nh, T, T)


def _heads(t2d, B, T, nh, hs):
    return t2d.reshape(B, T, nh, hs).permute(0, 2, 1, 3)


def attn_fwd_tc(qkv, qkv_bf16, B, T, nh, hs, y32, y16, lse, scale, p_drop, seed_dev, seed_off):
    C = nh * hs
    x = torch.as_strided(qkv, (B * T, 3 * C), (3 * C, 1)).bfloat16().float()     # the tensor cores see bf16 operands
    q, k, v = (_heads(x[:, i * C:(i + 1) * C], B, T, nh, hs) for i in range(3))
    s = (q @ k.transpose(-1, -2)) * scale
    torch.as_strided(lse, (B, nh, T), (nh * T, T, 1)).copy_(torch.logsumexp(s, -1))
    pd = (torch.softmax(s, -1) * _attn_keep(seed_dev, seed_off, B, nh, T, p_drop)).bfloat16().float()
    y = (pd @ v).permute(0, 2, 1, 3).reshape(B * T, C)
    if y32 is not None:
        torch.as_strided(y32, (B * T, C), (C, 1)).copy_(y)
    if y16 is not None:
        torch.as_strided(y16, (B * T, C), (C, 1)).copy_(y)


def gemm_bf16_tc_out16(tb, M, N, K, A, lda, B, ldb, C16, ldc, bias, relu, alpha):
    tmp = torch.empty(M, N)
    gemm_bf16_tc(0, tb, M, N, K, A, lda, B, ldb, tmp, N, bias, relu, alpha, 0.0, 1)
    assert C16.dtype == torch.bfloat16 and ldc % 4 == 0
    torch.as_strided(C16, (M, N), (ldc, 1)).copy_(tmp)


def attn_bwd_tc(qkv, qkv_bf16, dy32, y32, y_bf16, lse, dsum, dy16, B, T, nh, hs, dqkv32, dqkv16, scale, p_drop, seed_dev, seed_off):
    C = nh * hs
    dy = dy32
    x = torch.as_strided(qkv, (B * T, 3 * C), (3 * C, 1)).bfloat16().float()
    q, k, v = (_heads(x[:, i * C:(i + 1) * C], B, T, nh, hs) for i in range(3))
    do = _heads(torch.as_strided(dy, (B * T, C), (C, 1)).bfloat16().float(), B, T, nh, hs)
    keep = _attn_keep(seed_dev, seed_off, B, nh, T, p_drop)
    p = torch.exp((q @ k.transpose(-1, -2)) * scale - torch.as_strided(lse, (B, nh, T), (nh * T, T, 1)).unsqueeze(-1))
    D = (_heads(torch.as_strided(dy32, (B * T, C), (C, 1)), B, T, nh, hs) * _heads(torch.as_strided(y32, (B * T, C), (C, 1)), B, T, nh, hs)).sum(-1, keepdim=True)
    dv = (p * keep).bfloat16().float().transpose(-1, -2) @ do
    ds = (scale * p * ((do @ v.transpose(-1, -2)) * keep - D)).bfloat16().float()
    dq, dk = ds @ k, ds.transpose(-1, -2) @ q
    out = torch.cat([t.permute(0, 2, 1, 3).reshape(B * T, C) for t in (dq, dk, dv)], dim=1)
    if dqkv32 is not None:
        torch.as_strided(dqkv32, (B * T, 3 * C), (3 * C, 1)).copy_(out)
    if dqkv16 is not None:
        torch.as_strided(dqkv16, (B * T, 3 * C), (3 * C, 1)).copy_(out)


class WithTensorCoreStandins:
    """Wraps the emulated library: the three tensor-core entry points go to the stand-ins above, everything else to the emulation."""

    def __init__(self, emul):
        self.emul = emul
        self.log = emul.log
        self.launches = 0
        self.profiler = None
        self.fns = {'tfb_gemm_bf16_tc': gemm_bf16_tc, 'tfb_gemm_bf16_tc_stats': gemm_bf16_tc_stats, 'tfb_gemm_bf16_tc_out16': gemm_bf16_tc_out16, 'tfb_conv3x3_tc': conv3x3_tc, 'tfb_conv3x3_tc_strided': conv3x3_tc_strided, 'tfb_gemm_bf16_tc_wgrad_batched': gemm_bf16_tc_wgrad_batched,
                    'tfb_attn_fwd_tc': attn_fwd_tc, 'tfb_attn_bwd_tc': attn_bwd_tc}

    def call(self, name, *args):
        fn = self.fns.get(name)
        if fn is None:
            return self.emul.call(name, *args)
        self.log.append(name)
        self.launches += 1
        fn(*args)
