"""CPU self-tests of the exact-operand references in tests/tc_ref.py (no GPU): the attention reference against fp64 softmax
attention and autograd, the hand-written backward against autograd of the forward, and the restated dropout hash."""
import math

import torch

import tc_ref as R


def _qkv(B, T, nh, hs, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B * T, 3 * nh * hs, generator=g, dtype=torch.float64)


def test_unrounded_reference_is_softmax_attention():
    B, T, nh, hs = 2, 37, 3, 10
    qkv, scale = _qkv(B, T, nh, hs, 1), R.scale_for(hs)
    dy = torch.randn(B * T, nh * hs, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    ones = torch.ones(B, nh, T, T, dtype=torch.float64)
    f = R.attn_fwd_ref(qkv, B, T, nh, hs, scale, ones, rounding=False)
    q, k, v = R.split_heads(qkv, B, T, nh, hs)
    s = scale * q @ k.transpose(-1, -2)
    y = R.merge_heads(torch.softmax(s, -1) @ v)
    assert (f['y'] - y).abs().max() < 1e-12
    assert (f['lse'] - torch.logsumexp(s, -1)).abs().max() < 1e-12
    b = R.attn_bwd_ref(qkv, dy, f['y'], f['lse'], B, T, nh, hs, scale, ones, rounding=False)
    g = R.attn_plain_grads(qkv, dy, B, T, nh, hs, scale, ones)
    assert (b['dqkv'] - g).abs().max() < 1e-12


def test_backward_is_autograd_of_forward_with_dropout():
    """With a fixed mask (and the backward given y = the forward's output), the restated backward is the exact gradient of
    (softmax * drop) v, including the D = rowsum(dy * y) form of the softmax backward under dropout."""
    B, T, nh, hs, p = 1, 29, 2, 6, 0.3
    qkv, scale = _qkv(B, T, nh, hs, 3), R.scale_for(hs)
    drop = R.drop_factor(11, B, nh, T, p)
    assert 0 < (drop == 0).double().mean() < 1
    dy = torch.randn(B * T, nh * hs, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    f = R.attn_fwd_ref(qkv, B, T, nh, hs, scale, drop, rounding=False)
    yp, _, _ = R.attn_plain(qkv, B, T, nh, hs, scale, drop)
    assert (f['y'] - yp.detach()).abs().max() < 1e-12
    b = R.attn_bwd_ref(qkv, dy, f['y'], f['lse'], B, T, nh, hs, scale, drop, rounding=False)
    g = R.attn_plain_grads(qkv, dy, B, T, nh, hs, scale, drop)
    assert (b['dqkv'] - g).abs().max() < 1e-12


def test_rounded_reference_stays_near_the_plain_one():
    """The rounding points move the result by bf16-operand amounts (~1e-2 relative), not more: the two references cannot share
    a structural mistake the rounded one would hide."""
    B, T, nh, hs = 2, 50, 2, 18
    qkv, scale = _qkv(B, T, nh, hs, 5), R.scale_for(hs)
    drop = R.drop_factor(3, B, nh, T, 0.1)
    dy = torch.randn(B * T, nh * hs, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    f = R.attn_fwd_ref(qkv, B, T, nh, hs, scale, drop)
    yp, _, _ = R.attn_plain(qkv, B, T, nh, hs, scale, drop)
    assert 1e-4 < R.rel_l2(f['y'], yp.detach()) < 2e-2
    b = R.attn_bwd_ref(qkv, dy, f['y'], f['lse'], B, T, nh, hs, scale, drop)
    assert R.rel_l2(b['dqkv'], R.attn_plain_grads(qkv, dy, B, T, nh, hs, scale, drop)) < 3e-2


def _hash_scalar(seed, idx, p):
    """Plain-integer restatement of drop_scale (one element at a time, Python ints masked to 32 bits)."""
    M = 0xFFFFFFFF
    x = (idx * 0x9E3779B1 + (seed & M)) & M
    x ^= x >> 16
    x = (x * 0x85EBCA6B) & M
    x ^= (seed >> 32) & M
    x ^= x >> 13
    x = (x * 0xC2B2AE35) & M
    x ^= x >> 16
    u = (x >> 8) / 16777216.0                     # exact in float32 (24 bits)
    return not (u < float(torch.tensor(p, dtype=torch.float32)))


def test_mask_tensor_form_matches_scalar_form():
    g = torch.Generator().manual_seed(0)
    idx = torch.randint(0, 2 ** 32, (2000,), generator=g, dtype=torch.int64)
    for seed in (0, 12345, (7 << 32) + 99, 2 ** 64 - 1):
        m = R.keep_mask(seed, idx, 0.1)
        assert [bool(v) for v in m] == [_hash_scalar(seed, int(i), 0.1) for i in idx]


def test_drop_fraction_within_5_sigma():
    for p, seed in ((0.1, 0), (0.5, 77), (0.1, 2 ** 40 + 5)):
        n = 4 * 4 * 174 * 174
        frac = (R.drop_factor(seed, 4, 4, 174, p) == 0).double().mean().item()
        assert abs(frac - p) < 5 * math.sqrt(p * (1 - p) / n), (p, seed, frac)
    assert R.keep_scale(0.1) == float(torch.tensor(1.0, dtype=torch.float32) / (1 - torch.tensor(0.1, dtype=torch.float32)))


def test_forward_and_backward_index_conventions_agree():
    """BWD_Q looks up (query tok, key c) at ((bh*T + tok)*T + c), BWD_K looks up (query c, key tok) at ((bh*T + c)*T + tok): both
    must read the forward's mask entry [b, h, query, key]."""
    B, nh, T, p, seed = 2, 3, 23, 0.5, 99
    fwd = R.drop_factor(seed, B, nh, T, p)
    for bh in range(B * nh):
        b, h = divmod(bh, nh)
        for tok in range(0, T, 5):
            c = torch.arange(T, dtype=torch.int64)
            bwd_q = R.keep_mask(seed, (bh * T + tok) * T + c, p)          # row = query tok, columns = keys c
            bwd_k = R.keep_mask(seed, (bh * T + c) * T + tok, p)          # row = key tok, columns = queries c
            assert torch.equal(bwd_q, fwd[b, h, tok, :] != 0)
            assert torch.equal(bwd_k, fwd[b, h, :, tok] != 0)
    # the counter wraps mod 2^32 as the kernel's uint32 does
    big = torch.tensor([2 ** 32 + 5], dtype=torch.int64)
    assert torch.equal(R.keep_mask(seed, big, p), R.keep_mask(seed, big - 2 ** 32, p))


def test_check_catches_single_element_and_row_errors():
    g = torch.Generator().manual_seed(1)
    a, b = torch.randn(64, 200, generator=g), torch.randn(200, 48, generator=g)
    ref, mag = R.contract(a, b)
    out = (R.bf(a).float() @ R.bf(b).float())                         # fp32 accumulation of the same operands
    R.check(out, ref, mag, 200, 1e-5)
    for bad in (out.clone().index_put_((torch.tensor(5), torch.tensor(7)), torch.tensor(0.0)), out * (1 + 1e-4)):
        try:
            R.check(bad, ref, mag, 200, 1e-3)
        except AssertionError:
            continue
        raise AssertionError('check() missed a perturbation')


def test_flip_allowance_is_one_ulp_near_midpoints_only():
    x = torch.tensor([1.0 + 2 ** -8, 1.0 + 2 ** -9, 3.0], dtype=torch.float64)   # a midpoint, off it, exact
    r, f = R.bf_flip(x, torch.full_like(x, 1e-9))
    assert f.tolist() == [2 ** -7, 0.0, 0.0]
    assert torch.equal(r, x.bfloat16().double())
