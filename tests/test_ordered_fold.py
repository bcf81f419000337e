"""The fixed-order cross-CTA sums (ordered_fold in csrc/common.cuh): split-K tiles, the BatchNorm statistics of the GEMM epilogue and
the BatchNorm backward column reductions. Their bits must not depend on which CTA or block finishes a sum, nor on whether a split-K
tile is folded inside the GEMM kernel or by ordered_sum_kernel after it."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _call(name, *a):
    from transfuser_b200 import _lib
    _lib.call(name, *a)


def _bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int64).cpu()


def _randn(*shape, seed):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV)


# (splits, M, N, K): the kernel folds a tile itself while splits * min(M, 128) * min(N, tile width) * 4 bytes stays within 256 KB,
# otherwise ordered_sum_kernel folds after the launch
SPLITK = [(2, 256, 256, 2 * 64 * 3), (33, 32, 32, 33 * 64 * 2), (33, 72, 72, 64 * 64 + 40), (132, 8, 32, 132 * 64), (132, 72, 72, 132 * 64)]


@pytest.mark.parametrize('splits,M,N,K', SPLITK)
def test_splitk_is_left_fold_of_single_split_launches(splits, M, N, K):
    """y = x W^T with `splits` K splits equals the fp32 left fold, in split order, of one single-split launch per split's K range."""
    A = _randn(M, K, seed=1).to(torch.bfloat16)
    B = _randn(N, K, seed=2).to(torch.bfloat16)
    bias = _randn(N, seed=3)
    num_kb = (K + 63) // 64
    kbps = (num_kb + splits - 1) // splits
    assert (num_kb + kbps - 1) // kbps == splits
    ref = torch.zeros(M, N, device=DEV)
    for s in range(splits):
        k0, k1 = s * kbps * 64, min(K, (s + 1) * kbps * 64)
        part = torch.full((M, N), float('nan'), device=DEV)
        _call('tfb_gemm_bf16_tc', 0, 1, M, N, k1 - k0, A[:, k0:], K, B[:, k0:], K, part, N, bias if s == 0 else None, 0, 1.0, 0.0, 1)
        ref = ref + part
    runs = []
    for _ in range(2):
        C = torch.full((M, N), float('nan'), device=DEV)     # beta = 0: C must not be read
        _call('tfb_gemm_bf16_tc', 0, 1, M, N, K, A, K, B, K, C, N, bias, 0, 1.0, 0.0, splits)
        runs.append(C)
    torch.cuda.synchronize()
    assert torch.equal(_bits(runs[0]), _bits(ref))
    assert torch.equal(_bits(runs[1]), _bits(ref))
    # beta = 1 adds the same fold to C
    C = ref.clone()
    _call('tfb_gemm_bf16_tc', 0, 1, M, N, K, A, K, B, K, C, N, bias, 0, 1.0, 1.0, splits)
    assert torch.equal(_bits(C), _bits(ref + ref))


@pytest.mark.parametrize('N', [72, 1512])
def test_gemm_stats_same_bits_and_value(N):
    """Per-column statistics of y = x W^T out of the GEMM epilogue: folded by one CTA per column block, the same bits on every call."""
    M, K = 4400, 576
    A = _randn(M, K, seed=4).to(torch.bfloat16)
    B = _randn(N, K, seed=5).to(torch.bfloat16)
    outs = []
    for _ in range(2):
        y = torch.empty(M, N, device=DEV)
        st = torch.zeros(2 * N, dtype=torch.float64, device=DEV)
        _call('tfb_gemm_bf16_tc_stats', M, N, K, A, K, B, K, y, N, st)
        outs.append((y, st))
    torch.cuda.synchronize()
    assert torch.equal(_bits(outs[0][1]), _bits(outs[1][1]))
    y = outs[0][0].double()
    ref = torch.cat([y.sum(0), (y * y).sum(0)])
    assert ((outs[0][1] - ref).norm() / ref.norm()).item() < 1e-6


@pytest.mark.parametrize('M,C', [(70400, 72), (4400, 1512)])
def test_bn_bwd_params_same_bits_and_value(M, C):
    """dgamma / dbeta of the BatchNorm backward: many row splits (C = 72) or many 128-channel slabs (C = 1512), each slab folded by
    its own last block."""
    x = _randn(M, C, seed=6)
    dy = _randn(M, C, seed=7)
    gamma, beta = _randn(C, seed=8), _randn(C, seed=9)
    mean = x.mean(0)
    invstd = 1.0 / (x.var(0, unbiased=False) + 1e-5).sqrt()
    outs = []
    for _ in range(2):
        dx = torch.empty_like(x)
        dgamma, dbeta = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
        ws = torch.zeros(2 * C + 1, dtype=torch.float64, device=DEV)
        _call('tfb_bn_bwd', x, dy, dx, M, C, gamma, beta, mean, invstd, 0, dgamma, dbeta, ws, None, None, None)
        outs.append((dgamma, dbeta, dx, ws))
    torch.cuda.synchronize()
    for a, b in zip(outs[0][:3], outs[1][:3]):
        assert torch.equal(_bits(a), _bits(b))
    assert torch.count_nonzero(outs[0][3]).item() == 0      # the workspace is left zero
    xh = ((x - mean) * invstd).double()
    rg = (dy.double() * xh).sum(0)
    rb = dy.double().sum(0)
    assert ((outs[0][0].double() - rg).norm() / rg.norm()).item() < 1e-5
    assert ((outs[0][1].double() - rb).norm() / rb.norm()).item() < 1e-5
