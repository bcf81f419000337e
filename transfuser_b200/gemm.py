"""Host wrappers over the GEMM entry points of the C-ABI (csrc/gemm_simt.cu, csrc/gemm_tc.cu)."""
import os

import torch

from . import _lib

# 'simt' (exact fp32 CUDA cores: the parity mode and the import-time default), 'bf16' (wgmma bf16 tensor cores, fp32
# accumulate: the throughput mode bench.py / Trainer select), 'bf16x3' / 'bf16x6' (the tensor-core PARITY modes: every fp32 operand
# is split into 2 / 3 bf16 terms — 16 / 24 of its mantissa bits — and a product runs as 3 / 6 tensor-core bf16 GEMMs, smallest terms
# first, accumulated in fp32: ~1e-5 relative per product for x3, fp32-grade for x6; the sidecar / fusion machinery of 'bf16' is
# off), 'tf32' (wgmma tf32 for K-major operands only)
MODE = os.environ.get('TFB_GEMM', 'simt')
MULTI_TERM = {'bf16x3': 2, 'bf16x6': 3}      # mode -> bf16 terms per operand


def set_mode(mode):
    global MODE
    assert mode in ('tf32', 'simt', 'bf16', 'bf16x3', 'bf16x6')
    MODE = mode


def multi_term():
    """True in the tensor-core parity modes."""
    return MODE in MULTI_TERM


def _ld(t):
    assert t.dim() == 2 and t.stride(1) == 1, 'row-major 2-D view required'
    return t.stride(0)


def gemm(a, b, out, trans_a=False, trans_b=False, bias=None, relu=False, alpha=1.0, beta=0.0, splits=1, mode=None):
    """out[M,N] = alpha * op(a) @ op(b) + beta*out (+bias) (relu). a, b, out: fp32 CUDA 2-D views with unit inner stride."""
    M, N = out.shape
    K = a.shape[0] if trans_a else a.shape[1]
    if MODE in MULTI_TERM and x3_ok(M, N, K, trans_a, trans_b):    # (also for callers that pin mode='simt': that means "exact")
        return gemm_x3(split_bf16(a), split_bf16(b), out, trans_a, trans_b, bias, relu, alpha, beta)
    mode = mode or MODE
    lda, ldb, ldc = _ld(a), _ld(b), _ld(out)
    use_tc = (mode == 'tf32' and not trans_a and trans_b and lda % 4 == 0 and ldb % 4 == 0 and a.data_ptr() % 16 == 0 and b.data_ptr() % 16 == 0
              and M >= 1 and N >= 8 and K >= 8)
    if use_tc:
        _lib.call('tfb_gemm_tf32_tc', int(trans_a), int(trans_b), M, N, K, a, lda, b, ldb, out, ldc, bias, int(relu),
                  float(alpha), float(beta), int(splits))
    else:
        _lib.call('tfb_gemm_f32_simt', int(trans_a), int(trans_b), M, N, K, a, lda, b, ldb, out, ldc, bias, int(relu),
                  float(alpha), float(beta), 1, 1, 0, 0, 0, 0, 0, 0)
    return out


def x3_ok(M, N, K, trans_a, trans_b):
    """Shapes the three-term bf16 product takes: the tensor-core kernel's minimum tile and 16-byte aligned rows of the (contiguous)
    split operands; everything else stays on the exact fp32 kernel."""
    lda, ldb = (M if trans_a else K), (K if trans_b else N)
    return M >= 16 and N >= 16 and K >= 16 and lda % 8 == 0 and ldb % 8 == 0


def split_bf16(x, terms=None):
    """fp32 2-D view (unit inner stride) -> tuple of `terms` contiguous bf16 matrices (default: the current mode's count) with
    x = t0 + t1 (+ t2): 16 (24) mantissa bits of x."""
    terms = terms or MULTI_TERM.get(MODE, 2)
    rows, cols = x.shape
    t = [torch.empty((rows, cols), dtype=torch.bfloat16, device=x.device) for _ in range(terms)]
    _lib.call('tfb_split_bf16', x, _ld(x), rows, cols, t[0], t[1], t[2] if terms > 2 else None, None, None, None)
    return tuple(t)


def gemm_x3(a, b, out, trans_a=False, trans_b=False, bias=None, relu=False, alpha=1.0, beta=0.0):
    """out = alpha * op(a) @ op(b) + beta*out (+bias) (relu) from pre-split operands a = (a0, a1[, a2]), b = (b0, b1[, b2]) (largest
    term first): the term-by-term tensor-core bf16 GEMMs whose order i + j is below the number of terms (3 products for 2 terms, 6 for 3;
    the dropped ones are below 2^-16 / 2^-24 of the result), smallest first, accumulated in fp32 in `out` (reduction epilogue)."""
    M, N = out.shape
    K = a[0].shape[0] if trans_a else a[0].shape[1]
    ldc = _ld(out)
    terms = len(a)
    pairs = sorted(((i, j) for i in range(terms) for j in range(terms) if i + j < terms), key=lambda p: (-(p[0] + p[1]), -p[0]))
    for n, (i, j) in enumerate(pairs):
        last = n == len(pairs) - 1
        _lib.call('tfb_gemm_bf16_tc', int(trans_a), int(trans_b), M, N, K, a[i], _ld(a[i]), b[j], _ld(b[j]), out, ldc,
                  bias if n == 0 else None, int(relu and last), float(alpha), float(beta if n == 0 else 1.0), 1)
    return out


def bgemm(a, b, out, M, N, K, lda, ldb, ldc, trans_a, trans_b, batch_outer, batch_inner, sa, sb, sc, alpha=1.0, beta=0.0):
    """Two-level strided-batched fp32 GEMM on raw (tensor-with-offset) operands: sa/sb/sc = (outer stride, inner stride)."""
    _lib.call('tfb_gemm_f32_simt', int(trans_a), int(trans_b), M, N, K, a, lda, b, ldb, out, ldc, None, 0, float(alpha), float(beta),
              batch_outer, batch_inner, sa[0], sa[1], sb[0], sb[1], sc[0], sc[1])
    return out


# ---------------------------------------------------------------------------------------------------------------------
# bf16 tensor-core mode: operands are bf16 copies (weights: maintained by the fused AdamW kernel inside the flat bf16 buffer;
# activations: cast once by the producing op and kept for backward instead of the fp32 tensor), accumulation and outputs fp32.
_FLAT = [None]
_WCACHE = {}


def attach_bf16_weights(flat_params):
    """flat_params: transfuser_b200.optim.FlatParams. Creates / refreshes the bf16 mirror of the flat fp32 weight buffer."""
    fp = flat_params
    if fp.bf16 is None:
        fp.bf16 = torch.empty(fp.total, dtype=torch.bfloat16, device=fp.flat.device)
    _lib.call('tfb_cast_bf16', fp.flat, fp.bf16, fp.total)
    _FLAT[0] = fp
    return fp.bf16


def to_bf16(x):
    """fp32 contiguous CUDA tensor -> bf16 copy (one HBM pass: 4 B read + 2 B written per element)."""
    assert x.is_contiguous() and x.dtype == torch.float32
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _lib.call('tfb_cast_bf16', x, y, x.numel())
    return y


def weight_bf16(w):
    """bf16 view of a weight: straight out of the flat mirror when the parameter lives in the flat buffer, else a cached cast
    (keyed on the tensor's in-place version counter)."""
    fp = _FLAT[0]
    if fp is not None:
        off = (w.data_ptr() - fp.flat.data_ptr()) // 4
        if 0 <= off < fp.total and w.is_contiguous():
            return fp.bf16[off:off + w.numel()].view(w.shape)
    key = id(w)
    hit = _WCACHE.get(key)
    if hit is not None and hit[0] == w._version and hit[1] == w.data_ptr():
        return hit[2]
    wb = to_bf16(w.detach().contiguous())
    _WCACHE[key] = (w._version, w.data_ptr(), wb)
    return wb


def tc_ok(M, N, K, *lds):
    """Shapes the tensor-core bf16 kernel takes (TMA: 16-byte aligned leading dimensions); everything else runs on the SIMT kernel."""
    return MODE == 'bf16' and M >= 32 and N >= 16 and K >= 16 and all(ld % 8 == 0 for ld in lds)


def gemm_bf16(a, b, out, trans_a=False, trans_b=False, bias=None, relu=False, alpha=1.0, beta=0.0, splits=1):
    """out[M,N] (fp32) = alpha * op(a) @ op(b) + beta*out (+bias) (relu); a, b bf16 2-D views with unit inner stride."""
    M, N = out.shape
    K = a.shape[0] if trans_a else a.shape[1]
    _lib.call('tfb_gemm_bf16_tc', int(trans_a), int(trans_b), M, N, K, a, _ld(a), b, _ld(b), out, _ld(out), bias, int(relu),
              float(alpha), float(beta), int(splits))
    return out
