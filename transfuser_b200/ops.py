"""torch.autograd.Function wrappers over the C-ABI kernels (include/tfb200.h): every forward AND backward below is a
hand-written sm_90a kernel launch; torch supplies device memory, the current stream and the autograd graph only.

Activations are NHWC fp32 ([N, H, W, C], contiguous); parameters keep the reference's PyTorch layouts so that the
reference's state_dicts load unchanged (SURVEY.md §8b)."""
import contextlib
import os
import weakref

import torch
import torch.distributed as dist
from torch.autograd import Function

from . import _lib
from . import gemm as G
from .gemm import bgemm, gemm

call = _lib.call

# Dropout randomness = hash(device base seed + call-site offset, element index). The base seed is a device-resident uint64
# advanced once per training step by `tick()` (a kernel, so it also advances inside a replayed CUDA graph); the offsets
# below are plain Python ints that identify the call site.
_SEED = {'off': 0, 'base': 0x5EED0000, 'dev': {}}


def manual_seed(seed):
    _SEED['base'] = int(seed) & 0x7FFFFFFFFFFF
    _SEED['dev'].clear()


def seed_state(device):
    t = _SEED['dev'].get(device)
    if t is None:
        t = torch.tensor([_SEED['base']], dtype=torch.int64, device=device)
        _SEED['dev'][device] = t
    return t


# Per-step arena of accumulators that kernels ADD into (BatchNorm statistics written by conv / GEMM epilogues, squeeze-excite pooling
# sums): one buffer per device, cleared by ONE memset at the start of the step (tick) and handed out in call order, so every step
# (and a captured CUDA graph) uses the same addresses and no kernel needs a clearing pass or a last-block clean-up of its own.
_ARENA = {}
ARENA_BYTES = 8 << 20


def _arena_take(device, nbytes, dtype):
    """A zeroed [nbytes / itemsize] tensor of `dtype` out of the step arena, or None when the arena is exhausted / not armed."""
    dev = torch.device(device)
    if dev.type == 'cuda' and dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    a = _ARENA.get(dev)
    if a is None:
        return None
    off = (a['off'] + 15) // 16 * 16
    if off + nbytes > ARENA_BYTES:
        return None
    a['off'] = off + nbytes
    # an independent tensor on the arena's storage (set_, not a view): it does not share the arena's version counter, so clearing
    # the arena at the next tick() never invalidates a tensor autograd saved from here
    item = torch.empty(0, dtype=dtype).element_size()
    return torch.empty(0, dtype=dtype, device=a['buf'].device).set_(a['buf'].untyped_storage(), off // item, (nbytes // item,))


def tick(device):
    """Advance the device-side dropout seed (call once per training step)."""
    call('tfb_step_tick', seed_state(device), None)
    dev = torch.device(device)
    if dev.type == 'cuda' and dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    a = _ARENA.get(dev)
    if a is None:
        a = _ARENA[dev] = dict(buf=torch.zeros(ARENA_BYTES, dtype=torch.uint8, device=dev), off=0, armed=True)
    if a['off'] > 0:
        a['buf'][:a['off']].zero_()          # what the last step handed out; everything beyond is still zero
    a['off'] = 0
    s = _SYNC.get(dev)
    if s is not None:
        s['chunk'], s['off'] = 0, 0
    _SEED['off'] = 0
    _BWD16.clear()
    _COL_CACHE.clear()
    _prepack_all(device)


# Per-step arena of the synchronized BatchNorms' fp64 slices (a rank's [sum x | sum x^2 | count] / [sum g | sum g*xhat], the W gathered
# slices, the folded sums): handed out in call order and rewound by tick(), so every step and a captured CUDA graph use the same
# addresses. Grown by whole chunks (kept for good) when a step needs more; nothing here is read before it is written.
_SYNC = {}
SYNC_CHUNK_BYTES = 4 << 20


def _sync_take(device, n, dtype=torch.float64):
    dev = torch.device(device)
    a = _SYNC.setdefault(dev, dict(chunks=[], chunk=0, off=0))
    item = torch.empty(0, dtype=dtype).element_size()
    nbytes = (n * item + 15) // 16 * 16
    while True:
        if a['chunk'] == len(a['chunks']):
            a['chunks'].append(torch.empty(max(SYNC_CHUNK_BYTES, nbytes), dtype=torch.uint8, device=dev))
        buf = a['chunks'][a['chunk']]
        if a['off'] + nbytes <= buf.numel():
            break
        a['chunk'], a['off'] = a['chunk'] + 1, 0
    off, a['off'] = a['off'], a['off'] + nbytes
    return torch.empty(0, dtype=dtype, device=dev).set_(buf.untyped_storage(), off // item, (n,))


def sync_group(bn):
    """The process group a training-mode BatchNorm normalises over: that of an nn.SyncBatchNorm (its `process_group`, WORLD when
    None) once a default process group exists, else None (per-rank statistics, plain nn.BatchNorm2d)."""
    if not isinstance(bn, torch.nn.SyncBatchNorm) or not (dist.is_available() and dist.is_initialized()):
        return None
    return bn.process_group if bn.process_group is not None else dist.group.WORLD


def _gather_slices(slice_, group):
    """[W * n] = the n-value slices of the W ranks of `group`, in rank order (all-gather: every rank then folds the same values in the
    same order, whatever algorithm the collective uses). gloo gathers CUDA tensors through host memory."""
    W = dist.get_world_size(group)
    out = _sync_take(slice_.device, W * slice_.numel())
    if slice_.is_cuda and dist.get_backend(group) == 'gloo':
        host = torch.empty(W * slice_.numel(), dtype=slice_.dtype)
        dist.all_gather_into_tensor(host, slice_.cpu(), group=group)
        out.copy_(host)
    else:
        dist.all_gather_into_tensor(out, slice_, group=group)
    return out, W


def _bn_fwd(x, y, M, C, weight, bias, momentum, eps, relu, running_mean, running_var, mean, invstd, stats, y16, residual, pooled,
            pool_batch, group):
    """Training-mode BatchNorm forward (see batch_norm); returns the synchronized BatchNorm's folded sums + total count, or None."""
    if group is None:
        if stats is not None:
            call('tfb_bn_fwd_stats', x, y, M, C, weight, bias, float(eps), float(momentum), int(relu), running_mean, running_var, mean, invstd,
                 stats, y16, residual, pooled, pool_batch)
        else:
            call('tfb_bn_fwd', x, y, M, C, weight, bias, float(eps), float(momentum), int(relu), running_mean, running_var, mean, invstd,
                 _ws(x.device), y16, residual, pooled, pool_batch)
        return None
    sl = _sync_take(x.device, 2 * C + 1)
    call('tfb_bn_sync_slice', x, M, C, stats, sl, _ws(x.device))
    g, W = _gather_slices(sl, group)
    folded = _sync_take(x.device, 2 * C + 1)
    call('tfb_bn_fwd_sync', x, y, M, C, weight, bias, float(eps), float(momentum), int(relu), running_mean, running_var, mean, invstd, g, W,
         folded, int(stats is not None), y16, residual, pooled, pool_batch)
    return folded


def _bn_bwd(x, dy, dx, M, C, weight, bias, mean, invstd, relu, dg, db, dx16, ymask=None, gmasked=None, se_gate=None, se_dpool=None, hw=1,
            group=None, folded=None):
    """Training-mode BatchNorm backward; `folded` / `group` from the synchronized forward (_bn_fwd)."""
    if group is None:
        if se_gate is not None:
            call('tfb_bn_bwd_se', x, dy, dx, M, C, weight, bias, mean, invstd, int(relu), dg, db, _ws(x.device), dx16, se_gate, se_dpool, hw)
        else:
            call('tfb_bn_bwd', x, dy, dx, M, C, weight, bias, mean, invstd, int(relu), dg, db, _ws(x.device), dx16, ymask, gmasked)
        return
    sl = _sync_take(x.device, 2 * C)
    call('tfb_bn_bwd_sync_reduce', x, dy, M, C, weight, bias, mean, invstd, int(relu), dg, db, _ws(x.device), ymask, se_gate, se_dpool, hw, sl)
    g, W = _gather_slices(sl, group)
    gsum = _sync_take(x.device, 2 * C, torch.float32)
    call('tfb_bn_bwd_sync_apply', x, dy, dx, M, C, weight, bias, mean, invstd, int(relu), g, W, folded[2 * C:], gsum, dx16, ymask, gmasked,
         se_gate, se_dpool, hw)


def next_seed():
    _SEED['off'] += 0x10000000
    return _SEED['off']


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


# bf16 sidecars: in bf16 mode the producer of a tensor-core operand (BatchNorm, SE gating, residual add, LayerNorm) writes the bf16
# copy in the same pass as its fp32 output; it travels as the `_tfb16` attribute of the fp32 tensor and the consuming GEMM / conv
# takes it instead of running a cast pass of its own. SIDECARS = False restores the separate cast launches.
SIDECARS = os.environ.get('TFB_SIDECARS', '1') == '1'
QKV_FUSED = os.environ.get('TFB_QKV_FUSED', '1') == '1'           # one q|k|v GEMM when the flat buffer packs the three weights
BN_ADD_FUSED = os.environ.get('TFB_BN_ADD_FUSED', '1') == '1'     # conv3.bn + shortcut add + ReLU as one BatchNorm call
SE_POOL_FUSED = os.environ.get('TFB_SE_POOL_FUSED', '1') == '1'   # SE average pool inside the preceding BatchNorm's pass
SE_FUSED_BWD = os.environ.get('TFB_SE_FUSED_BWD', '1') == '1'   # tfb_se_mlp_bwd (2 launches) instead of 8 small ones
CONV_S2_TC = os.environ.get('TFB_CONV_S2_TC', '1') == '1'       # bf16 mode: stride-2 3x3 convs forward on the tensor-core kernel (TMA element strides)
WGRAD_STREAM = os.environ.get('TFB_WGRAD_STREAM', '1') == '1'   # bf16 mode: weight-gradient GEMMs on a third stream (they only feed AdamW)
BN_STATS_FUSED = os.environ.get('TFB_BN_STATS_FUSED', '1') == '1'   # bf16 mode: BatchNorm statistics out of the producing conv / GEMM epilogue
# Weight-gradient GEMMs run on a side stream next to the critical dx chain. Letting their split-K fill every SM starves the chain;
# their persistent grid is capped at 64 CTAs (about half the chip) and the library picks tile width + split factor for THAT grid
# (csrc/gemm_tc.cu pick_bn).
WGRAD_AUTO_SPLIT = os.environ.get('TFB_WGRAD_AUTO_SPLIT', '1') == '1'
WGRAD_MAX_CTAS = int(os.environ.get('TFB_WGRAD_MAX_CTAS', '64'))
NARROW_DGRAD_TC = os.environ.get('TFB_NARROW_DGRAD_TC', '1') == '1'   # dgrad of 3x3 convs with < 8 output channels on the tensor cores (padded dy)
DECODER_STREAMS = os.environ.get('TFB_DECODER_STREAMS', '0') == '1'   # segmentation and depth decoders on two side streams (measured: no gain once
#                                                                        the upsample kernels were vectorised; off)
BN_SE_FUSED = os.environ.get('TFB_BN_SE_FUSED', '1') == '1'     # Bottleneck conv2.bn + squeeze-excite as one autograd node (SE gradient folded into BatchNorm backward)
ADD_LN_FUSED = os.environ.get('TFB_ADD_LN_FUSED', '1') == '1'   # GPT: residual add + dropout + the next LayerNorm in one launch
ATTN_FUSED = os.environ.get('TFB_ATTN_FUSED', '1') == '1'       # bf16 mode: fused tensor-core attention (csrc/attn_tc.cu), no T x T tensor in HBM
# bf16 mode: the weight gradients of the 3x3 convs made inside implicit_wgrad() (the model's forward) without the bf16 im2col
# matrix: the wgrad GEMM gathers its tiles from the activation (tfb_conv3x3_tc_wgrad)
IMPLICIT_WGRAD = os.environ.get('TFB_IMPLICIT_WGRAD', '1') == '1'
_IMPLICIT_SCOPE = [0]


@contextlib.contextmanager
def implicit_wgrad():
    """The 3x3 convs conv2d makes inside this context take the im2col-free weight gradient (tfb_conv3x3_tc_wgrad) when their
    backward runs on the tensor cores; outside it they keep im2col + the batched wgrad GEMM (the same bits)."""
    _IMPLICIT_SCOPE[0] += 1
    try:
        yield
    finally:
        _IMPLICIT_SCOPE[0] -= 1


def _emit16(x, want):
    """bf16 buffer for the sidecar of a tensor shaped like x, or None when not wanted."""
    if want and SIDECARS and G.MODE == 'bf16':
        return torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    return None


def _attach16(y, y16):
    if y16 is not None:
        y._tfb16, y._tfb16v = y16, y._version       # version stamp: an in-place edit of y afterwards invalidates the sidecar (_as16)
        y._tfb16e = None                            # written by y's own producer kernel: whoever may read y may read the sidecar
    return y


def _as16(x):
    """bf16 copy of the contiguous fp32 tensor x: its sidecar when the producer wrote one, else a cast pass."""
    s = getattr(x, '_tfb16', None)
    if s is not None and s.shape == x.shape and getattr(x, '_tfb16v', x._version) == x._version:
        evt = getattr(x, '_tfb16e', None)
        if evt is not None and x.is_cuda:
            # the copy was made lazily by an earlier consumer, possibly on ANOTHER stream (the image grid feeds the segmentation
            # decoder on one side stream and the depth decoder on a second one): order this stream behind that cast. Without it the
            # second decoder read the bf16 copy before it was written whenever the streams really ran concurrently (graph replay):
            # loss_depth came out doubled under CUDA-graph replay — found by tools/graph_vs_eager.py in round 2.
            cur = torch.cuda.current_stream(x.device)
            if cur.cuda_stream != evt[0]:
                cur.wait_event(evt[1])
                s.record_stream(cur)
        return s
    s = G.to_bf16(x)
    if SIDECARS:
        x._tfb16, x._tfb16v = s, x._version      # a tensor with several tensor-core consumers (p2 -> 8 head convs) is cast once
        if x.is_cuda:
            cur = torch.cuda.current_stream(x.device)
            evt = torch.cuda.Event()
            evt.record(cur)
            x._tfb16e = (cur.cuda_stream, evt)
    return s


# Backward sidecars: BatchNorm backward writes the bf16 copy of dx next to dx when the convolution in front of it runs its dgrad /
# wgrad on the tensor cores; that convolution's backward finds it here by (address, size) instead of running a cast pass over dy.
# An entry keeps a reference to the fp32 gradient, so its memory cannot be recycled (and the key cannot alias another live tensor)
# while the entry exists; entries are popped by the consumer and dropped wholesale at the start of the next step (tick()).
_BWD16 = {}


def _offer16(t, t16):
    if len(_BWD16) > 512:
        _BWD16.clear()
    _BWD16[(t.data_ptr(), t.numel())] = (t, t16, t._version)


def _take16(t):
    """bf16 sidecar of the contiguous fp32 gradient t (same memory as the tensor it was offered for), or None."""
    e = _BWD16.pop((t.data_ptr(), t.numel()), None)
    if e is None or e[0]._version != e[2] or t.dtype != torch.float32 or not t.is_contiguous():
        return None
    return e[1].view(t.shape)


def record_stream(t, stream):
    """Tensor.record_stream for a tensor that crosses streams, sidecar included."""
    t.record_stream(stream)
    s = getattr(t, '_tfb16', None)
    if s is not None:
        s.record_stream(stream)


def _view16(x, v):
    """v = a view (reshape) of x: carries x's sidecar over to v under the same reshape."""
    s = getattr(x, '_tfb16', None)
    if s is not None and v.is_contiguous() and x.is_contiguous():
        v._tfb16, v._tfb16e = s.view(v.shape), getattr(x, '_tfb16e', None)
    return v


_WS = {}
_SIDE = {}
TWO_STREAMS = os.environ.get('TFB_TWO_STREAMS', '1') == '1'


def side_stream(device):
    """The second CUDA stream on which independent branches of the step run (LiDAR trunk, auxiliary decoders)."""
    device = torch.device(device)
    s = _SIDE.get(device)
    if s is None:
        s = torch.cuda.Stream(device=device)
        _SIDE[device] = s
    return s


def side_stream2(device):
    """A further side stream (the depth decoder runs next to the segmentation decoder on it)."""
    device = torch.device(device)
    key = ('side2', device)
    s = _SIDE.get(key)
    if s is None:
        s = _SIDE[key] = torch.cuda.Stream(device=device)
    return s


def _capturing(stream):
    with torch.cuda.stream(stream):
        return torch.cuda.is_current_stream_capturing()


def side_streams(device):
    """The side streams on `device` that the caller may wait for: all of them normally; while the current stream is being captured
    into a CUDA graph only those that were forked into the same capture (waiting for an event of a stream outside the capture
    invalidates it — a stream created by an earlier model / configuration and not used by this step is simply skipped)."""
    device = torch.device(device)
    out = [s for s in _SIDE.values() if s.device == device or (device.index is None and s.device.type == device.type)]
    if out and torch.cuda.is_current_stream_capturing():
        out = [s for s in out if _capturing(s)]
    return out


def join_side_streams():
    """Make the current stream wait for all work queued on the side streams (used before NCCL calls issued from autograd hooks)."""
    if not _SIDE:
        return
    cur = torch.cuda.current_stream()
    for s in side_streams(cur.device):
        cur.wait_stream(s)



_JOIN_QUEUED = [False]


def _join_after_backward():
    _JOIN_QUEUED[0] = False
    join_side_streams()


class _OnWgradStream:
    """`with _OnWgradStream(dev, t1, t2, ...):` — runs the enclosed launches on the weight-gradient stream. Weight gradients feed
    nothing but the optimizer, so their GEMMs (split-K, a few dozen CTAs each) need not sit on the critical dx chain: they run next
    to it and are joined (join_side_streams) before the gradient all-reduce / AdamW. The listed tensors are the ones the launches
    read or write; record_stream keeps the caching allocator from recycling them while the side stream still uses them."""

    def __init__(self, device, *tensors):
        self.on = WGRAD_STREAM and G.MODE == 'bf16' and torch.device(device).type == 'cuda'
        self.device, self.tensors = device, tensors

    def __enter__(self):
        if self.on:
            device = torch.device(self.device)
            if not _JOIN_QUEUED[0] and torch._C._current_graph_task_id() != -1:
                # inside a backward pass: make the caller's stream wait for the side streams when this backward() returns
                _JOIN_QUEUED[0] = True
                torch.autograd.Variable._execution_engine.queue_callback(_join_after_backward)
            key = ('wgrad', device)
            s = _SIDE.get(key)
            if s is None:
                s = _SIDE[key] = torch.cuda.Stream(device=device)
            s.wait_stream(torch.cuda.current_stream(device))
            for t in self.tensors:
                if t is not None:
                    t.record_stream(s)
            self.ctx = torch.cuda.stream(s)
            self.ctx.__enter__()
            if WGRAD_MAX_CTAS > 0:
                call('tfb_gemm_set_max_ctas', WGRAD_MAX_CTAS)
        return self

    def __exit__(self, *exc):
        if self.on:
            if WGRAD_MAX_CTAS > 0:
                call('tfb_gemm_set_max_ctas', 0)
            self.ctx.__exit__(*exc)
        return False


def _ws(device):
    """The per-device reduction workspace (fp64 sums + arrival counter) shared by every BatchNorm / bias-gradient reduction:
    the kernels require it to be zero on entry and leave it zero on exit (last-block finalisation), so it is zeroed only once."""
    key = (device, torch.cuda.current_stream(device).cuda_stream)   # one workspace per stream: kernels of a stream run in order
    t = _WS.get(key)
    if t is None:
        t = torch.zeros(2 * 8192 + 8, dtype=torch.float64, device=device)
        _WS[key] = t
    return t


def _gbuf(p):
    """Output buffer for the gradient of parameter `p`. When the model was flattened (optim.flatten) and p.grad is None
    (zero_grad(set_to_none=True)), this is p's view of the flat gradient buffer: the backward kernel writes the gradient in
    place, autograd adopts the tensor as p.grad without a copy, and the fused AdamW / all-reduce read the flat buffer."""
    info = getattr(p, '_tfb_flat', None)
    if info is not None and p.grad is None:
        fp, off = info
        if off not in fp.taken:                      # a second producer in the same backward (shared parameter) must not overwrite
            fp.taken.add(off)                        # the first one's result: it gets a fresh buffer and autograd adds the two
            return fp.grad[off:off + p.numel()].view(p.shape)
    return torch.empty(p.shape, dtype=torch.float32, device=p.device)


def _pack3(a, b, c):
    """The tensor that three equally-shaped contiguous tensors form when they lie back to back in ONE storage (the q|k|v packs
    of optim.FlatParams): shape [3 * a.shape[0], ...]. None when they do not."""
    if a is None or b is None or c is None or not (a.shape == b.shape == c.shape):
        return None
    if not (a.is_contiguous() and b.is_contiguous() and c.is_contiguous()):
        return None
    n = a.numel() * a.element_size()
    base = a.untyped_storage().data_ptr()
    if b.data_ptr() != a.data_ptr() + n or c.data_ptr() != b.data_ptr() + n or c.untyped_storage().data_ptr() != base:
        return None
    return a.detach().as_strided((3 * a.shape[0],) + tuple(a.shape[1:]), a.stride())


def _gbuf3(pq, pk, pv):
    """Gradient buffer of a q|k|v pack as ONE [3n, ...] tensor: the pack's span of the flat gradient buffer when all three
    parameters are flat and have no .grad yet (their gradients are then views of it, adopted by autograd without a copy)."""
    infos = [getattr(p, '_tfb_flat', None) for p in (pq, pk, pv)]
    n = pq.numel()
    if all(i is not None for i in infos) and all(p.grad is None for p in (pq, pk, pv)) \
            and infos[1][1] == infos[0][1] + n and infos[2][1] == infos[1][1] + n \
            and not any(i[1] in infos[0][0].taken for i in infos):
        fp, off = infos[0]
        fp.taken.update(i[1] for i in infos)
        return fp.grad[off:off + 3 * n].view((3 * pq.shape[0],) + tuple(pq.shape[1:]))
    return torch.empty((3 * pq.shape[0],) + tuple(pq.shape[1:]), dtype=torch.float32, device=pq.device)


def _colsum(x2d, out=None):
    M, C = x2d.shape
    if out is None:
        out = torch.empty(C, dtype=torch.float32, device=x2d.device)
    ws = _ws(x2d.device)
    ld = C if x2d.is_contiguous() else x2d.stride(0)
    assert x2d.is_contiguous() or x2d.stride(1) == 1
    call('tfb_colsum', x2d, ld, M, C, out, ws)
    return out


def _grad_prep(dy2d, y2d, want32, want16, bias_p):
    """One pass over dy: ReLU mask (y2d given), fp32 / bf16 copies as requested, bias gradient. Returns (g32, g16, db)."""
    M, C = dy2d.shape
    dev = dy2d.device
    g32 = torch.empty((M, C), dtype=torch.float32, device=dev) if (want32 and y2d is not None) else None
    g16 = torch.empty((M, C), dtype=torch.bfloat16, device=dev) if want16 else None
    db = _gbuf(bias_p) if bias_p is not None else None
    ws = _ws(dev) if db is not None else None
    if g32 is not None or g16 is not None or db is not None:
        call('tfb_grad_prep', dy2d, y2d, g32, g16, db, ws, M, C)
    if want32 and g32 is None:
        g32 = dy2d
    return g32, g16, db


def _relu_bwd(y, dy):
    g = torch.empty_like(dy)
    call('tfb_relu_bwd', y, dy, g, dy.numel())
    return g


# ------------------------------------------------------------------ dense layers (GEMM) and convolutions
def _wgrad_splits(M, N, K):
    """split-K factor for dW[N,K] = dy^T x with a long contraction (M rows): aim for >= 2 waves of 128x128 tiles."""
    if WGRAD_AUTO_SPLIT:
        return 0          # the library picks tile width and split factor together (csrc/gemm_tc.cu pick_bn: one wave of SMs, >= 4 k-blocks per CTA)
    tiles = ((N + 127) // 128) * ((K + 127) // 128)
    return max(1, min(64, (296 + tiles - 1) // tiles, M // 2048 if M >= 4096 else 1))


class LinearFn(Function):
    """y[M,N] = x[M,K] @ w[N,K]^T + b (ReLU). nn.Linear (transfuser.py:498-506, 538-543) and 1x1 nn.Conv2d as a GEMM.
    bf16 mode: x is cast once (kept for backward instead of the fp32 tensor), the weight comes from the bf16 mirror, and
    forward / dgrad / wgrad all run on the tensor-core kernel (K-major / MN-major operand descriptors, no transposes)."""

    @staticmethod
    def forward(ctx, x, w, bias, relu, want_stats=False):
        x = _c(x)
        w2 = w.view(w.shape[0], -1)
        M, K = x.shape
        N = w2.shape[0]
        y = torch.empty((M, N), dtype=torch.float32, device=x.device)
        ctx.tc = G.tc_ok(M, N, K, K, N)
        if ctx.tc:
            xs = _as16(x)
            st = _arena_take(x.device, 2 * N * 8, torch.float64) if (want_stats and bias is None and not relu and N % 4 == 0) else None
            if st is not None:
                # training-mode BatchNorm follows: its per-channel sum / sum of squares come out of this GEMM's epilogue
                wb = G.weight_bf16(w2)
                call('tfb_gemm_bf16_tc_stats', M, N, K, xs, xs.stride(0), wb, wb.stride(0), y, N, st)
                y._tfb_stats = st
            else:
                G.gemm_bf16(xs, G.weight_bf16(w2), y, trans_b=True, bias=bias, relu=relu)
        else:
            xs = x
            if M <= 16:
                call('tfb_gemm_small_m', 1, M, N, K, x, K, w2, K, y, N, bias, 1 if relu else 0)
            else:
                gemm(x, w2, y, trans_b=True, bias=bias, relu=relu, mode='simt')
        ctx.save_for_backward(xs, w, y if relu else None, bias)
        ctx.relu, ctx.has_bias = relu, bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        xs, w, y, bias_p = ctx.saved_tensors
        dy = _c(dy)
        w2 = w.view(w.shape[0], -1)
        M, K = xs.shape
        N = w2.shape[0]
        want_db = ctx.has_bias and ctx.needs_input_grad[2]
        gb = _take16(dy) if (ctx.tc and not ctx.relu and not want_db) else None
        if gb is not None:
            g, db = None, None              # dy's producer (BatchNorm backward) already wrote its bf16 copy: no pass over dy here
        else:
            g, gb, db = _grad_prep(dy, y if ctx.relu else None, not ctx.tc, ctx.tc, bias_p if want_db else None)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty((M, K), dtype=torch.float32, device=dy.device)
            if ctx.tc:
                G.gemm_bf16(gb, G.weight_bf16(w2), dx, trans_b=False)
            elif M <= 16:
                call('tfb_gemm_small_m', 0, M, K, N, g, N, w2, K, dx, K, None, 0)
            else:
                gemm(g, w2, dx, trans_b=False, mode='simt')
        if ctx.needs_input_grad[1]:
            dw = _gbuf(w)
            if ctx.tc:
                with _OnWgradStream(dy.device, gb, xs, dw):
                    G.gemm_bf16(gb, xs, dw.view(w2.shape), trans_a=True, splits=_wgrad_splits(M, N, K))
            elif M >= 4096 and not (G.multi_term() and G.x3_ok(N, K, M, True, False)):
                # long contraction, narrow output (head 1x1 convs): the pixel-split direct-conv wgrad kernel (k = 1)
                call('tfb_conv2d_wgrad', xs, g, dw, None, 1, M, 1, K, N, 1, 1, 1)
            else:
                gemm(g, xs, dw.view(w2.shape), trans_a=True, mode='simt')
        return dx, dw, db, None, None


def linear(x, w, bias=None, relu=False):
    lead = x.shape[:-1]
    y = LinearFn.apply(_view16(x, x.reshape(-1, x.shape[-1])), w, bias, relu)
    return y.view(*lead, y.shape[-1])


class Conv2dFn(Function):
    """NHWC conv, k in {1,3}, pad k//2, stride {1,2}, groups. 1x1/stride-1/groups-1 goes to LinearFn instead."""

    @staticmethod
    def forward(ctx, x, w, bias, stride, groups, relu, want_stats=False, implicit_wgrad=False):
        x = _c(x)
        N, H, W, Cin = x.shape
        Cout, ks = w.shape[0], w.shape[2]
        Ho, Wo = (H + 2 * (ks // 2) - ks) // stride + 1, (W + 2 * (ks // 2) - ks) // stride + 1
        plan = _conv_tc_plan(Cin, Cout, groups) if (G.MODE == 'bf16' and CONV_S2_TC and ks == 3 and stride == 2) else None
        ctx.x3 = _conv_x3_ok(x.shape, Cout, ks, stride, groups)
        if ctx.x3:
            # tensor-core parity mode, dense 3x3: im2col of the two bf16 terms of x, then the three-term GEMM against the split weights
            y = torch.empty((N, Ho, Wo, Cout), dtype=torch.float32, device=x.device)
            G.gemm_x3(_im2col_x3(x), G.split_bf16(w.view(Cout, Cin * 9)), y.view(-1, Cout), trans_b=True, bias=bias, relu=relu)
        elif plan is not None:
            # stride 2 on the tensor cores: same implicit-GEMM kernel, the TMA map steps two pixels per box element
            y = _conv_tc_run(_as16(x), w, bias, plan, 0, Cout, groups, relu, stride=2, want_stats=want_stats)
        else:
            y = torch.empty((N, Ho, Wo, Cout), dtype=torch.float32, device=x.device)
            call('tfb_conv2d_fwd', x, w, bias, y, N, H, W, Cin, Cout, ks, stride, groups, int(relu))
        ctx.save_for_backward(x, w, y if relu else None, bias)
        ctx.cfg = (N, H, W, Cin, Cout, ks, stride, groups, relu, bias is not None)
        ctx.implicit_wgrad = implicit_wgrad
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y, bias_p = ctx.saved_tensors
        N, H, W, Cin, Cout, ks, stride, groups, relu, has_bias = ctx.cfg
        dy = _c(dy)
        g = _relu_bwd(y, dy) if relu else dy
        dx = dw = db = None
        if ctx.x3:
            g = _c(g)
            if ctx.needs_input_grad[0]:
                # dgrad = the 3x3 conv of g with the transposed, tap-flipped weights: w'[ci][co][kh][kw] = w[co][ci][2-kh][2-kw]
                wt = w.detach().flip(2, 3).transpose(0, 1).contiguous().view(Cin, Cout * 9)
                dx = torch.empty_like(x)
                G.gemm_x3(_im2col_x3(g), G.split_bf16(wt), dx.view(-1, Cin), trans_b=True)
            if ctx.needs_input_grad[1]:
                dw = _gbuf(w)
                G.gemm_x3(G.split_bf16(g.view(-1, Cout)), _im2col_x3(x), dw.view(Cout, Cin * 9), trans_a=True)
                db = _colsum(g.view(-1, Cout), _gbuf(bias_p)) if has_bias else None
            return dx, dw, db, None, None, None, None, None
        if ctx.needs_input_grad[0]:
            plan = _conv_tc_plan(Cout, Cin, groups) if (G.MODE == 'bf16' and ks == 3 and stride == 2) else None
            if plan is not None:
                # stride-2 dgrad = stride-1 dgrad of the zero-dilated dy (tensor cores; 3/4 of the MMA work hits zeros, which is
                # cheaper than the CUDA-core kernel)
                up = torch.empty((N, H, W, Cout), dtype=torch.bfloat16, device=g.device)
                call('tfb_dilate2', g, up, N, H, W, Cout, 1)
                dx = _conv_tc_run(up, w, None, plan, 1, Cin, groups, False)
            else:
                dx = torch.empty_like(x)
                call('tfb_conv2d_dgrad', g, w, dx, N, H, W, Cin, Cout, ks, stride, groups)
        if ctx.needs_input_grad[1]:
            if G.MODE == 'bf16' and ks == 3 and Cout % 8 == 0 and _conv_wgrad_tc_ok(x.shape, Cout, groups, stride):
                g16 = _take16(dy) if not relu else None       # (the 3-channel stems stay on the direct kernel: no cast for them)
                dw = _conv_wgrad_tc(x, g16 if g16 is not None else G.to_bf16(g), w, groups, stride, ctx.implicit_wgrad)
                if dw is not None and has_bias:
                    db = _colsum(g.view(-1, Cout), _gbuf(bias_p))
            if dw is None:
                dw = _gbuf(w)
                db = _gbuf(bias_p) if has_bias else None
                call('tfb_conv2d_wgrad', x, g, dw, db, N, H, W, Cin, Cout, ks, stride, groups)
        return dx, dw, db, None, None, None, None, None


def _conv_x3_ok(x_shape, Cout, ks, stride, groups):
    """Dense 3x3 / stride-1 convs the 'bf16x3' parity mode runs on the tensor cores (im2col + three-term GEMM, forward, dgrad and
    wgrad); grouped 3x3 convs (24 channels per group: few FLOPs), the 3-channel stems and outputs narrower than 16 channels stay
    on the exact fp32 direct kernels."""
    N, H, W, Cin = x_shape
    return (G.multi_term() and ks == 3 and stride == 1 and groups == 1 and Cin % 8 == 0 and Cout % 8 == 0 and Cin >= 16 and Cout >= 16
            and N * H * W >= 32)


def _im2col_x3(x):
    """bf16 im2col matrices [N*H*W, 9*C] ((channel, tap) column order) of the 2 / 3 bf16 terms of the NHWC fp32 tensor x."""
    N, H, W, C = x.shape
    terms = G.MULTI_TERM[G.MODE]
    t32 = [torch.empty_like(x) for _ in range(terms)]
    call('tfb_split_bf16', x, C, N * H * W, C, None, None, None, t32[0], t32[1], t32[2] if terms > 2 else None)
    cols = []
    for t in t32:                    # (exactly bf16-representable fp32 values: the cast inside the im2col kernel is exact)
        col = torch.empty((N * H * W, 9 * C), dtype=torch.bfloat16, device=x.device)
        call('tfb_im2col3x3_bf16', t, col, N, H, W, C, 1, 1)
        cols.append(col)
    return tuple(cols)


def _conv_tc_plan(c_read, c_write, groups):
    """Tile plan of csrc/conv_tc.cu for a 3x3 stride-1 conv that READS a tensor with c_read channels and WRITES c_write
    channels (forward: Cin -> Cout; dgrad: Cout -> Cin). Returns None when the shape must stay on the direct kernel."""
    if c_read % 8 != 0:
        return None                                  # TMA needs 16-byte channel rows
    if groups > 1:
        cg_r, cg_w = c_read // groups, c_write // groups
        if cg_r != 24 or cg_w != 24:
            return None
        gblocks = (groups + 1) // 2                  # two 24-wide groups per CTA: N = 48, one 64-channel K window
        return dict(NB=48, KC=64, c_step=48, nchunks=1, nb_real=48, gblocks=gblocks)
    kc = 32 if c_read <= 32 else 64
    nchunks = (c_read + kc - 1) // kc
    nb = 16 if c_write <= 16 else 32 if c_write <= 32 else 64 if c_write <= 64 else 128
    if kc == 32 and nb > 64:
        return None                                  # (32-channel rows exist for NB <= 64 tiles only)
    gblocks = (c_write + nb - 1) // nb
    return dict(NB=nb, KC=kc, c_step=0, nchunks=nchunks, nb_real=nb if gblocks > 1 else c_write, gblocks=gblocks)


# Packed bf16 weights of the tensor-core 3x3 convs. Every (weight, direction) gets a persistent packed buffer on first use. Inside a
# training step (between tick() and the optimizer step) the weights do not change, so tick() re-packs ALL registered convs in one
# launch (tfb_conv3x3_pack_weights_batched) and the convs of that step's forward and backward reuse the buffers; anything else
# (eval, a weight whose tensor version moved, PACK_BATCHED off) packs per call as before. invalidate_packs() must follow every
# weight update that does not bump tensor versions (the fused AdamW kernel, CUDA-graph replays).
PACK_BATCHED = os.environ.get('TFB_PACK_BATCHED', '1') == '1'
_PACKS = {}                      # (id(weight), mode) -> _Pack
_PACK_STATE = {'epoch': 0, 'sig': None, 'table': None}


class _Pack:
    __slots__ = ('wref', 'ptr', 'wp', 'args', 'epoch', 'version')


def invalidate_packs():
    _PACK_STATE['epoch'] += 1


def _packed_weights(w, plan, mode, groups):
    args = (tuple(w.shape), groups, plan['NB'], plan['KC'], plan['c_step'], plan['nchunks'], plan['nb_real'], plan['gblocks'])
    key = (w.data_ptr(), mode)               # by address: the same parameter may reach forward and backward as different wrappers
    e = _PACKS.get(key)
    if e is not None and (e.wref() is None or e.args != args or e.wp.device != w.device):
        e = None
    if e is None:
        e = _Pack()
        e.wref, e.ptr, e.args, e.epoch, e.version = weakref.ref(w), w.data_ptr(), args, -1, -1
        e.wp = torch.empty((plan['gblocks'], plan['nchunks'], 9, plan['NB'], plan['KC']), dtype=torch.bfloat16, device=w.device)
        _PACKS[key] = e                        # (entries of dead weights are pruned by _prepack_all; nothing else is ever dropped:
        #                                        a captured CUDA graph may hold the addresses of the packed buffers)
        _PACK_STATE['sig'] = None
    return e


def _prepack_all(device):
    """One launch re-packs every registered conv weight that lives on `device` (called by tick() at the start of a training step)."""
    if not PACK_BATCHED:
        return
    device = torch.device(device)
    live = []
    for key, e in list(_PACKS.items()):
        w = e.wref()
        if w is None or w.data_ptr() != e.ptr:        # the parameter died or was re-homed (optim.flatten): forget the entry
            del _PACKS[key]
            _PACK_STATE['sig'] = None
        elif w.is_contiguous() and w.device.type == device.type and device.index in (None, w.device.index):
            live.append((key[1], e, w))
    if not live:
        return
    rows = []
    for mode, e, w in live:
        groups = e.args[1]
        rows.append([e.ptr, e.wp.data_ptr(), w.shape[0], w.shape[1] * groups, groups, mode] + list(e.args[2:]))
    sig = tuple(map(tuple, rows))
    if _PACK_STATE['sig'] != sig:
        if device.type == 'cuda' and torch.cuda.is_current_stream_capturing():
            return          # no host-to-device copy inside a graph capture: this step's convs pack per call (epoch not advanced)
        _PACK_STATE['table'] = torch.tensor(rows, dtype=torch.int64).to(device)
        _PACK_STATE.setdefault('keep', []).append(_PACK_STATE['table'])   # never freed: a captured graph may still read an old table
        _PACK_STATE['sig'] = sig
    call('tfb_conv3x3_pack_weights_batched', _PACK_STATE['table'], len(rows), 8)
    _PACK_STATE['epoch'] += 1
    for _, e, w in live:
        e.epoch, e.version = _PACK_STATE['epoch'], w._version


def _packed_current(w, plan, mode, groups):
    """The packed buffer of (w, mode), re-packed now unless the batched re-pack of this step already covered it."""
    Cout, Cin = (w.shape[0], w.shape[1] * groups)
    e = _packed_weights(w, plan, mode, groups)
    if not (PACK_BATCHED and e.epoch == _PACK_STATE['epoch'] and e.version == w._version):
        call('tfb_conv3x3_pack_weights', w, e.wp, Cout, Cin, groups, mode, plan['NB'], plan['KC'], plan['c_step'], plan['nchunks'],
             plan['nb_real'], plan['gblocks'])
    return e


def _conv_tc_run(x16, w, bias, plan, mode, c_write, groups, relu, stride=1, want_stats=False):
    N, H, W, c_read = x16.shape
    e = _packed_current(w, plan, mode, groups)
    y = torch.empty((N, (H - 1) // stride + 1, (W - 1) // stride + 1, c_write), dtype=torch.float32, device=x16.device)
    st = None
    if want_stats and bias is None and not relu and c_write % 4 == 0 and plan['nb_real'] % 4 == 0:
        st = _arena_take(x16.device, 2 * c_write * 8, torch.float64)
    if stride == 1 and st is None:
        call('tfb_conv3x3_tc', x16, e.wp, bias, y, N, H, W, c_read, c_write, plan['NB'], plan['KC'], plan['c_step'], plan['nchunks'], plan['nb_real'],
             plan['gblocks'], int(relu))
    else:
        call('tfb_conv3x3_tc_strided', x16, e.wp, bias, y, N, H, W, c_read, c_write, plan['NB'], plan['KC'], plan['c_step'], plan['nchunks'],
             plan['nb_real'], plan['gblocks'], int(relu), stride, st)
    if st is not None:
        y._tfb_stats = st
    return y


_COL_CACHE = {}     # (input address, shape, stride, groups) -> (input tensor, its bf16 im2col matrix, input version); dropped at tick()


def _conv_wgrad_tc_ok(x_shape, Cout, groups, stride):
    """Shapes _conv_wgrad_tc takes: 16-byte aligned channel windows and enough output pixels for a split-K GEMM."""
    N, H, W, Cin = x_shape
    Cig, Cog = Cin // groups, Cout // groups
    if Cig % 8 or (groups > 1 and Cog % 8):
        return False
    return N * ((H - 1) // stride + 1) * ((W - 1) // stride + 1) >= 512


def _conv_wgrad_tc(x, g16, w, groups, stride, implicit=False):
    """dW of a 3x3 conv on the tensor cores: one split-K GEMM per channel group (dW_g[Cog, Cig*9] = dy_g^T col_g, batched over groups
    in a single launch) over the bf16 im2col matrix col of x, written in PyTorch's [co][ci][kh][kw] layout into the gradient buffer.
    implicit: the GEMM's producer gathers each tile of col from the bf16 copy of x (tfb_conv3x3_tc_wgrad) instead of reading a matrix that
    tfb_im2col3x3_bf16 wrote; same tiles, split and fold, so the same bits. Returns None when the shape does not fit (channel
    windows must be 16-byte aligned)."""
    N, H, W, Cin = x.shape
    Cout = w.shape[0]
    Cig, Cog = Cin // groups, Cout // groups
    if not _conv_wgrad_tc_ok(x.shape, Cout, groups, stride):
        return None
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    M = N * Ho * Wo
    ldg = g16.shape[-1]                      # > Cout when dy was zero-padded to 8 channels (the 7- / 1-channel decoder outputs)
    rows = max(Cout, ldg) if groups == 1 else Cout
    ntiles = groups * ((9 * Cig + 127) // 128)
    splits = 0 if WGRAD_AUTO_SPLIT else max(1, min(128, (2 * 132 + ntiles - 1) // ntiles, M // 256))
    dw = _gbuf(w)
    if implicit and IMPLICIT_WGRAD and 'tfb_conv3x3_tc_wgrad' in _lib.lib().fns:
        x16 = _as16(x)                       # (the producers' bf16 copies round to nearest, as the im2col kernel does)
        with _OnWgradStream(x.device, x16, g16, dw):
            work = torch.empty(rows * 9 * Cig, dtype=torch.float32, device=x.device)
            call('tfb_conv3x3_tc_wgrad', x16, g16, dw, work, N, H, W, Cin, Cout, ldg, groups, stride, splits)
        return dw
    # the seven CenterNet heads and the BEV head all convolve the same p2 map: its im2col matrix is built once per backward
    key = (x.data_ptr(), tuple(x.shape), stride, groups)
    with _OnWgradStream(x.device, x, g16, dw):
        hit = _COL_CACHE.get(key)
        if hit is not None and hit[2] == x._version:          # (the entry pins the input it was built from: the address cannot be reused)
            col = hit[1]
        else:
            col = torch.empty((M, 9 * Cin), dtype=torch.bfloat16, device=x.device)
            call('tfb_im2col3x3_bf16', x, col, N, H, W, Cin, stride, groups)
            if col.numel() * 2 <= (128 << 20):                # small maps only (p2: 47 MB); the 160x704 decoder maps are not shared anyway
                if len(_COL_CACHE) >= 2:
                    _COL_CACHE.pop(next(iter(_COL_CACHE)))
                _COL_CACHE[key] = (x, col, x._version)
        dwp = dw.view(Cout, 9 * Cig) if rows == Cout else torch.empty((rows, 9 * Cig), dtype=torch.float32, device=x.device)
        call('tfb_gemm_bf16_tc_wgrad_batched', Cog if groups > 1 else rows, 9 * Cig, M, g16, ldg, Cog if groups > 1 else 0, col, 9 * Cin,
             9 * Cig if groups > 1 else 0, dwp, 9 * Cig, Cog * 9 * Cig, groups, splits)
        if rows != Cout:
            call('tfb_scale_dev', dwp, None, 1.0, dw, Cout * 9 * Cig, 0)      # the first Cout rows are the gradient; the rest is padding
    return dw


class Conv3x3TCFn(Function):
    """3x3 / stride 1 conv in bf16 mode: forward and dgrad as implicit GEMMs on the wgmma tensor cores (csrc/conv_tc.cu:
    TMA tap-shifted NHWC tiles, no im2col); wgrad on the fp32 direct kernel."""

    @staticmethod
    def forward(ctx, x, w, bias, groups, relu, want_stats=False, implicit_wgrad=False):
        x = _c(x)
        Cout, Cin = w.shape[0], w.shape[1] * groups
        y = _conv_tc_run(_as16(x), w, bias, _conv_tc_plan(Cin, Cout, groups), 0, Cout, groups, relu, want_stats=want_stats)
        ctx.save_for_backward(x, w, y if relu else None, bias)
        ctx.cfg = (groups, relu, bias is not None)
        ctx.implicit_wgrad = implicit_wgrad
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y, bias_p = ctx.saved_tensors
        groups, relu, has_bias = ctx.cfg
        N, H, W, Cin = x.shape
        Cout = w.shape[0]
        dy = _c(dy)
        dx = dw = db = None
        if Cout % 8 == 0:
            # everything downstream runs on the tensor cores: only the bf16 copy of g (and the bias gradient) is produced
            g16 = _take16(dy) if not (relu or has_bias) else None
            if g16 is not None:
                g = None
            else:
                g, g16, db = _grad_prep(dy.view(-1, Cout), y.view(-1, Cout) if relu else None, False, True, bias_p if has_bias else None)
            g16 = g16.view(N, H, W, Cout)
        else:
            g = _relu_bwd(y, dy) if relu else dy
            if groups == 1 and Cin % 8 == 0:     # narrow dy (7 / 1 channels): zero-pad to 8 so the rows are TMA-loadable
                g16 = torch.empty((N, H, W, 8), dtype=torch.bfloat16, device=g.device)
                call('tfb_cast_bf16_pad', g, g16, N * H * W, Cout, 8)
            else:
                g16 = None
        if ctx.needs_input_grad[0]:
            # narrow outputs (the 7- / 1-channel decoder heads at 160 x 704): dgrad on the tensor cores too, reading the dy that was
            # zero-padded to 8 channels for the wgrad GEMM (the packed dgrad weights are zero beyond the real Cout)
            plan = _conv_tc_plan(Cout, Cin, groups) if Cout % 8 == 0 else (_conv_tc_plan(8, Cin, 1) if (g16 is not None and NARROW_DGRAD_TC) else None)
            if plan is not None:
                dx = _conv_tc_run(g16, w, None, plan, 1, Cin, groups, False)
            else:
                if g is None:
                    g = _relu_bwd(y, dy) if relu else dy
                dx = torch.empty_like(x)
                call('tfb_conv2d_dgrad', g, w, dx, N, H, W, Cin, Cout, 3, 1, groups)
        if ctx.needs_input_grad[1]:
            dw = _conv_wgrad_tc(x, g16, w, groups, 1, ctx.implicit_wgrad) if g16 is not None else None
            if dw is not None:
                if has_bias and db is None:
                    db = _colsum(g.view(-1, Cout), _gbuf(bias_p))
            else:
                if g is None:
                    g = _relu_bwd(y, dy) if relu else dy
                dw = _gbuf(w)
                db = (_gbuf(bias_p) if db is None else db) if has_bias else None
                call('tfb_conv2d_wgrad', x, g, dw, db, N, H, W, Cin, Cout, 3, 1, groups)
        return dx, dw, db, None, None, None, None


class Subsample2Fn(Function):
    """x[:, ::2, ::2, :] — the input view of a 1x1 / stride-2 conv (RegNet downsample shortcut), so the conv itself is a GEMM."""

    @staticmethod
    def forward(ctx, x):
        x = _c(x)
        N, H, W, C = x.shape
        xs = torch.empty((N, (H + 1) // 2, (W + 1) // 2, C), dtype=torch.float32, device=x.device)
        xs16 = _emit16(xs, True)                   # the only consumer is the shortcut's 1x1 GEMM
        call('tfb_subsample2', x, xs, N, H, W, C, xs16)
        ctx.shape = (N, H, W, C)
        return _attach16(xs, xs16)

    @staticmethod
    def backward(ctx, d):
        N, H, W, C = ctx.shape
        dx = torch.empty((N, H, W, C), dtype=torch.float32, device=d.device)
        call('tfb_dilate2', _c(d), dx, N, H, W, C, 0)
        return dx


class Conv7x7Fn(Function):
    """The ResNet stem conv: 7x7 / stride 2 / pad 3, no bias, <= 4 input channels (csrc/resnet_stem.cu), exact fp32 in every mode.
    Forward and weight gradient only: the trunk inputs (image, LiDAR BEV) never need a gradient."""

    @staticmethod
    def forward(ctx, x, w):
        x = _c(x)
        N, H, W, Cin = x.shape
        y = torch.empty((N, (H - 1) // 2 + 1, (W - 1) // 2 + 1, w.shape[0]), dtype=torch.float32, device=x.device)
        call('tfb_conv7x7s2_fwd', x, _c(w), y, N, H, W, Cin, w.shape[0])
        ctx.save_for_backward(x, w)
        return y

    @staticmethod
    def backward(ctx, dy):
        if ctx.needs_input_grad[0]:
            raise RuntimeError('the 7x7 stem conv has no input gradient (csrc/resnet_stem.cu): its input must not require grad')
        x, w = ctx.saved_tensors
        N, H, W, Cin = x.shape
        dw = None
        if ctx.needs_input_grad[1]:
            dw = _gbuf(w)
            call('tfb_conv7x7s2_wgrad', x, _c(dy), dw, N, H, W, Cin, w.shape[0])
        return None, dw


class MaxPool2dFn(Function):
    """max_pool2d(x, 3, stride 2, padding 1) with PyTorch's semantics (csrc/resnet_stem.cu): the forward keeps a one-byte argmax
    tap per output element, the backward gathers each input element's gradient from the <= 4 windows that selected it."""

    @staticmethod
    def forward(ctx, x, emit16):
        x = _c(x)
        N, H, W, C = x.shape
        y = torch.empty((N, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C), dtype=torch.float32, device=x.device)
        y16 = _emit16(y, emit16)
        arg = torch.empty(y.shape, dtype=torch.uint8, device=x.device)
        call('tfb_maxpool3x3s2_fwd', x, y, y16, arg, N, H, W, C)
        ctx.save_for_backward(arg)
        ctx.shape = (N, H, W, C)
        return _attach16(y, y16)

    @staticmethod
    def backward(ctx, dy):
        arg, = ctx.saved_tensors
        N, H, W, C = ctx.shape
        dx = torch.empty((N, H, W, C), dtype=torch.float32, device=dy.device)
        call('tfb_maxpool3x3s2_bwd', _c(dy), arg, dx, N, H, W, C)
        return dx, None


def max_pool2d(x, emit16=False):
    """3x3 / stride-2 / pad-1 max-pool of the NHWC tensor x. emit16: the output feeds a tensor-core conv next (bf16 mode: its bf16
    copy is written in the same pass)."""
    return MaxPool2dFn.apply(x, emit16)


def conv2d(x, w, bias=None, stride=1, groups=1, relu=False, bn_stats=False):
    """bn_stats: a training-mode BatchNorm consumes the result next — on the tensor-core paths (bf16 mode) the producing kernel's
    epilogue then accumulates the per-channel sum / sum of squares (y._tfb_stats) and batch_norm skips its statistics pass.
    Inside implicit_wgrad() a 3x3 conv's tensor-core weight gradient skips the im2col matrix (see _conv_wgrad_tc)."""
    if w.shape[2] == 7:
        if not (stride == 2 and groups == 1 and bias is None and not relu and w.shape[1] <= 4):
            raise RuntimeError('7x7 convs are implemented for the ResNet stem only (stride 2, no bias / ReLU, <= 4 input channels)')
        return Conv7x7Fn.apply(x, w)
    bn_stats = bn_stats and BN_STATS_FUSED and G.MODE == 'bf16' and bias is None and not relu
    if w.shape[2] == 1 and stride == 2 and groups == 1 and (G.MODE == 'bf16' or G.multi_term()):
        x, stride = Subsample2Fn.apply(x), 1
    if w.shape[2] == 1 and stride == 1 and groups == 1:
        N, H, W, C = x.shape
        y2 = LinearFn.apply(_view16(x, x.reshape(-1, C)), w, bias, relu, bn_stats)
        y = y2.view(N, H, W, w.shape[0])
        st = getattr(y2, '_tfb_stats', None)
        if st is not None:
            y._tfb_stats = st
        return y
    implicit = _IMPLICIT_SCOPE[0] > 0
    if G.MODE == 'bf16' and w.shape[2] == 3 and stride == 1 and _conv_tc_plan(w.shape[1] * groups, w.shape[0], groups) is not None:
        return Conv3x3TCFn.apply(x, w, bias, groups, relu, bn_stats, implicit)
    return Conv2dFn.apply(x, w, bias, stride, groups, relu, bn_stats, implicit)


# ------------------------------------------------------------------ eval-mode BatchNorm in the conv / GEMM epilogue
def bn_epilogue_path(x, w, stride, groups, residual):
    """Which tensor-core launch computes bn(conv(x)) of an eval-mode BatchNorm in its epilogue: 'gemm' (1x1 convs, after the
    stride-2 subsample), 'conv3' (3x3 convs, stride 1 or 2) or None (the conv and batch_norm run as two launches). It follows
    conv2d's choice of kernel in bf16 mode, so the fused launch has the plain launch's tile plan and gives its bits."""
    if G.MODE != 'bf16' or x.dim() != 4 or w.shape[0] % 4 != 0:
        return None
    if torch.is_grad_enabled() and (x.requires_grad or w.requires_grad):
        return None                                   # (batch_norm refuses it: eval-mode BatchNorm has no backward)
    if residual is not None and not BN_ADD_FUSED:
        return None
    N, H, W, Cin = x.shape
    ks, Cout = w.shape[2], w.shape[0]
    if ks == 1 and groups == 1 and stride in (1, 2):
        Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
        return 'gemm' if G.tc_ok(N * Ho * Wo, Cout, Cin, Cin, Cout) else None
    if ks == 3 and (stride == 1 or (stride == 2 and CONV_S2_TC)) and _conv_tc_plan(Cin, Cout, groups) is not None:
        return 'conv3'
    return None


def conv_bn_eval(x, w, bn, stride=1, groups=1, relu=False, residual=None, emit16=False):
    """relu?(bn(conv(x)) + residual) of an eval-mode BatchNorm (running statistics) as ONE tensor-core launch whose epilogue
    normalises, adds the residual, applies the ReLU and writes the fp32 result (and its bf16 sidecar when emit16): the same bits as
    conv2d + batch_norm, without the unnormalised conv output in memory. None when bn_epilogue_path finds no such launch."""
    path = bn_epilogue_path(x, w, stride, groups, residual)
    if path is None:
        return None
    invstd = torch.rsqrt(bn.running_var + bn.eps)
    res = _c(residual) if residual is not None else None
    Cout = w.shape[0]
    if path == 'gemm':
        if stride == 2:
            x = Subsample2Fn.apply(x)
        N, H, W, C = x.shape
        xs = _as16(_c(_view16(x, x.reshape(-1, C))))
        wb = G.weight_bf16(w.view(Cout, -1))
        y = torch.empty((N, H, W, Cout), dtype=torch.float32, device=x.device)
        y16 = _emit16(y, emit16)
        call('tfb_gemm_bf16_tc_bn_eval', N * H * W, Cout, C, xs, xs.stride(0), wb, wb.stride(0), y, Cout, bn.running_mean, invstd, bn.weight,
             bn.bias, res, int(relu), y16)
        return _attach16(y, y16)
    x = _c(x)
    N, H, W, Cin = x.shape
    plan = _conv_tc_plan(Cin, Cout, groups)
    x16 = _as16(x)
    e = _packed_current(w, plan, 0, groups)
    y = torch.empty((N, (H - 1) // stride + 1, (W - 1) // stride + 1, Cout), dtype=torch.float32, device=x.device)
    y16 = _emit16(y, emit16)
    call('tfb_conv3x3_tc_bn_eval', x16, e.wp, y, N, H, W, Cin, Cout, plan['NB'], plan['KC'], plan['c_step'], plan['nchunks'], plan['nb_real'],
         plan['gblocks'], stride, bn.running_mean, invstd, bn.weight, bn.bias, res, int(relu), y16)
    return _attach16(y, y16)


# ------------------------------------------------------------------ normalisation
class BatchNormTrainFn(Function):
    """BatchNorm2d in training mode (+ fused ReLU): batch statistics, running-stat update (momentum, unbiased var)."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, momentum, eps, relu, emit16=False, bwd16=False, pool=False, stats=None,
                group=None):
        x = _c(x)
        C = x.shape[-1]
        M = x.numel() // C
        y = torch.empty_like(x)
        pool = pool and SE_POOL_FUSED and x.dim() == 4
        y16 = _emit16(y, emit16 and not pool)
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        invstd = torch.empty(C, dtype=torch.float32, device=x.device)
        # pool: the squeeze-excite average pool of the output comes out of the normalise pass (SEFn picks it up from y._tfb_pooled)
        pooled = None
        if stats is not None and pool:
            pooled = _arena_take(x.device, x.shape[0] * C * 4, torch.float32)      # accumulated into: must start at zero
            if pooled is None:
                stats = None
            else:
                pooled = pooled.view(x.shape[0], C)
        if stats is None and pool:
            pooled = torch.empty((x.shape[0], C), dtype=torch.float32, device=x.device)
        # stats: the conv / GEMM that produced x already accumulated sum x, sum x^2 per channel in its epilogue: one launch, one pass
        folded = _bn_fwd(x, y, M, C, weight, bias, momentum, eps, relu, running_mean, running_var, mean, invstd, stats, y16, None, pooled,
                         x.shape[0] if pool else 0, group)
        ctx.save_for_backward(x, weight, bias, mean, invstd, folded)
        ctx.relu, ctx.bwd16, ctx.group = relu, bwd16, group
        if pool:
            y._tfb_pooled = pooled
        return _attach16(y, y16)

    @staticmethod
    def backward(ctx, dy):
        x, weight, bias, mean, invstd, folded = ctx.saved_tensors
        dy = _c(dy)
        C = x.shape[-1]
        M = x.numel() // C
        dx = torch.empty_like(x)
        dg = _gbuf(weight)
        db = _gbuf(bias)
        dx16 = _emit16(dx, ctx.bwd16)
        _bn_bwd(x, dy, dx, M, C, weight, bias, mean, invstd, ctx.relu, dg, db, dx16, group=ctx.group, folded=folded)
        if dx16 is not None:
            _offer16(dx, dx16)
        return dx, dg, db, None, None, None, None, None, None, None, None, None, None


class BatchNormAddReluFn(Function):
    """relu(BatchNorm2d(x) + residual), training mode: the tail of timm's Bottleneck (conv3.bn -> + shortcut -> ReLU) with the add
    and the ReLU inside BatchNorm's normalise pass (forward) and the ReLU mask + the shortcut's gradient inside BatchNorm's backward
    passes — two launches and four passes over the block-sized activation fewer than BatchNorm, add+ReLU, ReLU', BatchNorm'."""

    @staticmethod
    def forward(ctx, x, res, weight, bias, running_mean, running_var, momentum, eps, emit16=False, bwd16=False, stats=None, group=None):
        x, res = _c(x), _c(res)
        C = x.shape[-1]
        M = x.numel() // C
        y = torch.empty_like(x)
        y16 = _emit16(y, emit16)
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        invstd = torch.empty(C, dtype=torch.float32, device=x.device)
        folded = _bn_fwd(x, y, M, C, weight, bias, momentum, eps, 1, running_mean, running_var, mean, invstd, stats, y16, res, None, 0, group)
        ctx.save_for_backward(x, weight, bias, mean, invstd, y, folded)
        ctx.bwd16, ctx.group = bwd16, group
        return _attach16(y, y16)

    @staticmethod
    def backward(ctx, dy):
        x, weight, bias, mean, invstd, y, folded = ctx.saved_tensors
        dy = _c(dy)
        C = x.shape[-1]
        M = x.numel() // C
        dx, g = torch.empty_like(x), torch.empty_like(x)
        dg, db = _gbuf(weight), _gbuf(bias)
        dx16 = _emit16(dx, ctx.bwd16)
        _bn_bwd(x, dy, dx, M, C, weight, bias, mean, invstd, 0, dg, db, dx16, ymask=y, gmasked=g, group=ctx.group, folded=folded)
        if dx16 is not None:
            _offer16(dx, dx16)
        return dx, g, dg, db, None, None, None, None, None, None, None, None


def batch_norm(x, bn, relu, training, emit16=False, bwd16=False, residual=None, pool=False):
    """bn: an nn.BatchNorm2d used as a parameter/buffer container; an nn.SyncBatchNorm in training mode normalises with the
    statistics of all ranks of its process group once one is initialised (sync_group). residual: act(bn(x) + residual) in the same pass (relu required).
    pool: the output feeds a squeeze-excite module next — its global average pool is accumulated in the normalise pass (training). emit16: the output feeds a tensor-core GEMM / conv next, so
    (bf16 mode) its bf16 copy is written in the same pass. bwd16: the same for dx in backward (the convolution in front of this
    BatchNorm has no bias / ReLU of its own and runs dgrad + wgrad on the tensor cores)."""
    if residual is not None and not (relu and BN_ADD_FUSED):
        return add(batch_norm(x, bn, False, training, False, bwd16), residual, relu=relu, emit16=emit16)
    if training:
        stats = getattr(x, '_tfb_stats', None)        # accumulated by the producing conv / GEMM epilogue (conv2d(..., bn_stats=True))
        if stats is not None and (stats.numel() != 2 * x.shape[-1] or x.shape[-1] > 2048):
            stats = None
        group = sync_group(bn)
        if residual is not None:
            return BatchNormAddReluFn.apply(x, residual, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps, emit16,
                                            bwd16, stats, group)
        return BatchNormTrainFn.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps, relu, emit16, bwd16,
                                      pool, stats, group)
    if torch.is_grad_enabled() and x.requires_grad:
        raise RuntimeError('eval-mode BatchNorm backward is not implemented (training path only)')
    C = x.shape[-1]
    y = torch.empty_like(x)
    y16 = _emit16(y, emit16)
    invstd = torch.rsqrt(bn.running_var + bn.eps)
    call('tfb_bn_apply', _c(x), y, x.numel() // C, C, bn.weight, bn.bias, bn.running_mean, invstd, int(relu), y16,
         _c(residual) if residual is not None else None)
    return _attach16(y, y16)


class LayerNormFn(Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps, emit16=False):
        x = _c(x)
        C = x.shape[-1]
        R = x.numel() // C
        y = torch.empty_like(x)
        y16 = _emit16(y, emit16)
        mean = torch.empty(R, dtype=torch.float32, device=x.device)
        rstd = torch.empty(R, dtype=torch.float32, device=x.device)
        call('tfb_layernorm_fwd', x, y, R, C, weight, bias, float(eps), mean, rstd, y16)
        ctx.save_for_backward(x, weight, mean, rstd, bias)
        return _attach16(y, y16)

    @staticmethod
    def backward(ctx, dy):
        x, weight, mean, rstd, bias = ctx.saved_tensors
        dy = _c(dy)
        C = x.shape[-1]
        R = x.numel() // C
        dx = torch.empty_like(x)
        dg = _gbuf(weight)
        db = _gbuf(bias)
        call('tfb_layernorm_bwd', x, dy, dx, R, C, weight, mean, rstd, dg, db, 0, _ws(x.device))
        return dx, dg, db, None, None


def layer_norm(x, ln, emit16=False):
    return LayerNormFn.apply(x, ln.weight, ln.bias, ln.eps, emit16)


# ------------------------------------------------------------------ squeeze-excite, residual
class SEFn(Function):
    """timm SEModule: x * sigmoid(fc2(relu(fc1(mean_hw(x))))) — pooling, two tiny GEMMs and the gating, fwd + bwd."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, emit16=False):
        x = _c(x)
        N, H, W, C = x.shape
        Cr = w1.shape[0]
        dev = x.device
        pooled = getattr(x, '_tfb_pooled', None)             # written by the BatchNorm in front (batch_norm(..., pool=True))
        if pooled is None or pooled.shape != (N, C):
            pooled = torch.empty((N, C), dtype=torch.float32, device=dev)
            call('tfb_pool_hw_fwd', x, pooled, N, H * W, C)
        h = torch.empty((N, Cr), dtype=torch.float32, device=dev)
        gate = torch.empty((N, C), dtype=torch.float32, device=dev)
        if N <= 16:
            call('tfb_gemm_small_m', 1, N, Cr, C, pooled, C, w1, C, h, Cr, b1, 1)
            call('tfb_gemm_small_m', 1, N, C, Cr, h, Cr, w2, Cr, gate, C, b2, 2)
        else:
            gemm(pooled, w1.view(Cr, C), h, trans_b=True, bias=b1, relu=True, mode='simt')
            s = torch.empty((N, C), dtype=torch.float32, device=dev)
            gemm(h, w2.view(C, Cr), s, trans_b=True, bias=b2, mode='simt')
            call('tfb_sigmoid_fwd', s, gate, s.numel())
        y = torch.empty_like(x)
        y16 = _emit16(y, emit16)
        call('tfb_se_scale_fwd', x, gate, y, N, H * W, C, y16)
        ctx.save_for_backward(x, w1, w2, pooled, h, gate, b1, b2)
        return _attach16(y, y16)

    @staticmethod
    def backward(ctx, dy):
        x, w1, w2, pooled, h, gate, b1, b2 = ctx.saved_tensors
        dy = _c(dy)
        N, H, W, C = x.shape
        Cr = w1.shape[0]
        dev = x.device
        dgate = torch.empty((N, C), dtype=torch.float32, device=dev)
        call('tfb_se_bwd_reduce', x, dy, dgate, N, H * W, C)
        dw2, db2, dw1, db1 = _gbuf(w2), _gbuf(b2), _gbuf(w1), _gbuf(b1)
        dpool = torch.empty((N, C), dtype=torch.float32, device=dev)
        if N <= 16 and Cr <= 512 and SE_FUSED_BWD:
            # the whole MLP backward (sigmoid', both weight / bias gradients, both skinny GEMMs, relu') in two launches
            part = torch.empty(((C + 63) // 64, N, Cr), dtype=torch.float32, device=dev)
            call('tfb_se_mlp_bwd', dgate, gate, h, pooled, w1, w2, dw1, db1, dw2, db2, dpool, part, N, C, Cr)
        else:
            ds = torch.empty_like(dgate)
            call('tfb_sigmoid_bwd', gate, dgate, ds, ds.numel())
            gemm(ds, h, dw2.view(C, Cr), trans_a=True, mode='simt')
            _colsum(ds, db2)
            dh = torch.empty((N, Cr), dtype=torch.float32, device=dev)
            if N <= 16:
                call('tfb_gemm_small_m', 0, N, Cr, C, ds, C, w2, Cr, dh, Cr, None, 0)
            else:
                gemm(ds, w2.view(C, Cr), dh, trans_b=False, mode='simt')
            dh = _relu_bwd(h, dh)
            gemm(dh, pooled, dw1.view(Cr, C), trans_a=True, mode='simt')
            _colsum(dh, db1)
            if N <= 16:
                call('tfb_gemm_small_m', 0, N, C, Cr, dh, Cr, w1, C, dpool, C, None, 0)
            else:
                gemm(dh, w1.view(Cr, C), dpool, trans_b=False, mode='simt')
        dx = torch.empty_like(x)
        call('tfb_se_bwd_apply', dy, gate, dpool, dx, N, H * W, C)
        return dx, dw1, db1, dw2, db2, None


class BNSEFn(Function):
    """relu(BatchNorm2d(x)) followed by the squeeze-excite module it feeds (timm Bottleneck: conv2.bn -> se), training mode, as ONE
    autograd node: forward = BatchNormTrainFn(pool=True) + SEFn, launch for launch; backward folds the squeeze-excite gradient
    dy * gate + dpool / HW into BatchNorm's backward passes (tfb_bn_bwd_se) instead of materialising it (tfb_se_bwd_apply): one
    launch, one write and one read of the block-sized map fewer per bottleneck."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, momentum, eps, w1, b1, w2, b2, bwd16, stats, group=None):
        x = _c(x)
        N, H, W, C = x.shape
        M, Cr, dev = N * H * W, w1.shape[0], x.device
        y2 = torch.empty_like(x)
        mean = torch.empty(C, dtype=torch.float32, device=dev)
        invstd = torch.empty(C, dtype=torch.float32, device=dev)
        pooled = None
        if stats is not None:
            pooled = _arena_take(dev, N * C * 4, torch.float32)               # accumulated into: must start at zero
            pooled = pooled.view(N, C) if pooled is not None else None
        if pooled is None:
            stats, pooled = None, torch.empty((N, C), dtype=torch.float32, device=dev)
        folded = _bn_fwd(x, y2, M, C, weight, bias, momentum, eps, 1, running_mean, running_var, mean, invstd, stats, None, None, pooled, N, group)
        h = torch.empty((N, Cr), dtype=torch.float32, device=dev)
        gate = torch.empty((N, C), dtype=torch.float32, device=dev)
        call('tfb_gemm_small_m', 1, N, Cr, C, pooled, C, w1, C, h, Cr, b1, 1)
        call('tfb_gemm_small_m', 1, N, C, Cr, h, Cr, w2, Cr, gate, C, b2, 2)
        y = torch.empty_like(x)
        y16 = _emit16(y, True)                               # the gated output always feeds the 1x1 conv3 GEMM
        call('tfb_se_scale_fwd', y2, gate, y, N, H * W, C, y16)
        ctx.save_for_backward(x, weight, bias, mean, invstd, y2, w1, w2, pooled, h, gate, b1, b2, folded)
        ctx.bwd16, ctx.group = bwd16, group
        return _attach16(y, y16)

    @staticmethod
    def backward(ctx, dy):
        x, weight, bias, mean, invstd, y2, w1, w2, pooled, h, gate, b1, b2, folded = ctx.saved_tensors
        dy = _c(dy)
        N, H, W, C = x.shape
        M, Cr, dev = N * H * W, w1.shape[0], x.device
        dgate = torch.empty((N, C), dtype=torch.float32, device=dev)
        call('tfb_se_bwd_reduce', y2, dy, dgate, N, H * W, C)
        dw2, db2, dw1, db1 = _gbuf(w2), _gbuf(b2), _gbuf(w1), _gbuf(b1)
        dpool = torch.empty((N, C), dtype=torch.float32, device=dev)
        part = torch.empty((N, Cr), dtype=torch.float32, device=dev)
        call('tfb_se_mlp_bwd', dgate, gate, h, pooled, w1, w2, dw1, db1, dw2, db2, dpool, part, N, C, Cr)
        dx = torch.empty_like(x)
        dg, db = _gbuf(weight), _gbuf(bias)
        dx16 = _emit16(dx, ctx.bwd16)
        _bn_bwd(x, dy, dx, M, C, weight, bias, mean, invstd, 1, dg, db, dx16, se_gate=gate, se_dpool=dpool, hw=H * W, group=ctx.group,
                folded=folded)
        if dx16 is not None:
            _offer16(dx, dx16)
        return dx, dg, db, None, None, None, None, dw1, db1, dw2, db2, None, None, None


def bn_se_ok(x, bn, fc1):
    """The fused BatchNorm + squeeze-excite node covers the training step's configuration (batch <= 16 per GPU, fused SE backward)."""
    return (BN_SE_FUSED and bn.training and SE_POOL_FUSED and SE_FUSED_BWD and x.dim() == 4 and x.shape[0] <= 16 and fc1.weight.shape[0] <= 512
            and x.shape[-1] % 4 == 0 and x.numel() < (1 << 31))


def bn_se(x, bn, fc1, fc2, bwd16=False):
    """relu(bn(x)) -> squeeze-excite(fc1, fc2), training mode (see BNSEFn)."""
    stats = getattr(x, '_tfb_stats', None)
    if stats is not None and (stats.numel() != 2 * x.shape[-1] or x.shape[-1] > 2048):
        stats = None
    return BNSEFn.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps, fc1.weight, fc1.bias, fc2.weight,
                        fc2.bias, bwd16, stats, sync_group(bn))


class AddFn(Function):
    """y = a + b (ReLU optional): the Bottleneck shortcut (timm) and the GPT residuals (transfuser.py:546-547)."""

    @staticmethod
    def forward(ctx, a, b, relu, emit16=False):
        a, b = _c(a), _c(b)
        y = torch.empty_like(a)
        y16 = _emit16(y, emit16)
        call('tfb_add_relu', a, b, y, a.numel(), int(relu), y16)
        ctx.relu = relu
        if relu:
            ctx.save_for_backward(y)
        return _attach16(y, y16)

    @staticmethod
    def backward(ctx, dy):
        dy = _c(dy)
        if ctx.relu:
            (y,) = ctx.saved_tensors
            dy = _relu_bwd(y, dy)
        return dy, dy, None, None


def add(a, b, relu=False, emit16=False):
    return AddFn.apply(a, b, relu, emit16)


class DropoutFn(Function):
    @staticmethod
    def forward(ctx, x, p, seed):
        x = _c(x)
        y = torch.empty_like(x)
        call('tfb_dropout', x, y, x.numel(), float(p), seed_state(x.device), seed, None)
        ctx.p, ctx.seed = p, seed
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = _c(dy)
        dx = torch.empty_like(dy)
        call('tfb_dropout', dy, dx, dy.numel(), float(ctx.p), seed_state(dy.device), ctx.seed, None)
        return dx, None, None


def dropout(x, p, training):
    if not training or p <= 0.0:
        return x
    return DropoutFn.apply(x, p, next_seed())


class BcastAddTokensFn(Function):
    """tok[B, T, C] + v[B, C] for every token: the velocity embedding of GPT.forward (transfuser.py:352-355, use_velocity=True)."""

    @staticmethod
    def forward(ctx, tok, v):
        tok, v = _c(tok), _c(v)
        B, T, C = tok.shape
        y = torch.empty_like(tok)
        call('tfb_bcast_add_nc', tok, v, y, B, T, C)
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = _c(dy)
        B, T, C = dy.shape
        mean = torch.empty((B, C), dtype=torch.float32, device=dy.device)
        call('tfb_pool_hw_fwd', dy, mean, B, T, C)
        dv = torch.empty_like(mean)
        call('tfb_scale_dev', mean, None, float(T), dv, mean.numel(), 0)
        return dy, dv


class VelEmbAddFn(Function):
    """x_k + vel_emb(v) for every token / pixel of each x_k [B, ..., C] (one or two tensors): the ego-speed embedding Linear(1, C)
    computed inside tfb_vel_emb_add, no [B, C] embedding tensor. One node per embedding, so its weight and bias gradients are
    written once per step, straight into the flat gradient buffer (tfb_vel_emb_bwd). The speed is an input: it gets no gradient."""

    @staticmethod
    def forward(ctx, velocity, weight, bias, *xs):
        B, C = xs[0].shape[0], xs[0].shape[-1]
        if len(xs) not in (1, 2) or any(x.shape[0] != B or x.shape[-1] != C for x in xs):
            raise ValueError('VelEmbAddFn takes one or two tensors [B, ..., C] of one batch and width')
        if velocity.numel() != B or tuple(weight.shape) != (C, 1) or tuple(bias.shape) != (C,):
            raise ValueError('VelEmbAddFn: the speed must be [B, 1] and the embedding Linear(1, %d)' % C)
        v = _c(velocity.reshape(B).to(torch.float32))
        xs = [_c(x) for x in xs]
        ys = [torch.empty_like(x) for x in xs]
        T = [x.numel() // (B * C) for x in xs]
        x1, y1, T1 = (xs[1], ys[1], T[1]) if len(xs) == 2 else (None, None, 0)
        call('tfb_vel_emb_add', v, weight, bias, xs[0], ys[0], T[0], x1, y1, T1, B, C)
        ctx.save_for_backward(v, weight, bias)
        ctx.T = T
        return ys[0] if len(ys) == 1 else tuple(ys)

    @staticmethod
    def backward(ctx, *dys):
        v, weight, bias = ctx.saved_tensors
        if ctx.needs_input_grad[0]:
            raise RuntimeError('VelEmbAddFn does not differentiate with respect to the speed input')
        dys = [_c(d) for d in dys]
        B, C = dys[0].shape[0], dys[0].shape[-1]
        dw, db = _gbuf(weight), _gbuf(bias)
        d1, T1 = (dys[1], ctx.T[1]) if len(dys) == 2 else (None, 0)
        call('tfb_vel_emb_bwd', v, dys[0], ctx.T[0], d1, T1, B, C, dw, db)
        return (None, dw, db) + tuple(dys)


def vel_emb_add(velocity, emb, *xs):
    """xs with the speed embedding `emb` (an nn.Linear(1, C)) added to every position, as VelEmbAddFn."""
    return VelEmbAddFn.apply(velocity, emb.weight, emb.bias, *xs)


class AddDropoutFn(Function):
    """res + dropout(x) in one pass (the GPT block's residual connections, transfuser.py:546-547); backward regenerates the mask."""

    @staticmethod
    def forward(ctx, res, x, p, seed):
        res, x = _c(res), _c(x)
        y = torch.empty_like(x)
        call('tfb_dropout', x, y, x.numel(), float(p), seed_state(x.device), seed, res)
        ctx.p, ctx.seed = p, seed
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = _c(dy)
        dx = torch.empty_like(dy)
        call('tfb_dropout', dy, dx, dy.numel(), float(ctx.p), seed_state(dy.device), ctx.seed, None)
        return dy, dx, None, None


def add_dropout(res, x, p, training):
    """res + dropout(x, p): one launch in training mode, a plain add otherwise."""
    if not training or p <= 0.0:
        return add(res, x)
    return AddDropoutFn.apply(res, x, p, next_seed())


class AddDropoutLNFn(Function):
    """(xnew, h) = (res + dropout(x, p), LayerNorm(xnew)) in one launch — a GPT residual connection together with the LayerNorm
    that reads it (transfuser.py:546-547, then 533/321). Backward: one row kernel takes the gradient of h and the gradient
    reaching xnew from the next residual connection and writes d res and d x (mask regenerated), plus the parameter reduction."""

    @staticmethod
    def forward(ctx, res, x, p, seed, weight, bias, eps, emit16):
        res, x = _c(res), _c(x)
        C = x.shape[-1]
        R = x.numel() // C
        xnew = torch.empty_like(x)
        h = torch.empty_like(x)
        h16 = _emit16(h, emit16)
        mean = torch.empty(R, dtype=torch.float32, device=x.device)
        rstd = torch.empty(R, dtype=torch.float32, device=x.device)
        call('tfb_add_dropout_ln_fwd', res, x, xnew, h, R, C, weight, bias, float(eps), float(p), seed_state(x.device), seed, mean, rstd, h16)
        ctx.save_for_backward(xnew, weight, mean, rstd, bias)
        ctx.p, ctx.seed = p, seed
        ctx.set_materialize_grads(False)
        return xnew, _attach16(h, h16)

    @staticmethod
    def backward(ctx, gx, dh):
        xnew, weight, mean, rstd, bias = ctx.saved_tensors
        C = xnew.shape[-1]
        R = xnew.numel() // C
        if dh is None:                                      # LayerNorm output unused: only the residual connection's gradient
            if gx is None:
                return (None,) * 8
            gx = _c(gx)
            dx = torch.empty_like(gx)
            call('tfb_dropout', gx, dx, gx.numel(), float(ctx.p), seed_state(gx.device), ctx.seed, None)
            return gx, dx, None, None, None, None, None, None
        dh = _c(dh)
        gx = _c(gx) if gx is not None else None
        dres = torch.empty_like(xnew)
        dx = torch.empty_like(xnew)
        dg = _gbuf(weight)
        db = _gbuf(bias)
        call('tfb_add_dropout_ln_bwd', xnew, dh, gx, dres, dx, R, C, weight, mean, rstd, float(ctx.p), seed_state(xnew.device), ctx.seed,
             dg, db, _ws(xnew.device))
        return dres, dx, None, None, dg, db, None, None


def add_dropout_ln(res, x, p, training, ln, emit16=False):
    """(res + dropout(x, p), ln(res + dropout(x, p))): fused unless TFB_ADD_LN_FUSED=0."""
    if not ADD_LN_FUSED:
        xnew = add_dropout(res, x, p, training)
        return xnew, layer_norm(xnew, ln, emit16=emit16)
    p = float(p) if training else 0.0
    return AddDropoutLNFn.apply(res, x, p, next_seed() if p > 0.0 else 0, ln.weight, ln.bias, ln.eps, emit16)


# ------------------------------------------------------------------ attention (SelfAttention.forward, transfuser.py:510-527)
class AttentionFn(Function):
    """h[B*T, C] -> softmax(q k^T / sqrt(hs)) v for n_head heads, with the key/query/value projections inside.
    The (b, head) products run as two-level strided-batched GEMMs straight on the packed [B*T, 3C] q|k|v buffer."""

    @staticmethod
    def forward(ctx, h, wq, bq, wk, bk, wv, bv, B, T, nh, p_drop, seed):
        h = _c(h)
        C = h.shape[1]
        hs = C // nh
        dev = h.device
        tc = G.tc_ok(B * T, C, C, C)
        fused = tc and ATTN_FUSED and T <= 192 and hs % 2 == 0
        w3, b3 = (_pack3(wq, wk, wv), _pack3(bq, bk, bv)) if QKV_FUSED else (None, None)
        packed = w3 is not None and b3 is not None
        q16 = fused and packed          # q|k|v straight out of the GEMM epilogue in bf16: the fused attention stages it with cp.async
        qkv = torch.empty((B * T, 3 * C), dtype=torch.bfloat16 if q16 else torch.float32, device=dev)
        hs_ = _as16(h) if tc else h
        if packed:
            # the three projections as ONE GEMM on the [3C, C] weight the flat parameter buffer holds contiguously
            if q16:
                wb = G.weight_bf16(w3)
                call('tfb_gemm_bf16_tc_out16', 1, B * T, 3 * C, C, hs_, hs_.stride(0), wb, wb.stride(0), qkv, 3 * C, b3, 0, 1.0)
            elif tc:
                G.gemm_bf16(hs_, G.weight_bf16(w3), qkv, trans_b=True, bias=b3)
            else:
                gemm(h, w3, qkv, trans_b=True, bias=b3, mode='simt')
        else:
            for i, (w_, b_) in enumerate(((wq, bq), (wk, bk), (wv, bv))):
                if tc:
                    G.gemm_bf16(hs_, G.weight_bf16(w_), qkv[:, i * C:(i + 1) * C], trans_b=True, bias=b_)
                else:
                    gemm(h, w_, qkv[:, i * C:(i + 1) * C], trans_b=True, bias=b_, mode='simt')
        scale = 1.0 / (hs ** 0.5)
        if fused:
            # one launch: scores in registers, softmax on the accumulator fragments, probabilities through shared memory (csrc/attn_tc.cu)
            y = torch.empty((B * T, C), dtype=torch.float32, device=dev)
            y16 = _emit16(y, True)                           # the output feeds the proj GEMM
            lse = torch.empty((B, nh, T), dtype=torch.float32, device=dev)
            call('tfb_attn_fwd_tc', qkv, int(q16), B, T, nh, hs, y, y16, lse, scale, float(p_drop), seed_state(dev), seed)
            ctx.save_for_backward(hs_, wq, wk, wv, qkv, y, lse, bq, bk, bv)      # y in fp32: D = rowsum(dy * y) keeps full precision
            ctx.cfg = (B, T, nh, p_drop, seed, scale, tc, packed, True)
            return _attach16(y, y16)
        S = torch.empty((B, nh, T, T), dtype=torch.float32, device=dev)
        q, k, v = qkv[:, 0:C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        bgemm(q, k, S, T, T, hs, 3 * C, 3 * C, T, False, True, B, nh, (T * 3 * C, hs), (T * 3 * C, hs), (nh * T * T, T * T))
        Pd = torch.empty_like(S) if p_drop > 0 else S
        call('tfb_softmax_fwd', S, S, Pd, B * nh * T, T, scale, float(p_drop), seed_state(dev), seed)
        y = torch.empty((B * T, C), dtype=torch.float32, device=dev)
        bgemm(Pd, v, y, T, hs, T, T, 3 * C, C, False, False, B, nh, (nh * T * T, T * T), (T * 3 * C, hs), (T * C, hs))
        ctx.save_for_backward(hs_, wq, wk, wv, qkv, S, Pd, bq, bk, bv)
        ctx.cfg = (B, T, nh, p_drop, seed, scale, tc, packed, False)
        return y

    @staticmethod
    def backward(ctx, dy):
        h, wq, wk, wv, qkv, P, Pd, bq, bk, bv = ctx.saved_tensors
        B, T, nh, p_drop, seed, scale, tc, packed, fused = ctx.cfg
        dy = _c(dy)
        C = h.shape[1]
        hs = C // nh
        dev = h.device
        dqkv = torch.empty(qkv.shape, dtype=torch.float32, device=dev)
        dq, dk, dv = dqkv[:, 0:C], dqkv[:, C:2 * C], dqkv[:, 2 * C:]
        d16 = None
        if fused:
            y, lse = P, Pd                                   # (saved in their place by the fused forward; y fp32 or its bf16 copy)
            d16 = torch.empty(dqkv.shape, dtype=torch.bfloat16, device=dev)
            dsum = torch.empty((B, nh, T), dtype=torch.float32, device=dev)
            dy16 = torch.empty((B * T, C), dtype=torch.bfloat16, device=dev)
            call('tfb_attn_bwd_tc', qkv, int(qkv.dtype == torch.bfloat16), dy, y, int(y.dtype == torch.bfloat16), lse, dsum, dy16,
                 B, T, nh, hs, dqkv, d16, scale, float(p_drop), seed_state(dev), seed)
        else:
            q, k, v = qkv[:, 0:C], qkv[:, C:2 * C], qkv[:, 2 * C:]
            sP, sQ, sY = (nh * T * T, T * T), (T * 3 * C, hs), (T * C, hs)
            dP = torch.empty_like(P)
            bgemm(dy, v, dP, T, T, hs, C, 3 * C, T, False, True, B, nh, sY, sQ, sP)          # dPd = dy v^T
            bgemm(Pd, dy, dv, T, hs, T, T, C, 3 * C, True, False, B, nh, sP, sY, sQ)         # dv  = Pd^T dy
            call('tfb_softmax_bwd', P, dP, dP, B * nh * T, T, scale, float(p_drop), seed_state(dev), seed)    # dS (in place)
            bgemm(dP, k, dq, T, hs, T, T, 3 * C, 3 * C, False, False, B, nh, sP, sQ, sQ)     # dq  = dS k
            bgemm(dP, q, dk, T, hs, T, T, 3 * C, 3 * C, True, False, B, nh, sP, sQ, sQ)      # dk  = dS^T q
        dh = torch.empty((B * T, C), dtype=torch.float32, device=dev)
        grads = []
        w3 = _pack3(wq, wk, wv) if packed else None
        if w3 is not None:
            # fused q|k|v: dh = dqkv W3 (one GEMM, K = 3C), dW3 = dqkv^T h (one GEMM), db3 = column sums of dqkv (one reduction)
            dw3, db3 = _gbuf3(wq, wk, wv), _gbuf3(bq, bk, bv)
            if tc:
                if d16 is not None:
                    _colsum(dqkv, db3)                       # the fused attention backward wrote the bf16 copy itself
                else:
                    # one pass over dqkv: its bf16 copy (operand of both GEMMs) and the three bias gradients (column sums)
                    d16 = torch.empty(dqkv.shape, dtype=torch.bfloat16, device=dev)
                    call('tfb_grad_prep', dqkv, None, None, d16, db3, _ws(dev), B * T, 3 * C)
                G.gemm_bf16(d16, G.weight_bf16(w3), dh, trans_b=False)
                with _OnWgradStream(dev, d16, h, dw3):
                    G.gemm_bf16(d16, h, dw3, trans_a=True, splits=_wgrad_splits(B * T, 3 * C, C))
            else:
                gemm(dqkv, w3, dh, trans_b=False, mode='simt')
                gemm(dqkv, h, dw3, trans_a=True, mode='simt')
                _colsum(dqkv, db3)
            for i in range(3):
                grads += [dw3[i * C:(i + 1) * C], db3[i * C:(i + 1) * C]]
        elif tc:
            if d16 is None:
                d16 = G.to_bf16(dqkv)
            for i, w_ in enumerate((wq, wk, wv)):
                G.gemm_bf16(d16[:, i * C:(i + 1) * C], G.weight_bf16(w_), dh, trans_b=False, beta=0.0 if i == 0 else 1.0)
            for i, (d, w_, b_) in enumerate(((dq, wq, bq), (dk, wk, bk), (dv, wv, bv))):
                dw = _gbuf(w_)
                G.gemm_bf16(d16[:, i * C:(i + 1) * C], h, dw, trans_a=True, splits=_wgrad_splits(B * T, C, C))
                grads += [dw, _colsum(d, _gbuf(b_))]
        else:
            for i, (d, w_, b_) in enumerate(((dq, wq, bq), (dk, wk, bk), (dv, wv, bv))):
                gemm(d, w_, dh, trans_b=False, beta=0.0 if i == 0 else 1.0, mode='simt')
                dw = _gbuf(w_)
                gemm(d, h, dw, trans_a=True, mode='simt')
                grads += [dw, _colsum(d, _gbuf(b_))]
        return (dh, *grads, None, None, None, None, None)


# ------------------------------------------------------------------ GPT token build / output view + upsample + add
class TokensFn(Function):
    """AdaptiveAvgPool2d of both feature maps -> (B, T, C) tokens + pos_emb, dropout (transfuser.py:150-151, 346-357)."""

    @staticmethod
    def forward(ctx, img, lid, pos_emb, ghi, gwi, ghl, gwl, p_drop, seed):
        img, lid = _c(img), _c(lid)
        N, Hi, Wi, C = img.shape
        _, Hl, Wl, _ = lid.shape
        T = ghi * gwi + ghl * gwl
        out = torch.empty((N, T, C), dtype=torch.float32, device=img.device)
        call('tfb_tokens_fwd', img, Hi, Wi, ghi, gwi, lid, Hl, Wl, ghl, gwl, pos_emb, out, N, C, float(p_drop), seed_state(img.device), seed)
        ctx.cfg = (N, Hi, Wi, Hl, Wl, C, ghi, gwi, ghl, gwl, p_drop, seed)
        ctx.save_for_backward(pos_emb)
        return out

    @staticmethod
    def backward(ctx, g):
        N, Hi, Wi, Hl, Wl, C, ghi, gwi, ghl, gwl, p_drop, seed = ctx.cfg
        g = _c(g)
        dimg = torch.empty((N, Hi, Wi, C), dtype=torch.float32, device=g.device)
        dlid = torch.empty((N, Hl, Wl, C), dtype=torch.float32, device=g.device)
        dpos = _gbuf(ctx.saved_tensors[0])
        call('tfb_tokens_bwd', g, dimg, Hi, Wi, ghi, gwi, dlid, Hl, Wl, ghl, gwl, dpos, N, C, float(p_drop), seed_state(g.device), seed, 0)
        return dimg, dlid, dpos, None, None, None, None, None, None


class GptUpAddFn(Function):
    """feat + bilinear_upsample(view(tokens)) for both branches; the token slab is *re-interpreted* as (C, gh, gw)
    exactly like the reference's `.contiguous().view(...)` (transfuser.py:363-364, then 154-157)."""

    @staticmethod
    def forward(ctx, img, lid, tok, ghi, gwi, ghl, gwl):
        img, lid, tok = _c(img), _c(lid), _c(tok)
        N, Hi, Wi, C = img.shape
        _, Hl, Wl, _ = lid.shape
        T = tok.shape[1]
        oi, ol = torch.empty_like(img), torch.empty_like(lid)
        oi16, ol16 = _emit16(oi, True), _emit16(ol, True)       # both feed the 1x1 convs of the next stage / the channel-change conv
        call('tfb_gpt_up_add_fwd', img, tok, oi, N, Hi, Wi, C, ghi, gwi, 0, T, oi16)
        call('tfb_gpt_up_add_fwd', lid, tok, ol, N, Hl, Wl, C, ghl, gwl, ghi * gwi, T, ol16)
        ctx.cfg = (N, Hi, Wi, Hl, Wl, C, ghi, gwi, ghl, gwl, T)
        return _attach16(oi, oi16), _attach16(ol, ol16)

    @staticmethod
    def backward(ctx, di, dl):
        N, Hi, Wi, Hl, Wl, C, ghi, gwi, ghl, gwl, T = ctx.cfg
        di, dl = _c(di), _c(dl)
        dtok = torch.empty((N, T, C), dtype=torch.float32, device=di.device)     # both calls together write every element once
        call('tfb_gpt_up_add_bwd', di, dtok, N, Hi, Wi, C, ghi, gwi, 0, T)
        call('tfb_gpt_up_add_bwd', dl, dtok, N, Hl, Wl, C, ghl, gwl, ghi * gwi, T)
        return di, dl, dtok, None, None, None, None


class UpsampleFn(Function):
    @staticmethod
    def forward(ctx, x, Ho, Wo, align_corners, emit16=False):
        x = _c(x)
        N, Hi, Wi, C = x.shape
        y = torch.empty((N, Ho, Wo, C), dtype=torch.float32, device=x.device)
        y16 = _emit16(y, emit16)
        call('tfb_upsample_bilinear_fwd', x, y, N, Hi, Wi, Ho, Wo, C, int(align_corners), y16)
        ctx.cfg = (N, Hi, Wi, Ho, Wo, C, int(align_corners))
        return _attach16(y, y16)

    @staticmethod
    def backward(ctx, dy):
        N, Hi, Wi, Ho, Wo, C, ac = ctx.cfg
        dy = _c(dy)
        dx = torch.empty((N, Hi, Wi, C), dtype=torch.float32, device=dy.device)
        call('tfb_upsample_bilinear_bwd', dy, dx, N, Hi, Wi, Ho, Wo, C, ac)
        return dx, None, None, None, None


def upsample(x, Ho, Wo, align_corners=False, emit16=False):
    """emit16: the result feeds a tensor-core conv next (decoders, FPN top-down): its bf16 copy is written in the same pass."""
    return UpsampleFn.apply(x, Ho, Wo, align_corners, emit16)


class AvgPoolGridFn(Function):
    """AdaptiveAvgPool2d((gh, gw)) on NHWC maps whose sides divide evenly (geometric_fusion.py:19-20)."""

    @staticmethod
    def forward(ctx, x, gh, gw):
        x = _c(x)
        N, H, W, C = x.shape
        out = torch.empty((N, gh, gw, C), dtype=torch.float32, device=x.device)
        call('tfb_avgpool_grid_fwd', x, out, N, H, W, C, gh, gw)
        ctx.cfg = (N, H, W, C, gh, gw)
        return out

    @staticmethod
    def backward(ctx, dout):
        N, H, W, C, gh, gw = ctx.cfg
        dout = _c(dout)
        dx = torch.empty((N, H, W, C), dtype=torch.float32, device=dout.device)
        call('tfb_avgpool_grid_bwd', dout, dx, N, H, W, C, gh, gw, 0)
        return dx, None, None


def avgpool_grid(x, gh, gw):
    return AvgPoolGridFn.apply(x, gh, gw)


class GatherSumFn(Function):
    """out[b,Y,X,:] = sum_j emb[b, pts[b,Y,X,j,1], pts[b,Y,X,j,0], :] — the B x B advanced index + diagonal + sum of
    geometric_fusion.py:145-148 as one gather; backward scatters with float atomics."""

    @staticmethod
    def forward(ctx, emb, pts):
        emb, pts = _c(emb), _c(pts)
        if pts.dtype != torch.int64 or pts.dim() != 5 or pts.shape[-1] != 2 or pts.shape[0] != emb.shape[0]:
            raise RuntimeError('correspondences must be int64 [B, H, W, P, 2], got %s %s' % (pts.dtype, tuple(pts.shape)))
        B, h, w, C = emb.shape
        _, H, W, P, _ = pts.shape
        out = torch.empty((B, H, W, C), dtype=torch.float32, device=emb.device)
        call('tfb_gather_sum_fwd', emb, pts, out, B, h, w, C, H * W, P)
        ctx.save_for_backward(pts)
        ctx.cfg = (B, h, w, C, H * W, P)
        return out

    @staticmethod
    def backward(ctx, dout):
        pts, = ctx.saved_tensors
        B, h, w, C, M, P = ctx.cfg
        dout = _c(dout)
        demb = torch.empty((B, h, w, C), dtype=torch.float32, device=dout.device)
        call('tfb_gather_sum_bwd', dout, pts, demb, B, h, w, C, M, P)
        return demb, None


def gather_sum(emb, pts):
    return GatherSumFn.apply(emb, pts)


def centernet_decode(preds, num_dir_bins, k=100, ratio=4.0):
    """preds: raw head output [B,H,W,9+num_dir_bins] (NHWC). Returns (boxes [B,k,8], labels [B,k] int64), model.py:436-497."""
    preds = _c(preds)
    B, H, W, C = preds.shape
    if C != 9 + num_dir_bins:
        raise RuntimeError('head output has %d channels, expected %d' % (C, 9 + num_dir_bins))
    boxes = torch.empty((B, k, 8), dtype=torch.float32, device=preds.device)
    labels = torch.empty((B, k), dtype=torch.int32, device=preds.device)
    call('tfb_centernet_decode', preds, B, H, W, num_dir_bins, k, float(ratio), boxes, labels)
    return boxes, labels.long()


class PoolHWFn(Function):
    @staticmethod
    def forward(ctx, x):
        x = _c(x)
        N, H, W, C = x.shape
        out = torch.empty((N, C), dtype=torch.float32, device=x.device)
        call('tfb_pool_hw_fwd', x, out, N, H * W, C)
        ctx.shape = (N, H, W, C)
        return out

    @staticmethod
    def backward(ctx, d):
        N, H, W, C = ctx.shape
        dx = torch.empty((N, H, W, C), dtype=torch.float32, device=d.device)
        call('tfb_pool_hw_bwd', _c(d), dx, N, H * W, C, 0)
        return dx


class TransposeFn(Function):
    """[N, A, B] -> [N, B, A]; used as NCHW <-> NHWC at the module boundary (the reference's tensors are NCHW)."""

    @staticmethod
    def forward(ctx, x):
        x = _c(x)
        N, A, B = x.shape
        y = torch.empty((N, B, A), dtype=torch.float32, device=x.device)
        call('tfb_transpose_last2', x, y, N, A, B)
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = _c(dy)
        N, B, A = dy.shape
        dx = torch.empty((N, A, B), dtype=torch.float32, device=dy.device)
        call('tfb_transpose_last2', dy, dx, N, B, A)
        return dx


def nchw_to_nhwc(x):
    N, C, H, W = x.shape
    return TransposeFn.apply(x.reshape(N, C, H * W)).view(N, H, W, C)


def nhwc_to_nchw(x):
    N, H, W, C = x.shape
    return TransposeFn.apply(x.reshape(N, H * W, C)).view(N, C, H, W)


def image_prep(img_nchw):
    """normalize_imagenet (transfuser.py:419-428) fused with the NCHW -> NHWC layout change. No gradient (input).
    A tensor produced by pipeline.InputPipeline.prepare(normalized_nhwc=True) is already in that form and passes through."""
    if getattr(img_nchw, '_tfb_nhwc_normalized', False):
        return img_nchw
    img = _c(img_nchw.detach())
    N, _, H, W = img.shape
    out = torch.empty((N, H, W, 3), dtype=torch.float32, device=img.device)
    call('tfb_image_prep', img, out, N, H, W)
    return out


# ------------------------------------------------------------------ losses
class CrossEntropyFn(Function):
    """k * sum_m w_m nll_m / den over NHWC logits. den: 'wsum' (sum of weights: F.cross_entropy's weighted mean),
    'count' (plain mean) — model.py:763, 786."""

    @staticmethod
    def forward(ctx, logits, target, class_w, den_mode, k):
        logits, target = _c(logits), _c(target)
        C = logits.shape[-1]
        M = logits.numel() // C
        acc = torch.empty(2, dtype=torch.float64, device=logits.device)
        call('tfb_ce_fwd', logits, target, M, C, class_w, None, 1, acc)
        out = torch.empty((), dtype=torch.float32, device=logits.device)
        den = acc[1:] if den_mode == 'wsum' else None
        kk = k if den_mode == 'wsum' else k / M
        call('tfb_ratio', acc, den, 0.0, float(kk), out)
        ctx.save_for_backward(logits, target, class_w, acc)
        ctx.cfg = (M, C, den_mode, kk)
        return out

    @staticmethod
    def backward(ctx, g):
        logits, target, class_w, acc = ctx.saved_tensors
        M, C, den_mode, kk = ctx.cfg
        d = torch.empty_like(logits)
        den = acc[1:] if den_mode == 'wsum' else None
        call('tfb_ce_bwd', logits, target, M, C, class_w, None, 1, _c(g), den, 0.0, float(kk), d)
        return d, None, None, None, None


class L1Fn(Function):
    """k * mean(|f(x) - t|), f = sigmoid or identity (model.py:765, 788 with transfuser.py:279)."""

    @staticmethod
    def forward(ctx, x, t, sigmoid, k):
        x, t = _c(x), _c(t)
        acc = torch.empty(1, dtype=torch.float64, device=x.device)
        call('tfb_l1_fwd', x, t, x.numel(), int(sigmoid), acc)
        out = torch.empty((), dtype=torch.float32, device=x.device)
        call('tfb_ratio', acc, None, 0.0, float(k) / x.numel(), out)
        ctx.save_for_backward(x, t)
        ctx.cfg = (int(sigmoid), float(k) / x.numel())
        return out

    @staticmethod
    def backward(ctx, g):
        x, t = ctx.saved_tensors
        d = torch.empty_like(x)
        call('tfb_l1_bwd', x, t, x.numel(), ctx.cfg[0], _c(g), ctx.cfg[1], d)
        return d, None, None, None


class CenterNetLossFn(Function):
    """get_targets + the seven head losses (model.py:149-374) on pred[B,H,W,21] (heat logit | wh | offset | yaw class x12 |
    yaw res | velocity | brake x2). Returns a [7] tensor in the order of the reference's loss dict."""

    @staticmethod
    def forward(ctx, pred, label, ratio_w, ratio_h, num_dir_bins):
        pred, label = _c(pred), _c(label)
        B, H, W, _ = pred.shape
        dev = pred.device
        tgt = torch.empty((B, 10, H, W), dtype=torch.float32, device=dev)
        count = torch.empty(1, dtype=torch.int32, device=dev)
        call('tfb_centernet_targets', label, B, label.shape[1], tgt, H, W, float(ratio_w), float(ratio_h), num_dir_bins, count)
        acc = torch.empty(7, dtype=torch.float64, device=dev)
        out = torch.empty(7, dtype=torch.float32, device=dev)
        call('tfb_centernet_loss_fwd', pred, tgt, B, H * W, count, acc, out)
        ctx.save_for_backward(pred, tgt, count)
        return out

    @staticmethod
    def backward(ctx, g):
        pred, tgt, count = ctx.saved_tensors
        B, H, W, _ = pred.shape
        d = torch.empty_like(pred)
        call('tfb_centernet_loss_bwd', pred, tgt, B, H * W, count, _c(g), d)
        return d, None, None, None, None


class GRUFn(Function):
    """forward_gru's autoregressive GRUCell loop (model.py:611-646) after the `join` MLP."""

    @staticmethod
    def forward(ctx, z0, target_point, w_ih, w_hh, b_ih, b_hh, w_out, b_out, steps, x_shift):
        z0, target_point = _c(z0), _c(target_point)
        B = z0.shape[0]
        wp = torch.empty((B, steps, 2), dtype=torch.float32, device=z0.device)
        save = torch.empty((B, steps, 5 * 64 + 4), dtype=torch.float32, device=z0.device)
        call('tfb_gru_fwd', z0, target_point, w_ih, w_hh, b_ih, b_hh, w_out, b_out, B, steps, float(x_shift), wp, save)
        ctx.save_for_backward(save, w_ih, w_hh, w_out, b_ih, b_hh, b_out)
        ctx.cfg = (B, steps)
        return wp

    @staticmethod
    def backward(ctx, d):
        save, w_ih, w_hh, w_out, b_ih, b_hh, b_out = ctx.saved_tensors
        B, steps = ctx.cfg
        dev = d.device
        dz0 = torch.empty((B, 64), dtype=torch.float32, device=dev)
        dw_ih, dw_hh, db_ih, db_hh, dw_out, db_out = [_gbuf(t) for t in (w_ih, w_hh, b_ih, b_hh, w_out, b_out)]
        call('tfb_gru_bwd', _c(d), save, w_ih, w_hh, w_out, B, steps, dz0, dw_ih, dw_hh, db_ih, db_hh, dw_out, db_out)
        return dz0, None, dw_ih, dw_hh, db_ih, db_hh, dw_out, db_out, None, None
