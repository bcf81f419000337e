"""ctypes binding of the C-ABI in include/tfb200.h (libtfb200.so, hand-written sm_90a CUDA).

There is deliberately NO fallback: if the library is missing or a kernel returns an error the call raises.
Signatures are parsed from the header so the header stays the single source of truth for the boundary."""
import ctypes
import os
import re

import torch  # noqa: F401  (loads libcudart before libtfb200.so resolves it)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libtfb200.so')
HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'tfb200.h')

_CTYPES = {
    'int': ctypes.c_int, 'int64_t': ctypes.c_int64, 'float': ctypes.c_float, 'double': ctypes.c_double,
    'uint64_t': ctypes.c_uint64, 'unsigned int': ctypes.c_uint, 'tfb_stream_t': ctypes.c_void_p,
}


def parse_header(path=HEADER):
    """Returns {name: (restype, [(ctype, argname)])} for every `TFB_EXPORT` declaration in the header."""
    src = open(path).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    src = re.sub(r'//[^\n]*', '', src)
    decls = {}
    for m in re.finditer(r'TFB_EXPORT\s+(const char\s*\*|int)\s+(\w+)\s*\((.*?)\)\s*;', src, flags=re.S):
        ret, name, args = m.group(1), m.group(2), m.group(3)
        params = []
        args = ' '.join(args.split())
        if args and args != 'void':
            for a in args.split(','):
                a = a.strip()
                pname = re.search(r'(\w+)$', a).group(1)
                ptype = a[:len(a) - len(pname)].strip()
                if '*' in ptype:
                    params.append((ctypes.c_void_p, pname))
                else:
                    params.append((_CTYPES[ptype.replace('const ', '')], pname))
        decls[name] = (ctypes.c_char_p if 'char' in ret else ctypes.c_int, params)
    return decls


HOST_ONLY = {'tfb_gemm_set_max_ctas'}      # entry points that change host-side state and launch nothing (not counted as launches)


class _Lib:
    def __init__(self):
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError('transfuser_b200: %s is missing — run `python -c "import __graft_entry__ as g; g.build()"`; '
                               'there is no CPU / eager fallback.' % LIB_PATH)
        self.cdll = ctypes.CDLL(LIB_PATH)
        self.decls = parse_header()
        self.fns = {}
        for name, (ret, params) in self.decls.items():
            fn = getattr(self.cdll, name)  # AttributeError if the header declares something the .so lacks
            fn.restype = ret
            fn.argtypes = [t for t, _ in params]
            self.fns[name] = (fn, params)
        self.launches = 0
        self.profiler = None

    def call(self, name, *args):
        """Calls tfb_<name>; torch tensors become device pointers; the trailing stream argument is filled in."""
        fn, params = self.fns[name]
        conv = []
        takes_stream = bool(params) and params[-1][1] == 'stream'
        n_user = len(params) - (1 if takes_stream else 0)
        if len(args) != n_user:
            raise TypeError('%s expects %d arguments, got %d' % (name, n_user, len(args)))
        for a, (t, pname) in zip(args, params):
            if t is ctypes.c_void_p:
                if a is None:
                    conv.append(None)
                elif isinstance(a, torch.Tensor):
                    conv.append(a.data_ptr())
                else:
                    conv.append(int(a))
            else:
                conv.append(a)
        if takes_stream:
            conv.append(torch.cuda.current_stream().cuda_stream)
        if self.profiler is not None:
            rc = self.profiler.timed(name, args, lambda: fn(*conv))
        else:
            rc = fn(*conv)
        if name not in HOST_ONLY:
            self.launches += 1
        if rc != 0:
            raise RuntimeError('%s failed with code %d: %s' % (name, rc, self.cdll.tfb_last_error().decode()))


_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        _LIB = _Lib()
    return _LIB


def call(name, *args):
    return lib().call(name, *args)


class Profiler:
    """Per-entry-point CUDA-event timing (events recorded on the launching stream around every C-ABI call) plus the
    algorithmic FLOPs / bytes of each call, used by bench.py for the live roofline of the dominant kernel."""

    # entry points that launch the same kernel: their times are added up when the dominant KERNEL of the step is picked
    FAMILY = {'tfb_gemm_bf16_tc': 'gemm_tc_kernel', 'tfb_gemm_bf16_tc_stats': 'gemm_tc_kernel', 'tfb_gemm_bf16_tc_out16': 'gemm_tc_kernel',
              'tfb_gemm_bf16_tc_wgrad_batched': 'gemm_tc_kernel', 'tfb_conv3x3_tc': 'conv3x3_tc_kernel', 'tfb_conv3x3_tc_strided': 'conv3x3_tc_kernel',
              'tfb_bn_fwd': 'bn_fwd (colreduce4 + bn_apply)', 'tfb_bn_fwd_stats': 'bn_apply_stats_kernel', 'tfb_attn_fwd_tc': 'attn_tc_kernel',
              'tfb_attn_bwd_tc': 'attn_tc_kernel'}

    def __init__(self, keep_calls=False):
        self.records = []
        self.calls = [] if keep_calls else None     # (name, args) of every call, tensors kept alive: replayed by bench.py's graph timing

    def timed(self, name, args, thunk):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = thunk()
        e1.record()
        self.records.append((name, self._work(name, args), e0, e1, self._key(name, args)))
        if self.calls is not None:
            self.calls.append((name, args))
        return rc

    @staticmethod
    def _key(name, a):
        if name == 'tfb_gemm_small_m':
            return '%s tb%d M%d N%d K%d' % (name, a[0], a[1], a[2], a[3])
        if name == 'tfb_gemm_bf16_tc_wgrad_batched':
            return '%s M%d N%d K%d batch%d splits%d' % (name, a[0], a[1], a[2], a[12], a[13])
        if name == 'tfb_gemm_bf16_tc_stats':
            return '%s M%d N%d K%d' % (name, a[0], a[1], a[2])
        if name == 'tfb_gemm_bf16_tc_out16':
            return '%s tb%d M%d N%d K%d' % (name, a[0], a[1], a[2], a[3])
        if name in ('tfb_attn_fwd_tc', 'tfb_attn_bwd_tc'):
            i0 = 2 if name.endswith('fwd_tc') else 8
            return '%s B%d T%d nh%d hs%d' % ((name,) + tuple(a[i0:i0 + 4]))
        if name == 'tfb_conv3x3_tc_strided':
            return '%s N%d H%d W%d Cx%d Cy%d NB%d KC%d chunks%d gblocks%d s%d' % (name, a[4], a[5], a[6], a[7], a[8], a[9], a[10], a[12], a[14], a[16])
        if name == 'tfb_conv3x3_tc':
            return '%s N%d H%d W%d Cx%d Cy%d NB%d KC%d chunks%d gblocks%d' % (name, a[4], a[5], a[6], a[7], a[8], a[9], a[10], a[12], a[14])
        if name in ('tfb_gemm_bf16_tc', 'tfb_gemm_f32_simt', 'tfb_gemm_tf32_tc'):
            return '%s ta%d tb%d M%d N%d K%d%s' % (name, a[0], a[1], a[2], a[3], a[4], (' batch%dx%d' % (a[15], a[16])) if name.endswith('simt') else '')
        if name.startswith('tfb_conv2d'):
            i0 = 3 if name.endswith('dgrad') else 4
            return '%s N%d H%d W%d Cin%d Cout%d k%d s%d g%d' % ((name,) + tuple(a[i0:i0 + 8]))
        return name

    @staticmethod
    def _work(name, a):
        """(flops, bytes) — algorithmic: 2*MAC for contractions, every tensor argument touched once for the rest."""
        if name == 'tfb_gemm_small_m':
            return 2.0 * a[1] * a[2] * a[3], 4.0 * (a[1] * a[3] + a[2] * a[3] + a[1] * a[2])
        if name == 'tfb_gemm_bf16_tc_wgrad_batched':
            return 2.0 * a[0] * a[1] * a[2] * a[12], 2.0 * a[2] * a[12] * (a[0] + a[1]) + 4.0 * a[0] * a[1] * a[12]
        if name == 'tfb_gemm_bf16_tc_stats':
            return 2.0 * a[0] * a[1] * a[2], 2.0 * (a[0] * a[2] + a[1] * a[2]) + 4.0 * a[0] * a[1]
        if name == 'tfb_gemm_bf16_tc_out16':
            return 2.0 * a[1] * a[2] * a[3], 2.0 * (a[1] * a[3] + a[2] * a[3]) + 2.0 * a[1] * a[2]
        if name == 'tfb_gemm_bf16_tc':
            return 2.0 * a[2] * a[3] * a[4], 2.0 * (a[2] * a[4] + a[3] * a[4]) + 4.0 * a[2] * a[3]
        if name in ('tfb_attn_fwd_tc', 'tfb_attn_bwd_tc'):
            i0 = 2 if name.endswith('fwd_tc') else 8
            B, T, nh, hs = a[i0:i0 + 4]
            mult = 1.0 if name.endswith('fwd_tc') else 2.5     # forward: S and PV; backward: S, dP, dV, dQ, dK
            return 4.0 * B * nh * T * T * hs * mult, 4.0 * B * T * nh * hs * 4 * mult
        if name in ('tfb_conv3x3_tc', 'tfb_conv3x3_tc_strided'):
            N, H, W, Cx, Cy, NB, KC, c_step, nchunks, nb_real, gblocks = a[4:15]
            # algorithmic (useful) MACs: each written channel contracts over its group's channels only
            cin_eff = Cx if c_step == 0 else 24
            st = a[16] if name == 'tfb_conv3x3_tc_strided' else 1
            Ho, Wo = (H - 1) // st + 1, (W - 1) // st + 1
            return 2.0 * N * Ho * Wo * Cy * cin_eff * 9, 2.0 * N * H * W * Cx + 4.0 * N * Ho * Wo * Cy
        if name in ('tfb_gemm_f32_simt', 'tfb_gemm_tf32_tc'):
            M, N, K = a[2], a[3], a[4]
            nb = a[15] * a[16] if name.endswith('simt') else 1
            return 2.0 * M * N * K * nb, 4.0 * nb * (M * K + N * K + M * N)
        if name.startswith('tfb_conv2d'):
            i0 = 3 if name.endswith('dgrad') else 4
            N, H, W, Cin, Cout, ks, stride, groups = a[i0:i0 + 8]
            Ho, Wo = (H + 2 * (ks // 2) - ks) // stride + 1, (W + 2 * (ks // 2) - ks) // stride + 1
            return 2.0 * N * Ho * Wo * Cout * (Cin // groups) * ks * ks, 4.0 * (N * H * W * Cin + N * Ho * Wo * Cout)
        b = sum(t.numel() * t.element_size() for t in a if isinstance(t, torch.Tensor))
        return 0.0, float(b)

    def summary(self, peaks_and_how):
        pk, how = peaks_and_how
        torch.cuda.synchronize()
        agg = {}
        self.detail = {}
        for name, (fl, by), e0, e1, key in self.records:
            d = agg.setdefault(name, [0.0, 0.0, 0.0, 0])
            dd = self.detail.setdefault(key, [0.0, 0, fl])
            dd[0] += e0.elapsed_time(e1)
            dd[1] += 1
            d[0] += e0.elapsed_time(e1)
            d[1] += fl
            d[2] += by
            d[3] += 1
        total = sum(v[0] for v in agg.values()) or 1.0
        fam = {}
        for name, v in agg.items():
            f = fam.setdefault(self.FAMILY.get(name, name), [0.0, 0.0, 0.0, 0, []])
            for i in range(4):
                f[i] += v[i]
            f[4].append(name)
        self.families = fam
        top = sorted(((k, v[:4]) for k, v in fam.items()), key=lambda kv: -kv[1][0])
        name, (ms, fl, by, n) = top[0]
        self.top_entry_points = fam[name][4]
        tensor = fl > 0
        if tensor:
            ach, peak, unit = fl / (ms * 1e-3) / 1e12, pk['bf16_tflops_sustained'], 'TFLOP/s'
        else:
            ach, peak, unit = by / (ms * 1e-3) / 1e9, pk['hbm_gbs'], 'GB/s'
        return {'kernel': name, 'bound': 'tensor' if tensor else 'hbm', 'achieved': round(ach, 3), 'peak': peak, 'unit': unit,
                'frac': round(ach / peak, 5), 'traffic': None, 'of': how, 'launches': n, 'avg_ms': round(ms / n, 4),
                'share_of_step': round(ms / total, 4),
                'top5_ms': {k: round(v[0], 3) for k, v in top[:5]}, 'step_kernel_ms': round(total, 3)}
