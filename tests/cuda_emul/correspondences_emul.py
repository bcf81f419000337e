"""TEST INFRASTRUCTURE ONLY. tests/cuda_emul/_build/libtfb200_correspondences_emul.so: csrc/correspondences.cu (with api.cu for
the error text) compiled for the host against the emulation header, as bev_label_emul.py builds the BEV-label kernel, with
-ffp-contract=off so that the compiler fuses no multiply-add either. The intrinsics the kernel spells out (__dmul_rn, __dadd_rn,
__dsub_rn, __ddiv_rn; __fadd_rn / __fmul_rn come from cuda_emul.h) are plain IEEE operations here. `call` has stem_emul's
convention."""
import ctypes
import hashlib
import os
import subprocess

from transfuser_b200 import _lib

from . import build_emul

FILES = ('api.cu', 'correspondences.cu')
LIB = os.path.join(build_emul.OUT, 'libtfb200_correspondences_emul.so')
PRELUDE = ('#include "cuda_emul.h"\n'
           'static inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }\n'
           'static inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }\n'
           'static inline double __dsub_rn(double a, double b) { volatile double r = a - b; return r; }\n'
           'static inline double __ddiv_rn(double a, double b) { volatile double r = a / b; return r; }\n')


def build():
    os.makedirs(build_emul.OUT, exist_ok=True)
    srcs, h = [], hashlib.sha1(PRELUDE.encode())
    for extra in ('cuda_emul.h', 'build_emul.py', 'correspondences_emul.py'):
        h.update(open(os.path.join(build_emul.HERE, extra), 'rb').read())
    for hdr in sorted(f for f in os.listdir(build_emul.CSRC) if f.endswith('.cuh')):
        h.update(open(os.path.join(build_emul.CSRC, hdr), 'rb').read())
    h.update(open(os.path.join(build_emul.ROOT, 'include', 'tfb200.h'), 'rb').read())
    for f in FILES:
        text = build_emul.transpile(open(os.path.join(build_emul.CSRC, f)).read())
        if f == 'correspondences.cu':
            text = PRELUDE + text
        h.update(text.encode())
        dst = os.path.join(build_emul.OUT, f.replace('.cu', '_correspondences_emul.cpp'))
        if not os.path.exists(dst) or open(dst).read() != text:
            open(dst, 'w').write(text)
        srcs.append(dst)
    stamp = LIB + '.stamp'
    if os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest():
        return LIB
    cmd = ['g++', '-O1', '-std=c++20', '-ffp-contract=off', '-fPIC', '-shared', '-pthread', '-Wno-unknown-pragmas', '-Wno-attributes',
           '-I', build_emul.HERE, '-I', build_emul.CSRC, '-I', os.path.join(build_emul.ROOT, 'include')] + srcs + ['-o', LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('emulation build failed:\n' + r.stderr[-6000:])
    open(stamp, 'w').write(h.hexdigest())
    return LIB


_FNS = {}


def call(name, *args):
    """Calls the emulated tfb_<name> (CPU tensors become pointers; no stream)."""
    if not _FNS:
        cdll = ctypes.CDLL(build())
        for fname, (ret, params) in _lib.parse_header().items():
            fn = getattr(cdll, fname, None)
            if fn is not None:
                fn.restype = ret
                fn.argtypes = [t for t, _ in params]
                _FNS[fname] = (fn, params)
        _FNS['_cdll'] = (cdll, None)
    fn, params = _FNS[name]
    takes_stream = bool(params) and params[-1][1] == 'stream'
    if len(args) != len(params) - (1 if takes_stream else 0):
        raise TypeError('%s expects %d arguments, got %d' % (name, len(params) - takes_stream, len(args)))
    conv = []
    for a, (t, _) in zip(args, params):
        if t is ctypes.c_void_p:
            conv.append(a.data_ptr() if hasattr(a, 'data_ptr') else (None if a is None else int(a)))
        else:
            conv.append(a)
    if takes_stream:
        conv.append(None)
    rc = fn(*conv)
    if rc != 0:
        raise RuntimeError('%s failed with code %d: %s' % (name, rc, _FNS['_cdll'][0].tfb_last_error().decode()))
