"""In-tree build of the sm_90a CUDA library (libtfb200.so) with nvcc — no torch headers, no JIT cache.

The objects (csrc/build/) and the .so are build products: git-ignored, rebuilt whenever a source, a header or the flags change."""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(CSRC, 'build')
LIB = os.path.join(HERE, 'libtfb200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC,-fvisibility=hidden',
         '--expt-relaxed-constexpr', '-I', CSRC, '-I', os.path.join(os.path.dirname(HERE), 'include')]


def _stamp(path, deps):
    h = hashlib.sha1(' '.join(FLAGS).encode())
    for d in [path] + deps:
        h.update(open(d, 'rb').read())
    return h.hexdigest()


def _compile(src, headers, verbose):
    obj = os.path.join(OBJ, os.path.basename(src)[:-3] + '.o')
    stamp_file = obj + '.stamp'
    stamp = _stamp(src, headers)
    if os.path.exists(obj) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return obj, False
    cmd = [NVCC] + FLAGS + ['-c', src, '-o', obj]
    if verbose:
        print(' '.join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
    if r.stderr.strip() and verbose:
        print(r.stderr, file=sys.stderr)
    open(stamp_file, 'w').write(stamp)
    return obj, True


def build(verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))
    headers = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cuh'))
    inc = os.path.join(os.path.dirname(HERE), 'include')
    headers += sorted(os.path.join(inc, f) for f in os.listdir(inc) if f.endswith('.h'))
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 2)) as ex:
        res = list(ex.map(lambda s: _compile(s, headers, verbose), srcs))
    objs = [o for o, _ in res]
    if any(changed for _, changed in res) or not os.path.exists(LIB):
        cmd = [NVCC, '-shared', '-cudart', 'shared', '-o', LIB] + objs + ['-Xlinker', '-rpath,/usr/local/cuda/lib64']
        if verbose:
            print(' '.join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    return LIB


if __name__ == '__main__':
    print(build(verbose=True))
