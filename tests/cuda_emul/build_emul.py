"""TEST INFRASTRUCTURE ONLY. Builds tests/cuda_emul/_build/libtfb200_emul.so: the SIMT .cu files of transfuser_b200/csrc
compiled for the host against the emulation header (see cuda_emul.h). The only source transformation is the launch syntax:
    kernel<<<grid, block, smem, stream>>>(args);   ->   emul_launch(grid, block, [=] { kernel(args); });
The tensor-core files (gemm_tc.cu, conv_tc.cu: wgmma / TMA / mbarrier PTX) cannot be emulated and are left out, so their
entry points are absent from the emulated library."""
import hashlib
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, 'transfuser_b200', 'csrc')
OUT = os.path.join(HERE, '_build')
LIB = os.path.join(OUT, 'libtfb200_emul.so')
FILES = ('api.cu', 'bev_hist.cu', 'conv_pack.cu', 'conv_simt.cu', 'decode.cu', 'elementwise.cu', 'gemm_simt.cu', 'geometric.cu', 'gru_adamw.cu',
         'input_prep.cu', 'losses.cu', 'norm.cu')
def _split_top(s):
    parts, depth, cur = [], 0, ''
    for ch in s:
        if ch in '([{':
            depth += 1
        elif ch in ')]}':
            depth -= 1
        if ch == ',' and depth == 0:
            parts.append(cur.strip())
            cur = ''
        else:
            cur += ch
    parts.append(cur.strip())
    return parts


def transpile(text):
    """Rewrites every `name<targs><<<cfg>>>(args)` (balanced parentheses, optional template arguments) in place."""
    out, pos = '', 0
    while True:
        i = text.find('<<<', pos)
        if i < 0:
            break
        j = i                                              # walk back over the kernel name and its template arguments
        while j > 0 and text[j - 1].isspace():
            j -= 1
        if text[j - 1] == '>':
            depth = 0
            while True:
                j -= 1
                depth += 1 if text[j] == '>' else -1 if text[j] == '<' else 0
                if depth == 0:
                    break
        while j > 0 and (text[j - 1].isalnum() or text[j - 1] == '_'):
            j -= 1
        k = text.index('>>>', i)
        cfg = _split_top(text[i + 3:k])
        p0 = text.index('(', k)
        depth, p1 = 0, p0
        while True:
            depth += 1 if text[p1] == '(' else -1 if text[p1] == ')' else 0
            if depth == 0:
                break
            p1 += 1
        kern, args = text[j:i].strip(), text[p0 + 1:p1]
        out += text[pos:j] + 'emul_launch(dim3(%s), dim3(%s), [=] { %s(%s); })' % (cfg[0], cfg[1], kern, args)
        pos = p1 + 1
    out += text[pos:]
    assert '<<<' not in out
    return out


def build():
    os.makedirs(OUT, exist_ok=True)
    srcs, h = [], hashlib.sha1()
    for extra in ('cuda_emul.h', 'build_emul.py'):
        h.update(open(os.path.join(HERE, extra), 'rb').read())
    for hdr in sorted(f for f in os.listdir(CSRC) if f.endswith('.cuh')):
        h.update(open(os.path.join(CSRC, hdr), 'rb').read())
    for f in FILES:
        text = transpile(open(os.path.join(CSRC, f)).read())
        h.update(text.encode())
        dst = os.path.join(OUT, f.replace('.cu', '_emul.cpp'))
        if not os.path.exists(dst) or open(dst).read() != text:
            open(dst, 'w').write(text)
        srcs.append(dst)
    stamp = os.path.join(OUT, 'stamp')
    if os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest():
        return LIB
    cmd = ['g++', '-O1', '-std=c++20', '-ffp-contract=off', '-fPIC', '-shared', '-pthread', '-Wno-unknown-pragmas', '-Wno-attributes',
           '-I', HERE, '-I', CSRC, '-I', os.path.join(ROOT, 'include')] + srcs + ['-o', LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('emulation build failed:\n' + r.stderr[-6000:])
    open(stamp, 'w').write(h.hexdigest())
    return LIB


if __name__ == '__main__':
    print(build())
