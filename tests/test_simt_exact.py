"""The exact-fp32 CUDA-core convolution and GEMM kernels (csrc/conv_simt.cu, csrc/gemm_simt.cu) on the H100, against the float64
references of tests/simt_ref.py (cases: tests/simt_cases.py; the same cases at reduced size under the CPU emulation:
tests/test_simt_emulated.py). Besides the emulated shapes and larger tiles, every call these five entry points receive in one
eager bf16 training step of each benchmarked backbone is run (simt_cases.BENCH), and one test re-spies those steps so that a new
call site cannot arrive untested. Every case runs twice into NaN-filled, sentinel-guarded outputs and must give the same bits.
Each test prints its worst allowance ratio per check (1.0 = at the bound; exact checks print 0)."""
import os
import sys

import pytest
import torch

sys.path[:0] = [os.path.dirname(os.path.abspath(__file__)), os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import simt_cases as K  # noqa: E402
from test_simt_emulated import EMUL_CONV, EMUL_GEMM, EMUL_SMALL_M, LAYOUTS, gemm_args  # noqa: E402

pytestmark = pytest.mark.gpu

# larger than the emulation can afford: many pixel splits on 132 SMs, several 128 x 64 tiles and K slabs
CONV = [(4, 40, 88, 64, 64, 3, 1, 1, True, True), (4, 20, 88, 216, 216, 3, 2, 9, True, False), (2, 33, 35, 3, 32, 3, 2, 1, True, True),
        (10, 64, 64, 64, 3, 1, 1, 1, True, False), (3, 30, 41, 130, 16, 1, 1, 1, False, False), (2, 17, 19, 72, 144, 1, 2, 1, False, False)]
GEMM = [(1000, 700, 515, 'exact', 1.0, 0.0, True, True, {}), (513, 257, 1024, 'gauss', 0.5, 1.0, False, False, dict(pad=(2, 4, 8))),
        (300, 200, 129, 'shift', 1.0, 0.0, True, False, dict(pad=(1, 0, 0))),
        (174, 174, 64, 'exact', 0.5, 0.0, False, False, dict(batch=(10, 4), gap=2, offs=(2, 2)))]


@pytest.fixture(scope='module')
def ctx():
    from transfuser_b200 import _lib
    return K.Ctx(_lib.call, 'cuda', torch.cuda.get_device_properties(0).multi_processor_count)


def _show(what, res):
    print('%s: %s' % (what, {k: '%.4f' % v for k, v in res.items()}))


def _fresh(ctx):
    ctx.res = {}
    return ctx


@pytest.mark.parametrize('shape', EMUL_CONV + CONV)
def test_conv_exact(ctx, shape):
    for kind in K.KINDS:
        _show('conv %s %s' % (shape, kind), K.conv(_fresh(ctx), *shape, kind, seed=sum(shape[:8])))


@pytest.mark.parametrize('ta,tb', LAYOUTS)
@pytest.mark.parametrize('M,N,Kd,kind,alpha,beta,bias,relu,extra', EMUL_GEMM + GEMM)
def test_gemm_exact(ctx, ta, tb, M, N, Kd, kind, alpha, beta, bias, relu, extra):
    _show('gemm ta %d tb %d M %d N %d K %d %s' % (ta, tb, M, N, Kd, kind),
          K.gemm(_fresh(ctx), ta, tb, M, N, Kd, kind, alpha, beta, bias, relu, seed=M + N + Kd, **gemm_args(M, N, Kd, ta, tb, extra)))


@pytest.mark.parametrize('tb,M,N,Kd,act,bias', EMUL_SMALL_M + [(1, 10, 1512, 144, 2, True), (1, 10, 144, 1512, 1, True),
                                                               (0, 16, 1512, 144, 0, False), (1, 16, 1000, 1536, 2, True)])
def test_small_m_exact(ctx, tb, M, N, Kd, act, bias):
    for kind in K.KINDS:
        _show('small_m tb %d M %d N %d K %d act %d %s' % (tb, M, N, Kd, act, kind),
              K.small_m(_fresh(ctx), tb, M, N, Kd, act, bias, kind, seed=M + N + Kd))


@pytest.mark.parametrize('key', K.BENCH, ids=lambda k: '-'.join(str(v) for v in k))
def test_bench_call_exact(ctx, key):
    for kind in K.kinds_for(key):
        _show('%s %s' % (key, kind), K.run_key(_fresh(ctx), key, kind))


def test_bench_call_sites_are_listed():
    """Every call of the five entry points in one eager bf16 step of each SPY_STEPS configuration has its key in BENCH. Each step
    runs in a fresh process (spy_keys below), so it has the device to itself whatever the session has left resident."""
    import ast
    import gc
    import subprocess
    gc.collect()
    torch.cuda.empty_cache()
    here = os.path.dirname(os.path.abspath(__file__))
    listed, missing = set(K.BENCH), {}
    for backbone, B in K.SPY_STEPS:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), backbone, str(B)], cwd=os.path.dirname(here), capture_output=True,
                           text=True, timeout=1200)
        lines = [l for l in r.stdout.splitlines() if l.startswith('KEYS ')]
        assert r.returncode == 0 and len(lines) == 1, '%s: the spied step failed\n%s' % (backbone, r.stderr[-4000:])
        keys = ast.literal_eval(lines[0][5:])
        print('%s batch %d: %d calls of the CUDA-core convolutions and GEMMs, %d distinct' % (backbone, B, len(keys), len(set(keys))))
        for k in keys:
            if k not in listed:
                missing.setdefault(k, backbone)
    assert not missing, 'calls not in simt_cases.BENCH:\n' + '\n'.join('    %r,   # %s' % (k, b) for k, b in missing.items())


def spy_keys(backbone, B):
    """The call keys (simt_cases.call_key) of one eager bf16 training step, in call order."""
    import numpy as np
    from bench import make_host_batch
    from test_tc_exact import _spy
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    torch.manual_seed(0)
    raw = backbone != 'latentTF'
    tr = Trainer(TrainConfig(), 'cuda', gemm_mode='bf16', lr=1e-4, seed=0, backbone=backbone, raw_inputs=raw)
    host = make_host_batch(B, seed=100, torch=torch, np=np, backbone=backbone, raw=raw)
    dev = {k: v.cuda() for k, v in host.items()}
    _, calls = _spy(lambda: tr.step(dev))
    torch.cuda.synchronize()
    return [K.call_key(n, a) for n, a in calls if n in K.SPIED]


def test_argument_checks(ctx):
    """Refused on the host: nothing is launched."""
    K.refusals(ctx)


def test_pool_misaligned_operands_refused():
    """The max-pool's misaligned operands are refused on the host: nothing misaligned is ever launched."""
    K.pool_refusals(_lib_call, 'cuda')


def _lib_call(name, *args):
    from transfuser_b200 import _lib
    return _lib.call(name, *args)


if __name__ == '__main__':
    print('KEYS %r' % (spy_keys(sys.argv[1], int(sys.argv[2])),))
