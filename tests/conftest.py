import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    import torch
    # the torch ops used as fp32 references must really be fp32 (cuDNN / cuBLAS default to TF32 for convs)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100: sm_90a)')


@pytest.fixture(scope='session', autouse=True)
def _built_library():
    """The C-ABI library is a build product (git-ignored): build it once per session if it is not there yet
    (nvcc cross-compiles sm_90a without a GPU)."""
    from transfuser_b200 import build as b
    if not os.path.isfile(b.LIB):
        b.build(verbose=False)
    yield


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device in this container')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _reset_numerics_mode():
    """Every test starts in the exact-fp32 ('simt') GEMM mode; tests of the bf16 tensor-core mode switch it on themselves."""
    try:
        from transfuser_b200 import gemm
    except Exception:
        yield
        return
    gemm.set_mode('simt')
    gemm._FLAT[0] = None
    gemm._WCACHE.clear()
    yield
    gemm.set_mode('simt')
    gemm._FLAT[0] = None
    gemm._WCACHE.clear()
