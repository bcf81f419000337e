"""The kernel-level GPU tests of tests/test_widen.py and tests/test_pipeline.py, executed at their full sizes on the CPU emulation of the unchanged kernel sources — see
tests/cuda_emul/ and tests/test_ops_emulated.py. The module-level ones (whole networks) are too slow for the emulation inside
the test suite; tools/emulated_module_checks.py runs them by hand. Test infrastructure only."""
import pytest

import test_pipeline as P
import test_widen as W
from cuda_emul import loader


@pytest.fixture(autouse=True)
def _emulated_kernels(monkeypatch):
    from transfuser_b200 import pipeline
    lib = loader.patch_product(monkeypatch)
    monkeypatch.setattr(W, 'DEV', 'cpu')
    monkeypatch.setattr(P, 'DEV', 'cpu')
    monkeypatch.setattr(pipeline.InputPipeline, '_require_cuda', lambda self: None)
    yield
    assert lib.log, 'the test did not reach the emulated C-ABI'


@pytest.mark.parametrize('shape,grid', [((2, 72, 40, 176), (5, 22)), ((2, 216, 32, 32), (8, 8)), ((1, 1512, 5, 22), (5, 22)), ((2, 6, 16, 24), (4, 3))])
def test_avgpool_grid(shape, grid):
    W.test_avgpool_grid_matches_torch(shape, grid)


@pytest.mark.parametrize('B,hw,HW,C', [(2, (5, 22), (8, 8), 512), (3, (8, 8), (5, 22), 512), (1, (4, 4), (2, 3), 8)])
def test_gather_sum(B, hw, HW, C):
    W.test_gather_sum_matches_torch_index(B, hw, HW, C)


@pytest.mark.parametrize('case', [0, 1, 2, 3])
def test_centernet_decode(case):
    W.test_centernet_decode_matches_oracle(case)


def test_fused_adamw():
    W.test_fused_adamw_matches_torch_adamw_on_device()


def test_input_pipeline_full_size():
    P.test_input_pipeline_matches_oracle()


def test_target_point_map():
    P.test_target_point_map_borders_and_overflow()
