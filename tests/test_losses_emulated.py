"""The loss tests of tests/test_losses.py (cross-entropy, L1, tfb_ratio, the CenterNet targets and head losses against float64
references) executed WITHOUT a GPU: the same test functions, with the C-ABI calls routed to the CPU emulation of the unchanged
kernel source (tests/cuda_emul/), on CPU tensors and with the two largest row counts made smaller (one OS thread per CUDA thread).
The `-m gpu` run of test_losses.py on an H100 remains the test proper: this run checks the kernel source's indexing, control flow and
arithmetic, not the device compiler. Test infrastructure only."""
import pytest

import test_losses as L
from cuda_emul import loader
from test_losses import (test_centernet_classification_terms_confident, test_centernet_losses, test_centernet_saturated_heatmap_logits,  # noqa: F401
                         test_centernet_targets_edge_cases, test_cross_entropy_logit_regimes, test_cross_entropy_position_weights,
                         test_cross_entropy_sizes, test_cross_entropy_zero_weights_and_ratio_clamp, test_l1, test_loss_entry_points_refuse_bad_shapes)


@pytest.fixture(autouse=True)
def _emulated_kernels(monkeypatch):
    lib = loader.patch_product(monkeypatch)
    monkeypatch.setattr(L, 'DEV', 'cpu')
    monkeypatch.setattr(L, 'CE_M', (1, 255, 257, 2053, 40960))
    monkeypatch.setattr(L, 'L1_N', (1, 3, 1027, 40960))
    yield
    assert lib.log, 'the test did not reach the emulated C-ABI'
