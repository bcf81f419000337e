"""tests/test_bf16x3.py on the CPU: the CUDA-core kernels (operand split, im2col, reductions) run on the emulation of their sources,
the tensor-core GEMM is replaced by its torch stand-in (bf16 operands, fp32 accumulate — tests/cuda_emul/tc_standins.py). Checks the
host logic of the three-term mode (operand order, transposes, the flipped dgrad weights, accumulation, gradient buffers) — the
`-m gpu` run of test_bf16x3.py is the parity test proper. Test infrastructure only."""
import pytest

import test_bf16x3 as T
from cuda_emul import loader, tc_standins
from test_bf16x3 import (test_attention_x3, test_conv_x3_fwd_bwd, test_grouped_and_narrow_convs_stay_exact, test_linear_x3_fwd_bwd,  # noqa: F401
                         test_split_is_exact_to_two_bf16_terms, x3_mode)
from transfuser_b200 import _lib

pytestmark = []          # (overrides the gpu mark of the imported module: these run without a GPU)


@pytest.fixture(autouse=True)
def _emulated(monkeypatch):
    emul = loader.patch_product(monkeypatch)
    wrapped = tc_standins.WithTensorCoreStandins(emul)
    monkeypatch.setattr(_lib, '_LIB', wrapped)
    monkeypatch.setattr(T, 'DEV', 'cpu')
    yield


def test_conv_trunk_x3_mode_matches_fp32_mode(x3_mode):
    """A RegNetY stage in miniature + decoder-like heads (tests/test_bf16_host_emulated._Net): outputs and every gradient of the
    three-term mode against the exact-fp32 mode. With fp32-grade products the two agree to ~1e-5 (gradients through the batch-2
    BatchNorms a little less), where the plain bf16 mode sits at 3e-2 / 0.25."""
    import torch
    if x3_mode == 'bf16x3':
        pytest.skip('same host code as bf16x6 (only the number of terms differs); the per-op tests above run in both modes')
    from test_bf16_host_emulated import _Net, _run, rel
    from transfuser_b200 import gemm, optim
    gemm.set_mode('simt')
    torch.manual_seed(0)
    ref = _Net().train()
    state = {k: v.clone() for k, v in ref.state_dict().items()}
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 32, 32, 32, generator=g)
    r1, r2 = torch.randn(2, 16, 16, 16, generator=g), torch.randn(2, 16, 16, 7, generator=g)
    want = _run(ref, x.clone().requires_grad_(True), r1, r2)
    gemm.set_mode(x3_mode)
    net = _Net().train()
    net.load_state_dict(state)
    optim.flatten(net)
    lib = _lib.lib()
    lib.log.clear()
    got = _run(net, x.clone().requires_grad_(True), r1, r2)
    log = list(lib.log)
    names = ['head1 out', 'narrow out', 'dx'] + [n for n, _ in net.named_parameters()]
    for i, (n, a, b) in enumerate(zip(names, got, want)):
        assert rel(a, b) < (1e-4 if i < 2 else 2e-3), (n, rel(a, b))
    assert log.count('tfb_gemm_bf16_tc') >= T.NPROD[x3_mode] * 12 and log.count('tfb_split_bf16') >= 20
    assert 'tfb_conv3x3_tc' not in log and 'tfb_gemm_bf16_tc_stats' not in log       # none of the bf16-mode fusions
