"""One training forward + backward of the whole LidarCenterNet in the bf16 tensor-core MODE on the CPU (build container, no GPU):
every CUDA-core kernel runs on the emulation (tests/cuda_emul/), the tensor-core entry points are torch stand-ins written from
their C-ABI contract (tests/cuda_emul/tc_standins.py). Run twice on the same weights and batch — with the host-side options of
DESIGN.md 4b (sidecars, fused SE backward, q|k|v pack, BatchNorm+add+ReLU, batched weight pack) on and off — and against the fp32
CPU oracle. By hand:   python tools/emulated_bf16_step.py [transFuser|late_fusion]      (tens of minutes; test infrastructure)"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import pytest  # noqa: E402
import torch  # noqa: E402

from cuda_emul import loader, tc_standins  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402
from transfuser_b200 import LidarCenterNet, _lib, gemm, ops, optim  # noqa: E402
from transfuser_b200.config import TrainConfig  # noqa: E402

FLAGS = ('SIDECARS', 'SE_FUSED_BWD', 'SE_POOL_FUSED', 'QKV_FUSED', 'BN_ADD_FUSED', 'PACK_BATCHED')


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


def main(backbone, second=False):
    """second = True: the reference run keeps the options ON too — measures the run-to-run noise of the step itself (fp32 atomics land
    in thread-scheduling order on the emulation, as they do in warp-scheduling order on the GPU) that the on/off comparison sits in."""
    mp = pytest.MonkeyPatch()
    emul = loader.patch_product(mp)
    lib = tc_standins.WithTensorCoreStandins(emul)
    mp.setattr(_lib, '_LIB', lib)
    cfg = TrainConfig(embd_pdrop=0.0, attn_pdrop=0.0, resid_pdrop=0.0)
    batch = O.synthetic_batch(1, seed=5)
    w = dict(zip(cfg.detailed_losses, cfg.detailed_losses_weights))
    proto = LidarCenterNet(cfg, 'cpu', backbone, 'regnety_032', 'regnety_032', use_velocity=False)
    names = [(n, tuple(p.shape)) for n, p in list(proto.named_parameters()) + list(proto.named_buffers()) if not n.startswith('_bev')]
    state = O.deterministic_state(names, seed=2)
    proto.load_state_dict(state, strict=False)
    P = {k: v.clone() for k, v in proto.state_dict().items()}
    res = {}
    for on in (True, False):
        for f in FLAGS:
            setattr(ops, f, on or second)
        gemm.set_mode('bf16')
        ops._PACKS.clear()
        ops._PACK_STATE.update(sig=None, table=None)
        net = LidarCenterNet(cfg, 'cpu', backbone, 'regnety_032', 'regnety_032', use_velocity=False)
        net.load_state_dict(state, strict=False)
        net.train()
        fp = optim.flatten(net)
        gemm.attach_bf16_weights(fp)
        t = time.time()
        lib.log.clear()
        out = net(batch['rgb'], batch['lidar'], ego_waypoint=batch['ego_waypoint'], target_point=batch['target_point'],
                  target_point_image=batch['target_point_image'], ego_vel=batch['ego_vel'], bev=batch['bev'], label=batch['label'],
                  depth=batch['depth'], semantic=batch['semantic'])
        sum(w[k] * out[k] for k in out).backward()
        stray = [n for (n, p), o in zip(net.named_parameters(), [dict(zip(map(id, fp.params), fp.offsets))[id(p)] for p in net.parameters()])
                 if p.grad is not None and p.grad.data_ptr() != fp.grad.data_ptr() + 4 * o]
        res[on] = ({k: float(v) for k, v in out.items()}, {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None},
                   len(lib.log))
        print('options %-3s: %d C-ABI calls, %.0f s, %d gradients outside the flat buffer %s' %
              ('on' if on else 'off', len(lib.log), time.time() - t, len(stray), stray[:3]), flush=True)
    (l1, g1, n1), (l0, g0, n0) = res[True], res[False]
    worst = max(abs(l1[k] - l0[k]) / max(abs(l0[k]), 0.1) for k in l0)
    errs = sorted((rel(g1[n], g0[n]), n) for n in g0 if 'key.bias' not in n)
    print('losses, options on vs off: worst relative difference %.2e' % worst)
    print('gradients, options on vs off: median %.2e  p95 %.2e  max %.2e (%s)' %
          (errs[len(errs) // 2][0], errs[int(len(errs) * 0.95)][0], errs[-1][0], errs[-1][1]))
    print('C-ABI calls per forward+backward: %d -> %d' % (n0, n1))
    # where the gap appears: parameters grouped by depth (backward runs from the heads at the top of this list towards the stems)
    import re
    order = ['head|pred_bev|join|decoder|output', 'change_channel|up_conv|c5_conv', 'transformer4', r'\.s4\.|layer4', 'transformer3', r'\.s3\.|layer3',
             'transformer2', r'\.s2\.|layer2', 'transformer1', r'\.s1\.|layer1', 'stem|conv1|bn1']
    left = dict(errs and [(n, e) for e, n in errs])
    for pat in order:
        sel = sorted(e for n, e in left.items() if re.search(pat, n))
        for n in [n for n in left if re.search(pat, n)]:
            del left[n]
        if sel:
            print('  %-44s %4d tensors  median %.2e  max %.2e' % (pat, len(sel), sel[len(sel) // 2], sel[-1]))
    if left:
        sel = sorted(left.values())
        print('  %-44s %4d tensors  median %.2e  max %.2e' % ('(other)', len(sel), sel[len(sel) // 2], sel[-1]))

    class C(O.Cfg):
        embd_pdrop = attn_pdrop = resid_pdrop = 0.0
    if backbone == 'transFuser':
        with torch.no_grad():
            ref = O.forward(P, batch, C, train=True)
        for k in ref:
            print('%-22s fp32 oracle %.6f  bf16 mode %.6f  rel %.2e' % (k, float(ref[k]), l1[k], abs(l1[k] - float(ref[k])) / max(abs(float(ref[k])), 1e-9)))
    ok = worst < 2e-3 and errs[int(len(errs) * 0.95)][0] < 2e-2
    print('RESULT', 'PASSED' if ok else 'FAILED')


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else 'transFuser', second=len(sys.argv) > 2 and sys.argv[2] == 'noise')
