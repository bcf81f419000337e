"""Simulated ranks of a synchronized BatchNorm, shared by tests/test_sync_bn.py (CPU emulation) and tests/test_sync_bn_gpu.py (H100):
each rank's slice from its own rows, the slices concatenated in rank order as an all-gather leaves them, every rank's apply pass on
its own rows. Checked against an fp64 restatement of BatchNorm over the concatenated rows, against a host fold of the kernels' own
slices, and (one rank) bit for bit against the unsynchronized entry points."""
import torch

TOL_Y, TOL_DX = 2e-5, 2e-5       # fp32 kernels vs the fp64 restatement, relative to the largest magnitude of the compared tensor
EPS, MOM = 1e-5, 0.1


def _rand(shape, seed, dev, scale=1.0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale + shift).to(dev)


def _ref(xs, gamma, beta, relu, res, dys, gates, dpools, hw):
    """fp64 BatchNorm over the concatenated rows: y per rank, mean, invstd, unbiased var, dx per rank."""
    x = torch.cat(xs).double()
    N = x.shape[0]
    mean = x.mean(0)
    var = x.var(0, unbiased=False)
    invstd = 1.0 / torch.sqrt(var + EPS)
    xh = (x - mean) * invstd
    z = xh * gamma.double() + beta.double()
    if res is not None:
        z = z + torch.cat(res).double()
    y = torch.relu(z) if relu else z
    g = torch.cat(dys).double()
    if gates is not None:
        # gradient of the SE output -> gradient of the BatchNorm output: dy * gate[n] + dpool[n] / hw
        gate = torch.cat(gates).double().repeat_interleave(hw, 0)
        dp = torch.cat(dpools).double().repeat_interleave(hw, 0)
        g = g * gate + dp / hw
    if relu:
        g = g * (z > 0).double()
    dx = gamma.double() * invstd * (g - g.mean(0) - xh * (g * xh).mean(0))
    split = [t.shape[0] for t in xs]
    return dict(y=list(torch.split(y, split)), mean=mean, invstd=invstd, var_unbiased=x.var(0, unbiased=True), dx=list(torch.split(dx, split)),
                dbeta=[t.sum(0) for t in torch.split(g, split)], dgamma=[t.sum(0) for t in torch.split(g * xh, split)])


def _fold(slices):
    """The host fold of the ranks' slices in rank order from +0 (the kernels' rule)."""
    acc = [0.0] * slices[0].numel()
    for s in slices:
        acc = [a + v for a, v in zip(acc, s.tolist())]
    return acc


def run(call, dev, world, variant, from_stats, C=8, hw=6, seed=0):
    """variant: 'plain', 'relu', 'residual' (relu(bn(x) + res), ymask backward), 'pool' (SE pool forward, SE-gated backward).
    from_stats: the forward slice from epilogue-style statistics (fp64 sums of the rank's rows) instead of the statistics pass."""
    ns = [(2 + 3 * w) % 5 + 1 for w in range(world)]            # unequal samples per rank
    xs = [_rand((n * hw, C), seed + 10 * w, dev, 2.0, 0.5) for w, n in enumerate(ns)]
    dys = [_rand((n * hw, C), seed + 10 * w + 1, dev) for w, n in enumerate(ns)]
    res = [_rand((n * hw, C), seed + 10 * w + 2, dev) for w, n in enumerate(ns)] if variant == 'residual' else None
    se = variant == 'pool'
    gates = [torch.sigmoid(_rand((n, C), seed + 10 * w + 3, dev)) for w, n in enumerate(ns)] if se else None
    dpools = [_rand((n, C), seed + 10 * w + 4, dev) for w, n in enumerate(ns)] if se else None
    gamma, beta = _rand((C,), seed + 5, dev, 0.3, 1.0), _rand((C,), seed + 6, dev, 0.2)
    relu = variant != 'plain'
    ws = torch.zeros(2 * 8192 + 8, dtype=torch.float64, device=dev)
    f32 = lambda n: torch.empty(n, dtype=torch.float32, device=dev)
    stats = [torch.cat([x.double().sum(0), (x.double() ** 2).sum(0)]) for x in xs] if from_stats else [None] * world

    slices = []
    for w in range(world):
        sl = torch.empty(2 * C + 1, dtype=torch.float64, device=dev)
        call('tfb_bn_sync_slice', xs[w], xs[w].shape[0], C, stats[w], sl, ws)
        slices.append(sl)
    gathered = torch.cat(slices)
    out = []
    for w in range(world):
        M = xs[w].shape[0]
        o = dict(y=torch.empty_like(xs[w]), mean=f32(C), invstd=f32(C), rm=torch.zeros(C, device=dev), rv=torch.ones(C, device=dev),
                 folded=torch.empty(2 * C + 1, dtype=torch.float64, device=dev), pooled=f32(ns[w] * C).view(ns[w], C) if se else None)
        call('tfb_bn_fwd_sync', xs[w], o['y'], M, C, gamma, beta, EPS, MOM, int(relu), o['rm'], o['rv'], o['mean'], o['invstd'], gathered, world,
             o['folded'], int(from_stats), None, res[w] if res else None, o['pooled'], ns[w] if se else 0)
        out.append(o)
    bslices = []
    for w in range(world):
        M = xs[w].shape[0]
        o = out[w]
        o['dg'], o['db'], sl = f32(C), f32(C), torch.empty(2 * C, dtype=torch.float64, device=dev)
        call('tfb_bn_bwd_sync_reduce', xs[w], dys[w], M, C, gamma, beta, o['mean'], o['invstd'], int(relu and not res), o['dg'], o['db'], ws,
             o['y'] if res else None, gates[w] if se else None, dpools[w] if se else None, hw, sl)
        bslices.append(sl)
    bgathered = torch.cat(bslices)
    for w in range(world):
        M = xs[w].shape[0]
        o = out[w]
        o['dx'], o['gm'] = torch.empty_like(xs[w]), torch.empty_like(xs[w]) if res else None
        call('tfb_bn_bwd_sync_apply', xs[w], dys[w], o['dx'], M, C, gamma, beta, o['mean'], o['invstd'], int(relu and not res), bgathered, world,
             o['folded'][2 * C:], f32(2 * C), None, o['y'] if res else None, o['gm'], gates[w] if se else None, dpools[w] if se else None, hw)

    ref = _ref(xs, gamma, beta, relu, res, dys, gates, dpools, hw)
    rel = lambda a, b: ((a.double().cpu() - b.cpu()).abs().max() / b.abs().max().clamp_min(1e-30)).item()
    fold, N = _fold(slices), sum(x.shape[0] for x in xs)
    assert fold[2 * C] == N
    for w in range(world):
        o = out[w]
        # every rank: the same bits, and exactly the host fold of the kernels' own slices
        assert torch.equal(o['mean'], out[0]['mean']) and torch.equal(o['invstd'], out[0]['invstd'])
        assert torch.equal(o['rm'], out[0]['rm']) and torch.equal(o['rv'], out[0]['rv'])
        assert o['folded'].tolist() == fold
        hm = [s0 / N for s0 in fold[:C]]
        hv = [max(s1 / N - m * m, 0.0) for s1, m in zip(fold[C:2 * C], hm)]
        assert o['mean'].tolist() == torch.tensor(hm, dtype=torch.float32).tolist()
        assert o['invstd'].tolist() == torch.tensor([1.0 / (v + EPS) ** 0.5 for v in hv], dtype=torch.float32).tolist()
        assert rel(o['y'], ref['y'][w]) < TOL_Y
        assert rel(o['dx'], ref['dx'][w]) < TOL_DX
        assert rel(o['db'], ref['dbeta'][w]) < TOL_DX and rel(o['dg'], ref['dgamma'][w]) < TOL_DX
        if se:
            pooled_ref = ref['y'][w].view(ns[w], hw, C).mean(1)
            assert rel(o['pooled'], pooled_ref) < TOL_Y
    assert rel(out[0]['mean'], ref['mean']) < TOL_Y and rel(out[0]['invstd'], ref['invstd']) < TOL_Y
    assert rel(out[0]['rm'], MOM * ref['mean']) < TOL_Y
    assert rel(out[0]['rv'], (1 - MOM) + MOM * ref['var_unbiased']) < TOL_Y

    if world == 1:
        # one rank: the bits of the unsynchronized entry points
        M = xs[0].shape[0]
        p = dict(y=torch.empty_like(xs[0]), mean=f32(C), invstd=f32(C), rm=torch.zeros(C, device=dev), rv=torch.ones(C, device=dev),
                 pooled=f32(ns[0] * C).view(ns[0], C).zero_() if se else None)
        args = (xs[0], p['y'], M, C, gamma, beta, EPS, MOM, int(relu), p['rm'], p['rv'], p['mean'], p['invstd'])
        tail = (None, res[0] if res else None, p['pooled'], ns[0] if se else 0)
        if from_stats:
            call('tfb_bn_fwd_stats', *args, stats[0], *tail)
        else:
            call('tfb_bn_fwd', *args, ws, *tail)
        for k in ('y', 'mean', 'invstd', 'rm', 'rv') + (('pooled',) if se else ()):
            assert torch.equal(p[k], out[0][k]), k
        dx, dg, db, gm = torch.empty_like(xs[0]), f32(C), f32(C), torch.empty_like(xs[0]) if res else None
        if se:
            call('tfb_bn_bwd_se', xs[0], dys[0], dx, M, C, gamma, beta, p['mean'], p['invstd'], 1, dg, db, ws, None, gates[0], dpools[0], hw)
        else:
            call('tfb_bn_bwd', xs[0], dys[0], dx, M, C, gamma, beta, p['mean'], p['invstd'], int(relu and not res), dg, db, ws, None,
                 p['y'] if res else None, gm)
        assert torch.equal(dx, out[0]['dx']) and torch.equal(dg, out[0]['dg']) and torch.equal(db, out[0]['db'])
        if res:
            assert torch.equal(gm, out[0]['gm'])
    return out
