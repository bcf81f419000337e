"""bench.py — TransFuser training-step throughput (samples/s of RGB+LiDAR pairs) on N H100s of one node.

  python bench.py --gpus 1 --steps 20 --warmup 3          # this repo's CUDA path (default)
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...
  python bench.py --impl reference ...                    # the reference's CPU PyTorch path (oracle port) on the host cores

One "step" = BASELINE.json configs[1]: LidarCenterNet (TransFuser, RegNetY-3.2GF) forward + backward + AdamW on a batch of
10 samples per GPU (160x704 RGB + 40k LiDAR points -> 2x256x256 BEV histogram on the GPU + target-point image), dropout on,
all 11 losses, synthetic data, random-init weights. Prints ONE JSON line (rank 0).

  python bench.py ... --dump-outputs DIR                  # also write what the last timed step computed to DIR/<name>.npy

Inputs and initial weights are seeded, so two builds run with the same arguments can be compared output for output."""
import argparse
import json
import math
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FLOP_PER_SAMPLE_TRAIN = 230.3e9   # SURVEY.md §8(d): 3 x 76.8 GFLOP forward (2*MAC)
# BASELINE.json configs[1..4] -> (backbone, per-GPU batch, algorithmic train-step GFLOP per sample (SURVEY.md §8d), label)
CONFIGS = {2: ('transFuser', 10, 230.3e9, 'TransFuser RegNetY-3.2GF'), 3: ('transFuser', 12, 230.3e9, 'TransFuser RegNetY-3.2GF + all aux heads'),
           4: ('geometric_fusion', 12, 109.1e9, 'GeometricFusion'), 5: ('late_fusion', 16, 93.1e9, 'LateFusion (conv-only)')}
METRIC = 'training samples/sec (RGB+LiDAR pairs)'


def peaks():
    """Roofline peaks: H100 SXM data sheet (700 W card; dense BF16), never reached figures."""
    return dict(hbm_gbs=3350.0, bf16_tflops=989.0, bf16_tflops_sustained=989.0), 'H100 SXM data sheet'


def gpu_identity(index=0):
    """Card name and power limit, read in the same run as the measurement they qualify."""
    try:
        r = subprocess.run(['nvidia-smi', '-i', str(index), '--query-gpu=name,power.limit', '--format=csv,noheader,nounits'],
                           capture_output=True, text=True, timeout=30)
        name, limit = [c.strip() for c in r.stdout.strip().split(',')[:2]]
        return {'name': name, 'power_limit_w': float(limit)}
    except Exception:  # noqa: BLE001
        import torch
        return {'name': torch.cuda.get_device_name(index), 'power_limit_w': None}


class ClockSampler:
    Q = 'clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap'

    def __init__(self, index=0):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(['nvidia-smi', '-i', str(self.index), '--query-gpu=' + self.Q, '--format=csv,noheader,nounits', '-lms', '100'],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(',')])

    def stop(self):
        if self.proc is None:
            return dict(sm_mhz=None, sm_max_mhz=None, reasons=['nvidia-smi unavailable'])
        self.proc.terminate()
        self.proc.wait()
        sm = sorted(float(r[0]) for r in self.rows if r and r[0].replace('.', '').isdigit())
        reasons = set()
        names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap']
        for r in self.rows:
            for n, v in zip(names, r[3:7]):
                if v.lower().startswith('active'):
                    reasons.add(n)
        mx = max((float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace('.', '').isdigit()), default=None)
        return dict(sm_mhz=sm[len(sm) // 2] if sm else None, sm_max_mhz=mx, reasons=sorted(reasons), samples=len(sm))


def make_host_batch(B, seed, torch, np, backbone='transFuser', raw=False):
    """Synthetic inputs of SURVEY.md §8(d) in PINNED host memory (the e2e arm copies them every step)."""
    from oracle import bev_oracle, torch_oracle as O
    b = O.synthetic_batch(B, seed=seed)
    if backbone == 'geometric_fusion':
        b['bev_points'], b['cam_points'] = O.synthetic_correspondences(B, seed=seed)
    pts = np.stack([bev_oracle.synthetic_points(40000, 1000 * seed + i, np.float32, edge_cases=False) for i in range(B)])
    b['points'] = torch.from_numpy(pts)
    del b['lidar']
    if raw:
        # the compact form of the same batch (what the dataset holds on disk): uint8 camera / depth / semantic frames, the pose
        # transform of align() (identity: no second LiDAR sweep in the synthetic batch), the float64 target point; the expanded
        # fp32 / int64 tensors they replace are built on the GPU by pipeline.InputPipeline inside the step
        g = torch.Generator().manual_seed(4000 + seed)
        b['rgb_u8'] = b.pop('rgb').permute(0, 2, 3, 1).contiguous().to(torch.uint8)
        b['depth_u8'] = torch.randint(0, 256, (B, 160, 704, 3), dtype=torch.uint8, generator=g)
        b['depth_u8'][..., 0] = torch.randint(0, 13, (B, 160, 704), dtype=torch.uint8, generator=g)   # 24-bit depth code, mostly inside the 0.05 clip
        b['seg_u8'] = torch.randint(0, 28, (B, 160, 704), dtype=torch.uint8, generator=g)
        b['crop_shift'] = torch.zeros(B, dtype=torch.int32)
        b['transforms'] = torch.eye(4, dtype=torch.float64).reshape(1, 4, 4).repeat(B, 1, 1)
        b['target_point64'] = b.pop('target_point').double()
        for k in ('depth', 'semantic', 'target_point_image'):
            del b[k]
    return {k: v.pin_memory() for k, v in b.items()}


def run_b200(args):
    import numpy as np
    import torch
    import torch.distributed as dist
    from transfuser_b200 import _lib
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer

    rank, world, local = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1)), int(os.environ.get('LOCAL_RANK', 0))
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault('NCCL_DEBUG_FILE', '/dev/stderr')   # NCCL's version / debug banner must not land on stdout (one JSON line)
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    dev = torch.device('cuda', local)
    backbone, cfg_batch, flop_per_sample, label = CONFIGS[args.config]
    B = args.batch or cfg_batch
    cfg = TrainConfig()
    torch.manual_seed(0)
    raw = bool(args.raw_inputs)
    tr = Trainer(cfg, dev, gemm_mode=args.gemm, lr=1e-4, seed=rank, backbone=backbone, raw_inputs=raw)
    host = make_host_batch(B, seed=100 + rank, torch=torch, np=np, backbone=backbone, raw=raw)

    def h2d():
        return {k: v.to(dev, non_blocking=True) for k, v in host.items()}

    step = tr.step

    def run_step(e2e):
        if tr.graph is None:
            return tr.step(h2d() if e2e else resident[0])
        if e2e:
            tr.load(host)
        return tr.replay()

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    resident = [None]
    last_loss = [None]               # the total-loss tensor of the latest timed step

    def timed(n, e2e):
        resident[0] = h2d()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = _lib.lib().launches
        e0.record()
        last = None
        for _ in range(n):
            loss = last_loss[0] = run_step(e2e)
            if e2e:
                last = float(loss.item())  # device -> host read of the step's result
        e1.record()
        barrier()
        ms = e0.elapsed_time(e1)
        if world > 1:
            t = torch.tensor([ms], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
        launches = tr.graph_launches * n if tr.graph is not None else _lib.lib().launches - l0
        return ms, launches, last

    for _ in range(max(args.warmup, 3)):
        step(h2d())
    if args.graph:
        if tr.capture(host):
            for _ in range(2):
                run_step(True)
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    ms_dev, launches, _ = timed(args.steps, e2e=False)
    ms_e2e, _, e2e_loss = timed(args.steps, e2e=True)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, tr, last_loss[0], torch, np)

    # ---- roofline of the dominant kernel: per-entry-point CUDA-event timing over one extra step (rank 0) ----
    roof = None
    prof = _lib.Profiler(keep_calls=True) if rank == 0 else None
    _lib.lib().profiler = prof
    torch.cuda.synchronize()

    def profiler_bracket(fn):        # cudaProfilerStart / Stop: no-ops without an attached profiler; never allowed to fail the bench
        try:
            fn()
        except Exception:  # noqa: BLE001
            pass

    profiler_bracket(torch.cuda.profiler.start)   # `ncu --profile-from-start off` captures exactly this eager step (process-wide: the
    step(h2d())                      # backward kernels are launched by the autograd thread, which a per-thread NVTX range would miss).
    torch.cuda.synchronize()         # Every rank runs the step (it contains the gradient all-reduce); only rank 0 instruments.
    profiler_bracket(torch.cuda.profiler.stop)
    _lib.lib().profiler = None
    if rank == 0:
        roof = prof.summary(peaks())
        try:
            roof.update(graph_timed_roofline(prof, torch, _lib))
        except Exception as e:  # noqa: BLE001 — the eager-event figures stay in the line; say why the graph timing is missing
            roof['graph_timing_error'] = repr(e)[:200]
        prof.calls = None
    h2d_bytes = sum(v.numel() * v.element_size() for v in host.values())
    if rank == 0:
        pk, how = peaks()
        total = B * world
        value = total * args.steps / (ms_dev / 1e3)
        e2e_v = total * args.steps / (ms_e2e / 1e3)
        line = {
            'metric': METRIC, 'value': round(value, 3), 'unit': 'samples/s', 'n_gpus': world, 'steps': args.steps, 'warmup': max(args.warmup, 3),
            'ms_per_step': round(ms_dev / args.steps, 3), 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
            'dtype': {'bf16': 'bf16', 'bf16x3': 'bf16x3 (fp32 operands as two bf16 terms, three tensor-core products, fp32 accumulate)',
                      'bf16x6': 'bf16x6 (fp32 operands as three bf16 terms, six tensor-core products, fp32 accumulate)'}.get(args.gemm, 'fp32'),
            'data': 'synthetic',
            'config': {'workload': '%s LidarCenterNet full train step (fwd+bwd+AdamW), all aux heads, dropout 0.1, '
                                   '160x704 RGB + 40k-point LiDAR->BEV, batch %d per GPU (BASELINE configs[%d])' % (label, B, args.config - 1),
                       'global_batch': total, 'parallelism': 'dp%d' % world, 'gemm_mode': args.gemm,
                       'inputs': ('raw (uint8 frames, points, pose transform, target point): model inputs built by the GPU input pipeline inside the step'
                                  if raw else 'expanded fp32 / int64 tensors as the reference DataLoader ships them; LiDAR points -> BEV histogram on the GPU'), 'cuda_graph': tr.graph is not None, 'cuda_graph_error': tr.graph_error,
                       'l2': 'working set (672 MB weights + activations) exceeds the 50 MB L2; no explicit flush'},
            'e2e': {'value': round(e2e_v, 3), 'unit': 'samples/s', 'ms_per_step': round(ms_e2e / args.steps, 3),
                    'h2d_bytes_per_step': h2d_bytes, 'd2h_bytes_per_step': 4, 'last_loss': e2e_loss},
            'gpu': gpu_identity(local), 'gpu_launches': launches, 'clocks': clocks,
            'step_tensor_roofline': {'achieved_tflops': round(flop_per_sample * value / 1e12, 2), 'peak_tflops': pk['bf16_tflops_sustained'],
                                     'frac': round(flop_per_sample * value / 1e12 / pk['bf16_tflops_sustained'], 4), 'of': how},
            'roofline': roof,
        }
        if not args.no_cpu_baseline and world == 1:
            line['cpu_baseline'] = cpu_baseline_subprocess()
        print(json.dumps(line), flush=True)
    if world > 1:
        torch.cuda.synchronize()
        dist.barrier()
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)   # skip process-group teardown: destroying a communicator that a live CUDA graph captured can block


def graph_timed_roofline(prof, torch, _lib, replays=5):
    """The dominant kernel's launches of ONE step (every C-ABI call of its entry points, original order and operands) captured into a
    dedicated CUDA graph and timed with CUDA events: per-launch device time without the host launch path that eager per-call events
    include. achieved = algorithmic FLOPs (or bytes) of those launches / that time. `roof_frac` compares with the BINDING roofline
    of each launch — max(FLOPs / tensor peak, algorithmic bytes / HBM peak) — because the same kernel serves tensor-bound GPT GEMMs
    and HBM-bound 72..576-channel 1x1 convs."""
    pk, how = peaks()
    names = set(prof.top_entry_points)
    calls = [(n, a) for n, a in prof.calls if n in names]
    call = _lib.lib().call
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for n, a in calls:
            call(n, *a)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for n, a in calls:
            call(n, *a)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / replays
    work = [_lib.Profiler._work(n, a) for n, a in calls]
    fl, by = sum(w[0] for w in work), sum(w[1] for w in work)
    ideal_ms = sum(max(w[0] / (pk['bf16_tflops_sustained'] * 1e12), w[1] / (pk['hbm_gbs'] * 1e9)) for w in work) * 1e3
    out = {'timing': 'dedicated CUDA graph of the %d launches of one step (CUDA events, %d replays)' % (len(calls), replays),
           'launches': len(calls), 'avg_ms': round(ms / len(calls), 5), 'kernel_ms_per_step': round(ms, 3)}
    if fl > 0:
        ach = fl / (ms * 1e-3) / 1e12
        out.update(bound='tensor', achieved=round(ach, 3), peak=pk['bf16_tflops_sustained'], unit='TFLOP/s', frac=round(ach / pk['bf16_tflops_sustained'], 5))
    else:
        ach = by / (ms * 1e-3) / 1e9
        out.update(bound='hbm', achieved=round(ach, 3), peak=pk['hbm_gbs'], unit='GB/s', frac=round(ach / pk['hbm_gbs'], 5))
    out['roof_frac'] = round(ideal_ms / ms, 5)        # time at the binding roofline of every launch / measured time
    # the large tensor-bound launches on their own (>= 10 GFLOP: the C = 1512 GPT GEMMs)
    big = [(n, a, w) for (n, a), w in zip(calls, work) if w[0] >= 1e10]
    if len(big) >= 4:
        gb = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gb):
            for n, a, _ in big:
                call(n, *a)
        gb.replay()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(replays):
            gb.replay()
        e1.record()
        torch.cuda.synchronize()
        msb = e0.elapsed_time(e1) / replays
        achb = sum(w[0] for _, _, w in big) / (msb * 1e-3) / 1e12
        out['large_launches'] = {'what': 'launches with >= 10 GFLOP (the C = 1512 GPT GEMMs)', 'launches': len(big), 'ms_per_step': round(msb, 3),
                                 'achieved': round(achb, 2), 'unit': 'TFLOP/s', 'frac': round(achb / pk['bf16_tflops_sustained'], 4)}
    return out


def dump_outputs(out_dir, tr, loss, torch, np, n_sample=1 << 20):
    """Writes what the last timed step computed, as a caller of Trainer.step receives it: the weighted total loss, the 11 loss
    terms, and the parameters and gradients the step left in the flat buffers (the same seeded sample of n_sample elements of
    each; 8 MB in all). float64 for the losses, float32 for the rest."""
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    np.save(os.path.join(out_dir, 'loss_total.npy'), np.array([float(loss.detach())], dtype=np.float64))
    for k, v in tr.last_losses.items():
        np.save(os.path.join(out_dir, '%s.npy' % k), np.array([float(v)], dtype=np.float64))
    total = tr.flat.total
    idx = np.unique(np.random.default_rng(0).integers(0, total, size=min(n_sample, total)))
    it = torch.from_numpy(idx).to(tr.flat.flat.device)
    np.save(os.path.join(out_dir, 'params_sample.npy'), tr.flat.flat[it].float().cpu().numpy())
    np.save(os.path.join(out_dir, 'grads_sample.npy'), tr.flat.grad[it].float().cpu().numpy())


def effective_cores():
    """Host cores this process may really use: CPU affinity capped by the cgroup CPU quota (a container can see 128 logical
    CPUs while being throttled to a handful — spinning 128 OpenMP threads there is orders of magnitude slower)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, 'sched_getaffinity') else (os.cpu_count() or 1)
    try:
        q, p = open('/sys/fs/cgroup/cpu.max').read().split()
        if q != 'max':
            n = min(n, max(1, int(float(q) / float(p))))
    except Exception:
        pass
    return max(1, n)


def cpu_reference(steps, warmup, batch, budget_s=150.0):
    """The reference's CPU PyTorch path (oracle port: oracle/torch_oracle.py, pinned to the verbatim reference) —
    forward + backward + torch.optim.AdamW on the host cores, bounded sample of the same workload (stops early when the
    time budget is used up; at least one timed step)."""
    import torch
    from oracle import torch_oracle as O
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    cores = effective_cores()
    threads = min(cores, 32)
    torch.set_num_threads(threads)
    t_start = time.time()
    with torch.device('meta'):   # names / shapes only; values come from the seeded generator below
        net = LidarCenterNet(TrainConfig(), 'meta', 'transFuser', 'regnety_032', 'regnety_032', use_velocity=False)
    names = [(k, tuple(v.shape)) for k, v in net.state_dict().items()]
    P = {k: v.requires_grad_(v.dtype.is_floating_point and 'running' not in k and 'num_batches' not in k)
         for k, v in O.deterministic_state(names, seed=3).items()}
    params = [v for v in P.values() if v.requires_grad]
    opt = torch.optim.AdamW(params, lr=1e-4)
    batch_d = O.synthetic_batch(batch, seed=7)
    drop = lambda t, p: torch.nn.functional.dropout(t, p, True)
    cfg = TrainConfig()
    w = dict(zip(cfg.detailed_losses, cfg.detailed_losses_weights))

    def one():
        opt.zero_grad(set_to_none=True)
        losses = O.forward(P, batch_d, O.Cfg, train=True, drop=drop)
        sum(w[k] * v for k, v in losses.items()).backward()
        opt.step()

    for _ in range(warmup):
        if time.time() - t_start < budget_s * 0.4:
            one()
    done, t0 = 0, time.time()
    while done < steps and (done == 0 or time.time() - t_start < budget_s):
        one()
        done += 1
    dt = time.time() - t0
    return {'value': round(batch * done / dt, 4), 'unit': 'samples/s', 'cores': threads, 'host_cores_visible': os.cpu_count(),
            'host_cores_usable': cores, 'kind': 'port', 'ms_per_step': round(dt / done * 1e3, 1),
            'sample': '%d step(s) of batch %d (fwd+bwd+AdamW, fp32, %d torch threads)' % (done, batch, threads)}


def cpu_baseline_subprocess(timeout_s=300):
    """Runs cpu_reference() in a child process (own OpenMP pool, hard timeout) so the GPU line is printed no matter what."""
    try:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), '--impl', 'cpu_baseline'], capture_output=True, text=True, timeout=timeout_s)
        for ln in reversed(r.stdout.strip().splitlines()):
            if ln.startswith('{'):
                return json.loads(ln)
        return {'value': None, 'error': (r.stderr or 'no output')[-300:]}
    except subprocess.TimeoutExpired:
        return {'value': None, 'error': 'cpu baseline exceeded %d s' % timeout_s}


def run_reference(args):
    rank = int(os.environ.get('RANK', 0))
    if rank != 0:
        return
    steps = max(1, min(args.steps, 3))
    warm = 1 if args.warmup > 0 else 0
    cb = cpu_reference(steps=steps, warmup=warm, batch=2)
    line = {'impl': 'reference', 'metric': METRIC, 'value': cb['value'], 'unit': 'samples/s', 'n_gpus': int(os.environ.get('WORLD_SIZE', args.gpus)),
            'steps': steps, 'warmup': warm, 'ms_per_step': cb['ms_per_step'], 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
            'dtype': 'fp32', 'data': 'synthetic',
            'config': {'workload': 'TransFuser RegNetY-3.2GF LidarCenterNet full train step (fwd+bwd+AdamW) on the host CPU, bounded sample: batch 2'},
            'cpu_baseline': cb, 'e2e': {'value': cb['value'], 'unit': 'samples/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--config', type=int, default=2, choices=sorted(CONFIGS), help='BASELINE.json configs[] entry (1-based): 2 = TransFuser batch 10 '
                    '(the headline), 3 = TransFuser batch 12, 4 = GeometricFusion batch 12, 5 = LateFusion batch 16')
    ap.add_argument('--batch', type=int, default=0, help='samples per GPU (default: the batch of --config; configs[1]: 10)')
    ap.add_argument('--impl', default='b200', choices=['b200', 'reference', 'cpu_baseline'])
    ap.add_argument('--gemm', default=os.environ.get('TFB_GEMM', 'bf16'), choices=['simt', 'bf16', 'bf16x3', 'bf16x6'],
                    help="bf16: wgmma bf16 operands (the benched mode); bf16x6 / bf16x3: the tensor-core parity modes (fp32 operands as three / two bf16 terms, six / three "
                         "wgmma products per fp32 product); simt: exact fp32 on the CUDA cores")
    ap.add_argument('--no-cpu-baseline', action='store_true')
    ap.add_argument('--raw-inputs', type=int, default=int(os.environ.get('TFB_RAW_INPUTS', '1')),
                    help='1: feed the step with what is on disk (uint8 frames, raw points, pose transform; 1.6 MB per sample over PCIe) and '
                         'build the model inputs on the GPU inside the step; 0: the expanded fp32 / int64 tensors of the reference DataLoader (3.8 MB)')
    ap.add_argument('--graph', type=int, default=1, help='1: capture the whole step (incl. the NCCL gradient all-reduce when N > 1) in a CUDA graph; 0: eager')
    ap.add_argument('--dump-outputs', default=None, metavar='DIR', help='write the losses, parameters and gradients of the last timed step to DIR/<name>.npy')
    args = ap.parse_args()
    if args.impl == 'cpu_baseline':
        print(json.dumps(cpu_reference(steps=2, warmup=0, batch=1, budget_s=120.0)), flush=True)
    elif args.impl == 'reference':
        run_reference(args)
    else:
        run_b200(args)


if __name__ == '__main__':
    main()
