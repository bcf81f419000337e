"""One data-parallel training step of the hot path — BEV histogram, LidarCenterNet forward, weighted loss sum, backward,
gradient all-reduce, fused AdamW — as a reusable object, optionally captured into ONE CUDA graph and replayed.

This is the body of the reference's `Engine.train()` loop (train.py:304-316) with the synchronising `.item()` calls moved
out of the step; bench.py and the tests drive it. `Validator` is the reference's `Engine.validate()` / `log_losses`
(train.py:321-379): the eval-mode forward and its loss bookkeeping, also as one CUDA graph."""
import torch
import torch.distributed as dist

from . import _lib, bev, gemm, ops, optim
from .model import LidarCenterNet

import os

OVERLAP_ADAMW = os.environ.get('TFB_OVERLAP_ADAMW', '1') == '1'   # AdamW per gradient span from inside backward (captured step only)

INPUT_KEYS = ('rgb', 'points', 'target_point_image', 'target_point', 'ego_vel', 'ego_waypoint', 'bev', 'semantic', 'depth', 'label')
# raw_inputs=True: what is on disk instead of the expanded tensors (uint8 frames, raw points, one pose transform, the target point);
# the GPU input pipeline (pipeline.InputPipeline, csrc/input_prep.cu) builds the model inputs inside the step — 1.6 MB instead of
# 3.8 MB per sample over PCIe
RAW_KEYS = ('rgb_u8', 'depth_u8', 'seg_u8', 'crop_shift', 'points', 'transforms', 'target_point64', 'ego_vel', 'ego_waypoint', 'bev', 'label')
# raw_inputs='dataset': the batches of dataset.CarlaRawDataset / dataset.collate — the raw inputs with the sweep's point count and, in
# place of the finished BEV label, the topdown plane and the augmentation's rotation matrix (rotated inside the step, csrc/bev_label.cu)
DATASET_KEYS = tuple(k for k in RAW_KEYS if k != 'bev') + ('n_valid', 'bev_u8', 'bev_matrix')


class Trainer:
    def __init__(self, cfg, device, gemm_mode='bf16', lr=1e-4, seed=0, n_chunks=int(os.environ.get('TFB_GRAD_CHUNKS', '8')), backbone='transFuser',
                 raw_inputs=False, image_architecture='regnety_032', lidar_architecture='regnety_032', use_velocity=False,
                 sync_batch_norm=False):
        """sync_batch_norm: every BatchNorm normalises with the statistics of the global batch (train.py --sync_batch_norm 1): the model
        is converted with nn.SyncBatchNorm.convert_sync_batchnorm and each trunk's BatchNorms get a process group of their own, apart
        from the gradient all-reduce's, so one trunk's statistics never queue behind the other trunk's or behind the gradients. Needs an
        initialised default process group (world size 1 included)."""
        self.cfg, self.device = cfg, device
        self.raw_inputs = raw_inputs
        if raw_inputs not in (False, True, 'dataset'):
            raise ValueError("raw_inputs must be False, True or 'dataset'")
        # the geometric-fusion backbone consumes two more inputs per sample, the LiDAR <-> camera correspondences
        # (train.py:279-288); in dataset mode they are built inside the step from the sweep and a per-sample seed (csrc/correspondences.cu)
        geo = backbone == 'geometric_fusion'
        self.input_keys = (DATASET_KEYS + (('corr_seed',) if geo else ()) if raw_inputs == 'dataset' else
                           (RAW_KEYS if raw_inputs else INPUT_KEYS) + (('bev_points', 'cam_points') if geo else ()))
        if raw_inputs:
            from .pipeline import InputPipeline
            self.pipe = InputPipeline(cfg, device)
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        gemm.set_mode(gemm_mode)
        ops.manual_seed(1234 + seed)
        self.net = LidarCenterNet(cfg, device, backbone, image_architecture, lidar_architecture, use_velocity=use_velocity).train()
        if sync_batch_norm:
            if not dist.is_initialized():
                raise RuntimeError('sync_batch_norm=True needs an initialised process group (torch.distributed.init_process_group)')
            self.net = torch.nn.SyncBatchNorm.convert_sync_batchnorm(self.net)
            # new_group is collective: every rank creates both groups here, before any step is captured
            groups = {'image': dist.new_group(), 'lidar': dist.new_group()}
            for name, m in self.net.named_modules():
                if isinstance(m, torch.nn.SyncBatchNorm):
                    m.process_group = groups['lidar' if 'lidar_encoder' in name else 'image']
        self.flat = optim.flatten(self.net)
        if self.world > 1:
            # replicas start identical whatever the caller's RNG state: rank 0's parameters and buffers win (DDP does the same at
            # construction, train.py:134)
            dist.broadcast(self.flat.flat, 0)
            for buf in self.net.buffers():
                if buf.is_floating_point() or buf.dtype == torch.int64:
                    dist.broadcast(buf, 0)
        if gemm_mode == 'bf16':
            gemm.attach_bf16_weights(self.flat)
        self.opt = optim.FusedAdamW(self.net.parameters(), lr=lr, grad_scale=1.0 / self.world)
        self.reducer = optim.GradAllReducer(self.flat, n_chunks=n_chunks, opt=self.opt if OVERLAP_ADAMW else None)
        self.weights = dict(zip(cfg.detailed_losses, cfg.detailed_losses_weights))
        self.graph = None
        self.static = None
        self.static_loss = None
        self.graph_launches = 0
        self.graph_error = None
        self._stream = None

    def step(self, d):
        """Eager step on device-resident inputs `d` (dict with INPUT_KEYS). Returns the weighted total loss (0-dim tensor).

        Never runs on the legacy default stream: autograd pins every parameter's AccumulateGrad node to the stream of its first
        backward, the gradient hooks keep those nodes alive, and a later CUDA-graph capture cannot fork the legacy stream
        (cudaErrorStreamCaptureImplicit — the round-1 "AccumulateGrad node's stream does not match" warning, fatal once the hooks
        also drive the pipelined AdamW). When called on the default stream the step runs on a stream of the trainer's own, ordered
        after the caller's work, and the caller's stream is ordered after the step."""
        dev = self.device
        if torch.device(dev).type == 'cuda' and not torch.cuda.is_current_stream_capturing():
            cur = torch.cuda.current_stream(dev)
            if cur == torch.cuda.default_stream(dev):
                if self._stream is None:
                    self._stream = torch.cuda.Stream(device=dev)
                own = self._stream
                own.wait_stream(cur)
                for t in d.values():
                    if isinstance(t, torch.Tensor) and t.is_cuda:
                        t.record_stream(own)
                with torch.cuda.stream(own):
                    loss = self._step(d)
                cur.wait_stream(own)
                loss.record_stream(cur)
                return loss
        return self._step(d)

    def expand_inputs(self, d):
        """(model inputs, LiDAR BEV) from a batch of `input_keys`: the GPU input pipeline on raw batches, the BEV histogram else."""
        if self.raw_inputs:
            # crop + CHW / normalise, depth decode, class LUT, align + BEV histogram, target-point map: three launches on the raw batch
            raw = dict(rgb=d['rgb_u8'], depth=d['depth_u8'], seg=d['seg_u8'], crop_shift=d['crop_shift'], points=d['points'],
                       transforms=d['transforms'], target_point=d['target_point64'])
            if self.raw_inputs == 'dataset':
                raw.update(n_valid=d['n_valid'], bev_u8=d['bev_u8'], bev_matrix=d['bev_matrix'])   # + the BEV-label rotation
                if 'corr_seed' in d:
                    raw['corr_seed'] = d['corr_seed']                                                # + the correspondences
            p = self.pipe.prepare(raw, normalized_nhwc=True)
            d = dict(d, rgb=p['rgb'], depth=p['depth'], semantic=p['semantic'], target_point=p['target_point'],
                     target_point_image=p['target_point_image'], bev=p.get('bev', d.get('bev')),
                     bev_points=p.get('bev_points', d.get('bev_points')), cam_points=p.get('cam_points', d.get('cam_points')))
            lidar = p['lidar']
        else:
            lidar = bev.lidar_to_histogram_features_batched(d['points'])
        return d, lidar

    def _step(self, d):
        d, lidar = self.expand_inputs(d)
        self.opt.zero_grad()
        if self.reducer.pipeline:
            self.opt.begin_step()        # AdamW spans are launched from the backward pass (optim.FusedAdamW.step_span)
        losses = self.forward_losses(d, lidar)
        self.last_losses = losses          # the 11 scalars of this step (device tensors; static buffers under graph replay)
        loss = None
        for k, v in losses.items():
            loss = v * self.weights[k] if loss is None else loss + v * self.weights[k]
        loss.backward()
        self.opt.step(chunks=self.reducer.chunks())
        if not self.reducer.replanned and self.graph is None and not torch.cuda.is_current_stream_capturing():
            self.reducer.replan()       # once, after the first backward pass showed the order in which gradients complete
        return loss

    def forward_losses(self, d, lidar):
        """The model's 11 losses (dict in the model's order) on the expanded inputs."""
        return self.net(d['rgb'], lidar, ego_waypoint=d['ego_waypoint'], target_point=d['target_point'],
                        target_point_image=d['target_point_image'], ego_vel=d['ego_vel'], bev=d['bev'], label=d['label'],
                        depth=d['depth'], semantic=d['semantic'], bev_points=d.get('bev_points'), cam_points=d.get('cam_points'))

    def capture(self, example):
        """Captures step() into a CUDA graph over static input buffers shaped like `example` (host or device tensors).
        The dropout base seed and the optimizer step count live in device memory and are advanced by kernels inside the graph,
        so every replay is a genuinely new step. Returns True on success (falls back to eager otherwise)."""
        try:
            self.static = {k: torch.empty(example[k].shape, dtype=example[k].dtype, device=self.device) for k in self.input_keys}
            self.load(example)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    self.step(self.static)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            self.opt.check_grads = False
            self.reducer.pipeline = OVERLAP_ADAMW    # every gradient is known to land in the flat buffer: update spans as they complete
            g = torch.cuda.CUDAGraph()
            l0 = _lib.lib().launches
            with torch.cuda.graph(g):
                self.static_loss = self.step(self.static)
            self.graph, self.graph_launches = g, _lib.lib().launches - l0
            return True
        except Exception as e:  # noqa: BLE001 — keep the eager path, report why
            import traceback
            self.graph, self.graph_error = None, repr(e)[:300]
            self.graph_traceback = traceback.format_exc()
            if os.environ.get('TFB_CAPTURE_DEBUG') == '1':
                print(self.graph_traceback, flush=True)
            torch.cuda.synchronize()
            return False

    def load(self, batch):
        """Copies a batch (pinned host or device tensors) into the static input buffers of the captured graph."""
        for k in self.input_keys:
            self.static[k].copy_(batch[k], non_blocking=True)

    def replay(self):
        self.opt.sync_hparams()       # lr / weight-decay edits of param_groups reach the captured AdamW kernel through device scalars
        self.graph.replay()
        ops.invalidate_packs()        # the replayed optimizer kernel changed the weights behind Python's back
        return self.static_loss


def average_over_ranks(means):
    """The per-rank means (CPU fp64 tensor) averaged over the ranks of the process group, as log_losses averages the gathered rank
    means (train.py:344-379): a SUM all-reduce divided by the world size. Without a process group (or with one rank) the means."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return means
    world = dist.get_world_size()
    t = means.to('cuda') if dist.get_backend() == 'nccl' else means.clone()
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t.cpu() / world


class Validator:
    """Validation of a Trainer's network: the eval-mode forward and the 11 losses of each batch, accumulated on the device as
    Engine.validate does (train.py:321-342) by tfb_val_accumulate, so a batch needs no host read-back; finish() reads the sums once.

        val = Validator(tr); val.capture(example)
        for batch in loader: val.load(batch); val.replay()      # (a batch of another size: val.step(batch))
        means = val.finish()                                    # {'loss_total', 'loss_wp', ...}, averaged over ranks; resets

    It shares the trainer's network, loss weights, input mode and input pipeline, and touches no training state: no tick(), no
    dropout seed, no running statistics, no optimizer."""

    def __init__(self, trainer):
        self.tr = trainer
        self.device = trainer.device
        self.acc = None
        self.order = None                  # the model's loss-dict order, fixed by the first forward
        self.graph = None
        self.static = None
        self.graph_launches = 0

    def _losses(self, d):
        """The eval-mode forward of batch d (input_keys) under no_grad: the packed conv weights are refreshed first by ONE batched
        re-pack launch (the weights may have changed since the last validation), then the model's losses."""
        net = self.tr.net
        was = net.training
        net.eval()
        try:
            with torch.no_grad():
                ops._prepack_all(self.device)
                d, lidar = self.tr.expand_inputs(d)
                return self.tr.forward_losses(d, lidar)
        finally:
            net.train(was)

    def _accumulate(self, losses, table):
        if self.order is None:
            self.order = list(losses)
            self.w32 = torch.tensor([self.tr.weights[k] for k in self.order], dtype=torch.float32, device=self.device)
            self.acc = torch.zeros(len(self.order) + 2, dtype=torch.float64, device=self.device)
        if list(losses) != self.order:
            raise RuntimeError('the model returned its losses in another order')
        if table is None:
            table = torch.tensor([losses[k].data_ptr() for k in self.order], dtype=torch.int64).to(self.device)
        _lib.call('tfb_val_accumulate', table, self.w32, len(self.order), self.acc)

    def step(self, batch):
        """One validation batch, eagerly (any batch size); batch tensors on the host or the device."""
        d = {k: batch[k].to(self.device, non_blocking=True) for k in self.tr.input_keys}
        losses = self._losses(d)
        self._accumulate(losses, None)
        return losses

    def capture(self, example):
        """Captures one validation batch (re-pack, eval forward, losses, accumulation) as ONE CUDA graph over static input buffers
        shaped like `example`. The sums it accumulates during the warm-up are cleared."""
        self.static = {k: torch.empty(example[k].shape, dtype=example[k].dtype, device=self.device) for k in self.tr.input_keys}
        self.load(example)
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(2):             # registers every packed weight and the batched re-pack table, loads the modules
                self.step(self.static)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        table = torch.empty(len(self.order), dtype=torch.int64, device=self.device)
        g = torch.cuda.CUDAGraph()
        l0 = _lib.lib().launches
        with torch.cuda.graph(g):
            self.static_losses = self._losses(self.static)
            self._accumulate(self.static_losses, table)
        self.graph, self.graph_launches = g, _lib.lib().launches - l0
        # the graph's losses live at fixed addresses: the table the captured accumulation reads is written once, after the capture
        table.copy_(torch.tensor([self.static_losses[k].data_ptr() for k in self.order], dtype=torch.int64))
        self._table = table
        self.acc.zero_()
        torch.cuda.synchronize(self.device)
        return True

    def load(self, batch):
        for k in self.tr.input_keys:
            self.static[k].copy_(batch[k], non_blocking=True)

    def replay(self):
        self.graph.replay()
        return self.static_losses

    def finish(self):
        """{'loss_total', 'loss_<name>', ...}: the per-batch means of the validation so far, averaged over the ranks, as log_losses
        logs them. Resets the sums."""
        if self.acc is None:
            raise RuntimeError('no validation batch was run')
        a = self.acc.cpu()
        n = len(self.order)
        if a[n + 1] == 0:
            raise RuntimeError('no validation batch was run')
        means = torch.cat([a[n:n + 1], a[:n]]) / a[n + 1]
        means = average_over_ranks(means)
        self.acc.zero_()
        return dict(zip(['loss_total'] + self.order, means.tolist()))
