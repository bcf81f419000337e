"""GPU drop-in for `lidar_to_histogram_features` (team_code_transfuser/data.py:446-470).

Same name, same argument meaning (an (N, >=4) point array: x, y, z, intensity) and same result
((2, 256, 256) float32, channel 0 = above, channel 1 = below), computed by the sm_90a kernel in csrc/bev_hist.cu."""
import numpy as np
import torch

from . import _lib


def lidar_to_histogram_features_batched(points, n_valid=None):
    """points: CUDA tensor [B, N, 4] float32/float64 (padded), n_valid: optional CUDA int32 [B] -> CUDA [B, 2, 256, 256] float32."""
    if not points.is_cuda:
        raise RuntimeError('points must be a CUDA tensor (no CPU fallback)')
    if points.dim() != 3 or points.shape[2] != 4 or points.dtype not in (torch.float32, torch.float64):
        raise ValueError('points must be [B, N, 4] float32/float64')
    points = points.contiguous()
    b, n = points.shape[0], points.shape[1]
    counts = torch.empty((b, 2, 256, 256), dtype=torch.int32, device=points.device)
    out = torch.empty((b, 2, 256, 256), dtype=torch.float32, device=points.device)
    if n_valid is not None:
        n_valid = n_valid.to(device=points.device, dtype=torch.int32).contiguous()
    _lib.call('tfb_bev_histogram', points, 1 if points.dtype == torch.float64 else 0, n_valid, b, n, counts, out)
    return out


def lidar_to_histogram_features(lidar, device='cuda'):
    """Reference-shaped call: one (N, >=4) numpy / torch point cloud -> (2,256,256) float32 numpy array (data.py:446)."""
    is_np = isinstance(lidar, np.ndarray)
    t = torch.as_tensor(lidar)
    if t.dtype not in (torch.float32, torch.float64):
        t = t.to(torch.float64)
    t = t[:, :4].contiguous() if t.shape[1] >= 4 else torch.nn.functional.pad(t, (0, 4 - t.shape[1]))
    out = lidar_to_histogram_features_batched(t.to(device).unsqueeze(0))[0]
    return out.cpu().numpy() if is_np else out
