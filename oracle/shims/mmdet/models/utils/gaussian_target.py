"""ORACLE / TEST INFRASTRUCTURE ONLY. Minimal stand-in for the un-vendored dependency named by the
package path (mmcv-full==1.5.3 / mmdet==2.25.0, environment.yml:27-28); restates only the
symbols imported at team_code_transfuser/model.py:20-30. parity unpinned (source absent)."""
from math import sqrt

import torch
import torch.nn.functional as F


def gaussian2D(radius, sigma=1, dtype=torch.float32, device='cpu'):
    x = torch.arange(-radius, radius + 1, dtype=dtype, device=device).view(1, -1)
    y = torch.arange(-radius, radius + 1, dtype=dtype, device=device).view(-1, 1)
    h = (-(x * x + y * y) / (2 * sigma * sigma)).exp()
    h[h < torch.finfo(h.dtype).eps * h.max()] = 0
    return h


def gen_gaussian_target(heatmap, center, radius, k=1):
    diameter = 2 * radius + 1
    kern = gaussian2D(radius, sigma=diameter / 6, dtype=heatmap.dtype, device=heatmap.device)
    x, y = center
    height, width = heatmap.shape[:2]
    left, right = min(x, radius), min(width - x, radius + 1)
    top, bottom = min(y, radius), min(height - y, radius + 1)
    masked_heatmap = heatmap[y - top:y + bottom, x - left:x + right]
    masked_gaussian = kern[radius - top:radius + bottom, radius - left:radius + right]
    torch.max(masked_heatmap, masked_gaussian * k, out=heatmap[y - top:y + bottom, x - left:x + right])
    return heatmap


def gaussian_radius(det_size, min_overlap):
    """CornerNet radius: min over the three overlap cases (roots of three quadratics)."""
    height, width = det_size
    a1 = 1
    b1 = (height + width)
    c1 = width * height * (1 - min_overlap) / (1 + min_overlap)
    r1 = (b1 - sqrt(b1 ** 2 - 4 * a1 * c1)) / (2 * a1)
    a2 = 4
    b2 = 2 * (height + width)
    c2 = (1 - min_overlap) * width * height
    r2 = (b2 - sqrt(b2 ** 2 - 4 * a2 * c2)) / (2 * a2)
    a3 = 4 * min_overlap
    b3 = -2 * min_overlap * (height + width)
    c3 = (min_overlap - 1) * width * height
    r3 = (b3 + sqrt(b3 ** 2 - 4 * a3 * c3)) / (2 * a3)
    return min(r1, r2, r3)


def get_local_maximum(heat, kernel=3):
    hmax = F.max_pool2d(heat, kernel, stride=1, padding=(kernel - 1) // 2)
    return heat * (hmax == heat).float()


def get_topk_from_heatmap(scores, k=20):
    batch, _, height, width = scores.size()
    topk_scores, topk_inds = torch.topk(scores.view(batch, -1), k)
    topk_clses = topk_inds // (height * width)
    topk_inds = topk_inds % (height * width)
    topk_ys = topk_inds // width
    topk_xs = (topk_inds % width).int().float()
    return topk_scores, topk_inds, topk_clses, topk_ys, topk_xs


def transpose_and_gather_feat(feat, ind):
    feat = feat.permute(0, 2, 3, 1).contiguous()
    feat = feat.view(feat.size(0), -1, feat.size(3))
    dim = feat.size(2)
    ind = ind.unsqueeze(2).repeat(1, 1, dim)
    return feat.gather(1, ind)
