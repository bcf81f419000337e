"""ORACLE SHIM — scikit-image 0.16.2's `rotate` / `warp` (the reference's pin) restated for what data.py uses: bilinear
interpolation (order 1), mode 'constant' with cval 0, clip=True, output shape = input shape, 2-D or 3-D float images.

- `rotation_matrix` composes translate(-centre) -> rotate -> translate(centre) the way `rotate` adds its SimilarityTransforms
  (tform3 + tform2 + tform1 = T1 . (R . T3)), each 3x3 product in scalar float64 as ((a0*b0 + a1*b1) + a2*b2). That equals skimage
  on a BLAS whose dgemm does not fuse multiply-adds; a BLAS that does may differ in the last bit of the matrix.
- `warp` is _warp_fast per channel in float64: (c', r') = ((M0*C + M1*R) + M2, (M3*C + M4*R) + M5), then
  bilinear_interpolation (floor / ceil taps, get_pixel2d in constant mode), then _clip_warp_output (clip to the input's
  [min, max], keeping cval pixels when cval lies outside that range). numpy applies every operation on its own, without FMA.
Parity against scikit-image itself is not pinned here (it is not installed); tests/test_dataset_reader.py checks this restatement
against scipy.ndimage.affine_transform and the fixture pins the reference's load_crop_bev_npy through it."""
import math

import numpy as np


def _mat3(a, b):
    return [[(a[i][0] * b[0][j] + a[i][1] * b[1][j]) + a[i][2] * b[2][j] for j in range(3)] for i in range(3)]


def _similarity(rotation=0.0, translation=(0.0, 0.0)):
    # SimilarityTransform(rotation=..., translation=...).params with scale 1
    return [[math.cos(rotation), -math.sin(rotation), float(translation[0])],
            [math.sin(rotation), math.cos(rotation), float(translation[1])],
            [0.0, 0.0, 1.0]]


def rotation_matrix(angle, rows, cols):
    """3x3 float64 output -> input matrix of rotate(image of shape (rows, cols, ...), angle) about the image centre."""
    cx, cy = cols / 2. - 0.5, rows / 2. - 0.5
    rad = angle * (math.pi / 180)           # np.deg2rad
    t1 = _similarity(translation=(cx, cy))
    t2 = _similarity(rotation=rad)
    t3 = _similarity(translation=(-cx, -cy))
    return np.array(_mat3(t1, _mat3(t2, t3)), dtype=np.float64)


def _warp_channel(img, M):
    rows, cols = img.shape
    R, C = np.meshgrid(np.arange(rows, dtype=np.float64), np.arange(cols, dtype=np.float64), indexing='ij')
    if not (M[2, 0] == 0 and M[2, 1] == 0 and M[2, 2] == 1):
        raise NotImplementedError('projective matrices are not used by the reference')
    c = (M[0, 0] * C + M[0, 1] * R) + M[0, 2]
    r = (M[1, 0] * C + M[1, 1] * R) + M[1, 2]
    minr, minc = np.floor(r), np.floor(c)
    maxr, maxc = np.ceil(r), np.ceil(c)
    dr, dc = r - minr, c - minc

    def px(rr, cc):
        ok = (rr >= 0) & (rr < rows) & (cc >= 0) & (cc < cols)
        ri = np.where(ok, rr, 0).astype(np.int64)
        ci = np.where(ok, cc, 0).astype(np.int64)
        return np.where(ok, img[ri, ci], 0.0)

    top = (1 - dc) * px(minr, minc) + dc * px(minr, maxc)
    bottom = (1 - dc) * px(maxr, minc) + dc * px(maxr, maxc)
    return (1 - dr) * top + dr * bottom


def warp(image, matrix, cval=0.0):
    img = np.asarray(image, dtype=np.float64)
    M = np.asarray(matrix, dtype=np.float64)
    if img.ndim == 2:
        out = _warp_channel(img, M)
    else:
        out = np.dstack([_warp_channel(np.ascontiguousarray(img[..., d]), M) for d in range(img.shape[2])])
    lo, hi = np.asarray(image).min(), np.asarray(image).max()
    keep = None if lo <= cval <= hi else (out == cval)
    np.clip(out, lo, hi, out=out)
    if keep is not None:
        out[keep] = cval
    return out


def rotate(image, angle, resize=False, center=None, order=1, mode='constant', cval=0, clip=True, preserve_range=False):
    if resize or center is not None or order != 1 or mode != 'constant' or not clip:
        raise NotImplementedError('the shim covers rotate(image, angle) as data.py calls it')
    image = np.asarray(image)
    if image.dtype.kind != 'f':
        raise NotImplementedError('the shim covers float images (data.py passes float32)')
    return warp(image, rotation_matrix(angle, image.shape[0], image.shape[1]), cval=float(cval))
