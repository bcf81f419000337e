"""ORACLE / TEST INFRASTRUCTURE ONLY — never imported by the product path.

numpy restatement of the per-sample input preparation of the reference's dataset class (CARLA_Data.__getitem__,
team_code_transfuser/data.py:103-356) for the pieces SURVEY.md §8f rank 2 moves to the GPU:
  align                 data.py:411-443   (+ utils.py:14-27 transforms)
  draw_target_point     data.py:616-630   (cv2.circle radius 5 thickness 3: restated as a 15x15 stamp, see STAMP below)
  crop_image_cv2        data.py:536-551,  crop_seg data.py:561-576, get_depth data.py:358-372, converter LUT data.py:235
  normalize_imagenet    transfuser.py:419-428
Pinned in tests/test_pipeline.py against the reference's own functions (exec'd from data.py with the real OpenCV) in the
build container, and through tests/golden/pipeline_golden.npz anywhere."""
import numpy as np

# cv2.circle(img, c, radius=5, color, thickness=3) as rasterised by OpenCV (4.13 in this image): rows c.y-7 .. c.y+7, bit j of
# a row = column c.x-7+j. Checked for translation invariance and plain border clipping over all 257 x 257 clipped centres
# (oracle/make_golden.py stamp); the CUDA kernel carries the same table.
STAMP = (992, 4088, 8188, 16382, 16382, 32319, 31775, 31775, 31775, 32319, 16382, 16382, 8188, 4088, 992)


def lidar_to_vehicle():
    T = np.eye(4)
    T[:3, :3] = np.array([[0, 1, 0], [-1, 0, 0], [0, 0, 1]], dtype=np.float32)
    T[0, 3], T[1, 3], T[2, 3] = 1.3, 0.0, 2.5
    return T


def align_transform(ego_matrix_0, ego_matrix_1, degree=0):
    """The 4x4 float64 matrix align() builds (data.py:413-431): frame-0 LiDAR -> frame-1 LiDAR, then the augmentation yaw."""
    m0, m1 = np.array(ego_matrix_0), np.array(ego_matrix_1)
    l2v = lidar_to_vehicle()
    T = np.linalg.inv(l2v) @ np.linalg.inv(m1) @ m0 @ l2v
    rad = np.deg2rad(degree)
    R = np.array([[np.cos(rad), np.sin(rad), 0, 0], [-np.sin(rad), np.cos(rad), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    return R @ T


def align_points(points, T):
    """data.py:432-441: homogeneous transform with the CARLA y flip before and after; intensity column restored."""
    p = points.copy()
    p[:, -1] = 1.
    p[:, 1] *= -1.
    p = (T @ p.T).T
    p[:, -1] = points[:, -1]
    p[:, 1] *= -1.
    return p


def draw_target_point(target_point):
    tp = np.array(target_point, dtype=np.float64).copy()
    tp[1] += 1.3
    pt = tp * 8.
    pt[1] *= -1
    pt[1] = 256 - pt[1]
    pt[0] += 128
    with np.errstate(invalid='ignore'):
        pt = np.clip(pt.astype(np.int32), 0, 256)
    img = np.zeros((256 + 16, 256 + 16), dtype=np.float64)
    rows = np.array([[(r >> j) & 1 for j in range(15)] for r in STAMP], dtype=np.float64)
    img[pt[1] + 8 - 7:pt[1] + 8 + 8, pt[0] + 8 - 7:pt[0] + 8 + 8] = rows
    return img[8:264, 8:264].reshape(1, 256, 256)


def crop_origin(H, W, crop, crop_shift):
    ch, cw = crop
    return H // 2 - ch // 2, W // 2 - cw // 2 + int(crop_shift)


def crop_rgb(image_hwc, crop, crop_shift=0):
    y0, x0 = crop_origin(image_hwc.shape[0], image_hwc.shape[1], crop, crop_shift)
    return np.transpose(image_hwc[y0:y0 + crop[0], x0:x0 + crop[1]], (2, 0, 1))


def depth_from_rgb(depth_chw):
    d = np.transpose(depth_chw, (1, 2, 0)).astype(np.float32)
    n = d[..., 0].astype(np.float64) * 65536.0 + d[..., 1].astype(np.float64) * 256.0 + d[..., 2].astype(np.float64)
    n = n / (256 * 256 * 256 - 1)
    return np.clip(n, 0.0, 0.05) * 20.0


def seg_classes(seg_hw, converter, crop, crop_shift=0):
    y0, x0 = crop_origin(seg_hw.shape[0], seg_hw.shape[1], crop, crop_shift)
    return np.uint8(converter)[seg_hw[y0:y0 + crop[0], x0:x0 + crop[1]]]


def normalize_nhwc(rgb_chw_float32):
    """normalize_imagenet (transfuser.py:419-428) in float32, then CHW -> HWC."""
    x = rgb_chw_float32.astype(np.float32)
    mean = np.array([0.485, 0.456, 0.406], dtype=np.float32).reshape(3, 1, 1)
    std = np.array([0.229, 0.224, 0.225], dtype=np.float32).reshape(3, 1, 1)
    return np.transpose(((x / np.float32(255.0)) - mean) / std, (1, 2, 0))


def synthetic_frame(seed, H=160, W=960, n_points=3000):
    """Seeded raw inputs of one sample in the reference's on-disk shapes / dtypes (after its scale step)."""
    rng = np.random.default_rng(seed)
    yaw0, yaw1 = rng.uniform(-np.pi, np.pi), rng.uniform(-0.2, 0.2)

    def pose(yaw, x, y):
        c, s = np.cos(yaw), np.sin(yaw)
        return [[c, -s, 0, x], [s, c, 0, y], [0, 0, 1, 0.03], [0, 0, 0, 1]]
    x, y = rng.uniform(-200, 200, 2)
    pts = np.concatenate([rng.uniform(-20, 36, (n_points, 1)), rng.uniform(-20, 20, (n_points, 1)), rng.uniform(-3.5, 1.0, (n_points, 1)),
                          rng.uniform(0, 1, (n_points, 1))], axis=1).astype(np.float32)
    return dict(
        rgb=rng.integers(0, 256, (H, W, 3), dtype=np.uint8), depth=rng.integers(0, 256, (H, W, 3), dtype=np.uint8),
        seg=rng.integers(0, 23, (H, W), dtype=np.uint8), points=pts,
        ego_matrix_0=pose(yaw0, x, y), ego_matrix_1=pose(yaw0 + yaw1, x + rng.uniform(-2, 2), y + rng.uniform(-2, 2)),
        degree=float(rng.uniform(-20, 20)), target_point=rng.uniform(-30, 30, 2))
