"""ORACLE / TEST INFRASTRUCTURE ONLY. Seeded writer of CARLA routes in the on-disk layout the reference's CARLA_Data reads
(data.py:46-85, 103-210): rgb / depth / semantics PNGs, topdown/encoded_*.png, the LiDAR sweep as the reference's pickled
[header, points] .npy, measurements and label_raw JSON. Every JSON float is a multiple of 2^-12 (dyadic), so json and ujson
parse the same double. The content exercises the reader's edge cases:
  - frame 3 lists the ego only (0 boxes); frame 5 has exactly 20 boxes that survive every rotation up to 20 degrees;
  - boxes near the 0..255 BEV-image border that the rotation pushes out, a box always clipped onto the border, a box with
    num_points == 1, vehicles that leave the future label files (identity-padded waypoints);
  - topdown planes with every bit random (rows 493-499 included: the 7-row shift drops them; bits other than 7 and 6 are ignored),
    a frame with solid rectangles, and the other two PNG planes random.

    python -m oracle.synthetic_route OUT_DIR        # the two routes of ROUTES under OUT_DIR"""
import json
import os
import sys

import numpy as np

Q = 2.0 ** -12


def _q(x):
    return np.round(np.asarray(x, dtype=np.float64) / Q) * Q


def _pose(yaw, x, y, z=0.0):
    c, s = _q(np.cos(yaw)), _q(np.sin(yaw))
    return [[float(c), float(-s), 0.0, float(_q(x))], [float(s), float(c), 0.0, float(_q(y))], [0.0, 0.0, 1.0, float(_q(z))], [0.0, 0.0, 0.0, 1.0]]


def _box(rng, vid, x, y, num_points=None):
    return dict(id=int(vid), num_points=int(rng.integers(2, 300) if num_points is None else num_points), distance=float(_q(np.hypot(x, y))),
                position=[float(_q(x)), float(_q(y)), float(_q(rng.uniform(-1, 1)))],
                extent=[float(_q(rng.uniform(0.5, 1.0))), float(_q(rng.uniform(1.5, 3.0))), float(_q(rng.uniform(0.8, 1.2)))],
                yaw=float(_q(rng.uniform(-3, 3))), speed=float(_q(rng.uniform(0, 12))), brake=float(rng.integers(0, 2)),
                ego_matrix=_pose(rng.uniform(-3, 3), rng.uniform(-100, 100), rng.uniform(-100, 100)))


def _labels(rng, f, ego):
    boxes = [dict(ego, id=0, num_points=0, position=[0.0, 0.0, 0.0], distance=0.0)]
    if f == 3:
        return boxes
    safe = 20 if f == 5 else int(rng.integers(1, 8))
    for i in range(safe):                                   # well inside: survive every rotation up to 20 degrees
        boxes.append(_box(rng, 1 + i, rng.uniform(8, 24), rng.uniform(-6, 6)))
    if f == 5:
        boxes.append(_box(rng, 40, 12.0, 1.0, num_points=1))
        boxes.append(_box(rng, 41, 60.0, 0.0))              # clipped onto the border: filtered at every angle
        return boxes
    boxes.append(_box(rng, 30, rng.uniform(0.0, 1.5), rng.uniform(-6, 6)))          # near the bottom edge
    boxes.append(_box(rng, 31, rng.uniform(8, 24), 15.75 + rng.uniform(-0.5, 0.5)))  # near the left / right edges
    boxes.append(_box(rng, 32, rng.uniform(8, 24), -15.75 + rng.uniform(-0.5, 0.5)))
    boxes.append(_box(rng, 33, 31.5 + rng.uniform(-1, 1), rng.uniform(-6, 6)))      # near the top edge
    boxes.append(_box(rng, 34, 12.0, 16.0))                                          # on the border at 0 degrees
    boxes.append(_box(rng, 35, 10.0, 2.0, num_points=1))
    keep = rng.random(len(boxes)) < 0.8                     # some vehicles leave the later label files
    keep[0] = True
    return [b for b, k in zip(boxes, keep) if k]


def write_route(path, seed, frames=14, cam=(160, 960), topdown=(500, 500), n_points=(2000, 3000)):
    import cv2
    rng = np.random.default_rng(seed)
    for sub in ('rgb', 'depth', 'semantics', 'topdown', 'lidar', 'measurements', 'label_raw'):
        os.makedirs(os.path.join(path, sub), exist_ok=True)
    H, W = cam
    x, y, yaw = rng.uniform(-200, 200), rng.uniform(-200, 200), rng.uniform(-np.pi, np.pi)
    for f in range(frames):
        x, y, yaw = x + rng.uniform(0, 2) * np.cos(yaw), y + rng.uniform(0, 2) * np.sin(yaw), yaw + rng.uniform(-0.05, 0.05)
        ego_matrix = _pose(yaw, x, y, 0.03)
        cv2.imwrite(os.path.join(path, 'rgb', '%04d.png' % f), rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        depth = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        depth[..., 2] = rng.integers(0, 13, (H, W), dtype=np.uint8)     # BGR on disk: the high byte of the 24-bit depth code
        cv2.imwrite(os.path.join(path, 'depth', '%04d.png' % f), depth)
        cv2.imwrite(os.path.join(path, 'semantics', '%04d.png' % f), rng.integers(0, 28, (H, W), dtype=np.uint8))
        top = rng.integers(0, 256, topdown + (3,), dtype=np.uint8)
        if f % 4 == 1:                                      # solid rectangles in the BEV bits, noise in the others
            plane = top[..., 0] & 0x3f
            for _ in range(12):
                r0, c0 = rng.integers(0, topdown[0] - 40), rng.integers(0, topdown[1] - 40)
                plane[r0:r0 + rng.integers(5, 40), c0:c0 + rng.integers(5, 40)] |= np.uint8(rng.choice([0x80, 0x40, 0xc0]))
            top[..., 0] = plane                             # cv2 writes BGR: plane 0 on disk is RGB plane 2 after BGR2RGB
        cv2.imwrite(os.path.join(path, 'topdown', 'encoded_%04d.png' % f), top)
        n = int(rng.integers(*n_points))
        pts = np.concatenate([rng.uniform(-20, 36, (n, 1)), rng.uniform(-20, 20, (n, 1)), rng.uniform(-3.5, 1.0, (n, 1)),
                              rng.uniform(0, 1, (n, 1))], axis=1).astype(np.float32)
        np.save(os.path.join(path, 'lidar', '%04d.npy' % f), np.array([f, pts], dtype=object), allow_pickle=True)
        m = dict(x=float(_q(x)), y=float(_q(y)), theta=float(_q(yaw)), speed=float(_q(rng.uniform(0, 10))), steer=float(_q(rng.uniform(-1, 1))),
                 throttle=float(_q(rng.uniform(0, 1))), brake=bool(rng.integers(0, 2)), light_hazard=bool(rng.integers(0, 2)),
                 x_command=float(_q(x + rng.uniform(-40, 40))), y_command=float(_q(y + rng.uniform(-40, 40))), ego_matrix=ego_matrix)
        with open(os.path.join(path, 'measurements', '%04d.json' % f), 'w') as fh:
            json.dump(m, fh)
        ego = _box(rng, 0, 0.0, 0.0)
        ego['ego_matrix'] = ego_matrix
        with open(os.path.join(path, 'label_raw', '%04d.json' % f), 'w') as fh:
            json.dump(_labels(rng, f, ego), fh)


ROUTES = (('route_a', 11, 14), ('route_b', 12, 15))      # (name, seed, frames)


def write_dataset(root, routes=ROUTES, **kw):
    """One dataset root with the given routes, plus a stray file at the root level (not a route: skipped by the index)."""
    os.makedirs(root, exist_ok=True)
    for name, seed, frames in routes:
        write_route(os.path.join(root, name), seed, frames, **kw)
    open(os.path.join(root, 'results.json'), 'w').write('{}')
    return root


if __name__ == '__main__':
    write_dataset(sys.argv[1])
