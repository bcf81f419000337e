"""ORACLE / TEST INFRASTRUCTURE ONLY — never imported by the product path.

numpy restatement of the geometric-fusion correspondences, lidar_bev_cam_correspondences (team_code_transfuser/data.py:675-842)
and correspondences_at_one_scale (data.py:632-673), with every floating-point operation spelled out elementwise (numpy ufuncs
round each operation; nothing is fused into an FMA):
  - the filter, the z shift and the BEV index in float32, the projections in float64 of the float32 inputs, the two rotations
    as ((r0*x + r1*y) + r2*z) per row, in the precisions numpy 2 (NEP 50) evaluates the reference in;
  - candidates in the reference's order (left, centre, right; sweep order within each);
  - cells_lists(): every cell's full candidate list; select(): the first 5 of a cell with at most 5 candidates, else the 5
    smallest keys (splitmix64(seed ^ (list << 62 | view << 32 | index)), view, index), the rule of csrc/correspondences.cu.
Pinned against the verbatim reference by tests/test_correspondences.py (tests/golden/reference_correspondences.npz,
oracle/make_golden_correspondences.py). Sweeps are the on-disk [N, >= 3] layout: y NOT negated."""
import numpy as np

N_BEV, N_CAM = (8, 8), (22, 5)
M64 = (1 << 64) - 1


def constants():
    """focal_x, focal_y, R_left, R_right by the reference's expressions (data.py:694-706, 740-745, 763-768)."""
    img_width, img_height, fov_width = 352, 160, 60
    fov_height = np.rad2deg(2.0 * np.arctan((img_height / img_width) * np.tan(0.5 * np.radians(fov_width))))
    focal_x = img_width / (2.0 * np.tan(np.deg2rad(fov_width) / 2.0))
    focal_y = img_height / (2.0 * np.tan(np.deg2rad(fov_height) / 2.0))
    rots = []
    for angle in (-60.0, 60.0):
        t = np.radians(angle)
        rots.append(np.array([[np.cos(t), -np.sin(t), 0.0], [np.sin(t), np.cos(t), 0.0], [0.0, 0.0, 1.0]]))
    return float(focal_x), float(focal_y), rots[0], rots[1]


def candidates(sweep):
    """-> view [K], index [K] (position in the sweep), bev [K, 2], cam [K, 2] int64, in the reference's candidate order."""
    w = np.asarray(sweep)[:, :3].astype(np.float32)
    fx, fy, r_left, r_right = constants()
    x = -w[:, 0]
    y, z = w[:, 1], w[:, 2]
    keep = (np.abs(x) < np.float32(16.0)) & (y < np.float32(32.0)) & (y > np.float32(0.0))
    idx = np.nonzero(keep)[0]
    x, y = x[keep], y[keep]
    z = z[keep] + np.float32(2.5 - 2.3)
    bx = ((x + np.float32(16.0)) * np.float32(8.0)).astype(np.int64)
    by = 255 - (y * np.float32(8.0)).astype(np.int64)
    X, Y, Z = x.astype(np.float64), y.astype(np.float64), z.astype(np.float64)
    out = []
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        for view in range(3):
            if view == 1:
                a, d, e = X, Y, Z
            else:
                R = r_left if view == 0 else r_right
                a, d, e = [(R[i, 0] * X + R[i, 1] * Y) + R[i, 2] * Z for i in range(3)]
            u = (fx * a) / d + 176.0
            v = (fy * e) / d + 80.0
            ok = (u > 0) & (u < 352.0) & (v > 0) & (v < 160.0)
            if view == 0:
                ok &= u >= 176.0
                u = u - 176.0
            elif view == 1:
                u = u + 176.0
            else:
                ok &= u < 176.0
                u = (u + 176.0) + 352.0
            cx = np.where(ok, u, 0.0).astype(np.int64)
            cy = 159 - np.where(ok, v, 0.0).astype(np.int64)
            ok &= (bx <= 255) & (cx <= 703)            # the two points the reference cannot index (it raises IndexError)
            out.append((np.full(int(ok.sum()), view), idx[ok], np.stack([bx[ok], by[ok]], 1), np.stack([cx[ok], cy[ok]], 1)))
    return tuple(np.concatenate([o[i] for o in out]).astype(np.int64).reshape((-1, 2) if i >= 2 else (-1,)) for i in range(4))


def cell_lists(sweep):
    """{('bev', i, j) / ('cam', i, j): (view [k], index [k], values [k, 2])} for every cell with candidates; values are what the
    reference appends (cam // 32 to a BEV cell, bev // 32 to a camera cell), in its order."""
    view, index, bev, cam = candidates(sweep)
    lists = {}
    for name, cell, val in (('bev', bev // 32, cam // 32), ('cam', cam // 32, bev // 32)):
        for i, j in sorted(set(map(tuple, cell.tolist()))):
            m = (cell[:, 0] == i) & (cell[:, 1] == j)
            lists[(name, i, j)] = (view[m], index[m], val[m])
    return lists


def splitmix64(x):
    z = (np.asarray(x, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def select(lists, seed):
    """bev_points [8,8,5,2], cam_points [22,5,5,2] int64 from cell_lists() under the selection rule, for one sample's seed."""
    bev_points = np.zeros(N_BEV + (5, 2), dtype=np.int64)
    cam_points = np.zeros(N_CAM + (5, 2), dtype=np.int64)
    for (name, i, j), (view, index, val) in lists.items():
        if len(view) > 5:
            L = 0 if name == 'bev' else 1
            with np.errstate(over='ignore'):
                h = splitmix64(np.uint64(int(seed) & M64) ^ ((np.uint64(L) << np.uint64(62)) | (view.astype(np.uint64) << np.uint64(32))
                                                              | index.astype(np.uint64)))
            order = np.lexsort((index, view, h))[:5]     # the last key is the primary one
            val = val[order]
        (bev_points if name == 'bev' else cam_points)[i, j, :len(val)] = val
    return bev_points, cam_points


def correspondences(sweep, seed):
    return select(cell_lists(sweep), seed)


# ---------------------------------------------------------------- the fixture's sweeps

def _boundary_points(rng):
    """Points that project onto (or next to) the image borders u in {0, 176, 352}, v in {0, 160} and the 32-pixel cell edges of
    each view, and onto the 0 / 16 / 32 m filters and the BEV cell edges: solved in float64, rounded to float32, then moved by
    -3..3 float32 ulps along the disk x (or z) axis."""
    fx, fy, r_left, r_right = constants()
    dz = np.float32(2.5 - 2.3)
    pts = []
    for view, R in ((0, r_left), (1, np.eye(3)), (2, r_right)):
        for depth in (1.5, 7.25, 13.0, 20.0):
            targets = [(u, 40.5) for u in (0.0, 176.0, 352.0) + tuple(32.0 * k - 176.0 * (view == 1) + 176.0 * (view == 0) for k in range(1, 12))]
            targets += [(100.0, v) for v in (0.0, 160.0, 16.0, 48.0, 80.0, 112.0, 144.0)]
            for u, v in targets:
                cam = np.array([(u - 176.0) * depth / fx, depth, (v - 80.0) * depth / fy])
                lid = R.T @ cam                               # cam = R . lidar
                base = np.array([-lid[0], lid[1], lid[2] - dz, 0.5], dtype=np.float32)
                for k in range(-3, 4):
                    p = base.copy()
                    axis = 0 if v == 40.5 or v == 100.0 else 2
                    for _ in range(abs(k)):
                        p[axis] = np.nextafter(p[axis], np.float32(np.inf if k > 0 else -np.inf))
                    pts.append(p)
    f32 = np.float32
    for xv in (f32(-16.0), f32(16.0), np.nextafter(f32(-16.0), f32(0)), f32(0.0), f32(-12.0), f32(-4.0), np.nextafter(f32(-4.0), f32(-8)),
               f32(4.0), np.nextafter(f32(4.0), f32(0)), f32(15.875), np.nextafter(f32(16.0), f32(0)) - f32(2.0 ** -19)):
        for yv in (f32(0.0), np.nextafter(f32(0.0), f32(1)), f32(4.0), np.nextafter(f32(4.0), f32(0)), f32(8.0), f32(31.875),
                   np.nextafter(f32(32.0), f32(0)), f32(32.0), f32(-1.0), f32(12.0)):
            pts.append(np.array([-xv, yv, rng.uniform(-2.5, 0.5), 0.25], dtype=np.float32))
    return np.array(pts, dtype=np.float32)


def random_sweep(n, seed):
    """On-disk layout [n, 4] float32 (x, y, z, intensity): x, y in CARLA's LiDAR frame, with points behind the side cameras."""
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.uniform(-24, 24, (n, 1)), rng.uniform(-8, 40, (n, 1)), rng.uniform(-3.0, 2.0, (n, 1)),
                           rng.uniform(0, 1, (n, 1))], axis=1).astype(np.float32)


def fixture_sweeps():
    """{name: [N, 4] float32 on-disk sweep} of tests/golden/reference_correspondences.npz (besides the routes)."""
    rng = np.random.default_rng(21)
    out = dict(rand20k=random_sweep(20000, 1), rand40k=random_sweep(40000, 2), empty=np.zeros((0, 4), np.float32),
               boundary=_boundary_points(rng))
    far = random_sweep(3000, 3)
    far[:1000, 1] = -np.abs(far[:1000, 1]) - 0.5          # behind the ego
    far[1000:2000, 0] = 16.0 + np.abs(far[1000:2000, 0])    # beyond 16 m to the side
    far[2000:, 1] = 32.0 + np.abs(far[2000:, 1])            # beyond 32 m ahead
    out['out_of_range'] = far
    pile = random_sweep(2000, 4)
    pile[:400, :3] = [-1.0, 10.0, -1.0]                     # one BEV cell and one camera cell with 400 identical candidates
    out['pile'] = pile
    return out
