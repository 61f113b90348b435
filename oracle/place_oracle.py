"""CPU restatement of the place-recognition chain (kintinuous_b200/csrc/kt_surf.cu, kt_place.cu, kt_place.hpp, cloud_fitness in kt_slice.cu).

numpy / scipy, FP64 wherever the device's result is a continuous quantity; the Hessian responses are formed in float32 exactly as the device
forms them (integer box sums, one float multiply per product), so that the detector's discrete decisions -- threshold, 3 x 3 x 3 maxima --
are the device's and only the continuous outputs (position, size, angle, descriptor) are compared with a tolerance.  cv2 pins the grey
conversion and the PnP pose; scipy's cKDTree pins the fitness.
"""
from __future__ import annotations

import numpy as np

OCTAVES, LAYERS = 4, 4
HESSIAN = 400.0
RATIO = 0.49


def grey(rgb):
    """cvtColor(RGB2GRAY) in fixed point as OpenCV 4 rounds 8-bit images: (9798 R + 19235 G + 3735 B + 2^14) >> 15."""
    r = rgb[..., 0].astype(np.int64); g = rgb[..., 1].astype(np.int64); b = rgb[..., 2].astype(np.int64)
    return ((9798 * r + 19235 * g + 3735 * b + (1 << 14)) >> 15).astype(np.int64)


def integral(g):
    rows, cols = g.shape
    I = np.zeros((rows + 1, cols + 1), np.int64)
    I[1:, 1:] = np.cumsum(np.cumsum(g, axis=0), axis=1)
    return I


def _box(I, x0, y0, x1, y1):
    return I[y1, x1] - I[y0, x1] - I[y1, x0] + I[y0, x0]


def size_of(o, l):
    return (9 + 6 * l) << o


def _fits(s, cx, cy, rows, cols):
    h = s // 2
    return (cx >= h) & (cy >= h) & (cx + (s - h) <= cols) & (cy + (s - h) <= rows)


def hessian(I, s, cx, cy):
    """det (float32, the device's rounding) and laplacian sign at centres (cx, cy) (arrays), filter side s."""
    L = s // 3
    x0 = cx - s // 2; y0 = cy - s // 2
    ya, yb = cy - (L - 1), cy + L
    xx = _box(I, x0, ya, x0 + s, yb) - 3 * _box(I, x0 + L, ya, x0 + 2 * L, yb)
    xa, xb = cx - (L - 1), cx + L
    yy = _box(I, xa, y0, xb, y0 + s) - 3 * _box(I, xa, y0 + L, xb, y0 + 2 * L)
    xy = (_box(I, cx - L, cy - L, cx, cy) - _box(I, cx + 1, cy - L, cx + 1 + L, cy)
          - _box(I, cx - L, cy + 1, cx, cy + 1 + L) + _box(I, cx + 1, cy + 1, cx + 1 + L, cy + 1 + L))
    inv = np.float32(1.0) / np.float32(s * s)
    dxx = xx.astype(np.float32) * inv; dyy = yy.astype(np.float32) * inv; dxy = xy.astype(np.float32) * inv
    det = dxx * dyy - np.float32(0.81) * (dxy * dxy)
    return det.astype(np.float32), np.where(xx + yy >= 0, 1, -1)


def response_maps(I, rows, cols):
    maps = {}
    for o in range(OCTAVES):
        step = 1 << o
        gr, gc = (rows + step - 1) // step, (cols + step - 1) // step
        jj, ii = np.meshgrid(np.arange(gc), np.arange(gr))
        cx, cy = jj << o, ii << o
        for l in range(LAYERS):
            s = size_of(o, l)
            ok = _fits(s, cx, cy, rows, cols)
            det = np.zeros((gr, gc), np.float32)
            if ok.any():
                d, _ = hessian(I, s, np.where(ok, cx, s // 2), np.where(ok, cy, s // 2))
                det[ok] = d[ok]
            maps[o, l] = det
    return maps


def detect(rgb, threshold=HESSIAN):
    """Every refined extremum: list of (key tuple, x, y, size, response, laplacian), strongest first."""
    rows, cols = rgb.shape[:2]
    I = integral(grey(rgb))
    maps = response_maps(I, rows, cols)
    out = []
    for o in range(OCTAVES):
        for l in (1, 2):
            R0, R1, R2 = maps[o, l - 1], maps[o, l], maps[o, l + 1]
            gr, gc = R1.shape
            s_hi = size_of(o, l + 1)
            cand = np.argwhere(R1 > np.float32(threshold))
            for i, j in cand:
                if i < 1 or j < 1 or i >= gr - 1 or j >= gc - 1:
                    continue
                if not (_fits(s_hi, (j - 1) << o, (i - 1) << o, rows, cols) and _fits(s_hi, (j + 1) << o, (i + 1) << o, rows, cols)):
                    continue
                v = R1[i, j]
                n0 = R0[i - 1:i + 2, j - 1:j + 2]; n1 = R1[i - 1:i + 2, j - 1:j + 2].copy(); n2 = R2[i - 1:i + 2, j - 1:j + 2]
                n1[1, 1] = -np.inf
                if (n0 >= v).any() or (n1 >= v).any() or (n2 >= v).any():
                    continue
                f = lambda R, di, dj: float(R[i + di, j + dj])
                dx = 0.5 * (f(R1, 0, 1) - f(R1, 0, -1)); dy = 0.5 * (f(R1, 1, 0) - f(R1, -1, 0)); ds = 0.5 * (f(R2, 0, 0) - f(R0, 0, 0))
                c2 = 2.0 * float(v)
                H = np.array([[f(R1, 0, 1) + f(R1, 0, -1) - c2, 0.25 * (f(R1, 1, 1) - f(R1, 1, -1) - f(R1, -1, 1) + f(R1, -1, -1)),
                               0.25 * (f(R2, 0, 1) - f(R2, 0, -1) - f(R0, 0, 1) + f(R0, 0, -1))],
                              [0, f(R1, 1, 0) + f(R1, -1, 0) - c2, 0.25 * (f(R2, 1, 0) - f(R2, -1, 0) - f(R0, 1, 0) + f(R0, -1, 0))],
                              [0, 0, f(R2, 0, 0) + f(R0, 0, 0) - c2]])
                H[1, 0] = H[0, 1]; H[2, 0] = H[0, 2]; H[2, 1] = H[1, 2]
                if np.linalg.det(H) == 0.0:
                    continue
                off = -np.linalg.solve(H, np.array([dx, dy, ds]))
                if np.any(np.abs(off) > 1.0):
                    continue
                _, lap = hessian(I, size_of(o, l), np.array(j << o), np.array(i << o))
                key = (-float(v), o, l - 1, int(i * gc + j))
                out.append((key, (j + off[0]) * (1 << o), (i + off[1]) * (1 << o), size_of(o, l) + off[2] * (6 << o), float(v), int(lap)))
    out.sort(key=lambda t: t[0])
    return out, I


def _haar(I, px, py, hs, rows, cols):
    h = hs // 2
    x0, y0 = px - h, py - h
    ok = (x0 >= 0) & (y0 >= 0) & (x0 + hs <= cols) & (y0 + hs <= rows)
    px_, py_, x0_, y0_ = [np.where(ok, a, h) for a in (px, py, x0, y0)]
    dx = _box(I, px_, y0_, x0_ + hs, y0_ + hs) - _box(I, x0_, y0_, px_, y0_ + hs)
    dy = _box(I, x0_, py_, x0_ + hs, y0_ + hs) - _box(I, x0_, y0_, x0_ + hs, py_)
    return np.where(ok, dx, 0).astype(np.float64), np.where(ok, dy, 0).astype(np.float64), ok


_DISC = [(i, j) for j in range(-6, 7) for i in range(-6, 7) if i * i + j * j < 36]


def describe(I, x, y, size, rows, cols):
    """(angle in radians, 64-d unit descriptor) of one keypoint, as kt_surf.cu's surf_describe_kernel."""
    x32, y32 = np.float32(x), np.float32(y)
    sigma = np.float32(1.2) * np.float32(size) / np.float32(9.0)
    ij = np.array(_DISC)
    hs_o = 2 * max(1, int(np.rint(np.float32(2.0) * sigma)))
    px = np.rint(x32 + ij[:, 0].astype(np.float32) * sigma).astype(np.int64)
    py = np.rint(y32 + ij[:, 1].astype(np.float32) * sigma).astype(np.int64)
    dx, dy, ok = _haar(I, px, py, hs_o, rows, cols)
    w = np.exp(-(ij[:, 0] ** 2 + ij[:, 1] ** 2) / (2.0 * 2.5 * 2.5))
    dx, dy = dx * w, dy * w
    ang = np.degrees(np.arctan2(dy, dx)); ang = np.where(ang < 0, ang + 360.0, ang)
    use = ~((dx == 0) & (dy == 0))
    best, bsx, bsy = -1.0, 0.0, 0.0
    for k in range(72):
        d = np.abs(ang - 5.0 * k)
        m = use & ((d < 30.0) | (d > 330.0))
        sx, sy = dx[m].sum(), dy[m].sum()
        if sx * sx + sy * sy > best:
            best, bsx, bsy = sx * sx + sy * sy, sx, sy
    th = float(np.arctan2(bsy, bsx))
    co, si = np.float32(np.cos(th)), np.float32(np.sin(th))
    u, v = np.meshgrid(np.arange(20), np.arange(20))
    ox = (u.astype(np.float32) - np.float32(9.5)) * sigma; oy = (v.astype(np.float32) - np.float32(9.5)) * sigma
    px = np.rint(x32 + co * ox - si * oy).astype(np.int64); py = np.rint(y32 + si * ox + co * oy).astype(np.int64)
    hs_d = 2 * max(1, int(np.rint(sigma)))
    dx, dy, ok = _haar(I, px, py, hs_d, rows, cols)
    w = np.exp(-(ox.astype(np.float64) ** 2 + oy.astype(np.float64) ** 2) / (2.0 * 3.3 * 3.3 * float(sigma) ** 2))
    c, s_ = np.cos(th), np.sin(th)
    rx = (dx * c + dy * s_) * w; ry = (-dx * s_ + dy * c) * w
    desc = np.zeros(64)
    for cv in range(4):
        for cu in range(4):
            bx = rx[cv * 5:cv * 5 + 5, cu * 5:cu * 5 + 5]; by = ry[cv * 5:cv * 5 + 5, cu * 5:cu * 5 + 5]
            desc[(cv * 4 + cu) * 4:(cv * 4 + cu) * 4 + 4] = [bx.sum(), by.sum(), np.abs(bx).sum(), np.abs(by).sum()]
    n = np.linalg.norm(desc)
    return th, desc / n if n > 0 else desc


def surf(rgb, max_features=1000, threshold=HESSIAN):
    """(kp [n, 6] = x, y, size, angle, response, laplacian; desc [n, 64]) in the device's order."""
    rows, cols = rgb.shape[:2]
    cands, I = detect(rgb, threshold)
    cands = cands[:max_features]
    kp = np.zeros((len(cands), 6)); desc = np.zeros((len(cands), 64))
    for k, (_, x, y, size, resp, lap) in enumerate(cands):
        th, d = describe(I, x, y, size, rows, cols)
        kp[k] = [x, y, size, th, resp, lap]; desc[k] = d
    return kp, desc


# ---- matching, lookup, candidate selection (kt_place.hpp) ----
def match_ratio(db, query, ratio=RATIO):
    """Per database row: nearest query index, d1, d2 (squared, FP64) and d1 < ratio d2."""
    db = np.asarray(db, np.float64); q = np.asarray(query, np.float64)
    D = (db * db).sum(1)[:, None] - 2.0 * db @ q.T + (q * q).sum(1)[None, :]
    o = np.argsort(D, axis=1, kind="stable")[:, :2]
    d1 = D[np.arange(len(db)), o[:, 0]]; d2 = D[np.arange(len(db)), o[:, 1]] if q.shape[0] > 1 else np.full(len(db), np.inf)
    return o[:, 0], d1, d2, (d1 < ratio * d2) & (q.shape[0] >= 2)


def select_candidate(passes, query, exclude_recent=20, min_passes=40):
    best, bp = -1, 0
    for k in range(0, query - exclude_recent + 1):
        if passes[k] > bp:
            best, bp = k, passes[k]
    return best if bp >= min_passes else -1


def unique_matches(best, d1, passes, n_new):
    owner = {}
    for i in range(len(best)):
        if not passes[i] or best[i] < 0 or best[i] >= n_new:
            continue
        j = int(best[i])
        if j not in owner or d1[i] < d1[owner[j]]:
            owner[j] = i
    js = sorted(owner)
    return np.array([owner[j] for j in js], np.int64), np.array(js, np.int64)


def match_3d(desc_old, desc_new, xyz_old, xyz_new, ratio=RATIO):
    """surfMatch3D's order: the ratio test over all features of both keyframes, one match per new feature, then the pairs without a 3-D
    point on either side dropped.  xyz_*: [n, 3] with NaN rows where a keypoint has no point.  Returns (old indices, new indices)."""
    best, d1, _, ps = match_ratio(desc_old, desc_new, ratio)
    oi, ni = unique_matches(best, d1, ps, len(desc_new))
    keep = ~np.isnan(np.asarray(xyz_old)[oi, 2]) & ~np.isnan(np.asarray(xyz_new)[ni, 2]) if len(oi) else np.zeros(0, bool)
    return oi[keep], ni[keep]


def lookup_3d(x, y, depth, intr):
    """+-0.5 px strict, depth != 0, z < 10 m; None without a point."""
    rows, cols = depth.shape
    x32, y32 = np.float32(x), np.float32(y)
    u = int(np.floor(x32 + np.float32(0.5))); v = int(np.floor(y32 + np.float32(0.5)))
    if not (abs(np.float32(u) - x32) < 0.5 and abs(np.float32(v) - y32) < 0.5):
        return None
    if u < 0 or v < 0 or u >= cols or v >= rows or depth[v, u] == 0:
        return None
    z = np.float32(depth[v, u]) / np.float32(1000.0)
    if not z < 10.0:
        return None
    fx, fy, cx, cy = [np.float32(a) for a in intr]
    return np.array([z * (np.float32(u) - cx) / fx, z * (np.float32(v) - cy) / fy, z], np.float32)


def is_keyframe(R_curr, R_last, g_curr, g_last, movement=0.15):
    from scipy.spatial.transform import Rotation
    ang = np.linalg.norm(Rotation.from_matrix(np.asarray(R_curr, np.float64).T @ np.asarray(R_last, np.float64)).as_rotvec())
    return 0.5 * (ang + np.linalg.norm(np.asarray(g_curr, np.float64) - np.asarray(g_last, np.float64))) >= movement


# ---- PnP ----
def _splitmix(seed, h, k):
    M = (1 << 64) - 1
    z = (seed + 0x9E3779B97F4A7C15 * (((h << 20) + k + 1) & M)) & M
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
    return ((z ^ (z >> 31)) >> 32) & 0xFFFFFFFF


def kabsch(a, b):
    """R, t with R a + t ~ b (FP64, SVD)."""
    ca, cb = a.mean(0), b.mean(0)
    U, _, Vt = np.linalg.svd((a - ca).T @ (b - cb))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(Vt.T @ U.T))])
    R = Vt.T @ D @ U.T
    return R, cb - R @ ca


def reproj_inliers(R, t, p_new, uv_old, intr, thr=2.0):
    fx, fy, cx, cy = intr
    X = p_new @ R.T + t
    with np.errstate(divide="ignore", invalid="ignore"):
        u = fx * X[:, 0] / X[:, 2] + cx; v = fy * X[:, 1] / X[:, 2] + cy
    e = (u - uv_old[:, 0]) ** 2 + (v - uv_old[:, 1]) ** 2
    return (X[:, 2] > 0) & (e <= thr * thr)


def refine(R, t, p_new, uv_old, intr, mask, iters=10):
    """Gauss-Newton on the reprojection error of the masked matches (left perturbation), FP64."""
    from scipy.spatial.transform import Rotation
    fx, fy, cx, cy = intr
    for _ in range(iters):
        X = p_new[mask] @ R.T + t
        ok = X[:, 2] > 0
        X = X[ok]; uv = uv_old[mask][ok]
        iz = 1.0 / X[:, 2]
        r = np.stack([fx * X[:, 0] * iz + cx - uv[:, 0], fy * X[:, 1] * iz + cy - uv[:, 1]], 1)
        P0 = np.stack([fx * iz, 0 * iz, -fx * X[:, 0] * iz * iz], 1); P1 = np.stack([0 * iz, fy * iz, -fy * X[:, 1] * iz * iz], 1)
        J = np.zeros((len(X), 2, 6))
        J[:, 0, :3] = P0; J[:, 1, :3] = P1
        J[:, 0, 3:] = np.cross(X, P0); J[:, 1, 3:] = np.cross(X, P1)
        A = np.einsum("nki,nkj->ij", J, J); b = np.einsum("nki,nk->i", J, r)
        x = -np.linalg.solve(A, b)
        dR = Rotation.from_rotvec(x[3:]).as_matrix()
        R, t = dR @ R, dR @ t + x[:3]
    return R, t


def pnp_ransac(p_new, p_old, uv_old, intr, iterations=500, thr=2.0, seed=0x4B696E74756F7573):
    """kt_place.cu's RANSAC restated: same samples, Kabsch by SVD, most inliers (ties: first), refinement, final inliers."""
    p_new = np.asarray(p_new, np.float64); p_old = np.asarray(p_old, np.float64); uv_old = np.asarray(uv_old, np.float64)
    n = len(p_new)
    best, bc = None, -1
    for h in range(iterations):
        pose = None
        for attempt in range(64):
            ids = [_splitmix(seed, h, attempt * 3 + m) % n for m in range(3)]
            if len(set(ids)) < 3:
                continue
            a = p_new[ids].astype(np.float32).astype(np.float64)
            if np.linalg.norm(np.cross(a[1] - a[0], a[2] - a[0])) ** 2 < 4e-8:
                continue
            pose = kabsch(a, p_old[ids])
            break
        if pose is None:
            continue
        c = int(reproj_inliers(*pose, p_new, uv_old, intr, thr).sum())
        if c > bc:
            best, bc = pose, c
    if best is None:
        return np.eye(3), np.zeros(3), np.zeros(n, bool)
    R, t = best
    m = reproj_inliers(R, t, p_new, uv_old, intr, thr)
    if m.sum() >= 6:
        R, t = refine(R, t, p_new, uv_old, intr, m)
    return R, t, reproj_inliers(R, t, p_new, uv_old, intr, thr)


# ---- fitness (PCL VoxelGrid + getFitnessScore) ----
def depth_cloud(depth, intr):
    fx, fy, cx, cy = [np.float32(a) for a in intr]
    rows, cols = depth.shape
    u, v = np.meshgrid(np.arange(cols, dtype=np.float32), np.arange(rows, dtype=np.float32))
    z = depth.astype(np.float32) / np.float32(1000.0)
    P = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], -1).reshape(-1, 3)
    return P[depth.reshape(-1) != 0]


def voxel_grid(P, leaf):
    """pcl::VoxelGrid: one centroid per occupied leaf, ascending leaf index."""
    P = np.asarray(P, np.float32)
    inv = np.float32(1.0) / np.float32(leaf)
    mn = np.floor(P.min(0) * inv).astype(np.int64); mx = np.floor(P.max(0) * inv).astype(np.int64)
    div = mx - mn + 1
    ijk = (np.floor(P * inv) - mn.astype(np.float32)).astype(np.int64)
    idx = (ijk[:, 2] * div[1] + ijk[:, 1]) * div[0] + ijk[:, 0]
    u, inv_i = np.unique(idx, return_inverse=True)
    C = np.zeros((len(u), 3)); np.add.at(C, inv_i, P.astype(np.float64))
    return C / np.bincount(inv_i)[:, None]


def fitness(src_depth, dst_depth, intr, leaf, T):
    from scipy.spatial import cKDTree
    S = voxel_grid(depth_cloud(src_depth, intr), leaf); D = voxel_grid(depth_cloud(dst_depth, intr), leaf)
    T = np.asarray(T, np.float64)
    S2 = S @ T[:3, :3].T + T[:3, 3]
    d, _ = cKDTree(D).query(S2, k=1)
    return float((d * d).mean()), len(S), len(D)
