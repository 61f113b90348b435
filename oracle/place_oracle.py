"""CPU restatement of the place-recognition chain (kintinuous_b200/csrc/kt_surf.cu, kt_place.cu, kt_place.hpp, cloud_fitness in kt_slice.cu).

numpy / scipy, FP64 wherever the device's result is a continuous quantity; the Hessian responses are formed in float32 exactly as the device
forms them (integer box sums, one float multiply per product), so that the detector's discrete decisions -- threshold, 3 x 3 x 3 maxima --
are the device's and only the continuous outputs (position, size, angle, descriptor) are compared with a tolerance.  cv2 pins the grey
conversion and the PnP pose; scipy's cKDTree pins the fitness.
"""
from __future__ import annotations

import math

import numpy as np

OCTAVES, LAYERS = 4, 4
HESSIAN = 400.0
RATIO = 0.49
U32 = 2.0 ** -24                            # float32 unit roundoff


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


def _to_half(p):
    """FP64 distance of positions p from the nearest rounding boundary of rint (k + 0.5)."""
    return np.abs(p - (np.floor(p) + 0.5))


def describe(I, x, y, size, rows, cols, margins=False):
    """(angle in radians, 64-d unit descriptor) of one keypoint, as kt_surf.cu's surf_describe_kernel.  margins: also a dict of how far
    the decisions float32 can flip lie from their edges --
      ori         the best 60 degree window's squared length minus the runner-up's (the best window with other members: windows with
                  the same members have the same sum on both sides), relative to the best; ori_bound: what float32 window sums can move it;
      ori_edge    degrees between a sample of the best window and the window's edge (samples on an axis, exact on both sides, excluded);
      sample      px between the FP64 position of any orientation or descriptor sample and a rint boundary (k + 0.5), the minimum;
      sample_slack  the same minus each position's float32 rounding bound (<= 0: a sample may round to the other pixel);
      sample_turn   the least change of the angle (radians) that moves a descriptor sample, float32 rounding included, across a boundary:
                  a device angle closer than that to the oracle's samples the same pixels."""
    x32, y32 = np.float32(x), np.float32(y)
    sigma = np.float32(1.2) * np.float32(size) / np.float32(9.0)
    ij = np.array(_DISC)
    hs_o = 2 * max(1, int(np.rint(np.float32(2.0) * sigma)))
    px = np.rint(x32 + ij[:, 0].astype(np.float32) * sigma).astype(np.int64)
    py = np.rint(y32 + ij[:, 1].astype(np.float32) * sigma).astype(np.int64)
    dx, dy, ok = _haar(I, px, py, hs_o, rows, cols)
    w = np.exp(-(ij[:, 0] ** 2 + ij[:, 1] ** 2) / (2.0 * 2.5 * 2.5))
    dx, dy = dx * w, dy * w
    dx_o, dy_o = dx, dy
    ang = np.degrees(np.arctan2(dy, dx)); ang = np.where(ang < 0, ang + 360.0, ang)
    use = ~((dx == 0) & (dy == 0))
    best, bsx, bsy, kb = -1.0, 0.0, 0.0, 0
    wins = np.zeros(72)
    for k in range(72):
        d = np.abs(ang - 5.0 * k)
        m = use & ((d < 30.0) | (d > 330.0))
        sx, sy = math.fsum(dx[m]), math.fsum(dy[m])           # correctly rounded: the same sum in any order
        wins[k] = sx * sx + sy * sy
        if sx * sx + sy * sy > best:
            best, bsx, bsy, kb = sx * sx + sy * sy, sx, sy, k
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
    desc = desc / n if n > 0 else desc
    if not margins:
        return th, desc
    # windows whose member set equals the best's have its sum on both sides: the runner-up is the best window with other members
    mem = [use & ((np.abs(ang - 5.0 * k) < 30.0) | (np.abs(ang - 5.0 * k) > 330.0)) for k in range(72)]
    other = [wins[k] for k in range(72) if not np.array_equal(mem[k], mem[kb])]
    ori = (best - max(other)) / best if best > 0 and other else (0.0 if best <= 0 else 1.0)
    # float32 sums of <= 109 terms: |d sx| <= 110 u sum |dx|, so s^2 moves by at most 2 (110 u) (sum|dx| + sum|dy|) / |s| relative
    mag = np.abs(dx_o[mem[kb]]).sum() + np.abs(dy_o[mem[kb]]).sum()
    rel = 110 * U32 * mag / np.sqrt(best) if best > 0 else np.inf
    e = np.abs(ang - 5.0 * kb)
    edge = np.minimum(np.abs(e - 30.0), np.abs(e - 330.0))
    exact = (dx_o == 0) | (dy_o == 0)                           # an axis direction: 0, 90, 180, 270 degrees on both sides
    ori_edge = float(edge[use & ~exact].min()) if (use & ~exact).any() else np.inf
    sig = float(sigma); x64, y64 = float(x32), float(y32)
    ox64, oy64 = ox.astype(np.float64), oy.astype(np.float64)
    po = [x64 + ij[:, 0] * sig, y64 + ij[:, 1] * sig]
    pd = [x64 + float(co) * ox64 - float(si) * oy64, y64 + float(si) * ox64 + float(co) * oy64]
    # float32 evaluation of a position, with any contraction: <= 4 roundings of magnitude |x| + |o|
    bo = [4 * U32 * (abs(x64) + np.abs(ij[:, 0]) * sig), 4 * U32 * (abs(y64) + np.abs(ij[:, 1]) * sig)]
    arm = np.abs(ox64) + np.abs(oy64)
    bd = [4 * U32 * (abs(x64) + arm), 4 * U32 * (abs(y64) + arm)]
    sample = float(min(_to_half(p_).min() for p_ in po + pd))
    slack = float(min((_to_half(p_) - b_).min() for p_, b_ in zip(po, bo)))
    # a descriptor sample moves by at most arm |d theta| when the angle changes: the least turn that can move one across a boundary
    turn = float(min(((_to_half(p_) - b_) / arm).min() for p_, b_ in zip(pd, bd)))
    return th, desc, dict(ori=float(ori), ori_bound=float(2 * rel), ori_edge=ori_edge, sample=sample, sample_slack=min(slack, turn * arm.max()),
                          sample_turn=turn)


def surf(rgb, max_features=1000, threshold=HESSIAN, margins=False):
    """(kp [n, 6] = x, y, size, angle, response, laplacian; desc [n, 64]) in the device's order.  margins: also a dict of arrays [n]
    (describe's ori, ori_edge and sample per keypoint)."""
    rows, cols = rgb.shape[:2]
    cands, I = detect(rgb, threshold)
    cands = cands[:max_features]
    kp = np.zeros((len(cands), 6)); desc = np.zeros((len(cands), 64))
    mg = {k: np.zeros(len(cands)) for k in ("ori", "ori_bound", "ori_edge", "sample", "sample_slack", "sample_turn")}
    for k, (_, x, y, size, resp, lap) in enumerate(cands):
        r = describe(I, x, y, size, rows, cols, margins)
        kp[k] = [x, y, size, r[0], resp, lap]; desc[k] = r[1]
        if margins:
            for key in mg:
                mg[key][k] = r[2][key]
    return (kp, desc, mg) if margins else (kp, desc)


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


def keypoints_3d(kp, depth, intr):
    """kt_place.cu keypoints_3d_kernel: [n, 3] float32, the rule of lookup_3d in the device's float32 order (z = d / 1000, then
    (z (u - cx)) / fx with one rounding per operation); NaN rows where a keypoint has no point."""
    kp = np.asarray(kp, np.float32).reshape(len(kp), -1)
    rows, cols = depth.shape
    f32 = np.float32
    x, y = kp[:, 0].astype(f32), kp[:, 1].astype(f32)
    u = np.floor(x + f32(0.5)).astype(np.int64); v = np.floor(y + f32(0.5)).astype(np.int64)
    ok = (np.abs(u.astype(f32) - x) < f32(0.5)) & (np.abs(v.astype(f32) - y) < f32(0.5)) & (u >= 0) & (v >= 0) & (u < cols) & (v < rows)
    d = np.where(ok, depth[np.clip(v, 0, rows - 1), np.clip(u, 0, cols - 1)], 0)
    z = d.astype(f32) / f32(1000.0)
    ok &= (d != 0) & (z < f32(10.0))
    fx, fy, cx, cy = [f32(a) for a in intr]
    out = np.stack([(z * (u.astype(f32) - cx)) / fx, (z * (v.astype(f32) - cy)) / fy, z], 1).astype(f32)
    out[~ok] = np.nan
    return out


def project_inliers(kp_new, kp_old, inlier, depth_new, depth_old, intr):
    """kt_place.hpp place_project_inliers: every inlier's keypoints back-projected at their TRUNCATED pixels, pairs where either
    depth is 0 (or a pixel is outside) dropped.  Returns (in_new [k, 3], in_old [k, 3]) float32."""
    rows, cols = depth_new.shape
    a, b = [], []
    ifx, ify = 1.0 / float(np.float32(intr[0])), 1.0 / float(np.float32(intr[1]))
    cx, cy = float(np.float32(intr[2])), float(np.float32(intr[3]))
    for i in np.flatnonzero(np.asarray(inlier)):
        u1, v1 = int(np.float32(kp_new[i][0])), int(np.float32(kp_new[i][1])); u2, v2 = int(np.float32(kp_old[i][0])), int(np.float32(kp_old[i][1]))
        if min(u1, v1, u2, v2) < 0 or u1 >= cols or u2 >= cols or v1 >= rows or v2 >= rows:
            continue
        z1 = float(np.float32(depth_new[v1, u1]) / np.float32(1000.0)); z2 = float(np.float32(depth_old[v2, u2]) / np.float32(1000.0))
        if z1 == 0.0 or z2 == 0.0:
            continue
        a.append([z1 * (u1 - cx) * ifx, z1 * (v1 - cy) * ify, z1]); b.append([z2 * (u2 - cx) * ifx, z2 * (v2 - cy) * ify, z2])
    return np.array(a, np.float32).reshape(-1, 3), np.array(b, np.float32).reshape(-1, 3)


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


# ---- the verification of one candidate (kt_tracker.cu place_process after retrieval) ----
RATIO32 = float(np.float32(RATIO))          # the device compares d1 < 0.49f d2
MIN_MATCHES, PNP_SEED = 40, 0x4B696E74756F7573
ICP_ITERS = (10, 5, 4, 0)                   # the tracker's ICP schedule, finest level first (ICPOdometry.cpp:42-55)


def dense_icp(maps_old, maps_new, R0, t0, intr, iterations=ICP_ITERS):
    """The dense check's point-to-plane ICP in FP64: the model is the old keyframe's maps with the camera at the identity, the current
    frame the new keyframe's maps moved by (R0, t0) (float32, as transform_maps_pyramid).  Levels coarse to fine, `iterations[l]`
    Gauss-Newton steps each, the systems of odometry_oracle.icp_system at the current pose (Rprev = I, tprev = 0), x = A^-1 b,
    resultRt <- [rodrigues(x[3:]) | x[:3]] resultRt, pose = resultRt^-1.  maps_*: per level (vmap, nmap) [3, rows, cols] float32.
    Returns (dT 4x4, ambiguous pixels summed over every step)."""
    from . import odometry_oracle as OO
    R0 = np.asarray(R0, np.float32).astype(np.float64); t0 = np.asarray(t0, np.float32).astype(np.float64)
    res = np.eye(4); amb = 0
    for level in range(len(iterations) - 1, -1, -1):
        if iterations[level] == 0:
            continue
        vo, no = (np.asarray(a, np.float32) for a in maps_old[level])
        vn, nn = (np.asarray(a, np.float64).reshape(3, -1) for a in maps_new[level])
        vn = (R0 @ vn + t0[:, None]).astype(np.float32).astype(np.float64); nn = (R0 @ nn).astype(np.float32).astype(np.float64)
        kl, _ = OO.level_intrinsics(*[np.float32(a) for a in intr], level)
        for _ in range(iterations[level]):
            T = np.linalg.inv(res)
            v = (T[:3, :3] @ vn + T[:3, 3:4]).reshape(vo.shape); n = (T[:3, :3] @ nn).reshape(vo.shape)
            S = OO.icp_system(v, n, vo, no, np.eye(3), np.zeros(3), kl)
            amb += S.extra["ambiguous"]
            x = np.linalg.solve(S.A, S.b)
            M = np.eye(4); M[:3, :3] = OO._rodrigues(x[3:]); M[:3, 3] = x[:3]
            res = M @ res
    return np.linalg.inv(res), amb


def verify(depth_old, kp_old, desc_old, depth_new, kp_new, desc_new, intr, maps_old, maps_new, voxel, inlier_ratio=0.35,
           iterations=ICP_ITERS, ratio=RATIO32):
    """place_process after retrieval, for candidate (old) and query (new) keyframes: 3-D matching, PnP, the inlier-ratio gate, the dense
    ICP check, C = inv(dT Tp), fitness at 2.5 voxels and the projected inliers.  Returns a dict with every stage's value, the stage
    where the chain stops (matches / inliers / fitness / loop, kt_place_result's names) and each gate's margin: matches - 40,
    inlier ratio - threshold, 0.01 - fitness."""
    out = dict(stage="matches")
    xo = keypoints_3d(kp_old, depth_old, intr); xn = keypoints_3d(kp_new, depth_new, intr)
    oi, ni = match_3d(desc_old, desc_new, xo, xn, ratio)
    m = len(oi)
    out.update(old_idx=oi, new_idx=ni, matches=m, margin_matches=m - MIN_MATCHES)
    if m < MIN_MATCHES:
        return out
    pn, po = xn[ni], xo[oi]
    uv = np.asarray(kp_old, np.float32)[oi, :2]
    Rp, tp, inl = pnp_ransac(pn, po, uv, intr)
    r = np.float32(inl.sum()) / np.float32(m)
    out.update(stage="inliers", R_pnp=Rp, t_pnp=tp, inliers=inl, n_inliers=int(inl.sum()), inlier_ratio=float(r),
               margin_ratio=float(r) - float(np.float32(inlier_ratio)))
    if not r > np.float32(inlier_ratio):
        return out
    Tp = np.eye(4); Tp[:3, :3] = Rp; Tp[:3, 3] = tp
    dT, amb = dense_icp(maps_old, maps_new, Rp, tp, intr, iterations)
    C = np.linalg.inv(dT @ Tp)
    leaf = float(np.float32(2.5) * np.float32(voxel))
    f, ns, nd = fitness(depth_old, depth_new, intr, leaf, C.astype(np.float32))          # the device moves the cloud by (float) C
    out.update(stage="fitness", dT=dT, C=C, icp_ambiguous=amb, fitness=f, n_src=ns, n_dst=nd, margin_fitness=0.01 - f)
    if not (f >= 0.0 and f < 0.01):
        return out
    kn = np.asarray(kp_new, np.float32)[ni, :2]; ko = uv
    a, b = project_inliers(kn, ko, inl, depth_new, depth_old, intr)
    out.update(stage="loop", inliers1=a, inliers2=b)
    return out
