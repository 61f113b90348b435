"""FP64 reference of the odometry's normal equations at iteration 0 of one pyramid level, with a forward error bound per entry.

At iteration 0 of a level that the tracker enters from the previous pose (every coarser level run for zero iterations), everything the
kernels compute is defined by their inputs alone:
  * the photometric warp is build_warp of resultRt = I (RGBDOdometry.cpp:209-231), so a pixel corresponds to itself;
  * ICP projects current pixel (x, y) back onto model pixel (x, y) (Rcurr = Rprev, tcurr = tprev).
This module rebuilds, from the same float inputs, what rgbd_frame_kernel / icp_frame_kernel and the per-iteration kernels sum:
  * photometric (rgb_precheck / rgb_correspond / rgb_pixel_row, cuda/reduce.cu:443-480, 709-764): the correspondence count and
    sum of (int)diff^2 wrapped to int32 as both sides do, sigma by the Q3 rule (RGBDOdometry.cpp:253), the weight 1 / (sigma + |diff|),
    the last-frame point rebuilt from its depth (projectToPointCloud, maps.cu:311-345), the seven row entries, summed in FP64;
  * point-to-plane ICP (icp_pixel_project / icp_pixel_finish, cuda/reduce.cu:211-316): the distance and angle tests, rows, residual
    and inlier count;
  * the -ri merge (A_rgb + 100 A_icp, b_rgb + 10 b_icp, RGBDOdometry.cpp:316-321), the FP64 solve and the pose composition.

Every entry comes with a bound on how far a correct float implementation may lie from the FP64 value:
    |dA_ij| <= sum_pix (|drow_i| |row_j| + |row_i| |drow_j|) + C_SUM 2^-24 S_ij + G 2^-24,      S_ij = sum_pix |row_i row_j|
where |drow_k| is a few ulps of the magnitudes that formed row k (for the ICP residual |n| (|s| + |d|): s - d cancels), C_SUM covers the
deepest float summation tree of either path, and G 2^-24 the fixed-point rounding of the whole-frame kernels' grid exchange.  Pixels
within that margin of a threshold test are counted as ambiguous: their whole contribution is added to the bound.  Test-only, numpy."""
import numpy as np

U = 2.0 ** -24          # unit roundoff of float
C_ROW = 16              # ulps of a row entry's magnitude (a handful of float products, an approximate division, float inputs rebuilt in double)
C_SUM = 160             # float additions along the deepest summation tree: <= 5 chunks per thread + warp tree (5) + 16 warps in the
                        # whole-frame kernels; <= 3 per thread + 5 + 8 + 66 partials + 8 in the per-iteration kernels at 640x480 on 132 SMs
G_MAX = 255             # CTAs of a whole-frame kernel (frame_grid)
SIN20 = float(np.sin(np.float32(20.0) * np.float32(3.14159254) / np.float32(180.0)))
MIN_GRADIENT = (12, 5, 3, 1)                      # RGBDOdometry.cpp:109-113
SOBEL_SCALE = 1.0 / 8.0
B_SLOTS = (6, 12, 17, 21, 24, 26)                # b components among the 27 products (internal.h:101-106)


def level_intrinsics(fx, fy, cx, cy, level):
    """(float Intr of the level, double IntrDoublePrecision of the level) as odom_level_args builds them."""
    div = 1 << level
    f = np.float32
    kl = (f(f(fx) / f(div)), f(f(fy) / f(div)), f(f(cx) / f(div)), f(f(cy) / f(div)))
    kd = (float(f(fx)) / div, float(f(fy)) / div, float(f(cx)) / div, float(f(cy)) / div)
    return kl, kd


def build_warp(T, Kfx, Kfy, Kcx, Kcy):
    """(K R K^-1, K t) of the inverse of the 4x4 double T, rounded to float (build_warp, kt_rgb.cu)."""
    T = np.asarray(T, np.float64).reshape(4, 4)
    R = T[:3, :3].T
    t = -R @ T[:3, 3]
    K = np.array([[Kfx, 0, Kcx], [0, Kfy, Kcy], [0, 0, 1.0]])
    Ki = np.array([[1.0 / Kfx, 0, -Kcx / Kfx], [0, 1.0 / Kfy, -Kcy / Kfy], [0, 0, 1.0]])
    return ((K @ R) @ Ki).astype(np.float32), (K @ t).astype(np.float32)


def _near(v, edge, margin):
    return np.abs(v - edge) <= margin


def photometric_correspondences(next_image, next_depth, dIdx, dIdy, last_depth, last_image, level, krk, kt, max_depth_delta=0.07):
    """Correspondences of every pixel for the float warp (krk, kt).  Returns a dict of per-pixel arrays: valid, ambiguous (a threshold
    test or a rounding lies within the float error of its edge), u0, v0, diff (float), gx, gy, d0."""
    rows, cols = next_image.shape
    ni = next_image.astype(np.int64)
    y, x = np.mgrid[0:rows, 0:cols]
    # 4x4 neighbourhood rows i-2..i+1, columns j-2..j+1, clipped to the image (reduce.cu:715-722)
    pos = np.pad(ni > 0, ((2, 1), (2, 1)), constant_values=True)
    nb = np.ones((rows, cols), bool)
    for du in range(4):
        for dv in range(4):
            nb &= pos[du:du + rows, dv:dv + cols]
    gx = dIdx.astype(np.int64); gy = dIdy.astype(np.int64)
    m2 = (gx * gx + gy * gy).astype(np.float32)
    min_scale = np.float32(MIN_GRADIENT[level] ** 2 / SOBEL_SCALE ** 2)
    d1 = next_depth.astype(np.float64)
    pre = (x < cols - 5) & (y < rows - 1) & nb & (m2 >= min_scale) & ~np.isnan(d1)
    k = krk.astype(np.float64); t = kt.astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        td1 = d1 * (k[2, 0] * x + k[2, 1] * y + k[2, 2]) + t[2]
        uf = (d1 * (k[0, 0] * x + k[0, 1] * y + k[0, 2]) + t[0]) / td1
        vf = (d1 * (k[1, 0] * x + k[1, 1] * y + k[1, 2]) + t[1]) / td1
    mag = C_ROW * U * (np.abs(uf) + np.abs(vf) + cols + rows)
    amb = pre & (_near(uf - np.floor(uf), 0.5, mag) | _near(vf - np.floor(vf), 0.5, mag))
    u0 = np.where(pre, np.rint(np.nan_to_num(uf)), -1).astype(np.int64)
    v0 = np.where(pre, np.rint(np.nan_to_num(vf)), -1).astype(np.int64)
    inb = pre & (u0 >= 0) & (v0 >= 0) & (u0 < cols) & (v0 < rows)
    uc, vc = np.clip(u0, 0, cols - 1), np.clip(v0, 0, rows - 1)
    d0 = last_depth.astype(np.float64)[vc, uc]
    il = last_image.astype(np.int64)[vc, uc]
    # The depth test |transformed_d1 - d0| <= maxDepthDelta is made in float.  Where every step of the float evaluation of transformed_d1
    # is exact (at the identity warp: d1 * 1 + 0), the kernel's value is that exact value however its products and sums are contracted,
    # and the float subtraction and comparison are reproduced bit for bit: no tie.  Elsewhere the test is ambiguous within a few ulps.
    td1_f, exact = _float_chain_if_exact(d1, x, y, k[2], t[2])
    thr = np.float32(max_depth_delta)
    with np.errstate(invalid="ignore"):
        dd_f = np.abs(td1_f.astype(np.float32) - last_depth.astype(np.float32)[vc, uc])
        dd = np.where(exact, dd_f.astype(np.float64), np.abs(td1 - d0))
        ok = inb & (d0 > 0) & (dd <= float(thr)) & (il != 0)
        amb |= inb & (d0 > 0) & (il != 0) & ~exact & _near(dd, float(thr), C_ROW * U * (np.abs(td1) + np.abs(d0)))
    diff = (ni - il).astype(np.float64)
    return dict(valid=ok, ambiguous=amb, u0=u0, v0=v0, diff=np.where(inb, diff, 0.0), gx=gx, gy=gy)


def _float_chain_if_exact(d1, x, y, k, t):
    """d1 * (k0 * x + k1 * y + k2) + t evaluated one float operation at a time, and whether every operation was exact."""
    f = lambda v: v.astype(np.float32).astype(np.float64)
    exact = np.ones(np.shape(d1), bool)
    def op(v):
        nonlocal exact
        r = f(v)
        with np.errstate(invalid="ignore"):
            exact &= (r == v) | np.isnan(v)
        return r
    inner = op(op(op(k[0] * x) + op(k[1] * y)) + float(k[2]))
    return op(op(d1 * inner) + float(t)), exact


def count_and_sigma(corr):
    """(count, sum of (int)diff^2 wrapped to int32) over the sure correspondences, and the number of ambiguous pixels."""
    ok = corr["valid"] & ~corr["ambiguous"]
    d2 = int((corr["diff"][ok].astype(np.int64) ** 2).sum())
    return int(ok.sum()), (d2 + 2 ** 31) % 2 ** 32 - 2 ** 31, int(corr["ambiguous"].sum())


def q3_sigma(count, sigma_sq):
    """sigmaVal = sqrt((float)sigma / rgbSize == 0 ? 1 : rgbSize) (RGBDOdometry.cpp:253), as a float: 1 when every diff is 0 (a repeated
    frame), sqrt(count) otherwise (0 without correspondences: 0 / 0 is NaN, not 0)."""
    return float(np.float32(np.sqrt(1.0 if (count != 0 and sigma_sq == 0) else float(count))))


def _products(rows7, mags7):
    """Upper-triangle products (the 27 of internal.h plus residual and count) of the rows, and the per-product error bound and S."""
    n = rows7.shape[0]
    P = np.zeros(29); S = np.zeros(29); E = np.zeros(29)
    pairs = [(a, b) for a in range(6) for b in range(a, 7)] + [(6, 6)]
    for k, (a, b) in enumerate(pairs):
        p = rows7[:, a] * rows7[:, b]
        P[k] = p.sum(); S[k] = np.abs(p).sum()
        E[k] = (mags7[:, a] * np.abs(rows7[:, b]) + np.abs(rows7[:, a]) * mags7[:, b] + mags7[:, a] * mags7[:, b]).sum()
    P[28] = n; S[28] = n
    return P, S, E


def unpack(v):
    """29 components -> A (6x6), b (6), residual, count (internal.h order)."""
    A = np.zeros((6, 6)); b = np.zeros(6)
    k = 0
    for i in range(6):
        for j in range(i, 7):
            if j == 6:
                b[i] = v[k]
            else:
                A[i, j] = A[j, i] = v[k]
            k += 1
    return A, b, v[27], v[28]


class System:
    """29 FP64 sums and their bounds; A / b / bound views."""

    def __init__(self, P, bound, count, extra=None):
        self.P, self.bound, self.count = P, bound, count
        self.A, self.b, self.residual, _ = unpack(P)
        self.dA, self.db, self.dres, _ = unpack(bound)
        self.extra = extra or {}


def _bound(S, E, amb_abs):
    bound = E + C_SUM * U * S + G_MAX * U + amb_abs
    bound[28] = amb_abs[28]
    return bound


def photometric_system(corr, sigma, last_depth_level, kl, kd, cloud=None):
    """Photometric normal equations of the correspondences corr at robust scale sigma (float).  kl: float (fx, fy, cx, cy) of the level,
    kd: double ones.  The last-frame point is rebuilt from its depth like rgbd_frame_kernel (or read from cloud [rows, cols, 3] when
    given: the reference's projectToPointCloud output)."""
    sure = corr["valid"] & ~corr["ambiguous"]
    amb = corr["ambiguous"]
    fx, fy = float(kl[0]), float(kl[1])
    Kfx, Kfy, Kcx, Kcy = kd
    invFx, invFy = 1.0 / Kfx, 1.0 / Kfy

    def rows_of(mask):
        u0 = corr["u0"][mask]; v0 = corr["v0"][mask]
        diff = corr["diff"][mask]; gx = corr["gx"][mask].astype(np.float64); gy = corr["gy"][mask].astype(np.float64)
        if cloud is not None:
            X, Y, Z = (cloud[v0, u0, c].astype(np.float64) for c in range(3))
        else:
            Z = last_depth_level[np.clip(v0, 0, None), np.clip(u0, 0, None)].astype(np.float64)
            X = (u0 - Kcx) * Z * invFx; Y = (v0 - Kcy) * Z * invFy
        w = 1.0 / (sigma + np.abs(diff))
        w = np.where(sigma + np.abs(diff) > 1.19209290e-07, w, 1.0)
        invz = 1.0 / Z
        v0r = w * SOBEL_SCALE * gx * fx * invz
        v1r = w * SOBEL_SCALE * gy * fy * invz
        v2r = -(v0r * X + v1r * Y) * invz
        r = np.stack([v0r, v1r, v2r, -Z * v1r + Y * v2r, Z * v0r - X * v2r, -Y * v0r + X * v1r, -w * diff], axis=1)
        m2 = (np.abs(v0r * X) + np.abs(v1r * Y)) * np.abs(invz)
        m = np.stack([np.abs(v0r), np.abs(v1r), m2, np.abs(Z * v1r) + np.abs(Y) * m2, np.abs(Z * v0r) + np.abs(X) * m2,
                      np.abs(Y * v0r) + np.abs(X * v1r), np.abs(w * diff)], axis=1) * (C_ROW * U)
        return r, m

    r, m = rows_of(sure)
    P, S, E = _products(r, m)
    rows_, cols_ = amb.shape
    u0, v0 = corr["u0"], corr["v0"]
    maybe = amb & (u0 >= 0) & (v0 >= 0) & (u0 < cols_) & (v0 < rows_)
    if cloud is None:                                   # a last-frame pixel without depth fails the test on both sides
        with np.errstate(invalid="ignore"):
            maybe &= last_depth_level[np.clip(v0, 0, rows_ - 1), np.clip(u0, 0, cols_ - 1)] > 0
    # either side of a test: the whole contribution goes to the bound
    ra, ma = rows_of(maybe) if maybe.any() else (np.zeros((0, 7)), np.zeros((0, 7)))
    _, Sa, Ea = _products(ra, ma)
    amb_abs = Sa + Ea
    amb_abs[28] = int(amb.sum())
    return System(P, _bound(S, E, amb_abs), int(sure.sum()), dict(ambiguous=int(amb.sum())))


def icp_system(vmap_curr, nmap_curr, vmap_g_prev, nmap_g_prev, Rprev, tprev, kl, dist_thres=0.10, angle_thres=SIN20):
    """Point-to-plane normal equations at Rcurr = Rprev, tcurr = tprev.  Maps are [3, rows, cols] float32 planes (NaN x = invalid):
    the current frame's in its camera, the model's in the volume frame."""
    _, rows, cols = vmap_curr.shape
    Rp = np.asarray(Rprev, np.float64).reshape(3, 3); tp = np.asarray(tprev, np.float64).reshape(3)
    Rpi = np.linalg.inv(Rp)
    fx, fy, cx, cy = (float(v) for v in kl)
    v = vmap_curr.reshape(3, -1).astype(np.float64).T; n = nmap_curr.reshape(3, -1).astype(np.float64).T
    vg = v @ Rp.T + tp                                   # vcurr_g
    s = (vg - tp) @ Rpi.T                                # vcurr_cp
    with np.errstate(invalid="ignore", divide="ignore"):
        uf = s[:, 0] * fx / s[:, 2] + cx; vf = s[:, 1] * fy / s[:, 2] + cy
    tmag = np.abs(tp).sum()
    smag = np.abs(v).sum(1) + tmag                       # the round trip through the volume frame rounds at |t|
    ok = ~np.isnan(v[:, 0])
    margin = C_ROW * U * (np.abs(uf) + np.abs(vf) + smag * (fx + fy) / np.maximum(np.abs(s[:, 2]), 1e-30))
    amb = ok & (_near(uf - np.floor(uf), 0.5, margin) | _near(vf - np.floor(vf), 0.5, margin))
    uk = np.rint(np.nan_to_num(uf)).astype(np.int64); vk = np.rint(np.nan_to_num(vf)).astype(np.int64)
    ok &= (uk >= 0) & (vk >= 0) & (uk < cols) & (vk < rows) & (s[:, 2] >= 0)
    j = np.clip(vk, 0, rows - 1) * cols + np.clip(uk, 0, cols - 1)
    vp = vmap_g_prev.reshape(3, -1).astype(np.float64).T[j]; npv = nmap_g_prev.reshape(3, -1).astype(np.float64).T[j]
    ok &= ~np.isnan(vp[:, 0]) & ~np.isnan(npv[:, 0]) & ~np.isnan(n[:, 0])
    ng = n @ Rp.T
    with np.errstate(invalid="ignore"):
        dist = np.linalg.norm(vp - vg, axis=1)
        sine = np.linalg.norm(np.cross(ng, npv), axis=1)
    dmag = np.abs(vp).sum(1) + tmag
    amb |= ok & (_near(dist, float(np.float32(dist_thres)), C_ROW * U * (dmag + smag)) | _near(sine, float(np.float32(angle_thres)), C_ROW * U * 4))
    inl = ok & (sine < float(np.float32(angle_thres))) & (dist <= float(np.float32(dist_thres)))
    d = (vp - tp) @ Rpi.T
    ncp = npv @ Rpi.T
    sxn = np.cross(s, ncp)
    res = np.einsum("ij,ij->i", ncp, s - d)
    nm = np.abs(ncp).sum(1); sm_abs = np.abs(s).sum(1)
    rows7 = np.concatenate([ncp, sxn, res[:, None]], axis=1)
    mags = np.concatenate([np.repeat(nm[:, None], 3, 1), np.repeat((2 * sm_abs * nm + smag * nm)[:, None], 3, 1),
                           (nm * (smag + dmag) + nm * np.abs(s - d).sum(1))[:, None]], axis=1) * (C_ROW * U)
    sure = inl & ~amb
    P, S, E = _products(rows7[sure], mags[sure])
    maybe = ok & amb
    _, Sa, Ea = _products(rows7[maybe], mags[maybe])
    amb_abs = Sa + Ea
    amb_abs[28] = int(maybe.sum())
    return System(P, _bound(S, E, amb_abs), int(sure.sum()), dict(ambiguous=int(maybe.sum())))


def merge(rgb, icp):
    """The -ri system: A_rgb + 100 A_icp, b_rgb + 10 b_icp (RGBDOdometry.cpp:316-321), with the bounds merged the same way."""
    w = np.array([10.0 if k in B_SLOTS else 100.0 for k in range(27)] + [0.0, 0.0])
    return System(rgb.P + w * icp.P, rgb.bound + w * icp.bound, rgb.count)


def _rodrigues(r):
    th = float(np.linalg.norm(r))
    if th == 0.0:
        return np.eye(3)
    k = r / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def pose_after_one_iteration(system, Rprev, tprev, guard=None):
    """Pose after one Gauss-Newton step from the previous pose, and its tolerance (rotation, translation): x = A^-1 b in FP64,
    resultRt = [rodrigues(x[3:]) | x[:3]], Rcurr = Rprev rot^T, tcurr = -Rprev rot^T tr + tprev (gauss_newton_update).  The tolerance
    propagates the entry bounds, |A^-1| (|dA| |x| + |db|), plus the float rounding of the composition.  guard: the photometric modes'
    0.3 m jump test (RGBDOdometry.cpp:383-387), which keeps the previous pose."""
    Rp = np.asarray(Rprev, np.float64).reshape(3, 3); tp = np.asarray(tprev, np.float64).reshape(3)
    A, b = system.A, system.b
    if not A.any():                                      # LDL^T of a zero matrix: zero increment
        x = np.zeros(6); dx = 0.0
    elif np.linalg.matrix_rank(A) < 6:                   # a rank-deficient system (a plane under ICP) pins no pose
        x = np.linalg.lstsq(A, b, rcond=None)[0]; dx = np.inf
    else:
        Ainv = np.linalg.inv(A)
        x = Ainv @ b
        dx = np.linalg.norm(Ainv, 2) * (np.linalg.norm(system.dA, 2) * np.linalg.norm(x) + np.linalg.norm(system.db))
    rot = _rodrigues(x[3:])
    Rc = Rp @ rot.T
    tc = -Rp @ rot.T @ x[:3] + tp
    fl = 16 * U * (np.abs(tp).sum() + np.abs(x[:3]).sum() + 1.0)
    tol_t = dx * (1.0 + np.linalg.norm(x[:3])) + fl
    tol_R = dx + 16 * U
    if guard is not None and np.linalg.norm(tc - tp) > guard:
        Rc, tc = Rp.copy(), tp.copy()
    return Rc, tc, tol_R, tol_t, x
