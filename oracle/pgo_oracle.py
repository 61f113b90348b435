"""CPU restatement (numpy / scipy, FP64) of loop closure's pose graph, the yardstick of kt_pgo.cu and kt_close_loop.

Written from the description of the reference's backend (src/backend/Deformation.cpp:130-346, iSAMInterface.cpp) and of iSAM's
Pose3d factors (slam3d.h, not in the checkout: restated, unpinned):
  select_nodes       Deformation::addCameraCamera (:130-171): every pose, or the -fl rule; loop poses and the last pose always
  odometry_z         addCameraCameraConstraint (iSAMInterface.cpp:44-83): prev^-1 curr in float32, M conjugation, float32 quaternion
  loop_z             addLoopConstraint (:85-105): M C M^-1 in FP64
  linearise          Pose3d_Pose3d_Factor: e = vector(p_i^-1 p_j) - z, angles wrapped to (-pi, pi], whitened by sqrt(1000)
  optimise           batch Gauss-Newton, J^T J solved by scipy.sparse spsolve, the stopping rule of kt_pgo.cu
Poses are 4 x 4 FP64, vector() = (x, y, z, yaw, pitch, roll), R = Rz(yaw) Ry(pitch) Rx(roll).  Update: t += rho, R <- R Exp(phi).
"""
import math

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import deform_oracle as D

M = np.array([[0, 0, 1], [-1, 0, 0], [0, -1, 0]], np.float64)     # transformation2isam
WHITEN = np.sqrt(1000.0)
MAX_LOOPS = 64


def wrap(a):
    r = np.fmod(np.asarray(a, np.float64) + np.pi, 2 * np.pi)
    r = np.where(r <= 0.0, r + 2 * np.pi, r)
    return r - np.pi


def ypr(R):
    R = np.asarray(R, np.float64)
    return np.stack([np.arctan2(R[..., 1, 0], R[..., 0, 0]),
                     np.arctan2(-R[..., 2, 0], np.sqrt(R[..., 2, 1] ** 2 + R[..., 2, 2] ** 2)),
                     np.arctan2(R[..., 2, 1], R[..., 2, 2])], -1)


def rot(v):
    v = np.asarray(v, np.float64)
    cy, sy, cp, spn, cr, sr = np.cos(v[..., 0]), np.sin(v[..., 0]), np.cos(v[..., 1]), np.sin(v[..., 1]), np.cos(v[..., 2]), np.sin(v[..., 2])
    R = np.empty(v.shape[:-1] + (3, 3))
    R[..., 0, 0] = cy * cp; R[..., 0, 1] = cy * spn * sr - sy * cr; R[..., 0, 2] = cy * spn * cr + sy * sr
    R[..., 1, 0] = sy * cp; R[..., 1, 1] = sy * spn * sr + cy * cr; R[..., 1, 2] = sy * spn * cr - cy * sr
    R[..., 2, 0] = -spn; R[..., 2, 1] = cp * sr; R[..., 2, 2] = cp * cr
    return R


def vector(X):
    X = np.asarray(X, np.float64)
    return np.concatenate([X[..., :3, 3], ypr(X[..., :3, :3])], -1)


def pose(v):
    v = np.asarray(v, np.float64)
    X = np.zeros(v.shape[:-1] + (4, 4)); X[..., :3, :3] = rot(v[..., 3:]); X[..., :3, 3] = v[..., :3]; X[..., 3, 3] = 1.0
    return X


def to_isam(P):
    """M P M^-1 in FP64 of float poses [..., 4, 4]."""
    P = np.asarray(P, np.float32).astype(np.float64)
    X = np.zeros(P.shape); X[..., :3, :3] = M @ P[..., :3, :3] @ M.T; X[..., :3, 3] = P[..., :3, 3] @ M.T; X[..., 3, 3] = 1.0
    return X


def from_isam(X):
    X = np.asarray(X, np.float64)
    P = np.zeros(X.shape); P[..., :3, :3] = M.T @ X[..., :3, :3] @ M; P[..., :3, 3] = X[..., :3, 3] @ M; P[..., 3, 3] = 1.0
    return P


def _quat_f32(m):
    """Eigen::Quaternionf(Matrix3f) in float32: (x, y, z, w)."""
    f = np.float32
    m = np.asarray(m, f)
    t = f(m[0, 0] + m[1, 1]) + m[2, 2]
    if t > f(0):
        t = np.sqrt(f(t + f(1)))
        w = f(0.5) * t
        t = f(0.5) / t
        return (f((m[2, 1] - m[1, 2]) * t), f((m[0, 2] - m[2, 0]) * t), f((m[1, 0] - m[0, 1]) * t), w)
    i = 0
    if m[1, 1] > m[0, 0]:
        i = 1
    if m[2, 2] > m[i, i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    t = np.sqrt(f(f(f(m[i, i] - m[j, j]) - m[k, k]) + f(1)))
    q = [f(0)] * 3
    q[i] = f(0.5) * t
    t = f(0.5) / t
    w = f((m[k, j] - m[j, k]) * t)
    q[j] = f((m[j, i] + m[i, j]) * t)
    q[k] = f((m[k, i] + m[i, k]) * t)
    return (q[0], q[1], q[2], w)


def odometry_z(prev, curr):
    """The measurement of the odometry factor prev -> curr (float32 4 x 4 tracked poses, world frame)."""
    f = np.float32
    p = np.asarray(prev, f); c = np.asarray(curr, f)
    inv = np.zeros((4, 4), f)
    inv[:3, :3] = p[:3, :3].T
    for r in range(3):
        inv[r, 3] = -f(f(p[0, r] * p[0, 3] + p[1, r] * p[1, 3]) + p[2, r] * p[2, 3])
    inv[3, 3] = 1
    d = np.zeros((4, 4), f)
    for r in range(4):
        for k in range(4):
            d[r, k] = f(f(f(inv[r, 0] * c[0, k] + inv[r, 1] * c[1, k]) + inv[r, 2] * c[2, k]) + inv[r, 3] * c[3, k])
    Mf = M.astype(f)
    Ri = (Mf @ d[:3, :3] @ Mf.T).astype(f)                # exact: one nonzero product per entry
    ti = (Mf @ d[:3, 3]).astype(f)
    x, y, z, w = (float(v) for v in _quat_f32(Ri))
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz, tyy, tyz, tzz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    R = np.array([[1 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1 - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, 1 - (txx + tyy)]])
    return np.concatenate([ti.astype(np.float64), _ypr_libm(R)])


def _ypr_libm(R):
    """ypr of one rotation through the C library's atan2 / sqrt, as kt_pgo.hpp computes it (numpy's arctan2 may differ by an ulp)."""
    R = [[float(v) for v in row] for row in R]
    return np.array([math.atan2(R[1][0], R[0][0]), math.atan2(-R[2][0], math.sqrt(R[2][1] * R[2][1] + R[2][2] * R[2][2])),
                     math.atan2(R[2][1], R[2][2])])


def loop_z(C):
    C = np.asarray(C, np.float64).reshape(4, 4)
    return np.concatenate([M @ C[:3, 3], _ypr_libm(M @ C[:3, :3] @ M.T)])


def check_constraint(C):
    """0 when C is finite with a rotation within 1e-3 of orthonormal; 1 not finite; 2 not orthonormal."""
    C = np.asarray(C, np.float64).reshape(4, 4)
    if not np.isfinite(C).all():
        return 1
    return 2 if np.abs(C[:3, :3].T @ C[:3, :3] - np.eye(3)).max() > 1e-3 else 0


def select_nodes(pos, flagged, pose_spacing):
    """Indices of the dense poses that are nodes (float32 positions)."""
    pos = np.asarray(pos, np.float32)
    n = len(pos)
    take = [0] if n else []
    for i in range(1, n):
        if pose_spacing == 0 or flagged[i] or D._dist_f32(pos[take[-1]], pos[i]) > np.float32(pose_spacing):
            take.append(i)
    if n and take[-1] != n - 1:
        take.append(n - 1)
    return np.array(take, np.int64)


def _skew(v):
    S = np.zeros(v.shape[:-1] + (3, 3))
    S[..., 0, 1] = -v[..., 2]; S[..., 0, 2] = v[..., 1]; S[..., 1, 0] = v[..., 2]
    S[..., 1, 2] = -v[..., 0]; S[..., 2, 0] = -v[..., 1]; S[..., 2, 1] = v[..., 0]
    return S


def linearise(X, fi, fj, fz):
    """Whitened errors [F, 6] and Jacobians J_i, J_j [F, 6, 6] (columns rho, phi) of the factors; fi = -1 is the prior at pose(fz)."""
    X = np.asarray(X, np.float64)
    prior = fi < 0
    Ti = np.where(prior[:, None, None], pose(fz), X[np.maximum(fi, 0)])
    Tj = X[fj]
    Ri, Rj = Ti[:, :3, :3], Tj[:, :3, :3]
    Re = np.swapaxes(Ri, 1, 2) @ Rj
    te = np.einsum("fji,fj->fi", Ri, Tj[:, :3, 3] - Ti[:, :3, 3])
    cp = np.sqrt(Re[:, 2, 1] ** 2 + Re[:, 2, 2] ** 2)
    ang = np.stack([np.arctan2(Re[:, 1, 0], Re[:, 0, 0]), np.arctan2(-Re[:, 2, 0], cp), np.arctan2(Re[:, 2, 1], Re[:, 2, 2])], 1)
    z = np.where(prior[:, None], 0.0, fz)
    e = np.concatenate([te - z[:, :3], wrap(ang - z[:, 3:])], 1) * WHITEN
    sr, cr, spn = np.sin(ang[:, 2]), np.cos(ang[:, 2]), -Re[:, 2, 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        G = np.zeros((len(fi), 3, 3))
        G[:, 0, 1] = sr / cp; G[:, 0, 2] = cr / cp; G[:, 1, 1] = cr; G[:, 1, 2] = -sr
        G[:, 2, 0] = 1.0; G[:, 2, 1] = sr * spn / cp; G[:, 2, 2] = cr * spn / cp
        Jj = np.zeros((len(fi), 6, 6)); Ji = np.zeros((len(fi), 6, 6))
        RiT = np.swapaxes(Ri, 1, 2)
        Jj[:, :3, :3] = RiT; Jj[:, 3:, 3:] = G
        Ji[:, :3, :3] = -RiT; Ji[:, :3, 3:] = _skew(te); Ji[:, 3:, 3:] = -G @ np.swapaxes(Re, 1, 2)
    return e, Ji * WHITEN, Jj * WHITEN


def exp_so3(w):
    th2 = (w * w).sum(-1); th = np.sqrt(th2)
    small = th < 1e-8
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.where(small, 1.0, np.sin(th) / th)
        b = np.where(small, 0.5, (1.0 - np.cos(th)) / th2)
    S = _skew(w)
    return np.eye(3) + a[..., None, None] * S + b[..., None, None] * (S @ S)


def update(X, dx):
    X = X.copy()
    dx = dx.reshape(-1, 6)
    X[:, :3, 3] += dx[:, :3]
    X[:, :3, :3] = X[:, :3, :3] @ exp_so3(dx[:, 3:])
    return X


def chain_factors(X0, loops):
    """(fi, fj, fz) of the chain graph kt_op_pgo_optimise takes: the prior on node 0 anchored at X0[0], odometry k-1 -> k with the
    relative poses of X0 as measurements, then loops = [(i, j, z6)]."""
    n = len(X0)
    fi = np.concatenate([[-1], np.arange(n - 1), [l[0] for l in loops]]).astype(np.int64)
    fj = np.concatenate([[0], np.arange(1, n), [l[1] for l in loops]]).astype(np.int64)
    rel = np.linalg.inv(X0[:-1]) @ X0[1:]
    fz = np.concatenate([vector(X0[:1]), vector(rel), np.array([l[2] for l in loops]).reshape(-1, 6)])
    return fi, fj, fz


def optimise(X0, fi, fj, fz, max_iter=100):
    """Gauss-Newton: (X, report dict with the fields of kt_pgo_report)."""
    X = np.asarray(X0, np.float64).copy()
    n, F = len(X), len(fi)
    rep = dict(nodes=n, factors=F, loops=F - n, iterations=0, solver_failed=0)
    e, Ji, Jj = linearise(X, fi, fj, fz)
    prev = float((e * e).sum())
    rep["chi2_initial"] = rep["chi2_final"] = prev
    prior = fi < 0
    for it in range(max_iter):
        rows = np.repeat(np.arange(6 * F).reshape(F, 6), 6, axis=1).reshape(F, 36)
        colj = (6 * fj[:, None] + np.arange(6)[None, :])
        coli = (6 * np.maximum(fi, 0)[:, None] + np.arange(6)[None, :])
        r_all = np.concatenate([rows.reshape(-1), rows[~prior].reshape(-1)])
        c_all = np.concatenate([np.tile(colj, (1, 6)).reshape(-1), np.tile(coli[~prior], (1, 6)).reshape(-1)])
        v_all = np.concatenate([Jj.reshape(-1), Ji[~prior].reshape(-1)])
        J = sp.csr_matrix((v_all, (r_all, c_all)), shape=(6 * F, 6 * n))
        H = (J.T @ J).tocsc()
        b = -(J.T @ e.reshape(-1))
        rep["iterations"] = it + 1
        if not np.isfinite(H.data).all():
            rep["solver_failed"] = 1
            break
        try:
            import scipy.linalg
            # SPD check on the dense matrix for small graphs; spsolve otherwise
            if 6 * n <= 3000:
                L = scipy.linalg.cholesky(H.toarray(), lower=True)
                dx = scipy.linalg.cho_solve((L, True), b)
            else:
                dx = spla.spsolve(H, b)
        except np.linalg.LinAlgError:
            rep["solver_failed"] = 1
            break
        X = update(X, dx)
        e, Ji, Jj = linearise(X, fi, fj, fz)
        chi2 = float((e * e).sum())
        rep["chi2_final"] = chi2
        dec = prev - chi2
        if dec < 1e-3 or dec < 1e-5 * prev:
            break
        prev = chi2
    return X, rep


# ---- kt_close_loop over a dense pose graph -------------------------------------------------------------------------------------
def close_loop(times, poses, loops, pose_spacing=0.0, isam_thresh=10.0):
    """times uint64 [n], poses float32 [n, 4, 4] (the dense pose graph); loops: [(time1, time2, C 4x4)], the accepted ones then the
    new one.  Returns (node indices, optimised node poses in the world frame [m, 4, 4], report, accepted)."""
    times = np.asarray(times, np.uint64); poses = np.asarray(poses, np.float32)
    at = {int(t): i for i, t in enumerate(times)}
    named = {at[int(t)] for l in loops for t in l[:2]}
    flagged = np.zeros(len(times), bool); flagged[list(named)] = True
    take = select_nodes(poses[:, :3, 3], flagged, pose_spacing)
    node_of = {int(k): q for q, k in enumerate(take)}
    X0 = to_isam(poses[take])
    n = len(take)
    fi = [-1] + list(range(n - 1)); fj = [0] + list(range(1, n))
    fz = [vector(X0[0])] + [odometry_z(poses[take[k - 1]], poses[take[k]]) for k in range(1, n)]
    for t1, t2, C in loops:
        fi.append(node_of[at[int(t1)]]); fj.append(node_of[at[int(t2)]]); fz.append(loop_z(C))
    X, rep = optimise(X0, np.array(fi), np.array(fj), np.array(fz))
    accepted = not rep["solver_failed"] and rep["chi2_final"] < isam_thresh
    return take, from_isam(X), rep, accepted


def synthetic_chain(seed, n, n_loops, step=0.05, drift=(2e-4, 1e-4)):
    """A seeded ground-truth trajectory (a wobbly circle), its drifted odometry-integrated estimate, and n_loops loop measurements
    from the ground truth between random far-apart nodes.  Returns (X_gt, X_drift, loops [(i, j, z6)]) in the isam frame."""
    rng = np.random.default_rng(seed)
    ang = np.arange(n) * step / 10.0
    v = np.zeros((n, 6))
    v[:, 0] = 10 * np.cos(ang); v[:, 1] = 10 * np.sin(ang); v[:, 2] = 0.3 * np.sin(5 * ang)
    v[:, 3] = ang + np.pi / 2; v[:, 4] = 0.05 * np.sin(3 * ang); v[:, 5] = 0.05 * np.cos(2 * ang)
    Xgt = pose(v)
    rel = np.linalg.inv(Xgt[:-1]) @ Xgt[1:]
    noise = np.concatenate([rng.normal(0, drift[0], (n - 1, 3)), rng.normal(0, drift[1], (n - 1, 3))], 1)
    Xd = np.empty_like(Xgt); Xd[0] = Xgt[0]
    for k in range(1, n):
        Xd[k] = Xd[k - 1] @ update(rel[k - 1][None], noise[k - 1])[0]
    loops = []
    for _ in range(n_loops):
        i = int(rng.integers(0, n // 4)); j = int(rng.integers(n // 2, n))
        loops.append((j, i, vector(np.linalg.inv(Xgt[j]) @ Xgt[i])))
    return Xgt, Xd, loops
